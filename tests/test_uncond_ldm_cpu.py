"""The unconditional attention-block LDM family on the host: the oracle (oracle/uncond_oracle.py) against the unmodified
reference's outputs (tests/golden/lsun.pt), the architecture tables, argument checks, and checkpoint ingest of the
LSUN-Churches config (scale_by_std buffer, EMA copies)."""
import pytest
import torch
import yaml

import helpers  # noqa: F401  (sys.path for the oracle)
import uncond_oracle as U
from helpers import golden, rel_l2, script
from sdb200 import arch

CFG = {"tiny_attn": arch.TINY_ATTN_UNET, "tiny_attn_plain": arch.TINY_ATTN_PLAIN_UNET, "lsun": arch.LSUN_CHURCHES_UNET}
_sd = {}


def _weights(tag, seed=11):
    if (tag, seed) not in _sd:
        _sd[(tag, seed)] = arch.random_state_dict(arch.unet_param_shapes(CFG[tag]), seed)
    return _sd[(tag, seed)]


@pytest.mark.parametrize("idx", range(6))
def test_oracle_unet_matches_reference(idx):
    case = golden("lsun.pt")["unet"][idx]
    eps = U.unet_forward(_weights(case["cfg"]), CFG[case["cfg"]], case["x"], case["t"])
    assert rel_l2(eps, case["eps"]) < 1e-5


def test_oracle_trajectories_match_reference():
    g = golden("lsun.pt")
    sd = _weights("tiny_attn")
    fn = lambda x, t: U.unet_forward(sd, arch.TINY_ATTN_UNET, x, t)
    d = g["ddim"]
    assert rel_l2(U.ddim_sample_uncond(fn, d["x_T"], g["sched_alphas_cumprod"], 10, 1.0, d["noise"]), d["sample"]) < 1e-5
    a = g["ancestral"]
    s, inter = U.progressive_denoising(fn, a["x_T"], U.ddpm_schedule(20), a["noise"])
    assert torch.equal(s, a["sample"]) and all(torch.equal(p, q) for p, q in zip(inter, a["intermediates"]))
    sched = U.ddpm_schedule(1000)
    for k in ("posterior_variance", "posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2",
              "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod"):
        assert torch.equal(sched[k], g["sched_" + k]), k


def test_oracle_ema_case():
    e = golden("lsun.pt")["ema"]
    out = U.unet_forward(_weights("tiny_attn", golden("lsun.pt")["ema_seed"]), arch.TINY_ATTN_UNET, e["x"], e["t"])
    assert rel_l2(out, e["eps_ema"]) < 1e-5 and rel_l2(e["eps_raw"], e["eps_ema"]) > 0.1


def test_arch_tables_match_reference_keys():
    """The reference LitEma names (every UNet parameter, dots removed) pin the key list of the tiny config; the LSUN
    table has the heads the reference builds (num_head_channels=-1: C / num_heads = 24, 48, 96)."""
    ema_keys = golden("lsun.pt")["ema"]["ema_keys"]
    names = sorted("model_ema.diffusion_model" + k.replace(".", "") for k in arch.unet_param_shapes(arch.TINY_ATTN_UNET))
    assert sorted(k for k in ema_keys if k not in ("model_ema.decay", "model_ema.num_updates")) == names
    plan = arch.unet_plan(arch.LSUN_CHURCHES_UNET)
    layers = [l for grp in plan["input"] + [plan["middle"]] + plan["output"] for l in grp]
    heads = sorted({(a["ch"], a["heads"], a["dhead"]) for k, _, a in layers if k == "attn"})
    assert heads == [(192, 8, 24), (384, 8, 48), (768, 8, 96)]
    assert sum(1 for k, _, a in layers if k == "res" and a["updown"] == "down") == 4
    assert sum(1 for k, _, a in layers if k == "res" and a["updown"] == "up") == 4
    shapes = arch.unet_param_shapes(arch.LSUN_CHURCHES_UNET)
    assert shapes["input_blocks.1.0.emb_layers.1.weight"] == (384, 768)       # [scale | shift]
    assert shapes["middle_block.1.qkv.weight"] == (2304, 768, 1)
    assert len(shapes) == 520
    plain = arch.unet_param_shapes(arch.TINY_ATTN_PLAIN_UNET)
    assert "input_blocks.2.0.op.weight" in plain and "output_blocks.1.2.conv.weight" in plain


def test_unet_argument_checks():
    import sdb200
    with pytest.raises(NotImplementedError):      # the transformer UNet still rejects scale-shift and up/down
        sdb200.UNetModel(**{**arch.TINY_UNET, "use_scale_shift_norm": True})
    with pytest.raises(NotImplementedError):
        sdb200.UNetModel(**{**arch.TINY_UNET, "resblock_updown": True})
    for bad in (dict(use_new_attention_order=True), dict(num_classes=10), dict(dims=3), dict(dropout=0.1),
                dict(num_heads=-1, num_head_channels=32)):
        with pytest.raises(NotImplementedError):
            sdb200.UNetModel(**{**arch.TINY_ATTN_UNET, **bad})
    net = sdb200.UNetModel(**arch.LSUN_CHURCHES_UNET)
    assert net.image_size == 32 and net.in_channels == 4 and not net.conditional
    net.W = {}
    with pytest.raises(RuntimeError):               # no CPU fallback
        net(torch.zeros(1, 4, 32, 32), torch.zeros(1))


def _lsun_yaml(tmp_path, unet_cfg, vae_cfg):
    node = script("sample_diffusion").lsun_churches_config(unet_cfg, vae_cfg)
    node["params"]["scheduler_config"] = {"target": "ldm.lr_scheduler.LambdaLinearScheduler",
                                          "params": {"warm_up_steps": [10000], "cycle_lengths": [10000000000000],
                                                     "f_start": [1.0e-6], "f_max": [1.0], "f_min": [1.0]}}
    cfg = {"model": {"base_learning_rate": 5.0e-5, **node}}
    p = tmp_path / "config.yaml"
    p.write_text(yaml.safe_dump(cfg))
    return str(p)


def test_load_lsun_config_with_scale_factor_and_ema(tmp_path):
    """A reference-style LSUN-Churches config (ldm.* targets, __is_unconditional__, scale_by_std, use_ema default) and a
    synthetic checkpoint: scale_factor is loaded, the EMA copies become the UNet's "ema" weight set."""
    from sdb200 import checkpoint
    cfg = _lsun_yaml(tmp_path, arch.TINY_ATTN_UNET, arch.TINY_VAE)
    raw, ema = _weights("tiny_attn"), _weights("tiny_attn", 31)
    sd = {"model.diffusion_model." + k: v for k, v in raw.items()}
    sd.update({"first_stage_model." + k: v for k, v in
               arch.random_state_dict(arch.vae_param_shapes(arch.TINY_VAE), 12).items()})
    sd.update({"model_ema." + ("diffusion_model." + k).replace(".", ""): v for k, v in ema.items()})
    sd["model_ema.decay"], sd["model_ema.num_updates"] = torch.tensor(0.9999), torch.tensor(1000, dtype=torch.int)
    sd["scale_factor"] = torch.tensor(0.37)
    ck = tmp_path / "model.ckpt"
    torch.save({"state_dict": sd, "global_step": 7}, ck)
    model = checkpoint.load_model_from_config(cfg, str(ck), device=None, allow_pickle=True)
    assert model.cond_stage_model is None and model.model.conditioning_key is None
    assert abs(float(model.scale_factor) - 0.37) < 1e-7 and model.use_ema
    unet = model.model.diffusion_model
    assert unet.has_weight_set("ema")
    k = "input_blocks.1.1.qkv.weight"
    assert torch.equal(unet._alt_sd["ema"][k], ema[k]) and torch.equal(unet._host_sd[k], raw[k])
    assert not [u for u in model.load_info["unexpected"] if u.startswith("model_ema.")]
    assert model.load_info["global_step"] == 7
