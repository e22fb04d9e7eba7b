"""The VQ-f4 latent diffusion models on the host: the oracle (oracle/vq_oracle.py) against the unmodified reference's
outputs (tests/golden/vq.pt), the architecture tables against the reference's key lists, the GEMM weight packing of
widths that are multiples of 32 only, argument checks, and config / checkpoint ingest of a CelebA-HQ-style model."""

import pytest
import torch
import yaml

import helpers  # noqa: F401  (sys.path for the oracle)
import uncond_oracle as U
import vq_oracle as V
from helpers import golden, rel_l2, script
from sdb200 import arch

UCFG = {"tiny_vq": arch.TINY_VQ_UNET, "celebahq": arch.CELEBAHQ_UNET}
VCFG = {"tiny_vq": arch.TINY_VQ, "vq_f4": arch.VQ_F4}


@pytest.mark.parametrize("idx", range(4))
def test_oracle_unet_matches_reference(idx):
    case = golden("vq.pt")["unet"][idx]
    sd = arch.random_state_dict(arch.unet_param_shapes(UCFG[case["cfg"]]), golden("vq.pt")["unet_seed"])
    assert rel_l2(V.unet_forward(sd, UCFG[case["cfg"]], case["x"], case["t"]), case["eps"]) < 1e-5


def test_oracle_quantizer_decode_encode_match_reference():
    g = golden("vq.pt")
    sds = {tag: arch.random_state_dict(arch.vq_param_shapes(cfg), g["vq_seed"]) for tag, cfg in VCFG.items()}
    for case in g["quantize"]:
        z_q, idx = V.quantize(case["z"], sds[case["cfg"]]["quantize.embedding.weight"])
        assert torch.equal(idx, case["indices"]) and torch.equal(z_q, case["z_q"])
    for case in g["decode"]:
        assert rel_l2(V.vq_decode(sds[case["cfg"]], case["h"], case["force_not_quantize"]), case["x"]) < 1e-5
    e = g["encode"]
    assert rel_l2(V.vq_encode(sds[e["cfg"]], e["x"]), e["h"]) < 1e-5


def test_oracle_ddim_trajectory_matches_reference():
    g = golden("vq.pt")
    d = g["ddim"]
    esd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_VQ_UNET), g["ema_seed"])
    fn = lambda x, t: V.unet_forward(esd, arch.TINY_VQ_UNET, x, t)
    s = U.ddim_sample_uncond(fn, d["x_T"], d["alphas_cumprod"], 10, 0.0, torch.zeros(10, *d["x_T"].shape))
    assert rel_l2(s, d["sample"]) < 1e-5
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ), g["vq_seed"])
    assert rel_l2(V.decode_first_stage(vsd, d["sample"]), d["x_dec"]) < 1e-5


def test_arch_tables_match_reference_keys():
    g = golden("vq.pt")
    assert [(k, tuple(s)) for k, s in arch.unet_param_shapes(arch.CELEBAHQ_UNET).items()] == \
        [(k, tuple(s)) for k, s in g["celebahq_unet_keys"]]
    assert [(k, tuple(s)) for k, s in arch.vq_param_shapes(arch.VQ_F4).items()] == [(k, tuple(s)) for k, s in g["vq_f4_keys"]]
    names = sorted("model_ema.diffusion_model" + k.replace(".", "") for k in arch.unet_param_shapes(arch.TINY_VQ_UNET))
    assert sorted(k for k in g["ddim"]["ema_keys"] if k not in ("model_ema.decay", "model_ema.num_updates")) == names
    plan = arch.unet_plan(arch.CELEBAHQ_UNET)
    layers = [l for grp in plan["input"] + [plan["middle"]] + plan["output"] for l in grp]
    assert sorted({(a["ch"], a["heads"], a["dhead"]) for k, _, a in layers if k == "attn"}) == \
        [(448, 14, 32), (672, 21, 32), (896, 28, 32)]


def test_codebook_init_rule():
    """The codebook draws N(0, 1) (the generic embedding rule's 0.02 would collapse every z_q towards 0); no other key of
    the existing tables matches the rule."""
    sd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ), 12)
    assert 0.8 < float(sd["quantize.embedding.weight"].std()) < 1.2
    for shapes in (arch.unet_param_shapes(arch.SD_V1_UNET), arch.vae_param_shapes(arch.SD_V1_VAE),
                   arch.clip_param_shapes(arch.SD_V1_CLIP), arch.safety_param_shapes(arch.SD_V1_SAFETY)):
        assert not [k for k in shapes if k.endswith("quantize.embedding.weight")]


def test_weight_packing_pads_32_aligned_widths():
    """Packed weights get zero columns up to whole 64-wide K steps per tap / per source; 64-aligned ones are unchanged."""
    from sdb200.unet import _pack_conv3, _pack_conv3_padk, _pack_hilo_1x1, _pack_hilo_conv3
    g = torch.Generator().manual_seed(0)
    w = torch.randn(8, 224, 3, 3, generator=g)
    p = _pack_conv3(w).view(8, 9, 256)
    assert torch.equal(p[:, :, :224], w.permute(0, 2, 3, 1).reshape(8, 9, 224).half())
    assert not p[:, :, 224:].any()
    w64 = torch.randn(8, 128, 3, 3, generator=g)
    assert torch.equal(_pack_conv3(w64), w64.permute(0, 2, 3, 1).reshape(8, -1).half())
    assert _pack_conv3_padk(torch.randn(8, 3, 3, 3, generator=g), 64).shape == (8, 64)
    w1 = torch.randn(5, 96, generator=g)
    h = _pack_hilo_1x1(w1).view(5, 3, 128)
    assert not h[:, :, 96:].any() and torch.equal(h[:, 0, :96], h[:, 1, :96])
    assert _pack_hilo_conv3(torch.randn(3, 224, 3, 3, generator=g)).shape == (3, 9 * 3 * 256)


def test_unet_argument_checks():
    import sdb200
    net = sdb200.UNetModel(**arch.CELEBAHQ_UNET)
    assert net.image_size == 64 and net.in_channels == 3 and not net.conditional and net._sg == 1
    sdb200.UNetModel(**{**arch.TINY_VQ_UNET, "legacy": False})
    for bad in (dict(use_scale_shift_norm=True), dict(resblock_updown=True), dict(use_new_attention_order=True)):
        with pytest.raises(NotImplementedError):
            sdb200.UNetModel(**{**arch.TINY_VQ_UNET, **bad})
    with pytest.raises(NotImplementedError):       # the transformer UNet keeps rejecting num_head_channels
        sdb200.UNetModel(**{**arch.TINY_UNET, "num_head_channels": 32})
    net.W = {}
    with pytest.raises(RuntimeError):               # no CPU fallback
        net(torch.zeros(1, 3, 64, 64), torch.zeros(1))


def test_vq_first_stage_arguments():
    import sdb200
    m = sdb200.VQModelInterface(**arch.VQ_F4, lossconfig={"target": "torch.nn.Identity"},
                                ckpt_path="configs/first_stage_models/vq-f4/model.yaml")
    assert m.n_embed == 8192 and m.embed_dim == 3
    with pytest.raises(NotImplementedError):
        sdb200.VQModelInterface(**arch.VQ_F4, remap="remap.npy")
    with pytest.raises(AssertionError):
        sdb200.VQModelInterface(**{**arch.VQ_F4, "ddconfig": {**arch.VQ_F4["ddconfig"], "double_z": True}})


def _celebahq_yaml(tmp_path):
    node = script("sample_diffusion").celebahq_config(arch.TINY_VQ_UNET, arch.TINY_VQ)
    p = tmp_path / "config.yaml"
    p.write_text(yaml.safe_dump({"model": {"base_learning_rate": 2.0e-06, **node}}))
    return str(p)


def test_load_celebahq_style_config_and_checkpoint(tmp_path):
    """A reference-style VQ-f4 LDM config (ldm.* targets incl. VQModelInterface, __is_unconditional__) and a synthetic
    checkpoint: the first stage is the sdb200 VQ model with the codebook loaded, loss keys are ignored."""
    import sdb200
    from sdb200 import checkpoint
    cfg = _celebahq_yaml(tmp_path)
    u = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_VQ_UNET), 11)
    v = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ), 12)
    sd = {"model.diffusion_model." + k: t for k, t in u.items()}
    sd.update({"first_stage_model." + k: t for k, t in v.items()})
    sd["first_stage_model.loss.logvar"] = torch.zeros(())
    ck = tmp_path / "model.ckpt"
    torch.save({"state_dict": sd, "global_step": 3}, ck)
    model = checkpoint.load_model_from_config(cfg, str(ck), device=None, allow_pickle=True)
    fs = model.first_stage_model
    assert isinstance(fs, sdb200.VQModelInterface) and model.cond_stage_model is None
    assert torch.equal(fs._host_sd["quantize.embedding.weight"], v["quantize.embedding.weight"])
    assert not [k for k in model.load_info["unexpected"] if k.startswith("first_stage_model.")]
    assert float(model.get_first_stage_encoding(torch.ones(2))[0]) == 1.0
