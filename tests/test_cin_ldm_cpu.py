"""The class-conditional ImageNet LDM (cin256-v2) on the host: the oracle (oracle/cin_oracle.py, ldm_oracle.unet_forward
with one head) against the unmodified reference's outputs (tests/golden/cin.pt), the architecture tables against the
reference's key list of the whole model, config resolution, checkpoint ingest and argument checks."""

import pytest
import torch
import yaml

import helpers  # noqa: F401  (sys.path for the oracle)
import cin_oracle as CO
import ldm_oracle as O
import vq_oracle as V
from helpers import golden, rel_l2, script
from sdb200 import arch

UCFG = {"tiny_cin": arch.TINY_CIN_UNET, "cin256": arch.CIN256_V2_UNET}
CCFG = {"tiny_cin": arch.TINY_CIN_COND, "cin256": arch.CIN256_V2_COND}


@pytest.mark.parametrize("idx", range(5))
def test_oracle_unet_matches_reference(idx):
    g = golden("cin.pt")
    case = g["unet"][idx]
    sd = arch.random_state_dict(arch.unet_param_shapes(UCFG[case["cfg"]]), g["unet_seed"])
    csd = arch.random_state_dict(arch.class_embedder_param_shapes(CCFG[case["cfg"]]), g["cond_seed"])
    c = CO.class_embed(csd, case["labels"])
    assert torch.equal(c, case["c"])
    assert rel_l2(O.unet_forward(sd, case["x"], case["t"], c, num_heads=1), case["eps"]) < 1e-5


def test_oracle_guided_ddim_trajectory_matches_reference():
    g = golden("cin.pt")
    d = g["ddim"]
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_CIN_UNET), g["unet_seed"])
    csd = arch.random_state_dict(arch.class_embedder_param_shapes(arch.TINY_CIN_COND), g["cond_seed"])
    fn = lambda x, t, ctx: O.unet_forward(usd, x, t, ctx, num_heads=1)
    uc = CO.class_embed(csd, torch.full_like(d["classes"], 1000))
    s = CO.ddim_sample_guided(fn, d["x_T"], CO.class_embed(csd, d["classes"]), uc, 3.0, d["alphas_cumprod"], 10)
    assert rel_l2(s, d["sample"]) < 1e-5
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ), g["vq_seed"])
    assert rel_l2(V.decode_first_stage(vsd, d["sample"]), d["x_dec"]) < 1e-5


def test_arch_tables_match_reference_keys():
    """Every parameter of the reference's cin256-v2 LatentDiffusion, by key and shape (the reference registers a
    BasicTransformerBlock's ff before attn2, so the orders differ); the rest of its state_dict is the schedule buffers
    (recomputed from the config)."""
    ref = [(k, tuple(s)) for k, s in golden("cin.pt")["cin256_keys"]]
    mine = [("model.diffusion_model." + k, tuple(s)) for k, s in arch.unet_param_shapes(arch.CIN256_V2_UNET).items()]
    mine += [("first_stage_model." + k, tuple(s)) for k, s in arch.vq_param_shapes(arch.VQ_F4).items()]
    mine += [("cond_stage_model." + k, tuple(s)) for k, s in arch.class_embedder_param_shapes(arch.CIN256_V2_COND).items()]
    stages = ("model.", "first_stage_model.", "cond_stage_model.")
    assert sorted(e for e in ref if e[0].startswith(stages)) == sorted(mine)
    assert ("cond_stage_model.embedding.weight", (1001, 512)) in ref
    assert all("." not in k for k, _ in ref if not k.startswith(stages))
    plan = arch.unet_plan(arch.CIN256_V2_UNET)
    layers = [l for grp in plan["input"] + [plan["middle"]] + plan["output"] for l in grp]
    sts = [(a["ch"], a["heads"], a["dhead"]) for k, _, a in layers if k == "st"]
    assert len(sts) == 16 and sorted(set(sts)) == [(384, 1, 384), (576, 1, 576), (960, 1, 960)]


def test_target_map_resolves_every_cin_target():
    from sdb200.util import TARGET_MAP, get_obj_from_str
    node = script("sample_imagenet").cin_config()
    targets = [node["target"]] + [node["params"][k]["target"] for k in ("unet_config", "first_stage_config",
                                                                           "cond_stage_config")]
    for t in targets:
        assert t in TARGET_MAP
        get_obj_from_str(TARGET_MAP[t])
    import sdb200
    assert get_obj_from_str(TARGET_MAP["ldm.modules.encoders.modules.ClassEmbedder"]) is sdb200.ClassEmbedder


def test_unet_accepts_cin_config_and_groupnorm_entries():
    """cin256-v2's UNet is accepted as configured; its 6 channels per GroupNorm group fuse statistics in entries of 2
    (no GEMM tile width is a multiple of 6), while SD-v1 keeps entries of 10."""
    import sdb200
    net = sdb200.UNetModel(**arch.CIN256_V2_UNET)
    assert net.conditional and net.num_heads == 1 and net._sg == 2
    assert sdb200.UNetModel(**arch.SD_V1_UNET)._sg == 10
    assert sdb200.UNetModel(**arch.TINY_CIN_UNET)._sg == 2


def test_class_embedder_interface():
    import sdb200
    m = sdb200.ClassEmbedder(512, n_classes=1001, key="class_label")
    assert m.key == "class_label" and m.shapes == {"embedding.weight": (1001, 512)}
    assert sdb200.ClassEmbedder(16).n_classes == 1000 and sdb200.ClassEmbedder(16).key == "class"
    sd = arch.random_state_dict(arch.class_embedder_param_shapes(arch.CIN256_V2_COND), 13)
    assert 0.9 < float(sd["embedding.weight"].std()) < 1.1          # nn.Embedding's N(0, 1)
    r = m.load_state_dict(sd, strict=False)
    assert not r.missing_keys and not r.unexpected_keys and torch.equal(m._host_sd["embedding.weight"], sd["embedding.weight"])


def test_load_tiny_cin_checkpoint(tmp_path):
    """A reference-style cin256-v2 config (tiny members) and a checkpoint written from random state dicts load through
    load_model_from_config with no missing or unexpected keys."""
    import sdb200
    from sdb200 import checkpoint
    node = script("sample_imagenet").cin_config(arch.TINY_CIN_UNET, arch.TINY_VQ, arch.TINY_CIN_COND)
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": {"base_learning_rate": 1.0e-04, **node}}))
    sd = {"model.diffusion_model." + k: t for k, t in
          arch.random_state_dict(arch.unet_param_shapes(arch.TINY_CIN_UNET), 11).items()}
    sd.update({"first_stage_model." + k: t for k, t in arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ), 12).items()})
    emb = arch.random_state_dict(arch.class_embedder_param_shapes(arch.TINY_CIN_COND), 13)
    sd.update({"cond_stage_model." + k: t for k, t in emb.items()})
    ck = tmp_path / "model.ckpt"
    torch.save({"state_dict": sd, "global_step": 7}, ck)
    model = checkpoint.load_model_from_config(str(cfg), str(ck), device=None, allow_pickle=True)
    info = model.load_info
    schedule = ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod")
    assert [k for k in info["missing"] if k not in schedule] == [] and info["unexpected"] == []
    assert isinstance(model.cond_stage_model, sdb200.ClassEmbedder) and model.cond_stage_key == "class_label"
    assert torch.equal(model.cond_stage_model._host_sd["embedding.weight"], emb["embedding.weight"])
    assert model.model.conditioning_key == "crossattn"
