"""The class-conditional ImageNet LDM-VQ-8 (models/ldm/cin256) on the host: the oracle (oracle/cin_f8_oracle.py) against
the unmodified reference's outputs (tests/golden/cin_f8.pt), the architecture tables against the reference's key list of
the whole model, both reference YAML nodes, checkpoint ingest with EMA weights, and argument checks."""

import pytest
import torch
import yaml

import helpers  # noqa: F401  (sys.path for the oracle)
import cin_f8_oracle as F8
import cin_oracle as CO
import uncond_oracle as U
from helpers import golden, rel_l2, script
from sdb200 import arch

UCFG = {"tiny": arch.TINY_CIN_F8_UNET, "cin256": arch.CIN256_F8_UNET}
CCFG = {"tiny": arch.TINY_CIN_F8_COND, "cin256": arch.CIN256_F8_COND}
VCFG = {"tiny": arch.TINY_VQ_F8, "vq_f8": arch.VQ_F8}


def _gen(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def _sub(x, g):
    """The pixels the golden stores of a decoded image: every g["image_stride"]-th in both directions."""
    k = g["image_stride"]
    return x[..., ::k, ::k]


@pytest.mark.parametrize("idx", range(5))
def test_oracle_unet_matches_reference(idx):
    g = golden("cin_f8.pt")
    case = g["unet"][idx]
    sd = arch.random_state_dict(arch.unet_param_shapes(UCFG[case["cfg"]]), g["unet_seed"])
    csd = arch.random_state_dict(arch.class_embedder_param_shapes(CCFG[case["cfg"]]), g["cond_seed"])
    c = CO.class_embed(csd, case["labels"])
    assert torch.equal(c, case["c"])
    assert rel_l2(F8.unet_forward(sd, _gen(case["shape"], case["x_seed"]), case["t"], c), case["eps"]) < 1e-5


def test_oracle_first_stage_matches_reference():
    """Decode through the 16384 x 4 quantizer and encode, with the level AttnBlocks (tiny: 128 and 512 wide)."""
    g = golden("cin_f8.pt")
    sds = {tag: arch.random_state_dict(arch.vq_param_shapes(cfg), g["vq_seed"]) for tag, cfg in VCFG.items()}
    for case in g["decode"]:
        x = F8.vq_decode(sds[case["cfg"]], _gen(case["shape"], case["seed"]))
        assert tuple(x.shape) == tuple(case["x_shape"]) and rel_l2(_sub(x, g), case["x"]) < 1e-5
    for case in g["encode"]:
        x = _gen(case["shape"], case["seed"]).clamp(-1, 1)
        assert rel_l2(F8.vq_encode(sds[case["cfg"]], x), case["h"]) < 1e-5
    assert {(c["cfg"], tuple(c["shape"])) for c in g["decode"]} >= {("vq_f8", (2, 4, 32, 32)), ("vq_f8", (1, 4, 16, 48))}


@pytest.mark.parametrize("eta", [0, 1])
def test_oracle_ddim_trajectory_matches_reference(eta):
    g = golden("cin_f8.pt")
    d = g["ddim"]
    r = d[f"eta{eta}"]
    esd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_CIN_F8_UNET), g["ema_seed"])
    csd = arch.random_state_dict(arch.class_embedder_param_shapes(arch.TINY_CIN_F8_COND), g["cond_seed"])
    x_T = _gen((2, 4, 16, 16), d["x_T_seed"])
    noises = torch.stack([_gen(x_T.shape, d["noise_seed"] + i) for i in range(r["n_noise"])])
    fn = lambda x, t: F8.unet_forward(esd, x, t, CO.class_embed(csd, d["classes"]))
    s = U.ddim_sample_uncond(fn, x_T, g["alphas_cumprod"], 10, float(eta), noises if eta else torch.zeros_like(noises))
    assert rel_l2(s, r["sample"]) < 1e-5
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F8), g["vq_seed"])
    assert rel_l2(_sub(F8.decode_first_stage(vsd, r["sample"]), g), r["x_dec"]) < 1e-5


def test_arch_tables_match_reference_keys():
    """Every parameter of the reference's cin256 LatentDiffusion by key and shape, its EMA copies (use_ema defaults to
    True) and the spatial-transformer plan."""
    g = golden("cin_f8.pt")
    ref = [(k, tuple(s)) for k, s in g["cin256_keys"]]
    ushapes = arch.unet_param_shapes(arch.CIN256_F8_UNET)
    vshapes = arch.vq_param_shapes(arch.VQ_F8)
    mine = [("model.diffusion_model." + k, tuple(s)) for k, s in ushapes.items()]
    mine += [("first_stage_model." + k, tuple(s)) for k, s in vshapes.items()]
    mine += [("cond_stage_model." + k, tuple(s)) for k, s in arch.class_embedder_param_shapes(arch.CIN256_F8_COND).items()]
    mine += [("model_ema.diffusion_model" + k.replace(".", ""), tuple(s)) for k, s in ushapes.items()]
    stages = ("model.", "first_stage_model.", "cond_stage_model.", "model_ema.diffusion_model")
    assert sorted(e for e in ref if e[0].startswith(stages)) == sorted(mine)
    assert {k for k, _ in ref if k.startswith("model_ema.") and not k.startswith(stages)} == \
        {"model_ema.decay", "model_ema.num_updates"}
    assert ("cond_stage_model.embedding.weight", (1000, 512)) in ref
    # the first stage in the reference's own registration order, level AttnBlocks included
    assert [e for e in ref if e[0].startswith("first_stage_model.")] == \
        [("first_stage_model." + k, tuple(s)) for k, s in vshapes.items()]
    for pre, n in (("encoder.down.3.attn", 2), ("decoder.up.3.attn", 3)):
        assert sorted({k[len(pre) + 1:].split(".")[0] for k in vshapes if k.startswith(pre + ".")}) == \
            [str(i) for i in range(n)]
    assert not [k for k in vshapes if ".attn." in k and not k.startswith(("encoder.down.3.", "decoder.up.3."))]
    plan = arch.unet_plan(arch.CIN256_F8_UNET)
    layers = [l for grp in plan["input"] + [plan["middle"]] + plan["output"] for l in grp]
    sts = [(a["ch"], a["heads"], a["dhead"]) for k, _, a in layers if k == "st"]
    assert len(sts) == 16 and sorted(set(sts)) == [(256, 8, 32), (512, 16, 32), (1024, 32, 32)]
    assert sts[6] == (1024, 32, 32)          # the middle block's


def test_tiny_members_level_attention():
    """The tiny first stage has level attention 128 wide (32x32: the per-image path) and 512 wide (8x8: the d = 512 flash
    path), one per ResnetBlock (the decoder has num_res_blocks + 1 of them); the tiny UNet has several heads of 32."""
    v = arch.vq_param_shapes(arch.TINY_VQ_F8)
    widths = {k.rsplit(".", 2)[0]: s[0] for k, s in v.items() if ".attn." in k and k.endswith(".q.weight")}
    assert widths == {"encoder.down.1.attn.0": 128, "encoder.down.3.attn.0": 512,
                      "decoder.up.1.attn.0": 128, "decoder.up.1.attn.1": 128,
                      "decoder.up.3.attn.0": 512, "decoder.up.3.attn.1": 512}
    plan = arch.unet_plan(arch.TINY_CIN_F8_UNET)
    layers = [l for grp in plan["input"] + [plan["middle"]] + plan["output"] for l in grp]
    assert sorted({(a["ch"], a["heads"], a["dhead"]) for k, _, a in layers if k == "st"}) == [(64, 2, 32), (128, 4, 32)]
    # attn_resolutions follow ddconfig.resolution: the same keys whatever size the stage later runs at
    assert not [k for k in arch.vq_param_shapes(arch.VQ_F4) if ".attn." in k]


@pytest.mark.parametrize("path", ["models/ldm/cin256/config.yaml", "configs/latent-diffusion/cin-ldm-vq-f8.yaml"])
def test_reference_yaml_nodes_resolve(path):
    """Both reference YAMLs' model nodes instantiate through TARGET_MAP with the parameters of the arch tables (the
    cin-ldm-vq-f8 first stage's ckpt_path points at a .yaml and is ignored), and the script's node is the same model."""
    import sdb200
    from sdb200.util import TARGET_MAP, instantiate_from_config, remap_config
    node = golden("cin_f8.pt")["yaml_nodes"][path]
    p = node["params"]
    assert p["unet_config"]["params"] == arch.CIN256_F8_UNET
    assert p["first_stage_config"]["params"]["ddconfig"] == arch.VQ_F8["ddconfig"]
    assert (p["first_stage_config"]["params"]["embed_dim"], p["first_stage_config"]["params"]["n_embed"]) == (4, 16384)
    assert p["cond_stage_config"]["params"] == {"embed_dim": 512, "key": "class_label"}
    assert "use_ema" not in p
    for t in [node["target"]] + [p[k]["target"] for k in ("unet_config", "first_stage_config", "cond_stage_config")]:
        assert t in TARGET_MAP
    m = instantiate_from_config(remap_config(node))
    assert isinstance(m.model.diffusion_model, sdb200.UNetModel) and m.model.diffusion_model.conditional
    assert isinstance(m.first_stage_model, sdb200.VQModelInterface) and m.first_stage_model.shapes == arch.vq_param_shapes(arch.VQ_F8)
    assert isinstance(m.cond_stage_model, sdb200.ClassEmbedder) and m.cond_stage_model.n_classes == 1000
    assert m.use_ema and m.cond_stage_key == "class_label" and m.model.conditioning_key == "crossattn"
    mine = script("sample_imagenet").cin256_f8_config()
    assert {k: v for k, v in mine["params"].items() if k not in ("unet_config", "first_stage_config", "cond_stage_config")} == \
        {k: v for k, v in p.items() if k not in ("unet_config", "first_stage_config", "cond_stage_config")}
    assert mine["params"]["unet_config"] == p["unet_config"]


def test_load_tiny_checkpoint_with_ema(tmp_path):
    """A cin256-style config (tiny members) and a checkpoint with model_ema.* load with no missing or unexpected keys;
    the EMA copies become the UNet's "ema" weight set."""
    import sdb200
    from sdb200 import checkpoint
    node = script("sample_imagenet").cin256_f8_config(arch.TINY_CIN_F8_UNET, arch.TINY_VQ_F8, arch.TINY_CIN_F8_COND)
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": {"base_learning_rate": 1.0e-06, **node}}))
    ushapes = arch.unet_param_shapes(arch.TINY_CIN_F8_UNET)
    u, e = arch.random_state_dict(ushapes, 11), arch.random_state_dict(ushapes, 31)
    sd = {"model.diffusion_model." + k: t for k, t in u.items()}
    sd.update({"model_ema.diffusion_model" + k.replace(".", ""): t for k, t in e.items()})
    sd.update({"model_ema.decay": torch.tensor(0.9999), "model_ema.num_updates": torch.tensor(7, dtype=torch.int)})
    sd.update({"first_stage_model." + k: t for k, t in
               arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F8), 12).items()})
    sd.update({"cond_stage_model." + k: t for k, t in
               arch.random_state_dict(arch.class_embedder_param_shapes(arch.TINY_CIN_F8_COND), 13).items()})
    ck = tmp_path / "model.ckpt"
    torch.save({"state_dict": sd, "global_step": 7}, ck)
    model = checkpoint.load_model_from_config(str(cfg), str(ck), device=None, allow_pickle=True)
    info = model.load_info
    schedule = ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod")
    assert [k for k in info["missing"] if k not in schedule] == [] and info["unexpected"] == []
    unet = model.model.diffusion_model
    assert model.use_ema and model.model_ema.loaded and unet.has_weight_set("ema")
    assert all(torch.equal(unet._alt_sd["ema"][k], e[k]) for k in ushapes)
    assert isinstance(model.first_stage_model, sdb200.VQModelInterface)
    assert any(k.startswith("decoder.up.3.attn.1.") for k in model.first_stage_model._host_sd)


def test_unet_arguments():
    """cin256's UNet is accepted (legacy True and False) with GroupNorm-statistics entries of 8 channels; the other
    spatial-transformer checks stay."""
    import sdb200
    net = sdb200.UNetModel(**arch.CIN256_F8_UNET)
    assert net.conditional and net._sg == 8 and net.num_heads == -1
    sdb200.UNetModel(**{**arch.CIN256_F8_UNET, "legacy": False})
    assert sdb200.UNetModel(**arch.TINY_CIN_F8_UNET)._sg == 2
    for bad in (dict(transformer_depth=2), dict(use_scale_shift_norm=True), dict(num_heads=8)):
        with pytest.raises(NotImplementedError):
            sdb200.UNetModel(**{**arch.CIN256_F8_UNET, **bad})


def test_unet_packs_heads_per_layer():
    """Every spatial transformer is packed with its own head count at d = 32; the SD-v1 tiny UNet keeps num_heads."""
    import sdb200
    net = sdb200.UNetModel(**arch.TINY_CIN_F8_UNET)
    net._host_sd = arch.random_state_dict(net.shapes, 11)
    net.pack_weights(torch.device("cpu"))
    assert [(s["ch"], s["heads"], s["d"], s["dpad"]) for s in net.W["st_list"]] == \
        [(64, 2, 32, 64), (128, 4, 32, 64), (128, 4, 32, 64), (128, 4, 32, 64), (128, 4, 32, 64), (64, 2, 32, 64),
         (64, 2, 32, 64)]
    sd1 = sdb200.UNetModel(**arch.TINY_UNET)
    sd1._host_sd = arch.random_state_dict(sd1.shapes, 11)
    sd1.pack_weights(torch.device("cpu"))
    assert {(s["heads"], s["d"]) for s in sd1.W["st_list"]} == {(2, 32), (2, 64)}


def test_first_stage_arguments():
    import sdb200
    m = sdb200.VQModelInterface(**arch.VQ_F8, lossconfig={"target": "torch.nn.Identity"},
                                ckpt_path="configs/first_stage_models/vq-f8/model.yaml")
    assert m.n_embed == 16384 and m.embed_dim == 4
    with pytest.raises(AssertionError):      # KL first stages with level attention stay out of scope
        sdb200.AutoencoderKL(ddconfig={**arch.SD_V1_VAE["ddconfig"], "attn_resolutions": [16]}, embed_dim=4)


def test_script_rejects_guidance_for_cin256():
    """cin256 has no unconditional label: any scale other than 1.0 is an error before anything is built."""
    mod = script("sample_imagenet")
    for scale in ("3", "0.5"):
        with pytest.raises(ValueError, match="unconditional"):
            mod.main(["--model", "cin256", "--scale", scale, "--random_init", "--tiny"])
    assert mod.MODELS["cin256"][2] == 1.0 and mod.MODELS["cin256-v2"][2] == 3.0
    assert mod.get_parser().parse_args([]).model == "cin256-v2"
