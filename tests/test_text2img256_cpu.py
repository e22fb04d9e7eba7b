"""The text-conditional LDM-VQ-4 (models/ldm/text2img256) on the host: the oracles (bert_oracle, cin_f8_oracle's UNet with
heads of num_head_channels, the samplers of ldm_oracle / uncond_oracle, vq_oracle's decode) against the unmodified
reference's outputs (tests/golden/text2img256.pt), the architecture tables against the reference's key list of the whole
model, checkpoint ingest from the unchanged YAML with the EMA set, and the host logic of scripts/txt2img.py for any
text-conditional config."""
import contextlib
import functools

import pytest
import torch
import yaml

import helpers  # noqa: F401  (sys.path for the oracle)
import bert_oracle as BO
import cin_f8_oracle as F8
import ldm_oracle as O
import uncond_oracle as U
import vq_oracle as VO
from helpers import golden, rel_l2, script
from sdb200 import arch

SCHEDULE = dict(linear_start=0.0015, linear_end=0.0195)      # text2img256/config.yaml
STAGES = ("model.", "first_stage_model.", "cond_stage_model.")


def tiny_node(g):
    """The YAML's `model:` node with the tiny members in place of the three stages' parameters."""
    node = {**g["yaml_node"], "params": dict(g["yaml_node"]["params"])}
    p = node["params"]
    p["unet_config"] = {**p["unet_config"], "params": dict(arch.TINY_TEXT2IMG256_UNET)}
    p["first_stage_config"] = {**p["first_stage_config"],
                               "params": {**arch.TINY_VQ_F4, "lossconfig": {"target": "torch.nn.Identity"}}}
    p["cond_stage_config"] = {**p["cond_stage_config"], "params": dict(arch.TINY_BERT)}
    return node


def tiny_state_dict(g, ema_seed=None):
    """A text2img256-layout checkpoint of the tiny model (reference keys, to_logits included), with the EMA copy of the
    UNet under model_ema.* (LitEma names) when ema_seed is given."""
    ushapes = arch.unet_param_shapes(arch.TINY_TEXT2IMG256_UNET)
    sd = {"model.diffusion_model." + k: t for k, t in arch.random_state_dict(ushapes, g["unet_seed"]).items()}
    sd.update({"first_stage_model." + k: t for k, t in
               arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F4), g["vq_seed"]).items()})
    sd.update({"cond_stage_model." + k: t for k, t in
               arch.random_state_dict(arch.bert_param_shapes(arch.TINY_BERT), g["bert_seed"]).items()})
    if ema_seed is not None:
        sd.update({"model_ema." + ("diffusion_model." + k).replace(".", ""): t
                   for k, t in arch.random_state_dict(ushapes, ema_seed).items()})
        sd["model_ema.decay"] = torch.tensor(0.9999)
        sd["model_ema.num_updates"] = torch.tensor(1000, dtype=torch.int32)
    return sd


# ------------------------------------------------------------------------------------------------ oracle vs reference
def test_oracle_full_bert_matches_reference():
    g = golden("text2img256.pt")
    d = g["bert"]
    sd = arch.random_state_dict(arch.bert_param_shapes(arch.TEXT2IMG256_BERT), g["bert_seed"])
    assert d["ids"][-1].tolist() == [101, 102] + [0] * 75
    assert rel_l2(BO.bert_embed(sd, d["ids"]), d["z"]) < 5e-4          # the reference output is stored as fp16


@pytest.mark.parametrize("idx", range(2))
def test_oracle_full_unet_matches_reference(idx):
    g = golden("text2img256.pt")
    case = g["unet"][idx]
    sd = arch.random_state_dict(arch.unet_param_shapes(arch.TEXT2IMG256_UNET), g["unet_seed"])
    x = torch.randn((1, 3, 64, 64), generator=torch.Generator().manual_seed(case["x_seed"])).repeat(2, 1, 1, 1)
    ctx = torch.randn((2, 77, 640), generator=torch.Generator().manual_seed(case["ctx_seed"]))
    assert rel_l2(F8.unet_forward(sd, x, case["t"], ctx), case["eps"]) < 1e-5


@contextlib.contextmanager
def _text2img256_schedule():
    """ldm_oracle's PLMS reads SD-v1's schedule from register_schedule(); text2img256 has its own."""
    orig = O.register_schedule
    O.register_schedule = functools.partial(orig, **SCHEDULE)
    try:
        yield
    finally:
        O.register_schedule = orig


@pytest.mark.parametrize("name", ["ddim_eta0", "ddim_eta1", "plms", "dpm_solver"])
def test_oracle_tiny_guided_trajectory_matches_reference(name):
    g = golden("text2img256.pt")
    d = g["tiny"]
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_TEXT2IMG256_UNET), g["unet_seed"])
    bsd = arch.random_state_dict(arch.bert_param_shapes(arch.TINY_BERT), g["bert_seed"])
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F4), g["vq_seed"])
    c, uc = BO.bert_embed(bsd, d["ids"]), BO.bert_embed(bsd, d["uc_ids"])
    fn = lambda x, t, ctx: F8.unet_forward(usd, x, t, ctx)
    S, scale, x_T = g["steps"], g["scale"], d["x_T"]
    sched = O.register_schedule(**SCHEDULE)
    assert torch.equal(sched["alphas_cumprod"], g["alphas_cumprod"])
    if name.startswith("ddim"):
        eta = int(name[-1])
        noises = torch.stack([torch.randn(x_T.shape, generator=torch.Generator().manual_seed(d["noise_seed"] + i))
                              for i in range(S)]) if eta else torch.zeros(S, *x_T.shape)
        guided = lambda x, t: O._guided_eps(fn, x, t, c, uc, scale)
        s = U.ddim_sample_uncond(guided, x_T, sched["alphas_cumprod"], S, float(eta), noises)
    elif name == "plms":
        with _text2img256_schedule():
            s = O.plms_sample(fn, x_T, c, uc, scale, S=S)
    else:
        s = O.dpm_solver_sample(fn, x_T, c, uc, scale, S=S, sched=sched)
    r = d[name]
    assert rel_l2(s, r["sample"]) < 1e-4
    assert rel_l2(VO.decode_first_stage(vsd, r["sample"]), r["x_dec"]) < 1e-5


# ------------------------------------------------------------------------------------------------ architecture, config
def test_arch_tables_match_reference_keys():
    """Every parameter of the reference's text2img256 LatentDiffusion, by key and shape, to_logits included; the EMA
    copy of every UNet parameter under LitEma's names; the rest of its state_dict is the schedule buffers."""
    g = golden("text2img256.pt")
    ref = [(k, tuple(s)) for k, s in g["keys"]]
    ushapes = arch.unet_param_shapes(arch.TEXT2IMG256_UNET)
    mine = [("model.diffusion_model." + k, tuple(s)) for k, s in ushapes.items()]
    mine += [("first_stage_model." + k, tuple(s)) for k, s in arch.vq_param_shapes(arch.VQ_F4).items()]
    bert = [("cond_stage_model." + k, tuple(s)) for k, s in arch.bert_param_shapes(arch.TEXT2IMG256_BERT).items()]
    assert sorted(e for e in ref if e[0].startswith(STAGES)) == sorted(mine + bert)
    assert [e for e in ref if e[0].startswith("cond_stage_model.")] == bert
    ema = sorted(("model_ema." + ("diffusion_model." + k).replace(".", ""), tuple(s)) for k, s in ushapes.items())
    assert sorted(e for e in ref if e[0].startswith("model_ema.") and e[0] not in
                  ("model_ema.decay", "model_ema.num_updates")) == ema
    assert ("model.diffusion_model.input_blocks.4.1.transformer_blocks.0.attn2.to_k.weight", (384, 640)) in ref
    assert ("cond_stage_model.transformer.to_logits.weight", (30522, 640)) in ref
    assert all("." not in k for k, _ in ref if not k.startswith(STAGES + ("model_ema.",)))
    n = sum(torch.Size(s).numel() for s in ushapes.values())
    assert round(n / 1e6, 1) == 403.6


def test_unchanged_yaml_builds_the_engine_classes():
    import sdb200
    from sdb200.util import instantiate_from_config, remap_config
    g = golden("text2img256.pt")
    m = instantiate_from_config(remap_config(g["yaml_node"]))
    assert isinstance(m, sdb200.LatentDiffusion) and m.use_ema and m.scale_factor == 1.0
    assert isinstance(m.cond_stage_model, sdb200.BERTEmbedder) and m.cond_stage_model.cfg == arch.TEXT2IMG256_BERT
    assert isinstance(m.first_stage_model, sdb200.VQModelInterface) and m.first_stage_model.n_embed == 8192
    u = m.model.diffusion_model
    assert isinstance(u, sdb200.UNetModel) and u.in_channels == 3 and u.shapes == arch.unet_param_shapes(
        arch.TEXT2IMG256_UNET)
    heads = [(a["heads"], a["dhead"]) for layers in u.plan["input"] + [u.plan["middle"]] + u.plan["output"]
             for kind, _, a in (layers if isinstance(layers, list) else [layers]) if kind == "st"]
    assert sorted(set(heads)) == [(12, 32), (18, 32), (30, 32)]
    assert torch.equal(m.alphas_cumprod, g["alphas_cumprod"])


@pytest.mark.parametrize("fmt", ["ckpt", "safetensors"])
def test_checkpoint_with_ema_loads_from_the_unchanged_yaml(tmp_path, fmt):
    """The YAML's node (tiny stage parameters) and a checkpoint with the reference's keys and model_ema.*: nothing is
    missing or unexpected, the EMA copy becomes the UNet's "ema" weight set and ema_scope() switches to it."""
    import sdb200
    from sdb200 import checkpoint
    g = golden("text2img256.pt")
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": tiny_node(g)}))
    sd = tiny_state_dict(g, ema_seed=31)
    if fmt == "ckpt":
        ck = tmp_path / "model.ckpt"
        torch.save({"state_dict": sd, "global_step": 7}, ck)
    else:
        ck = tmp_path / "model.safetensors"
        checkpoint.write_safetensors(str(ck), sd)
    model = checkpoint.load_model_from_config(str(cfg), str(ck), device=None)
    info = model.load_info
    schedule = ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod")
    assert [k for k in info["missing"] if k not in schedule] == [] and info["unexpected"] == []
    assert isinstance(model.cond_stage_model, sdb200.BERTEmbedder) and isinstance(model.first_stage_model,
                                                                                   sdb200.VQModelInterface)
    u = model.model.diffusion_model
    assert model.use_ema and model.model_ema.loaded and u.has_weight_set("ema")
    k = "input_blocks.3.1.transformer_blocks.0.attn2.to_k.weight"
    assert torch.equal(u._alt_sd["ema"][k], sd["model_ema.diffusion_model" + k.replace(".", "")])
    assert torch.equal(u._host_sd[k], sd["model.diffusion_model." + k]) and not torch.equal(u._host_sd[k],
                                                                                             u._alt_sd["ema"][k])
    assert u._active == "raw"
    with model.ema_scope():
        assert u._active == "ema"
    assert u._active == "raw"
    # a checkpoint without the EMA copy also loads; ema_scope() then keeps the raw weights
    ck2 = tmp_path / "raw.safetensors"
    checkpoint.write_safetensors(str(ck2), tiny_state_dict(g))
    raw = checkpoint.load_model_from_config(str(cfg), str(ck2), device=None)
    assert not raw.model.diffusion_model.has_weight_set("ema")
    with raw.ema_scope():
        assert raw.model.diffusion_model._active == "raw"


# ------------------------------------------------------------------------------------------------ scripts/txt2img.py
def _models():
    from sdb200 import pipeline
    from sdb200.util import instantiate_from_config, remap_config
    g = golden("text2img256.pt")
    bert = instantiate_from_config(remap_config(tiny_node(g)))
    clip = pipeline.build_model(arch.TINY_UNET, arch.TINY_VAE, arch.TINY_CLIP)
    return bert, clip


def test_txt2img_tokenizer_and_stand_in_ids_follow_the_cond_stage_class():
    import sdb200
    mod = script("txt2img")
    bert, clip = _models()
    assert mod.text_encoder_kind(bert) == "bert" and mod.text_encoder_kind(clip) == "clip"
    ids, un = mod.stand_in_ids("bert", bert.cond_stage_model, 3, 1234, "cpu")
    assert (ids[:, 0] == 101).all() and (ids[:, 20] == 102).all() and (ids[:, 21:] == 0).all()
    assert ((ids[:, 1:20] >= 103) & (ids[:, 1:20] < arch.TINY_BERT["vocab_size"])).all()
    assert un.tolist() == [[101, 102] + [0] * 75] * 3
    assert torch.equal(bert.cond_stage_model.check_ids(ids), ids)
    # the full-size vocabulary keeps the LAION stand-ins exactly
    assert torch.equal(mod.synthetic_bert_ids(2, 7, "cpu", 30522), mod.synthetic_bert_ids(2, 7, "cpu"))
    ids, un = mod.stand_in_ids("clip", clip.cond_stage_model, 2, 1234, "cpu")
    assert torch.equal(ids, mod.synthetic_ids(2, 1234, "cpu"))
    assert un.tolist() == [[49406] + [49407] * 76] * 2
    cin = sdb200.LatentDiffusion(
        first_stage_config={"target": "sdb200.vq.VQModelInterface", "params": arch.TINY_VQ_F4},
        cond_stage_config={"target": "sdb200.encoders.ClassEmbedder", "params": arch.TINY_CIN_COND},
        unet_config={"target": "sdb200.unet.UNetModel", "params": arch.TINY_CIN_UNET}, conditioning_key="crossattn")
    with pytest.raises(SystemExit, match="ClassEmbedder is not a text encoder"):
        mod.text_encoder_kind(cin)


def test_txt2img_rejects_latent_shape_flags_that_do_not_match_the_model():
    mod = script("txt2img")
    bert, clip = _models()
    mod.check_latent_shape(bert, 3, 4)            # TINY_TEXT2IMG256_UNET in_channels 3, TINY_VQ_F4 three levels
    mod.check_latent_shape(clip, 4, 2)            # TINY_VAE: two levels
    for C, f in ((4, 8), (3, 8), (4, 4)):
        with pytest.raises(SystemExit, match="pass --C 3 --f 4"):
            mod.check_latent_shape(bert, C, f)
    with pytest.raises(SystemExit, match="pass --C 4 --f 2"):
        mod.check_latent_shape(clip, 4, 8)


def test_txt2img_random_init_builds_the_model_the_config_names(tmp_path, monkeypatch):
    """--random_init instantiates --config; the built-in SD-v1 / LAION models stay the fallback for the reference's two
    default paths when those files are absent."""
    import sdb200
    mod = script("txt2img")
    g = golden("text2img256.pt")
    monkeypatch.chdir(tmp_path)
    seen = []
    monkeypatch.setattr(mod.pipeline, "load_random_weights", lambda m, dev, gen_device=None: seen.append(m) or m)
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": g["yaml_node"]}))
    m = mod.load_model_from_config(str(cfg), None, "cpu", random_init=True)
    assert m is seen[-1] and isinstance(m.cond_stage_model, sdb200.BERTEmbedder)
    assert isinstance(m.first_stage_model, sdb200.VQModelInterface) and m.model.diffusion_model.in_channels == 3
    mod.check_latent_shape(m, 3, 4)
    built = []
    monkeypatch.setattr(mod.pipeline, "build_model", lambda: built.append("sd-v1") or m)
    monkeypatch.setattr(mod.pipeline, "build_laion_model", lambda: built.append("laion") or m)
    mod.load_model_from_config(mod.DEFAULT_CONFIG, None, "cpu", random_init=True)
    mod.load_model_from_config(mod.LAION_CONFIG, None, "cpu", random_init=True)
    assert built == ["sd-v1", "laion"]
    with pytest.raises(FileNotFoundError):
        mod.load_model_from_config("configs/other.yaml", None, "cpu", random_init=True)


def test_txt2img_defaults_unchanged(monkeypatch):
    """The default command is SD-v1 (CLIP, 4 latent channels, f 8), --laion400m switches as before, and both pass the
    latent-shape check with the default --C 4 --f 8."""
    mod = script("txt2img")
    import argparse
    opt = argparse.Namespace(laion400m=False, config=mod.DEFAULT_CONFIG, ckpt="x.ckpt", outdir="o")
    assert vars(mod.apply_laion400m(opt)) == dict(laion400m=False, config=mod.DEFAULT_CONFIG, ckpt="x.ckpt", outdir="o")
    from sdb200 import pipeline
    from sdb200.util import instantiate_from_config, remap_config
    for node in (pipeline.v1_model_config(arch.TINY_UNET, arch.SD_V1_VAE, arch.TINY_CLIP),
                 pipeline.laion_model_config(arch.TINY_LAION_UNET, arch.SD_V1_VAE, arch.TINY_BERT)):
        m = instantiate_from_config(remap_config(node))
        mod.check_latent_shape(m, 4, 8)
    assert mod.text_encoder_kind(m) == "bert"
