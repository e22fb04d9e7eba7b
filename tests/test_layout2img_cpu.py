"""The layout-to-image LDM (models/ldm/layout2img-openimages256) on the host: the oracles (bert_oracle,
layout2img_oracle's UNet whose spatial transformers run every block of the state dict, uncond_oracle's DDIM loop,
vq_oracle's decode) against the unmodified reference's outputs (tests/golden/layout2img.pt), the architecture tables
against the reference's key list of the whole model and the YAML, checkpoint ingest from the unchanged YAML with the EMA set, the transformer depths the
engine accepts, and the host logic of scripts/layout2img.py."""

import numpy as np
import pytest
import torch
import yaml

import helpers  # noqa: F401  (sys.path for the oracle)
import bert_oracle as BO
import cin_f8_oracle as F8
import layout2img_oracle as L
import ldm_oracle as O
import uncond_oracle as U
import vq_oracle as VO
from helpers import golden, rel_l2, script
from sdb200 import arch

STAGES = ("model.", "first_stage_model.", "cond_stage_model.")


def tiny_node(g):
    """The YAML's `model:` node with the tiny members in place of the three stages' parameters."""
    node = {**g["yaml_node"], "params": dict(g["yaml_node"]["params"])}
    p = node["params"]
    p["unet_config"] = {**p["unet_config"], "params": dict(arch.TINY_LAYOUT2IMG_UNET)}
    p["first_stage_config"] = {**p["first_stage_config"],
                               "params": {**arch.TINY_VQ_F4, "lossconfig": {"target": "torch.nn.Identity"}}}
    p["cond_stage_config"] = {**p["cond_stage_config"],
                              "params": {**arch.TINY_LAYOUT2IMG_BERT, "use_tokenizer": False}}
    return node


def tiny_state_dict(g, ema=True):
    """A layout2img-layout checkpoint of the tiny model (reference keys, to_logits included), with the EMA copy of the
    UNet under model_ema.* (LitEma names) from the golden's EMA seed."""
    ushapes = arch.unet_param_shapes(arch.TINY_LAYOUT2IMG_UNET)
    sd = {"model.diffusion_model." + k: t for k, t in arch.random_state_dict(ushapes, g["unet_seed"]).items()}
    sd.update({"first_stage_model." + k: t for k, t in
               arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F4), g["vq_seed"]).items()})
    sd.update({"cond_stage_model." + k: t for k, t in
               arch.random_state_dict(arch.bert_param_shapes(arch.TINY_LAYOUT2IMG_BERT), g["bert_seed"]).items()})
    if ema:
        sd.update({"model_ema." + ("diffusion_model." + k).replace(".", ""): t
                   for k, t in arch.random_state_dict(ushapes, g["ema_seed"]).items()})
        sd["model_ema.decay"] = torch.tensor(0.9999)
        sd["model_ema.num_updates"] = torch.tensor(1000, dtype=torch.int32)
    return sd


# ------------------------------------------------------------------------------------------------ oracle vs reference
def test_oracle_full_bert_matches_reference():
    g = golden("layout2img.pt")
    d = g["bert"]
    sd = arch.random_state_dict(arch.bert_param_shapes(arch.LAYOUT2IMG_BERT), g["bert_seed"])
    assert d["ids"].shape == (2, 92) and d["z"].shape == (2, 92, 512)
    assert rel_l2(BO.bert_embed(sd, d["ids"]), d["z"]) < 5e-4          # the reference output is stored as fp16


@pytest.mark.parametrize("idx", range(2))
def test_oracle_full_unet_matches_reference(idx):
    g = golden("layout2img.pt")
    case = g["unet"][idx]
    sd = arch.random_state_dict(arch.unet_param_shapes(arch.LAYOUT2IMG_UNET), g["unet_seed"])
    x = torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(case["x_seed"]))
    ctx = torch.randn((2, 92, 512), generator=torch.Generator().manual_seed(case["ctx_seed"]))
    assert rel_l2(L.unet_forward(sd, x, case["t"], ctx), case["eps"]) < 1e-5


@pytest.mark.parametrize("eta", [0, 1])
def test_oracle_tiny_unguided_ddim_matches_reference(eta):
    """log_images' sampling on the tiny model: unguided DDIM inside ema_scope(), so on the EMA weight set."""
    g = golden("layout2img.pt")
    d = g["tiny"]
    esd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_LAYOUT2IMG_UNET), g["ema_seed"])
    bsd = arch.random_state_dict(arch.bert_param_shapes(arch.TINY_LAYOUT2IMG_BERT), g["bert_seed"])
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F4), g["vq_seed"])
    c = BO.bert_embed(bsd, d["ids"])
    S, x_T = g["steps"], d["x_T"]
    sched = O.register_schedule(linear_start=0.0015, linear_end=0.0205)
    assert torch.equal(sched["alphas_cumprod"], g["alphas_cumprod"])
    noises = torch.stack([torch.randn(x_T.shape, generator=torch.Generator().manual_seed(d["noise_seed"] + i))
                          for i in range(S)]) if eta else torch.zeros(S, *x_T.shape)
    s = U.ddim_sample_uncond(lambda x, t: L.unet_forward(esd, x, t, c), x_T, sched["alphas_cumprod"], S, float(eta),
                             noises)
    r = d[f"ddim_eta{eta}"]
    assert rel_l2(s, r["sample"]) < 1e-4
    assert rel_l2(VO.decode_first_stage(vsd, r["sample"]), r["x_dec"]) < 1e-5


def test_oracle_spatial_transformer_runs_every_block():
    """With one block, layout2img_oracle's spatial transformer and UNet equal ldm_oracle's / cin_f8_oracle's to the bit; a
    second block is run and changes the output."""
    sd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_TEXT2IMG256_UNET), 11)
    pre = "input_blocks.3.1"
    x = torch.randn((1, 128, 8, 8), generator=torch.Generator().manual_seed(1))
    ctx = torch.randn((1, 5, 128), generator=torch.Generator().manual_seed(2))
    one = L.spatial_transformer(sd, pre, x, ctx, 4)
    assert torch.equal(one, O.spatial_transformer(sd, pre, x, ctx, 4))
    xs, t, c = torch.randn((2, 3, 16, 16), generator=torch.Generator().manual_seed(3)), torch.tensor([981, 1]), \
        torch.randn((2, 7, 128), generator=torch.Generator().manual_seed(4))
    assert torch.equal(L.unet_forward(sd, xs, t, c), F8.unet_forward(sd, xs, t, c))
    deep = dict(sd)
    deep.update({k.replace(".transformer_blocks.0.", ".transformer_blocks.1."): v.flip(0) if v.dim() == 2 else v
                 for k, v in sd.items() if k.startswith(pre + ".transformer_blocks.0.")})
    y = O._conv(O._gn(x, sd, pre + ".norm", 1e-6), sd, pre + ".proj_in", padding=0).permute(0, 2, 3, 1).reshape(1, 64, 128)
    for i in range(2):
        y = O.basic_transformer_block(deep, f"{pre}.transformer_blocks.{i}", y, ctx, 4)
    y = O._conv(y.reshape(1, 8, 8, 128).permute(0, 3, 1, 2), sd, pre + ".proj_out", padding=0) + x
    two = L.spatial_transformer(deep, pre, x, ctx, 4)
    assert torch.equal(two, y) and not torch.equal(two, one)


# ------------------------------------------------------------------------------------------------ architecture, config
def test_arch_tables_match_reference_keys_and_yaml():
    """Every parameter of the reference's layout2img LatentDiffusion, by key and shape, to_logits included; the EMA copy
    of every UNet parameter under LitEma's names; the rest of its state_dict is the schedule buffers. The arch tables
    equal the YAML's parameters."""
    g = golden("layout2img.pt")
    node = g["yaml_node"]["params"]
    assert node["unet_config"]["params"] == arch.LAYOUT2IMG_UNET
    assert node["cond_stage_config"]["params"] == {**arch.LAYOUT2IMG_BERT, "use_tokenizer": False}
    assert {k: v for k, v in node["first_stage_config"]["params"].items() if k not in ("lossconfig", "monitor")} == \
        arch.VQ_F4
    ref = [(k, tuple(s)) for k, s in g["keys"]]
    ushapes = arch.unet_param_shapes(arch.LAYOUT2IMG_UNET)
    unet = [("model.diffusion_model." + k, tuple(s)) for k, s in ushapes.items()]
    vq = [("first_stage_model." + k, tuple(s)) for k, s in arch.vq_param_shapes(arch.VQ_F4).items()]
    bert = [("cond_stage_model." + k, tuple(s)) for k, s in arch.bert_param_shapes(arch.LAYOUT2IMG_BERT).items()]
    assert sorted(e for e in ref if e[0].startswith(STAGES)) == sorted(unet + vq + bert)
    assert [e for e in ref if e[0].startswith("cond_stage_model.")] == bert
    ema = sorted(("model_ema." + ("diffusion_model." + k).replace(".", ""), tuple(s)) for k, s in ushapes.items())
    assert sorted(e for e in ref if e[0].startswith("model_ema.") and e[0] not in
                  ("model_ema.decay", "model_ema.num_updates")) == ema
    # three blocks per spatial transformer, between proj_in and proj_out, in the reference's order of modules
    pre = "model.diffusion_model.input_blocks.4.1"
    rest = [k[len(pre) + 1:].split(".") for k, _ in ref if k.startswith(pre + ".")]
    sub = [".".join(r[:2]) if r[0] == "transformer_blocks" else r[0] for r in rest]
    assert list(dict.fromkeys(sub)) == ["norm", "proj_in", "transformer_blocks.0", "transformer_blocks.1",
                                        "transformer_blocks.2", "proj_out"]
    assert ("model.diffusion_model.input_blocks.4.1.transformer_blocks.2.attn2.to_k.weight", (256, 512)) in ref
    assert ("cond_stage_model.transformer.pos_emb.emb.weight", (92, 512)) in ref
    assert ("cond_stage_model.transformer.to_logits.weight", (8192, 512)) in ref
    plan = arch.unet_plan(arch.LAYOUT2IMG_UNET)
    sts = [(a["ch"], a["heads"], a["dhead"], a["depth"])
           for grp in plan["input"] + [plan["middle"]] + plan["output"] for k, _, a in grp if k == "st"]
    assert len(sts) == 16 and sorted(set(sts)) == [(256, 8, 32, 3), (384, 12, 32, 3), (512, 16, 32, 3)]


def test_depth_one_tables_unchanged():
    """Depth 1 keeps the key list (and so the seeded weights) of every depth-1 model."""
    for cfg in (arch.TEXT2IMG256_UNET, arch.SD_V1_UNET, arch.CIN256_F8_UNET):
        keys = list(arch.unet_param_shapes(cfg))
        assert not [k for k in keys if ".transformer_blocks.1." in k]
        assert keys == list(arch.unet_param_shapes({**cfg, "transformer_depth": 1}))
    deep = arch.unet_param_shapes(arch.TINY_LAYOUT2IMG_UNET)
    one = arch.unet_param_shapes(arch.TINY_TEXT2IMG256_UNET)
    assert [k for k in deep if ".transformer_blocks." not in k or ".transformer_blocks.0." in k] == list(one)


def test_unchanged_yaml_and_built_in_node_build_the_engine_classes():
    import sdb200
    from sdb200.util import instantiate_from_config, remap_config
    g = golden("layout2img.pt")
    assert script("layout2img").layout2img_config() == g["yaml_node"]
    m = instantiate_from_config(remap_config(g["yaml_node"]))
    assert isinstance(m, sdb200.LatentDiffusion) and m.use_ema and m.scale_factor == 1.0
    assert m.cond_stage_key == "coordinates_bbox"
    assert isinstance(m.cond_stage_model, sdb200.BERTEmbedder) and m.cond_stage_model.cfg == arch.LAYOUT2IMG_BERT
    assert not m.cond_stage_model.use_tknz_fn
    assert isinstance(m.first_stage_model, sdb200.VQModelInterface) and m.first_stage_model.n_embed == 8192
    u = m.model.diffusion_model
    assert isinstance(u, sdb200.UNetModel) and u.cfg["transformer_depth"] == 3
    assert u.shapes == arch.unet_param_shapes(arch.LAYOUT2IMG_UNET)
    assert torch.equal(m.alphas_cumprod, g["alphas_cumprod"])


def test_transformer_depths():
    """Depths 1 and 3 (the published ones) are accepted, 2 and 4 raise; the ClassEmbedder's one-token context is folded
    for depth 1 only."""
    import sdb200
    for depth in (1, 3):
        net = sdb200.UNetModel(**{**arch.TINY_LAYOUT2IMG_UNET, "transformer_depth": depth})
        net._host_sd = arch.random_state_dict(net.shapes, 11)
        net.pack_weights(torch.device("cpu"))
        assert [len(s["blocks"]) for s in net.W["st_list"]] == [depth] * len(net.W["st_list"])
        assert [b["tb"] for b in net.W["st_list"][0]["blocks"]] == \
            [f"input_blocks.3.1.transformer_blocks.{i}" for i in range(depth)]
    for depth in (2, 4):
        with pytest.raises(NotImplementedError, match="transformer_depth"):
            sdb200.UNetModel(**{**arch.TINY_LAYOUT2IMG_UNET, "transformer_depth": depth})
        with pytest.raises(AssertionError):
            arch.unet_param_shapes({**arch.TINY_LAYOUT2IMG_UNET, "transformer_depth": depth})
    with pytest.raises(NotImplementedError, match="one-token context"):
        net.context_kv(torch.zeros(2, 1, 128))


@pytest.mark.parametrize("fmt", ["ckpt", "safetensors"])
def test_checkpoint_with_ema_loads_from_the_unchanged_yaml(tmp_path, fmt):
    """The YAML's node (tiny stage parameters) and a checkpoint with the reference's keys and model_ema.*: nothing is
    missing or unexpected, to_logits is dropped, the EMA copy becomes the UNet's "ema" weight set and ema_scope()
    switches to it."""
    import sdb200
    from sdb200 import checkpoint
    g = golden("layout2img.pt")
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": tiny_node(g)}))
    sd = tiny_state_dict(g)
    assert "cond_stage_model.transformer.to_logits.weight" in sd
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
    bert = model.cond_stage_model
    assert isinstance(bert, sdb200.BERTEmbedder) and bert.cfg == arch.TINY_LAYOUT2IMG_BERT
    assert not [k for k in bert._host_sd if k.startswith("transformer.to_logits.")]
    u = model.model.diffusion_model
    assert model.use_ema and model.model_ema.loaded and u.has_weight_set("ema")
    k = "input_blocks.3.1.transformer_blocks.2.attn2.to_k.weight"
    assert torch.equal(u._alt_sd["ema"][k], sd["model_ema.diffusion_model" + k.replace(".", "")])
    assert torch.equal(u._host_sd[k], sd["model.diffusion_model." + k]) and not torch.equal(u._host_sd[k],
                                                                                             u._alt_sd["ema"][k])
    with model.ema_scope():
        assert u._active == "ema"
    assert u._active == "raw"


# ------------------------------------------------------------------------------------------------ scripts/layout2img.py
def _bert():
    import sdb200
    return sdb200.BERTEmbedder(**arch.TINY_LAYOUT2IMG_BERT, use_tokenizer=False)


def test_token_files(tmp_path):
    """.pt and .npy ids of shape [92] (repeated --n_samples times) or [B, 92]; anything else is rejected."""
    mod = script("layout2img")
    bert = _bert()
    row = torch.arange(92) * 89 % 8192
    torch.save(row, tmp_path / "one.pt")
    np.save(tmp_path / "rows.npy", np.stack([row.numpy(), row.flip(0).numpy(), row.numpy()]).astype(np.int32))
    ids = mod.check_layout_ids(bert, mod.read_token_file(str(tmp_path / "one.pt"), 4))
    assert ids.shape == (4, 92) and ids.dtype == torch.int64 and (ids == row).all()
    ids = mod.check_layout_ids(bert, mod.read_token_file(str(tmp_path / "rows.npy"), 4))
    assert ids.shape == (3, 92) and torch.equal(ids[1], row.flip(0))
    with pytest.raises(ValueError, match=".pt or .npy"):
        mod.read_token_file(str(tmp_path / "ids.txt"), 1)
    torch.save({"ids": row}, tmp_path / "dict.pt")
    with pytest.raises(TypeError, match="expected a tensor"):
        mod.read_token_file(str(tmp_path / "dict.pt"), 1)


@pytest.mark.parametrize("bad,err,match", [
    (torch.full((2, 92), 8192), IndexError, r"\[0, 8192\)"),
    (torch.full((2, 92), -1), IndexError, r"\[0, 8192\)"),
    (torch.zeros(2, 93, dtype=torch.long), ValueError, "n <= 92"),
    (torch.zeros(2, 77, dtype=torch.long), ValueError, "exactly 92"),
    (torch.zeros(91, dtype=torch.long), ValueError, "exactly 92"),
    (torch.zeros(2, 92), TypeError, "integer"),
    (torch.zeros(1, 2, 92, dtype=torch.long), TypeError, "2-D"),
])
def test_token_files_out_of_range_or_wrong_length_are_rejected(tmp_path, bad, err, match):
    mod = script("layout2img")
    path = tmp_path / "bad.pt"
    torch.save(bad, path)
    with pytest.raises(err, match=match):
        mod.check_layout_ids(_bert(), mod.read_token_file(str(path), 2))


def test_random_init_stand_in_ids_and_arguments():
    mod = script("layout2img")
    bert = _bert()
    ids = mod.stand_in_ids(bert, 3, 42)
    assert ids.shape == (3, 92) and torch.equal(ids, mod.stand_in_ids(bert, 3, 42))
    assert not torch.equal(ids, mod.stand_in_ids(bert, 3, 43)) and int(ids.min()) >= 0 and int(ids.max()) < 8192
    assert torch.equal(mod.check_layout_ids(bert, ids), ids)
    opt = mod.get_parser().parse_args([])
    assert (opt.ddim_steps, opt.ddim_eta, opt.config) == (200, 1.0, mod.DEFAULT_CONFIG)
    assert not hasattr(opt, "scale")
    with pytest.raises(SystemExit):
        mod.get_parser().parse_args(["--scale", "5.0"])
    with pytest.raises(SystemExit, match="--tokens"):
        mod.main([])


def test_random_init_builds_the_model_the_config_names(tmp_path, monkeypatch):
    """--random_init instantiates --config, or the built-in node when the default path is absent; another missing path is
    an error."""
    import sdb200
    mod = script("layout2img")
    g = golden("layout2img.pt")
    monkeypatch.chdir(tmp_path)
    seen = []
    monkeypatch.setattr(mod.pipeline, "load_random_weights", lambda m, dev, gen_device=None: seen.append(m) or m)
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": tiny_node(g)}))
    m = mod.load_model(str(cfg), None, "cpu", random_init=True)
    assert m is seen[-1] and m.model.diffusion_model.cfg["model_channels"] == 64
    m = mod.load_model(mod.DEFAULT_CONFIG, None, "cpu", random_init=True)
    assert isinstance(m.cond_stage_model, sdb200.BERTEmbedder) and m.cond_stage_model.cfg == arch.LAYOUT2IMG_BERT
    assert m.model.diffusion_model.shapes == arch.unet_param_shapes(arch.LAYOUT2IMG_UNET)
    with pytest.raises(FileNotFoundError):
        mod.load_model("configs/other.yaml", None, "cpu", random_init=True)
    with pytest.raises(FileNotFoundError, match="checkpoint"):
        mod.load_model(str(cfg), str(tmp_path / "missing.ckpt"), "cpu")
