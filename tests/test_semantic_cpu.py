"""The LDM semantic-synthesis models on the host: the cond-stage oracle (oracle/semantic_oracle.py) and the UNet oracle
against the unmodified reference (tests/golden/semantic.pt), both reference configs through TARGET_MAP, the
architecture tables against the reference's state-dict keys, the schedule, checkpoint ingest, and the host-side checks
of SpatialRescaler and scripts/semantic_synthesis.py (id validation, size rule, PNG modes, unsupported options)."""

import numpy as np
import pytest
import torch

import helpers  # noqa: F401  (sys.path for the oracle)
import semantic_oracle as SO
import uncond_oracle as U
from helpers import golden, rel_l2, script
from sdb200 import arch, checkpoint
from sdb200.util import instantiate_from_config, remap_config

# the `model:` nodes of models/ldm/semantic_synthesis256/config.yaml and semantic_synthesis512/config.yaml, as written
_VQ_PARAMS = {"embed_dim": 3, "n_embed": 8192, "ddconfig": {
    "double_z": False, "z_channels": 3, "resolution": 256, "in_channels": 3, "out_ch": 3, "ch": 128,
    "ch_mult": [1, 2, 4], "num_res_blocks": 2, "attn_resolutions": [], "dropout": 0.0},
    "lossconfig": {"target": "torch.nn.Identity"}}


def _yaml_model(image_size, monitor):
    vq = dict(_VQ_PARAMS)
    if monitor:
        vq = {"embed_dim": 3, "n_embed": 8192, "monitor": "val/rec_loss", "ddconfig": _VQ_PARAMS["ddconfig"],
              "lossconfig": _VQ_PARAMS["lossconfig"]}
    return {"base_learning_rate": 1.0e-06, "target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        "linear_start": 0.0015, "linear_end": 0.0205, "log_every_t": 100, "timesteps": 1000, "loss_type": "l1",
        "first_stage_key": "image", "cond_stage_key": "segmentation", "image_size": image_size, "channels": 3,
        "concat_mode": True, "cond_stage_trainable": True,
        "unet_config": {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": {
            "image_size": image_size, "in_channels": 6, "out_channels": 3, "model_channels": 128,
            "attention_resolutions": [32, 16, 8], "num_res_blocks": 2, "channel_mult": [1, 4, 8], "num_heads": 8}},
        "first_stage_config": {"target": "ldm.models.autoencoder.VQModelInterface", "params": vq},
        "cond_stage_config": {"target": "ldm.modules.encoders.modules.SpatialRescaler",
                              "params": {"n_stages": 2, "in_channels": 182, "out_channels": 3}}}}


SS256 = _yaml_model(64, monitor=False)
SS512 = _yaml_model(128, monitor=True)


def _cond_cfg(name):
    return {"full": arch.SEMANTIC_SYNTHESIS_COND, "tiny": arch.TINY_SEMANTIC_COND,
            "tiny_bias": golden("semantic.pt")["tiny_bias_cond"]}[name]


def case_input(e, n_classes):
    """The golden case's input, regenerated from its seed: (labels uint8 [1, h, w] or None, float map or None)."""
    if e["kind"] == "soft":
        return None, SO.soft_map((1, n_classes, e["h"], e["w"]), e["seed"])
    f = SO.voronoi_labels if e["kind"] == "voronoi" else SO.all_ids_labels
    return torch.from_numpy(f(e["h"], e["w"], n_classes, e["seed"]))[None], None


@pytest.mark.parametrize("idx", range(7))
def test_oracle_cond_bit_exact(idx):
    g = golden("semantic.pt")
    e = g["cond"][idx]
    cfg = _cond_cfg(e["cfg"])
    sd = arch.random_state_dict(arch.spatial_rescaler_param_shapes(cfg), g["cond_seed"])
    labels, soft = case_input(e, cfg["in_channels"])
    out = SO.cond_from_labels(labels, sd, cfg) if soft is None else SO.spatial_rescale(
        soft, cfg["n_stages"], sd["channel_mapper.weight"], sd.get("channel_mapper.bias"))
    assert torch.equal(out, e["c"]), e["tag"]
    if e["tag"] == "all_ids":
        assert set(labels.flatten().tolist()) == set(range(182))
    if e["tag"] == "voronoi30x46":
        assert tuple(out.shape) == (1, 3, 7, 11)


def test_oracle_unet_matches_reference():
    g = golden("semantic.pt")
    case = g["unet"][0]
    assert case["cfg"] == "tiny"
    sd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_SEMANTIC_UNET), g["unet_seed"])
    x = torch.randn(case["shape"], generator=torch.Generator().manual_seed(case["x_seed"]))
    eps = U.unet_forward(sd, arch.TINY_SEMANTIC_UNET, x, case["t"])
    assert rel_l2(eps, case["eps"]) < 1e-5


@pytest.mark.parametrize("node", [SS256, SS512], ids=["ss256", "ss512"])
def test_reference_configs_resolve_to_engine_classes(node):
    import sdb200
    model = instantiate_from_config(remap_config(node))
    assert isinstance(model, sdb200.LatentDiffusion) and model.model.conditioning_key == "concat"
    assert isinstance(model.model.diffusion_model, sdb200.UNetModel)
    assert isinstance(model.first_stage_model, sdb200.VQModelInterface)
    assert isinstance(model.cond_stage_model, sdb200.SpatialRescaler)
    assert model.cond_stage_key == "segmentation"
    # the schedule (linear_end 0.0205) equals the reference's buffers
    assert torch.equal(model.alphas_cumprod, golden("semantic.pt")["alphas_cumprod"])
    assert model.linear_end == 0.0205


def test_both_configs_share_param_shapes_and_match_reference_keys():
    keys = [(k, tuple(s)) for k, s in golden("semantic.pt")["ld_keys"]]
    sub = lambda pre: [(k[len(pre):], s) for k, s in keys if k.startswith(pre)]
    for node in (SS256, SS512):
        p = node["params"]
        u = {k: v for k, v in p["unet_config"]["params"].items() if k != "image_size"}
        assert u == {k: v for k, v in arch.SEMANTIC_SYNTHESIS_UNET.items() if k != "image_size"}
        assert p["cond_stage_config"]["params"] == arch.SEMANTIC_SYNTHESIS_COND
    assert sub("model.diffusion_model.") == [(k, tuple(s)) for k, s in
                                             arch.unet_param_shapes(arch.SEMANTIC_SYNTHESIS_UNET).items()]
    assert sub("first_stage_model.") == [(k, tuple(s)) for k, s in arch.vq_param_shapes(arch.VQ_F4).items()]
    assert sub("cond_stage_model.") == [("channel_mapper.weight", (3, 182, 1, 1))]
    assert sub("cond_stage_model.") == [(k, tuple(s)) for k, s in
                                        arch.spatial_rescaler_param_shapes(arch.SEMANTIC_SYNTHESIS_COND).items()]
    assert len(sub("model_ema.")) == len(sub("model.diffusion_model.")) + 2       # + decay, num_updates
    plan = arch.unet_plan(arch.SEMANTIC_SYNTHESIS_UNET)
    layers = [l for grp in plan["input"] + [plan["middle"]] + plan["output"] for l in grp]
    assert [(a["ch"], a["heads"], a["dhead"]) for k, _, a in layers if k == "attn"] == [(1024, 8, 128)]
    assert max(a["cin"] for k, _, a in layers if k == "res") == 2048


def _ckpt_sd(dtype=torch.float32):
    """A checkpoint with exactly the reference model's keys and shapes: stand-in weight values (the loader checks
    names and shapes), seeded channel-mapper weights, EMA copies, and the schedule buffers as the config computes
    them."""
    sched = instantiate_from_config(remap_config(SS256)).state_dict()
    mapper = arch.random_state_dict(arch.spatial_rescaler_param_shapes(arch.SEMANTIC_SYNTHESIS_COND), 13)
    sd = {}
    for k, shape in golden("semantic.pt")["ld_keys"]:
        if k.startswith("cond_stage_model."):
            t = mapper[k[len("cond_stage_model."):]]
        elif k == "model_ema.num_updates":
            t = torch.tensor(1000, dtype=torch.int32)
        elif k == "model_ema.decay":
            t = torch.tensor(0.9999)
        elif k.startswith(("model.", "first_stage_model.")):
            t = torch.full(shape, 0.5)
        elif k.startswith("model_ema."):
            t = torch.full(shape, 0.25)
        else:                                             # schedule buffers
            t = sched.get(k, torch.zeros(shape))
        assert tuple(t.shape) == tuple(shape), k
        sd[k] = t.to(dtype) if t.is_floating_point() else t
    return sd


@pytest.mark.parametrize("fmt", ["ckpt", "safetensors"])
def test_load_model_from_config_with_reference_key_set(tmp_path, fmt):
    import sdb200
    sd = _ckpt_sd(torch.float16 if fmt == "safetensors" else torch.float32)
    assert len(sd) == len(golden("semantic.pt")["ld_keys"])
    path = str(tmp_path / f"model.{fmt}")
    if fmt == "ckpt":
        torch.save({"state_dict": sd, "global_step": 1}, path)
    else:
        checkpoint.write_safetensors(path, sd)
    model = checkpoint.load_model_from_config({"model": SS256}, path, device=None)
    c = model.cond_stage_model
    assert isinstance(c, sdb200.SpatialRescaler)
    assert torch.equal(c._host_sd["channel_mapper.weight"], sd["cond_stage_model.channel_mapper.weight"])
    assert model.model.diffusion_model.has_weight_set("ema") and model.model_ema.loaded
    assert model.load_info["missing"] == []
    # left over: only schedule buffers the engine recomputes from the config; every weight and EMA copy is used
    unexpected = set(model.load_info["unexpected"])
    assert "log_one_minus_alphas_cumprod" in unexpected
    assert not [k for k in unexpected if k.startswith(("model.", "first_stage_model.", "cond_stage_model.", "model_ema."))]


def test_missing_or_misshaped_mapper_fails(tmp_path):
    sd = _ckpt_sd()
    path = str(tmp_path / "bad.ckpt")
    miss = dict(sd)
    del miss["cond_stage_model.channel_mapper.weight"]
    torch.save({"state_dict": miss}, path)
    with pytest.raises(RuntimeError, match="lacks 1 tensors"):
        checkpoint.load_model_from_config({"model": SS256}, path, device=None)
    shp = dict(sd)
    shp["cond_stage_model.channel_mapper.weight"] = torch.zeros(3, 181, 1, 1)
    torch.save({"state_dict": shp}, path)
    with pytest.raises(RuntimeError, match="size mismatch for cond_stage_model.channel_mapper.weight"):
        checkpoint.load_model_from_config({"model": SS256}, path, device=None)


def test_rescaler_state_dict_keys_and_options():
    import sdb200
    m = sdb200.SpatialRescaler(n_stages=1, in_channels=20, out_channels=3, bias=True)
    assert list(m.shapes) == ["channel_mapper.weight", "channel_mapper.bias"]
    assert sdb200.SpatialRescaler().shapes == {}                    # out_channels None: no channel mapper
    assert m.cpu() is m and m.to(torch.float32) is m and m.W is None     # host moves pack nothing
    for kw in ({"method": "nearest"}, {"method": "bicubic"}, {"multiplier": 0.25}, {"multiplier": 2},
               {"n_stages": 4}):
        with pytest.raises(NotImplementedError):
            sdb200.SpatialRescaler(**kw)
    with pytest.raises(AssertionError):
        sdb200.SpatialRescaler(n_stages=-1)


def test_rescaler_label_ids_checked_on_host():
    import sdb200
    m = sdb200.SpatialRescaler(n_stages=2, in_channels=182, out_channels=3)
    ok = torch.zeros(1, 8, 8, dtype=torch.uint8)
    ok[0, 0, 0] = 181
    assert m.check_labels(ok).dtype == torch.uint8
    for bad in (182, 255, -1):
        lab = torch.zeros(1, 8, 8, dtype=torch.int64)
        lab[0, 3, 5] = bad
        with pytest.raises(IndexError):
            m.check_labels(lab)
    with pytest.raises(TypeError):
        m.check_labels(torch.zeros(8, 8, dtype=torch.int64))           # [B, H, W]
    with pytest.raises(TypeError):
        m.check_labels(torch.zeros(1, 8, 8, dtype=torch.bool))
    # the one-hot / np.eye the reference builds fails the same way
    with pytest.raises(IndexError):
        np.eye(182)[np.array([[182]])]
    # label input needs a channel mapper (and, uint8 ids, at most 256 classes)
    m.W = {"device": torch.device("cpu"), "weight": None, "bias": None}
    with pytest.raises(NotImplementedError):
        sdb200.SpatialRescaler(n_stages=2, in_channels=182).load_weights({}, "cpu")(ok)
    big = sdb200.SpatialRescaler(n_stages=2, in_channels=300, out_channels=3)
    big.W = {"device": torch.device("cpu"), "weight": None, "bias": None}
    with pytest.raises(NotImplementedError):
        big(ok)


@pytest.mark.parametrize("h, w, ok", [(256, 256, True), (256, 512, True), (512, 1024, True), (64, 48, True),
                                      (16, 16, True), (1024, 2048, True),
                                      (250, 256, False), (256, 8, False), (24, 32, False), (0, 16, False)])
def test_size_rule(h, w, ok):
    check = script("semantic_synthesis").check_size
    if ok:
        check(h, w)
    else:
        with pytest.raises(ValueError, match="multiples of 16"):
            check(h, w)


def test_label_png_modes(tmp_path):
    from PIL import Image
    S = script("semantic_synthesis")
    lab = SO.voronoi_labels(32, 48, 182, 5)
    Image.fromarray(lab, mode="L").save(tmp_path / "l.png")
    assert np.array_equal(S.read_label_map(str(tmp_path / "l.png")), lab)
    p = Image.fromarray(lab, mode="L").convert("P")
    p.putdata(lab.reshape(-1).tolist())
    p.putpalette([i % 256 for i in range(768)])
    p.save(tmp_path / "p.png")
    assert Image.open(tmp_path / "p.png").mode == "P"
    assert np.array_equal(S.read_label_map(str(tmp_path / "p.png")), lab)
    Image.fromarray(np.stack([lab] * 3, -1)).save(tmp_path / "rgb.png")
    with pytest.raises(ValueError, match="mode L or P"):
        S.read_label_map(str(tmp_path / "rgb.png"))
    high = lab.copy()
    high[0, 0] = 200
    Image.fromarray(high, mode="L").save(tmp_path / "high.png")
    with pytest.raises(ValueError, match="out of range"):
        S.read_label_map(str(tmp_path / "high.png"))
    assert S.read_label_map(str(tmp_path / "high.png"), n_classes=256)[0, 0] == 200


def test_script_config_matches_reference_nodes():
    S = script("semantic_synthesis")
    for node, size in ((SS256, None), (SS512, 128)):
        assert S.semantic_config(image_size=size) == {k: v for k, v in node.items() if k != "base_learning_rate"}
    with pytest.raises(ValueError):
        S.main(["x.png"])                                        # no --ckpt / --random_init
    with pytest.raises(ValueError):
        S.main(["--random_init"])                                # no label map
