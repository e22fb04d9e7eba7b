"""The first-stage autoencoders of models/first_stage_models/* on the host: all nine YAMLs (stored in
tests/golden/first_stage.pt by oracle/make_golden_first_stage.py) through the config plumbing and the checkpoint loader,
the architecture tables against the reference's key lists, the oracle against the reference's outputs for the four
geometries no LDM uses, VQModel.decode_code's argument checks, scripts/autoencode.py's argument and size checks, and the
loud failure of the engine without CUDA."""
import os

import numpy as np
import pytest
import torch
import yaml

import helpers  # noqa: F401  (sys.path for the oracle)
import cin_f8_oracle as F8
import rdm_oracle as RO
import vq_oracle as VO
from helpers import golden, rel_l2, script
import sdb200
from sdb200 import arch, checkpoint
from sdb200.util import TARGET_MAP, instantiate_from_config, remap_config

NAMES = sorted(arch.FIRST_STAGES)
NEW = ["kl-f4", "kl-f32", "vq-f8-n256", "vq-f16"]


def _g():
    return golden("first_stage.pt")


def _shapes(cfg):
    return arch.vq_param_shapes(cfg) if "n_embed" in cfg else arch.vae_param_shapes(cfg)


def _write_yaml(tmp_path, name):
    path = tmp_path / f"{name}.yaml"
    path.write_text(yaml.safe_dump(_g()["yamls"][name]))
    return str(path)


def test_fixture_covers_nine_configs():
    g = _g()
    assert sorted(g["yamls"]) == sorted(g["keys"]) == NAMES and sorted(g["cases"]) == sorted(NEW)
    assert os.path.getsize(os.path.join(helpers.GOLDEN, "first_stage.pt")) < 2 << 20


@pytest.mark.parametrize("name", NAMES)
def test_yaml_instantiates_with_arch_params(name):
    """The unmodified YAML's model node (loss target and data node included) instantiates through TARGET_MAP with the
    arch table's parameters."""
    y = _g()["yamls"][name]
    assert "data" in y and "lossconfig" in y["model"]["params"]
    node = checkpoint.load_config(y)
    assert node["target"] in TARGET_MAP
    p = node["params"]
    cfg = arch.FIRST_STAGES[name]
    assert p["ddconfig"] == cfg["ddconfig"] and p["embed_dim"] == cfg["embed_dim"]
    assert p.get("n_embed") == cfg.get("n_embed")
    m = instantiate_from_config(remap_config(node))
    kind = sdb200.VQModel if name.startswith("vq") else sdb200.AutoencoderKL
    assert type(m) is kind and m.shapes == _shapes(cfg)


@pytest.mark.parametrize("name", NAMES)
def test_arch_tables_match_reference_keys(name):
    """Key, shape and registration order of the reference's AutoencoderKL / VQModel state dict."""
    ref = [(k, tuple(s)) for k, s in _g()["keys"][name]]
    assert [(k, tuple(s)) for k, s in _shapes(arch.FIRST_STAGES[name]).items()] == ref


def test_new_geometries_and_small_members():
    s = arch.vae_param_shapes(arch.KL_F32)
    assert s["quant_conv.weight"] == (128, 128, 1, 1) and s["post_quant_conv.weight"] == (64, 64, 1, 1)
    assert {k.split(".attn.")[0] for k in s if ".attn." in k} == {"encoder.down.4", "encoder.down.5", "decoder.up.4",
                                                                  "decoder.up.5"}
    assert arch.vq_param_shapes(arch.VQ_F16)["quantize.embedding.weight"] == (16384, 8)
    assert arch.vq_param_shapes(arch.VQ_F8_N256)["quantize.embedding.weight"] == (256, 4)
    assert arch.vae_param_shapes(arch.KL_F4)["quant_conv.weight"] == (6, 6, 1, 1)
    t = arch.vae_param_shapes(arch.TINY_KL_F32)
    assert t["quant_conv.weight"] == (128, 128, 1, 1) and len(arch.TINY_KL_F32["ddconfig"]["ch_mult"]) == 6
    assert {k.split(".attn.")[0] for k in t if ".attn." in k} == {"encoder.down.3", "encoder.down.4", "decoder.up.3",
                                                                  "decoder.up.4"}
    v = arch.vq_param_shapes(arch.TINY_VQ_F16)
    assert v["quantize.embedding.weight"] == (512, 8) and len(arch.TINY_VQ_F16["ddconfig"]["ch_mult"]) == 5
    assert {k.split(".attn.")[0] for k in v if ".attn." in k} == {"encoder.down.2", "decoder.up.2"}
    assert arch.vae_param_shapes(arch.TINY_KL_F4)["quant_conv.weight"] == (6, 6, 1, 1)


@pytest.mark.parametrize("name", ["kl-f32", "vq-f16"])
def test_load_model_from_config_unchanged_yaml(tmp_path, name):
    """load_model_from_config on the YAML file as published and a checkpoint carrying the training loss's tensors: the
    loss target and the data node are ignored, `loss.*` keys are dropped, every weight is adopted."""
    cfg = arch.FIRST_STAGES[name]
    sd = arch.random_state_dict(_shapes(cfg), 3)
    sd["loss.logvar"] = torch.zeros(())
    sd["loss.discriminator.main.0.weight"] = torch.zeros(64, 3, 4, 4)
    ckpt = tmp_path / "model.safetensors"
    checkpoint.write_safetensors(str(ckpt), sd)
    m = checkpoint.load_model_from_config(_write_yaml(tmp_path, name), str(ckpt), device=None)
    assert m.load_info["missing"] == [] and m.load_info["unexpected"] == []
    k = "quantize.embedding.weight" if name == "vq-f16" else "quant_conv.weight"
    assert torch.equal(m._host_sd[k], sd[k])


@pytest.mark.parametrize("name", NEW)
def test_oracle_matches_reference(name):
    g = _g()
    case = g["cases"][name]
    cfg = arch.FIRST_STAGES[name]
    sd = arch.random_state_dict(_shapes(cfg), g["weight_seed"])
    x = torch.randn(case["shape"], generator=torch.Generator().manual_seed(case["seed"])).clamp(-1, 1)
    if name.startswith("kl"):
        assert rel_l2(RO.kl_encode_moments(sd, x), case["moments"]) < 1e-5
        zc = cfg["embed_dim"]
        assert rel_l2(RO.kl_decode(sd, case["moments"][:, :zc]), case["dec"]) < 1e-5
        return
    k = g["image_stride"]
    assert rel_l2(F8.vq_encode(sd, x), case["h"]) < 1e-5
    e = sd["quantize.embedding.weight"]
    z_q, idx = VO.quantize(case["h"], e)
    assert torch.equal(idx, case["indices"])
    loss = 1.25 * torch.mean((e[idx] - case["h"].permute(0, 2, 3, 1).reshape(-1, e.shape[1])) ** 2)
    assert abs(float(loss) / float(case["emb_loss"]) - 1) < 1e-5
    assert rel_l2(F8.vq_decode(sd, case["h"])[..., ::k, ::k], case["dec"]) < 1e-5
    d = case["d_top2"]
    assert d.shape == (idx.numel(), 2) and bool((d[:, 1] >= d[:, 0]).all())


def test_decode_code_rejects_bad_codes():
    """Shape and dtype checks, then the index range, all before the device is needed."""
    m = sdb200.VQModel(**arch.TINY_VQ_F16)
    for bad in (torch.zeros(2, 4, dtype=torch.int64), torch.zeros(1, 2, 2, 1, dtype=torch.int64),
                torch.zeros(1, 2, 2, dtype=torch.int32), np.zeros((1, 2, 2), np.int64)):
        with pytest.raises(ValueError):
            m.decode_code(bad)
    for v in (-1, 512):
        code = torch.zeros(1, 2, 2, dtype=torch.int64)
        code[0, 1, 0] = v
        with pytest.raises(IndexError):
            m.decode_code(code)
    with pytest.raises(ValueError):
        m.get_codebook_entry(torch.zeros(4, dtype=torch.int64), (1, 2, 2, 4))     # e_dim 8
    with pytest.raises(AssertionError, match="CUDA only"):
        m.decode_code(torch.full((1, 2, 2), 511, dtype=torch.int64))


def test_vq_model_constructor_matches_interface():
    for cls in (sdb200.VQModel, sdb200.VQModelInterface):
        for kw in ({"remap": "x.npy"}, {"sane_index_shape": True}, {"use_ema": True}):
            with pytest.raises(NotImplementedError):
                cls(**arch.TINY_VQ_F16, **kw)
    assert issubclass(sdb200.VQModelInterface, sdb200.VQModel)
    assert TARGET_MAP["ldm.models.autoencoder.VQModel"] == "sdb200.vq.VQModel"


@pytest.mark.parametrize("cfg", ["TINY_VQ_F16", "TINY_KL_F32", "TINY_KL_F4"])
def test_fails_loudly_without_cuda(cfg):
    c = getattr(arch, cfg)
    m = sdb200.VQModel(**c) if "n_embed" in c else sdb200.AutoencoderKL(**c)
    m._host_sd = arch.random_state_dict(m.shapes, 0)
    x = torch.zeros(1, 3, 128, 128)
    calls = [lambda: m.encode(x), lambda: m.forward(x)] + (
        [lambda: m.encode_to_prequant(x), lambda: m.decode(torch.zeros(1, 8, 8, 8)),
         lambda: m.quantize(torch.zeros(1, 8, 8, 8))] if "n_embed" in c else
        [lambda: m.decode(torch.zeros(1, c["embed_dim"], 4, 4)), lambda: m.forward(x, sample_posterior=False)])
    for call in calls:
        with pytest.raises(AssertionError, match="CUDA only"):
            call()


def test_autoencode_arguments(tmp_path):
    S = script("autoencode")
    p = S.get_parser()
    cfg = _write_yaml(tmp_path, "kl-f32")
    with pytest.raises(ValueError, match="--ckpt, or --random_init"):
        S.check_args(p.parse_args(["--config", cfg]))
    with pytest.raises(ValueError, match="--ckpt, or --random_init"):
        S.check_args(p.parse_args(["--config", cfg, "--random_init", "--ckpt", "m.ckpt"]))
    with pytest.raises(SystemExit):
        p.parse_args(["--random_init"])                       # --config is required
    for hw in (["--H", "240"], ["--W", "100"]):               # KL-f32 downsamples by 32
        with pytest.raises(ValueError, match="downsampling factor 32"):
            S.check_args(p.parse_args(["--config", cfg, "--random_init", *hw]))
    with pytest.raises(ValueError, match="n_samples"):
        S.check_args(p.parse_args(["--config", cfg, "--random_init", "--n_samples", "0"]))
    node, inputs = S.check_args(p.parse_args(["--config", cfg, "--random_init", "--n_samples", "3", "--H", "64",
                                              "--W", "96", "--seed", "5"]))
    assert node["target"] == "ldm.models.autoencoder.AutoencoderKL" and S.downsampling_factor(node) == 32
    (name, u8), = inputs
    assert name == "synthetic" and u8.shape == (3, 64, 96, 3) and u8.dtype == torch.uint8
    assert torch.equal(u8, S.check_args(p.parse_args(["--config", cfg, "--random_init", "--n_samples", "3", "--H", "64",
                                                      "--W", "96", "--seed", "5"]))[1][0][1])


def test_autoencode_image_inputs(tmp_path):
    from PIL import Image
    S = script("autoencode")
    p = S.get_parser()
    cfg = _write_yaml(tmp_path, "vq-f8-n256")
    d = tmp_path / "imgs"
    d.mkdir()
    with pytest.raises(ValueError, match="no .png"):
        S.check_args(p.parse_args(["--config", cfg, "--random_init", "--indir", str(d)]))
    img = np.random.default_rng(0).integers(0, 256, (24, 40, 3), dtype=np.uint8)
    Image.fromarray(img).save(d / "a.png")
    (d / "notes.txt").write_text("not an image")
    _, inputs = S.check_args(p.parse_args(["--config", cfg, "--random_init", "--indir", str(d)]))
    assert [n for n, _ in inputs] == ["a"] and torch.equal(inputs[0][1][0], torch.from_numpy(img))
    x = S.preprocess(inputs[0][1])
    assert x.shape == (1, 3, 24, 40) and float(x.min()) >= -1 and float(x.max()) <= 1
    assert torch.equal(x[0, :, 3, 5], torch.from_numpy(img[3, 5]).float() / 127.5 - 1)
    assert np.array_equal(S.to_uint8(torch.tensor([[[[-2.0, -1.0, 0.0, 1.0, 3.0]]]]).expand(1, 3, 1, 5))[0, 0, :, 0],
                          [0, 0, 127, 255, 255])
    Image.fromarray(img[:20]).save(d / "b.jpg")
    with pytest.raises(ValueError, match="b.jpg: 20x40 is not a multiple"):
        S.check_args(p.parse_args(["--config", cfg, "--random_init", "--indir", str(d)]))
