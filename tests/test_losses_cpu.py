"""The denoising objective's host side without a GPU: the lvlb_weights / logvar buffers against the reference's
(tests/golden/losses.pt, oracle/make_golden_losses.py), the loss fields of every published YAML, the rejected options
and get_input keys, and the evaluation ABI (include/sdb200_eval.h)."""
import os
import re

import pytest
import torch

from helpers import ROOT, golden
import sdb200
from sdb200 import arch
from sdb200.util import instantiate_from_config, remap_config

G = golden("losses.pt")
L1_YAMLS = {"configs/latent-diffusion/lsun_churches-ldm-kl-8.yaml", "models/ldm/lsun_churches256/config.yaml",
            "models/ldm/semantic_synthesis256/config.yaml", "models/ldm/semantic_synthesis512/config.yaml",
            "models/ldm/inpainting_big/config.yaml", "models/ldm/layout2img-openimages256/config.yaml"}


def _model(name, **override):
    node = G["members"][name]["node"]
    node = {**node, "params": {**node["params"], **override}}
    return instantiate_from_config(remap_config(node))


@pytest.mark.parametrize("name", sorted(G["members"]))
def test_loss_buffers_equal_the_reference(name):
    m = _model(name)
    ref = G["members"][name]
    assert torch.equal(m.lvlb_weights, ref["lvlb_weights"]) and torch.equal(m.logvar, ref["logvar"])
    assert m.lvlb_weights.dtype == m.logvar.dtype == torch.float32
    assert torch.equal(m.lvlb_weights[0], m.lvlb_weights[1])
    assert m.loss_type == ref["node"]["params"].get("loss_type", "l2")


def test_loss_buffers_stay_out_of_the_checkpoint_keys():
    m = _model("lsun")
    keys = set(m.state_dict())
    assert "lvlb_weights" not in keys and "logvar" not in keys
    bufs = dict(m.named_buffers())
    assert "lvlb_weights" in bufs and "logvar" in bufs


def test_logvar_init_fills_the_table():
    m = _model("sd", logvar_init=-0.5)
    assert torch.equal(m.logvar, torch.full((1000,), -0.5))


def test_published_yaml_loss_fields():
    params = G["published_params"]
    assert len(params) >= 20 and L1_YAMLS <= set(params)
    for path, p in params.items():
        m = _model("sd", **{k: v for k, v in p.items() if k not in ("image_size", "channels")})
        assert m.loss_type == ("l1" if path in L1_YAMLS else "l2"), path
        assert (m.l_simple_weight, m.original_elbo_weight, m.learn_logvar) == (1.0, 0.0, False), path
        assert torch.equal(m.logvar, torch.zeros(m.num_timesteps)), path
        assert bool(torch.isfinite(m.lvlb_weights).all()), path


def test_learn_logvar_and_unknown_loss_type_are_rejected():
    with pytest.raises(NotImplementedError, match="learn_logvar"):
        _model("sd", learn_logvar=True)
    with pytest.raises(NotImplementedError, match="unknown loss type"):
        _model("sd", loss_type="huber")


@pytest.mark.parametrize("key", ["txt", "coordinates_bbox", "nix", "masked_image"])
def test_unsupported_get_input_keys(key):
    m = _model("bsr", cond_stage_key=key)
    batch = {"image": torch.zeros(1, 64, 64, 3), key: torch.zeros(1, 16, 16, 3)}
    with pytest.raises(NotImplementedError, match="inpaint" if key == "masked_image" else "get_input"):
        m.get_input(batch, "image", cond_key=key)


def test_get_loss_elementwise_is_not_materialized():
    with pytest.raises(NotImplementedError, match="sdb_diffusion_loss"):
        _model("sd").get_loss(torch.zeros(1, 4, 2, 2), torch.zeros(1, 4, 2, 2), mean=False)


def _eval_header_symbols():
    text = open(os.path.join(ROOT, "include", "sdb200_eval.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sdb_[a-z0-9_]+)\s*\(", text)))


def test_eval_abi_symbols_present():
    syms = _eval_header_symbols()
    assert syms == sorted(sdb200.lib.EVAL_SIGNATURES) == ["sdb_diffusion_loss", "sdb_q_sample_t"]
    assert not set(syms) & set(sdb200.lib.SIGNATURES)
    lib = sdb200.lib.load()
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/sdb200_eval.h but not exported"
        assert getattr(lib, s).argtypes == sdb200.lib.EVAL_SIGNATURES[s][0]


def test_eval_entry_points_are_tested_on_the_gpu():
    """Each evaluation entry point is called through ops in the GPU test file that checks it elementwise."""
    src = open(os.path.join(ROOT, "tests", "test_losses_gpu.py")).read()
    for s in _eval_header_symbols():
        assert re.search(r"\bops\.%s\(" % s[4:], src), s


def test_eval_entry_points_record_into_plans():
    src = open(os.path.join(ROOT, "stable-diffusion_b200", "csrc", "losses.cu")).read()
    for s in _eval_header_symbols():
        assert re.search(r"SDB_REC\(%s\(" % s, src), s


def test_tiny_member_shapes_are_consistent():
    for name, m in G["members"].items():
        n = m["x_start"].shape
        assert m["noise"].shape == n == m["x_noisy"].shape == m["model_output"].shape, name
        assert m["t"].tolist() == [0, 999, 381, 640]
        assert set(m["loss_dict"]) == {"val/loss_simple", "val/loss_vlb", "val/loss"}
    assert arch.TINY_UNET["context_dim"] == G["members"]["sd"]["cond"].shape[-1]
