"""The LDM super-resolution model on the host: the split path's weight / normalization tables and the oracle
(oracle/superres_oracle.py) against the unmodified reference (tests/golden/superres.pt), the LR conversion, the size
rule of scripts/superres.py, and the bsr_sr architecture tables against the reference's state-dict keys."""
import hashlib

import pytest
import torch

import helpers  # noqa: F401  (sys.path for the oracle)
import superres_oracle as S
from helpers import golden, script
from sdb200 import arch
from sdb200.diffusion import split_geometry, split_tables


def _sha(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def _check(e, key, t):
    t = t.view(e[key + "_shape"])
    if key + "_sha256" in e:
        assert _sha(t) == e[key + "_sha256"], (e["tag"], key)
    else:
        assert torch.equal(t, e[key]), (e["tag"], key)


@pytest.mark.parametrize("idx", range(9))
def test_engine_and_oracle_tables_bit_exact(idx):
    e = golden("superres.pt")["tables"][idx]
    p, uf = e["params"], e["uf"]
    ks, stride, grid = split_geometry(e["h"], e["w"], p, uf)
    weight, norm = split_tables(ks, stride, grid, p, uf)
    L, kh, kw = weight.shape
    _check(e, "weighting", weight.view(L, kh * kw).t())        # the reference's [1, 1, kh, kw, L]
    _check(e, "norm", norm)
    _, _, o_norm, o_w = S.get_fold_unfold((1, 3, e["h"], e["w"]), p["ks"], p["stride"], p, uf=uf)
    _check(e, "weighting", o_w)
    _check(e, "norm", o_norm)


def test_oracle_split_apply_and_decode_bit_exact():
    g = golden("superres.pt")["e2e"]
    a, d = g["apply"], g["decode"]
    x = torch.randn((1, 3, 24, 40), generator=torch.Generator().manual_seed(a["x_seed"]))
    c = S.lr_image(_lr_png(24, 40, a["lr_seed"]))
    tiles = list(a["eps_tiles"])
    assert torch.equal(S.split_apply(lambda xt, t, ct: tiles.pop(0), x, a["t"], c, g["params"]), a["eps"])
    z = torch.randn((1, 3, 12, 20), generator=torch.Generator().manual_seed(d["z_seed"]))
    dt = list(d["dec_tiles"])
    assert torch.equal(S.split_decode(lambda zt: dt.pop(0), z, d["params"]), d["dec"])
    assert not tiles and not dt


def _lr_png(h, w, seed):
    import numpy as np
    img = np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    img.reshape(-1)[:256] = np.arange(256, dtype=np.uint8)
    return img


@pytest.mark.parametrize("idx", range(2))
def test_lr_conversion_bit_exact(idx):
    case = golden("superres.pt")["lr"][idx]
    assert torch.equal(S.lr_image(case["image"].numpy()), case["c"])
    assert set(case["image"].flatten().tolist()) == set(range(256))


@pytest.mark.parametrize("h, w, path", [
    (16, 24, "plain"), (24, 24, "plain"),            # both sides < 32: the reference's plain path too
    (256, 256, "split"), (192, 320, "split"), (128, 128, "split"),
    (64, 64, "plain"), (32, 96, "plain"), (120, 256, "plain"),    # a side in [32, 128): the reference crashes
    (200, 256, ValueError), (256, 130, ValueError),  # uncovered strips: NaN in the reference
    (60, 60, ValueError),                             # plain path needs multiples of 8
])
def test_size_rule(h, w, path):
    choose = script("superres").choose_path
    if path is ValueError:
        with pytest.raises(ValueError):
            choose(h, w)
    else:
        assert choose(h, w) == path


def test_split_geometry_rejects_what_the_reference_cannot_compute():
    p = S.notebook_params()
    with pytest.raises(ValueError, match="larger than"):
        split_geometry(64, 64, p, 1)                     # apply_model does not reduce ks
    assert split_geometry(64, 64, p, 4) == ((64, 64), (64, 64), (1, 1))     # decode does ("reducing Kernel")
    with pytest.raises(ValueError, match="not square"):
        split_geometry(64, 200, p, 4)                    # reduced ks (64, 128) at uf 4
    with pytest.raises(ValueError, match="cover"):
        split_geometry(200, 256, p, 1)
    with pytest.raises(ValueError, match="tie_braker"):
        split_geometry(128, 256, S.notebook_params(tie_braker=True), 1)     # a single row of tiles: 0 / 0
    assert split_geometry(24, 40, S.notebook_params(16, 8), 1) == ((16, 16), (8, 8), (2, 4))


def test_arch_tables_match_reference_keys():
    keys = [(k, tuple(s)) for k, s in golden("superres.pt")["ld_keys"]]
    sub = lambda pre: [(k[len(pre):], s) for k, s in keys if k.startswith(pre)]
    assert sub("model.diffusion_model.") == [(k, tuple(s)) for k, s in arch.unet_param_shapes(arch.BSR_SR_UNET).items()]
    assert sub("first_stage_model.") == [(k, tuple(s)) for k, s in arch.vq_param_shapes(arch.VQ_F4).items()]
    assert not sub("cond_stage_model.")                 # torch.nn.Identity has no state
    plan = arch.unet_plan(arch.BSR_SR_UNET)
    layers = [l for grp in plan["input"] + [plan["middle"]] + plan["output"] for l in grp]
    assert {(a["ch"], a["heads"], a["dhead"]) for k, _, a in layers if k == "attn"} == {(640, 20, 32)}
    assert {a["cin"] for k, _, a in layers if k == "res"} >= {160, 480, 960, 1280}


def test_config_instantiates_with_identity_cond_stage_and_loads():
    import sdb200
    from sdb200.util import instantiate_from_config, remap_config
    node = script("superres").superres_config(arch.TINY_BSR_UNET, arch.TINY_VQ_F4)
    model = instantiate_from_config(remap_config(node))
    assert isinstance(model, sdb200.LatentDiffusion) and isinstance(model.cond_stage_model, torch.nn.Identity)
    assert model.model.conditioning_key == "concat" and model.cond_stage_key == "LR_image"
    u = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_BSR_UNET), 11)
    v = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F4), 12)
    sd = {"model.diffusion_model." + k: t for k, t in u.items()}
    sd.update({"first_stage_model." + k: t for k, t in v.items()})
    sd.update({k: t for k, t in model.state_dict().items() if "." not in k})
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert missing == [] and unexpected == []
    c = torch.randn(1, 3, 8, 8)
    assert model.get_learned_conditioning(c) is c
