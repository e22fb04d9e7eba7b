"""FrozenClipImageEmbedder and scripts/build_rdm_database.py on the host: the arch tables against the key list of
transformers' CLIPVisionModelWithProjection (tests/golden/clip_image.pt), a numpy restatement of the bicubic resize the
preprocessing kernel implements against F.interpolate, the database builder's manifest / shard / --resume logic, and the
constructor's errors."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import golden, script
from sdb200 import arch

A = -0.75


# ------------------------------------------------------------------------------------------------ arch tables
@pytest.mark.parametrize("tag,cfg", [("tiny", arch.TINY_CLIP_VISION_PROJ), ("vitl14", arch.CLIP_VISION_PROJ)])
def test_arch_tables_match_transformers_keys(tag, cfg):
    ref = [(k, tuple(s)) for k, s in golden("clip_image.pt")[tag]["keys"]]
    mine = [(k, tuple(s)) for k, s in arch.clip_vision_proj_param_shapes(cfg).items()]
    assert sorted(mine) == sorted(ref)


def test_vit_l14_is_the_safety_checkers_tower():
    """The full-size table is CLIP ViT-L/14's vision tower, the one the safety checker runs."""
    for k in ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "image_size", "patch_size",
              "projection_dim", "layer_norm_eps"):
        assert arch.CLIP_VISION_PROJ[k] == arch.SD_V1_SAFETY[k], k
    assert arch.TINY_CLIP_VISION_PROJ["projection_dim"] == arch.TINY_RDM_UNET["context_dim"]


# ------------------------------------------------------------------------------------------------ bicubic
def _cubic1(x, dt):
    return ((dt(A) + dt(2)) * x - (dt(A) + dt(3))) * x * x + dt(1)


def _cubic2(x, dt):
    return ((dt(A) * x - dt(5) * dt(A)) * x + dt(8) * dt(A)) * x - dt(4) * dt(A)


def _axis(n_in, n_out, dt):
    """(tap indices [n_out, 4], weights [n_out, 4]) of torch's align_corners bicubic along one axis, computed in dt as
    torch computes them for inputs of that type: scale = (in - 1) / (out - 1), source coordinate scale * dst, t its
    fraction, A = -0.75, taps clamped to the border."""
    one = dt(1)
    scale = dt(n_in - 1) / dt(n_out - 1) if n_out > 1 else dt(0)
    real = scale * np.arange(n_out, dtype=dt)
    i0 = np.floor(real).astype(np.int64)
    t = real - i0.astype(dt)
    w = np.stack([_cubic2(t + one, dt), _cubic1(t, dt), _cubic1(one - t, dt), _cubic2((one - t) + one, dt)], 1)
    idx = np.clip(i0[:, None] + np.arange(-1, 3)[None], 0, n_in - 1)
    return idx, w


def _interp(v, w):
    return ((v[..., 0] * w[..., 0] + v[..., 1] * w[..., 1]) + v[..., 2] * w[..., 2]) + v[..., 3] * w[..., 3]


def bicubic_np(x, size, dt=np.float32):
    """F.interpolate(x, (size, size), mode='bicubic', align_corners=True) of x [..., H, W] of numpy type dt: at each
    output pixel the four row interpolations at the source column, then the one down the column (the kernel's order);
    a copy when both sides already match."""
    H, W = x.shape[-2:]
    x = x.astype(dt)
    if (H, W) == (size, size):
        return x
    iy, wy = _axis(H, size, dt)
    ix, wx = _axis(W, size, dt)
    rows = _interp(x[..., :, ix], wx)                                         # [..., H, size]
    return _interp(np.moveaxis(rows[..., iy, :], -2, -1), wy[:, None, :])     # [..., size, size]


SIZES = [((64, 64), 224), ((512, 512), 224), ((1000, 333), 224), ((7, 513), 224), ((224, 224), 224), ((1, 300), 224),
         ((300, 1), 56), ((1, 1), 56), ((90, 70), 56)]


@pytest.mark.parametrize("hw,size", SIZES)
def test_bicubic_restatement_matches_interpolate(hw, size):
    """fp64 restatement vs F.interpolate on fp64 input: <= 1e-6 (it is ~1e-15). fp32: torch's CPU kernel rounds its
    own way (about 1e-6 from the exact value at these sizes), so the fp32 restatement, which follows the CUDA kernel's
    order, is held to the GPU kernel's 2e-6."""
    g = torch.Generator().manual_seed(hw[0] * 1000 + hw[1])
    x = torch.rand(2, 3, *hw, generator=g, dtype=torch.float64) * 2 - 1
    ref = F.interpolate(x, size=(size, size), mode="bicubic", align_corners=True).numpy()
    err64 = float(np.abs(bicubic_np(x.numpy(), size, np.float64) - ref).max())
    x32 = x.float()
    ref32 = F.interpolate(x32, size=(size, size), mode="bicubic", align_corners=True).numpy()
    err32 = float(np.abs(bicubic_np(x32.numpy(), size, np.float32) - ref32).max())
    assert err64 <= 1e-6 and err32 <= 2e-6, (err64, err32)


# ------------------------------------------------------------------------------------------------ builder host logic
def _tree(root, names):
    from PIL import Image
    for i, n in enumerate(names):
        p = os.path.join(root, n)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        Image.fromarray(np.full((4 + i, 5, 3), i, dtype=np.uint8)).save(p)


def test_manifest_lists_images_sorted_and_skips_other_files(tmp_path):
    mod = script("build_rdm_database")
    _tree(str(tmp_path), ["b/2.png", "a.jpg", "b/1.PNG", "c/d/e.webp"])
    (tmp_path / "notes.txt").write_text("x")
    assert mod.list_images(str(tmp_path)) == ["a.jpg", "b/1.PNG", "b/2.png", "c/d/e.webp"]
    out = tmp_path / "db"
    rows = mod.prepare_outdir(str(out), mod.list_images(str(tmp_path)), resume=False)
    assert (out / "manifest.txt").read_text().splitlines() == rows
    with pytest.raises(FileExistsError):                 # a second run without --resume
        mod.prepare_outdir(str(out), rows, resume=False)
    assert mod.prepare_outdir(str(out), rows, resume=True) == rows
    with pytest.raises(ValueError):                      # --resume over a different image list
        mod.prepare_outdir(str(out), rows[:-1], resume=True)


def test_shard_naming_and_ranges_keep_manifest_order():
    mod = script("build_rdm_database")
    assert mod.shard_ranges(10, 4) == [(0, 0, 4), (1, 4, 8), (2, 8, 10)]
    assert mod.shard_ranges(8, 4) == [(0, 0, 4), (1, 4, 8)]
    names = [mod.shard_name(k) for k in (0, 9, 10, 123456)]
    assert names == sorted(names) and names[0] == "shard_000000.npz"


def test_written_shards_load_through_retrieval_and_resume_check(tmp_path):
    from sdb200.retrieval import load_database
    mod = script("build_rdm_database")
    d = str(tmp_path)
    rng = np.random.default_rng(0)
    emb = rng.standard_normal((10, 768)).astype(np.float32)
    coords = np.array([(0, 0, 30 + i, 20 + i) for i in range(10)], dtype=np.int32)
    for k, s, e in mod.shard_ranges(10, 4):
        path = os.path.join(d, mod.shard_name(k))
        assert not mod.shard_complete(path, s, e)
        mod.write_shard(path, emb[s:e], np.arange(s, e), coords[s:e])
        assert mod.shard_complete(path, s, e)
        assert not mod.shard_complete(path, s, e + 1)
    assert not [f for f in os.listdir(d) if f.endswith(".partial")]
    db = load_database(d)
    assert db["embedding"].dtype == np.float32 and np.array_equal(db["embedding"], emb)
    assert db["img_id"].dtype == np.int64 and np.array_equal(db["img_id"], np.arange(10))
    assert db["patch_coords"].dtype == np.int32 and np.array_equal(db["patch_coords"], coords)
    # a truncated shard is not complete (an interrupted write of the old format, or a damaged file)
    p1 = os.path.join(d, mod.shard_name(1))
    with open(p1, "r+b") as f:
        f.truncate(100)
    assert not mod.shard_complete(p1, 4, 8)


def test_knn2img_database_dir_defaults_to_none():
    opt = script("knn2img").get_parser().parse_args([])
    assert opt.database_dir is None and opt.database == "artbench-surrealism"
    assert script("knn2img").get_parser().parse_args(["--database_dir", "x"]).database_dir == "x"


def test_builder_flags():
    mod = script("build_rdm_database")
    opt = mod.get_parser().parse_args(["--images", "a", "--outdir", "b"])
    assert (opt.batch, opt.shard_size, opt.resume, opt.clip_ckpt, opt.random_init) == (256, 100000, False, None, False)
    with pytest.raises(ValueError):
        mod.main(["--images", "a", "--outdir", "b", "--tiny"])


# ------------------------------------------------------------------------------------------------ constructor
def test_constructor_errors_and_target_map():
    import sdb200
    from sdb200.util import TARGET_MAP, get_obj_from_str, instantiate_from_config, remap_config
    with pytest.raises(NotImplementedError):
        sdb200.FrozenClipImageEmbedder("ViT-L/14", antialias=True)
    for name in ("ViT-B/32", "RN50", "ViT-L/14@336px"):
        with pytest.raises(NotImplementedError):
            sdb200.FrozenClipImageEmbedder(name)
    t = "ldm.modules.encoders.modules.FrozenClipImageEmbedder"
    assert get_obj_from_str(TARGET_MAP[t]) is sdb200.FrozenClipImageEmbedder
    e = instantiate_from_config(remap_config({"target": t, "params": {"model": "ViT-L/14", "jit": False}}))
    assert e.shapes == arch.clip_vision_proj_param_shapes(arch.CLIP_VISION_PROJ)


def test_weights_from_a_clip_model_state_dict():
    """The CLIPModel layout: the text tower's keys are present and ignored; the vision keys are adopted."""
    import sdb200
    cfg = arch.TINY_CLIP_VISION_PROJ
    e = sdb200.FrozenClipImageEmbedder("ViT-L/14", config=cfg)
    sd = arch.random_state_dict(e.shapes, 3)
    full = dict(sd)
    full.update({"text_model.embeddings.token_embedding.weight": torch.zeros(4, 4), "text_projection.weight":
                 torch.zeros(4, 4), "logit_scale": torch.zeros(()), "vision_model.embeddings.position_ids":
                 torch.zeros(1, 17, dtype=torch.long)})
    r = e.load_state_dict(full, strict=True)
    assert not r.missing_keys and not r.unexpected_keys
    assert set(e._host_sd) == set(sd)
