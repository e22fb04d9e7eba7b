"""FrozenClipImageEmbedder on the GPU: the preprocessing kernel (sdb_clip_resize_patches) against torch's
F.interpolate(bicubic, align_corners=True), ragged batches, the uint8 path, embeddings against transformers'
CLIPVisionModelWithProjection (tests/golden/clip_image.pt), batch invariance, agreement with the safety checker's tower,
a database built by scripts/build_rdm_database.py end to end through retrieval.Searcher and knn2img.py --database_dir,
and every GEMM plan at the tower's problems."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers
from helpers import golden, rel_l2, script
from sdb200 import arch, ops
from sdb200.clip_image import _table
from workloads import GEMM_MODEL_WORKLOADS

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

SIZES = [(64, 64), (512, 512), (1000, 333), (7, 513), (224, 224)]
MEAN = torch.tensor(arch.CLIP_IMAGE_MEAN).view(1, 3, 1, 1)
STD = torch.tensor(arch.CLIP_IMAGE_STD).view(1, 3, 1, 1)


def _embedder(cfg, dev, seed=16):
    import sdb200
    e = sdb200.FrozenClipImageEmbedder("ViT-L/14", config=cfg)
    return e.load_weights(arch.random_state_dict(e.shapes, seed), dev)


def _u8_to_x(u8):
    """uint8 numpy -> fp32 x / 127.5 - 1 with IEEE division (what the kernel's uint8 path computes)."""
    return torch.from_numpy(u8.astype(np.float32) / np.float32(127.5) - np.float32(1.0))


def _images(sizes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (3, h, w), dtype=np.uint8) for h, w in sizes]


def _pack_f32(xs, dev):
    flat = torch.cat([x.reshape(-1) for x in xs]).to(dev)
    return flat, _table([tuple(x.shape[-2:]) for x in xs], 3, flat.numel()).to(dev)


def _patches_from(resized, P, kpad):
    """fp16 patch rows of the normalised resized images, in CLIPVisionEmbeddings' flattening (torch ops)."""
    B, _, S, _ = resized.shape
    g = S // P
    v = ((resized + 1) / 2 - MEAN.to(resized.device)) / STD.to(resized.device)
    p = v.half().view(B, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(B * g * g, 3 * P * P)
    return F.pad(p, (0, kpad - 3 * P * P))


# ------------------------------------------------------------------------------------------------ preprocessing
def test_preprocess_matches_interpolate_and_is_ragged_exact(cuda_dev):
    S, P, kpad = 224, 14, 640
    xs = [_u8_to_x(u) for u in _images(SIZES, 0)]
    flat, table = _pack_f32(xs, cuda_dev)
    patches, resized = ops.clip_resize_patches(flat, table, S, P, kpad, arch.CLIP_IMAGE_MEAN, arch.CLIP_IMAGE_STD,
                                               want_resized=True)
    for i, x in enumerate(xs):
        ref = F.interpolate(x[None].to(cuda_dev), size=(S, S), mode="bicubic", align_corners=True)
        err = float((resized[i:i + 1] - ref).abs().max())
        print(f"{tuple(x.shape[-2:])} -> {S}²: max abs {err:.2e} vs F.interpolate")
        assert err <= 2e-6, (tuple(x.shape), err)
        # the same image alone: bit-equal to its rows of the ragged launch
        f1, t1 = _pack_f32([x], cuda_dev)
        p1, r1 = ops.clip_resize_patches(f1, t1, S, P, kpad, arch.CLIP_IMAGE_MEAN, arch.CLIP_IMAGE_STD, want_resized=True)
        assert torch.equal(r1[0], resized[i])
        assert torch.equal(p1, patches[i * 256:(i + 1) * 256])
    # the patch rows are the normalised resized values in the patch-embedding weight's flattening, zero-padded
    assert torch.equal(patches, _patches_from(resized, P, kpad))


def test_uint8_path_is_bit_equal_to_fp32_path(cuda_dev):
    S, P, kpad = 224, 14, 640
    u8s = _images(SIZES, 1)
    flat32, table32 = _pack_f32([_u8_to_x(u) for u in u8s], cuda_dev)
    p32, r32 = ops.clip_resize_patches(flat32, table32, S, P, kpad, arch.CLIP_IMAGE_MEAN, arch.CLIP_IMAGE_STD,
                                       want_resized=True)
    hwc = [torch.from_numpy(np.ascontiguousarray(u.transpose(1, 2, 0))) for u in u8s]
    flat8 = torch.cat([t.reshape(-1) for t in hwc]).to(cuda_dev)
    table8 = _table([tuple(t.shape[:2]) for t in hwc], 3, flat8.numel()).to(cuda_dev)
    p8, r8 = ops.clip_resize_patches(flat8, table8, S, P, kpad, arch.CLIP_IMAGE_MEAN, arch.CLIP_IMAGE_STD,
                                     want_resized=True)
    assert torch.equal(r8, r32) and torch.equal(p8, p32)


# ------------------------------------------------------------------------------------------------ embeddings
@pytest.mark.parametrize("tag,cfg", [("tiny", arch.TINY_CLIP_VISION_PROJ), ("vitl14", arch.CLIP_VISION_PROJ)])
def test_embeddings_vs_transformers_golden(cuda_dev, tag, cfg):
    case = golden("clip_image.pt")[tag]
    emb = _embedder(cfg, cuda_dev, case["seed"])
    u8 = case["images_u8"].numpy()
    z = emb(_u8_to_x(u8).to(cuda_dev))
    err = rel_l2(z.cpu(), case["image_embeds"].float())
    print(f"{tag}: image_embeds rel-L2 {err:.2e} vs CLIPVisionModelWithProjection")
    assert z.shape == case["image_embeds"].shape and err < 2e-3
    # the uint8 entry point (HWC images, host or device) gives the same bits
    hwc = [torch.from_numpy(np.ascontiguousarray(a.transpose(1, 2, 0))) for a in u8]
    assert torch.equal(emb.encode_uint8(hwc), z)
    assert torch.equal(emb.encode_uint8([t.to(cuda_dev) for t in hwc]), z)


def test_batch_invariance(cuda_dev):
    """Row i of a ragged batch of 37 against the same image alone."""
    emb = _embedder(arch.CLIP_VISION_PROJ, cuda_dev)
    rng = np.random.default_rng(5)
    sizes = [(int(rng.integers(100, 700)), int(rng.integers(100, 700))) for _ in range(37)]
    imgs = [torch.from_numpy(np.ascontiguousarray(u.transpose(1, 2, 0))) for u in _images(sizes, 6)]
    zb = emb.encode_uint8(imgs)
    worst = max(rel_l2(zb[i], emb.encode_uint8([im])[0]) for i, im in enumerate(imgs))
    print(f"batch 37 vs batch 1: worst row rel-L2 {worst:.2e}")
    assert worst < 1e-3


def test_matches_the_safety_checkers_tower(cuda_dev):
    """Same weights and pixel values through StableDiffusionSafetyChecker.image_embeds (per-image loops) and the
    batched path."""
    import sdb200
    emb = _embedder(arch.CLIP_VISION_PROJ, cuda_dev)
    sd = {("vision_model." + k if k.startswith("vision_model.") else k): v for k, v in emb._host_sd.items()}
    rest = arch.safety_param_shapes(arch.SD_V1_SAFETY)
    sd.update({k: v for k, v in arch.random_state_dict(rest, 14).items() if not k.startswith(("vision_model.", "visual_"))})
    chk = sdb200.StableDiffusionSafetyChecker(config=arch.SD_V1_SAFETY).load_weights(sd, cuda_dev)
    g = torch.Generator().manual_seed(7)
    x = (torch.rand(5, 3, 224, 224, generator=g) * 2 - 1).to(cuda_dev)       # 224²: the resize is a copy
    pix = ((x + 1) / 2 - MEAN.to(cuda_dev)) / STD.to(cuda_dev)
    err = rel_l2(emb(x), chk.image_embeds(pix))
    print(f"FrozenClipImageEmbedder vs safety checker tower: rel-L2 {err:.2e}")
    assert err < 1e-3


# ------------------------------------------------------------------------------------------------ database end to end
def synthetic_pngs(root, n=48, seed=0):
    """n seeded PNGs of different sizes under root/<i % 3>/: a random grid of 2-5 x 2-5 colour cells plus noise. (With
    the tiny random-weight tower the closest pair of these has cosine similarity 0.97, far from a tie.)"""
    from PIL import Image
    rng = np.random.default_rng(seed)
    for i in range(n):
        h, w = int(rng.integers(40, 160)), int(rng.integers(40, 160))
        cells = rng.integers(0, 256, (int(rng.integers(2, 6)), int(rng.integers(2, 6)), 3)).astype(np.float64)
        img = cells[(np.arange(h) * cells.shape[0]) // h][:, (np.arange(w) * cells.shape[1]) // w]
        img = np.clip(img + rng.normal(0, 20, (h, w, 3)), 0, 255).astype(np.uint8)
        d = os.path.join(root, str(i % 3))
        os.makedirs(d, exist_ok=True)
        Image.fromarray(img).save(os.path.join(d, f"img{i:03d}.png"))


def _run(script, args, cwd):
    cmd = [sys.executable, os.path.join(helpers.ROOT, "scripts", script)] + args
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"{script} failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    return r.stdout


def test_build_database_search_and_knn2img(cuda_dev, tmp_path):
    from sdb200.retrieval import Searcher, load_database
    from test_rdm_gpu import _tiny_vocab
    imgs, db = str(tmp_path / "imgs"), str(tmp_path / "db")
    synthetic_pngs(imgs)
    args = ["--images", imgs, "--outdir", db, "--random_init", "--tiny", "--batch", "16", "--shard_size", "20",
            "--workers", "2"]
    _run("build_rdm_database.py", args, str(tmp_path))
    shards = sorted(f for f in os.listdir(db) if f.endswith(".npz"))
    assert shards == ["shard_000000.npz", "shard_000001.npz", "shard_000002.npz"]
    data = load_database(db)
    manifest = open(os.path.join(db, "manifest.txt")).read().splitlines()
    assert len(manifest) == 48 and data["embedding"].shape == (48, 64)
    assert np.array_equal(data["img_id"], np.arange(48))
    from PIL import Image
    for i in (0, 17, 47):
        w, h = Image.open(os.path.join(imgs, manifest[i])).size
        assert tuple(data["patch_coords"][i]) == (0, 0, w, h)
    # the builder's embeddings are the embedder's on the decoded images
    emb = script("build_rdm_database").load_embedder(random_init=True, tiny=True, device=cuda_dev)
    some = [torch.from_numpy(np.asarray(Image.open(os.path.join(imgs, manifest[i])).convert("RGB"))) for i in (0, 1, 2)]
    assert rel_l2(emb.encode_uint8(some), torch.from_numpy(data["embedding"][:3])) < 1e-5
    # each image's own embedding finds that image first
    s = Searcher("own", device=cuda_dev, path=db)
    out = s.search(data["embedding"], 1)
    assert np.array_equal(out["img_ids"][:, 0], np.arange(48))
    # --resume keeps complete shards and rebuilds a missing one identically
    os.remove(os.path.join(db, shards[1]))
    with np.load(os.path.join(tmp_path, "db", shards[0])) as d0:
        first = d0["embedding"].copy()
    stdout = _run("build_rdm_database.py", args + ["--resume"], str(tmp_path))
    assert "2 complete shard(s) kept" in stdout
    again = load_database(db)
    assert np.array_equal(again["embedding"][:20], first)
    assert rel_l2(torch.from_numpy(again["embedding"]), torch.from_numpy(data["embedding"])) < 1e-6
    # knn2img.py samples with neighbours from the built database
    vocab = _tiny_vocab(str(tmp_path / "vocab"))
    _run("knn2img.py", ["--random_init", "--tiny", "--clip_vocab", vocab, "--outdir", str(tmp_path / "out"), "--H",
                        "256", "--W", "256", "--ddim_steps", "2", "--n_samples", "1", "--seed", "0", "--use_neighbors",
                        "--knn", "4", "--database_dir", db], str(tmp_path))
    assert len(os.listdir(tmp_path / "out" / "samples")) == 1


# ------------------------------------------------------------------------------------------------ GEMM plans
def test_every_plan_of_the_tower_gemm_problems(cuda_dev):
    """The ViT-L/14 tower's GEMMs at B = 1, 64 and 256 images (M = 256 B patch rows, 257 B token rows)."""
    from test_gemm_plans_gpu import catalogue, run_sweep
    problems = catalogue(GEMM_MODEL_WORKLOADS["clip_image"], cuda_dev)
    print(f"\nCLIP ViT-L/14 image tower at B = 1, 64, 256: {len(problems)} distinct GEMM problems")
    assert problems
    run_sweep(problems, cuda_dev, "clip_image")
    torch.cuda.empty_cache()
