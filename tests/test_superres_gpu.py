"""The LDM super-resolution model on the H100: the LR conversion bit-exact against get_cond (tests/golden/superres.pt),
the patch unfold bit-identical to nn.Unfold, the weighted stitch against fp64 fold(o·w)/fold(w), UNet / VQ-f4 / tiled
DDIM parity with the reference, the full model at 256² -> 1024² against per-tile calls stitched by the oracle, the size
rule, scripts/superres.py end to end, and every GEMM plan at the model's GEMM problems."""
import os

import pytest
import torch

import helpers  # noqa: F401
import superres_oracle as S
from helpers import golden, rel_l2, script
from sdb200 import arch, diffusion, ops, pipeline
from sdb200.diffusion import split_geometry, split_tables
from workloads import GEMM_MODEL_WORKLOADS

pytestmark = pytest.mark.gpu
UCFG = {"tiny": arch.TINY_BSR_UNET, "big": arch.BSR_SR_UNET}


def _gen(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


_UNETS = {}


def _unet(tag, dev):
    if tag not in _UNETS:
        import sdb200
        sd = arch.random_state_dict(arch.unet_param_shapes(UCFG[tag]), golden("superres.pt")["unet_seed"])
        _UNETS[tag] = sdb200.UNetModel(**UCFG[tag]).load_weights(sd, dev)
    return _UNETS[tag]


@pytest.mark.parametrize("idx", range(2))
def test_lr_prepare_bit_exact(cuda_dev, idx):
    case = golden("superres.pt")["lr"][idx]
    assert torch.equal(ops.lr_prepare(case["image"][None].to(cuda_dev)).cpu(), case["c"])


@pytest.mark.parametrize("shape, ks, stride", [((2, 3, 24, 40), (16, 16), (8, 8)), ((1, 6, 20, 28), (12, 12), (4, 4)),
                                               ((2, 3, 25, 42), (16, 8), (8, 5)), ((1, 3, 256, 256), (128, 128), (64, 64))])
def test_patch_unfold_bit_identical_to_unfold(cuda_dev, shape, ks, stride):
    x = torch.randn(shape, device=cuda_dev)
    ref = torch.nn.functional.unfold(x, ks, stride=stride)
    ref = ref.view(shape[0], shape[1], ks[0], ks[1], -1).permute(4, 0, 1, 2, 3).reshape(-1, shape[1], *ks)
    assert torch.equal(ops.patch_unfold(x, ks, stride), ref)


@pytest.mark.parametrize("tag", ["tiny_uf1", "tiny_uf4", "tiny_tie_uf1", "tiny_tie_uf4", "tiny_stride4_uf1",
                                 "nb256_uf1", "nb192_uf4"])
@pytest.mark.parametrize("nhwc", [False, True])
def test_patch_fold_matches_fp64_fold(cuda_dev, tag, nhwc):
    e = [t for t in golden("superres.pt")["tables"] if t["tag"] == tag][0]
    p, uf = e["params"], e["uf"]
    ks, stride, grid = split_geometry(e["h"], e["w"], p, uf)
    weight, norm = split_tables(ks, stride, grid, p, uf)
    L, kh, kw = weight.shape
    nb, c = (2, 3) if kh <= 64 else (1, 3)
    g = torch.Generator(device=cuda_dev).manual_seed(4)
    tiles = torch.randn((L * nb, c, kh, kw), generator=g, device=cuda_dev)
    st = (stride[0] * uf, stride[1] * uf)
    src = tiles.permute(0, 2, 3, 1).contiguous() if nhwc else tiles
    out = ops.patch_fold(src, weight.to(cuda_dev), norm.to(cuda_dev), grid, st, nhwc=nhwc)
    o = (tiles.double() * weight.to(cuda_dev).double().repeat_interleave(nb, 0)[:, None])
    o = o.view(L, nb, c * kh * kw).permute(1, 2, 0)
    size = tuple(norm.shape)
    w64 = weight.double().view(L, kh * kw).t()[None].to(cuda_dev)
    ref = torch.nn.functional.fold(o, size, (kh, kw), stride=st) / torch.nn.functional.fold(w64, size, (kh, kw), stride=st)
    err = rel_l2(out, ref)
    print(f"fold {tag} nhwc={nhwc}: rel-L2 {err:.2e} vs fp64")
    assert err < 1e-6 and bool(torch.isfinite(out).all())
    assert torch.equal(out, ops.patch_fold(src, weight.to(cuda_dev), norm.to(cuda_dev), grid, st, nhwc=nhwc))


def test_patch_fold_rejects_uncovered_output(cuda_dev):
    w = torch.ones(2, 4, 4, device=cuda_dev)
    with pytest.raises(RuntimeError, match="do not cover"):
        ops.patch_fold(torch.zeros(2, 3, 4, 4, device=cuda_dev), w, torch.ones(4, 9, device=cuda_dev), (1, 2), (4, 4))


@pytest.mark.parametrize("idx", range(4))
def test_unet_eps_matches_reference(cuda_dev, idx):
    case = golden("superres.pt")["unet"][idx]
    u = _unet(case["cfg"], cuda_dev)
    x, t = _gen(case["shape"], case["x_seed"]).to(cuda_dev), case["t"].to(cuda_dev)
    eps = u(x[:, :3].contiguous(), t, concat=x[:, 3:].contiguous())
    err = rel_l2(eps, case["eps"])
    print(f"unet {case['cfg']} {tuple(x.shape)}: eps rel-L2 {err:.2e}")
    assert err < 1e-3, (case["cfg"], tuple(x.shape), err)
    assert torch.equal(eps, u(x, t))
    if case["cfg"] == "tiny" or x.shape[-1] == 128:
        # graph replay on the default GEMM plans equals eager; with the autotuner's plans both routes still agree
        try:
            u.use_cuda_graph = True
            for tune in (False, True):
                u.autotune = tune
                u._graphs.clear()
                g = u(x[:, :3].contiguous(), t, concat=x[:, 3:].contiguous())
                assert torch.equal(g, u(x, t)) and (tune or torch.equal(g, eps))
                assert rel_l2(g, case["eps"]) < 1e-3
        finally:
            u.use_cuda_graph, u.autotune = False, True
            u._graphs.clear()


def test_vq_f4_decode(cuda_dev):
    import sdb200
    g = golden("superres.pt")
    m = sdb200.VQModelInterface(**arch.VQ_F4).load_weights(
        arch.random_state_dict(arch.vq_param_shapes(arch.VQ_F4), g["vq_seed"]), cuda_dev)
    err = rel_l2(m.decode(g["vq_f4"]["h"].to(cuda_dev)), g["vq_f4"]["dec"])
    print(f"vq_f4 decode: rel-L2 {err:.2e}")
    assert err < 2e-3


def _tiny_model(dev):
    Sc = script("superres")
    g = golden("superres.pt")
    m = Sc.load_model(random_init=True, tiny=True, device=dev)
    # load_model(random_init) draws on the device generator: load the CPU-drawn golden weights instead
    pipeline.load_random_weights(m, dev, seeds=(g["unet_seed"], g["vq_seed"]))
    return Sc, m


@pytest.mark.parametrize("eta", [0, 1])
@pytest.mark.parametrize("graph", [False, True])
def test_tiny_tiled_end_to_end_ddim10(cuda_dev, monkeypatch, eta, graph):
    from sdb200.samplers import DDIMSampler
    e = golden("superres.pt")["e2e"]
    Sc, m = _tiny_model(cuda_dev)
    assert torch.equal(m.alphas_cumprod.cpu(), e["alphas_cumprod"])
    m.model.diffusion_model.use_cuda_graph = graph
    r = e[f"eta{eta}"]
    x_T = _gen((1, 3, 24, 24), e["x_T_seed"]).to(cuda_dev)
    draws = [_gen((1, 3, 24, 24), e["noise_seed"] + i) for i in range(r["n_noise"])]
    if eta:
        monkeypatch.setattr(torch, "randn_like", lambda t, *a, **k: draws.pop(0).to(t.device))
    with m.ema_scope():
        x, c, s, path = Sc.superresolve(m, DDIMSampler(m), e["image"][None].to(cuda_dev), steps=10, eta=float(eta),
                                        x_T=x_T, return_latents=True, split=e["params"])
    monkeypatch.undo()
    assert path == "split" and (not eta or not draws)
    e_s, e_x = rel_l2(s, r["sample"]), rel_l2(x, r["x_dec"])
    # the tiled decode of the reference's own latent; the decode of ours matches too where the nearest-codebook search
    # picks the same codes (a near tie flips a code, and with it a whole 4x4 block of the image)
    e_d = rel_l2(m.decode_first_stage(r["sample"].to(cuda_dev)), r["x_dec"])
    q = m.first_stage_model.quantize
    same_codes = torch.equal(q(s)[2][2], q(r["sample"].to(cuda_dev))[2][2])
    print(f"tiled e2e eta {eta} graph {graph}: DDIM-10 latent rel-L2 {e_s:.2e}, decoded {e_x:.2e} (same codes "
          f"{same_codes}), tiled decode of the reference latent {e_d:.2e}")
    assert e_s < 1e-3 and e_d < 1e-3 and (e_x < 1e-3 or not same_codes)


def test_tiny_split_apply_and_decode_vs_oracle_and_chunks(cuda_dev, monkeypatch):
    """The engine's split apply_model / decode against the oracle stitching the engine's own per-tile calls, and the
    same results when memory forces one tile per chunk."""
    _, m = _tiny_model(cuda_dev)
    p = S.notebook_params(16, 8, tie_braker=True)
    m.split_input_params = p
    g = torch.Generator(device=cuda_dev).manual_seed(8)
    x = torch.randn(2, 3, 24, 40, generator=g, device=cuda_dev)
    c = torch.randn(2, 3, 24, 40, generator=g, device=cuda_dev)
    t = torch.tensor([700, 20], device=cuda_dev)
    eps = m.apply_model(x, t, c)
    unet = m.model.diffusion_model
    ref = S.split_apply(lambda xt, tt, ct: unet(xt.to(cuda_dev).contiguous(), t, concat=ct.to(cuda_dev).contiguous()).cpu(),
                        x.cpu(), t.cpu(), c.cpu(), p)
    z = torch.randn(1, 3, 24, 40, generator=g, device=cuda_dev)
    dec = m.decode_first_stage(z)
    ref_dec = S.split_decode(lambda zt: m.first_stage_model.decode(zt.to(cuda_dev).contiguous()).cpu(), z.cpu(), p)
    e_a, e_d = rel_l2(eps, ref), rel_l2(dec, ref_dec)
    print(f"tiny split vs oracle stitch of per-tile calls: apply {e_a:.2e}, decode {e_d:.2e}")
    assert e_a < 1e-3 and e_d < 1e-3
    monkeypatch.setattr(diffusion, "_UNET_TILE_BYTES", 1 << 60)
    monkeypatch.setattr(diffusion, "_DECODER_TILE_BYTES", 1 << 60)
    m._split_cache.clear()
    e_a1, e_d1 = rel_l2(m.apply_model(x, t, c), eps), rel_l2(m.decode_first_stage(z), dec)
    assert m._split_cache and all(v["chunk"] == 1 for v in m._split_cache.values())
    print(f"one tile per chunk vs one batch: apply {e_a1:.2e}, decode {e_d1:.2e}")
    assert e_a1 < 1e-3 and e_d1 < 1e-3


_FULL = {}


def _full(dev):
    if "m" not in _FULL:
        Sc = script("superres")
        _FULL["m"] = (Sc, Sc.load_model(random_init=True, device=dev))
    return _FULL["m"]


def test_full_model_256_to_1024(cuda_dev):
    """The reference workload's geometry: 3x3 tiles of 128² (one UNet batch of 9), 4 DDIM steps at eta 1 through the
    graph path, a tiled decode to 1024². One split evaluation matches the oracle's stitch of nine per-tile calls."""
    from sdb200.samplers import DDIMSampler
    Sc, m = _full(cuda_dev)
    unet = m.model.diffusion_model
    g = torch.Generator(device=cuda_dev).manual_seed(9)
    lr = torch.randint(0, 256, (1, 256, 256, 3), generator=g, device=cuda_dev, dtype=torch.uint8)
    try:
        unet.use_cuda_graph = True
        with m.ema_scope():
            x, c, s, path = Sc.superresolve(m, DDIMSampler(m), lr, steps=4, eta=1.0, return_latents=True)
        assert path == "split" and tuple(x.shape) == (1, 3, 1024, 1024) and bool(torch.isfinite(x).all())
        xt = torch.randn(1, 3, 256, 256, generator=g, device=cuda_dev)
        t = torch.tensor([500], device=cuda_dev)
        eps = m.apply_model(xt, t, c)
    finally:
        unet.use_cuda_graph = False
    ref = S.split_apply(lambda a, tt, b: unet(a.to(cuda_dev).contiguous(), t, concat=b.to(cuda_dev).contiguous()).cpu(),
                        xt.cpu(), t.cpu(), c.cpu(), m.split_input_params)
    err = rel_l2(eps, ref)
    print(f"full 256²: split apply_model (one batch of 9, graph) vs oracle stitch of 9 calls: rel-L2 {err:.2e}")
    assert err < 1e-3


def test_full_model_64_runs_plain_and_uncovered_sizes_raise(cuda_dev):
    from sdb200.samplers import DDIMSampler
    Sc, m = _full(cuda_dev)
    lr = torch.randint(0, 256, (1, 64, 64, 3), device=cuda_dev, dtype=torch.uint8)
    x, _, _, path = Sc.superresolve(m, DDIMSampler(m), lr, steps=4, return_latents=True)
    assert path == "plain" and not hasattr(m, "split_input_params")
    assert tuple(x.shape) == (1, 3, 256, 256) and bool(torch.isfinite(x).all())
    for h, w in ((200, 256), (256, 130)):
        with pytest.raises(ValueError, match="cover"):
            Sc.superresolve(m, DDIMSampler(m), torch.zeros(1, h, w, 3, device=cuda_dev, dtype=torch.uint8), steps=2)
    m.split_input_params = Sc.split_params()
    try:
        with pytest.raises(ValueError, match="larger than"):
            m.apply_model(torch.zeros(1, 3, 64, 64, device=cuda_dev), torch.tensor([1], device=cuda_dev),
                          torch.zeros(1, 3, 64, 64, device=cuda_dev))
    finally:
        del m.split_input_params


def test_script_tiny_writes_4x_png(cuda_dev, tmp_path):
    import numpy as np
    from PIL import Image
    indir, outdir = tmp_path / "in", tmp_path / "out"
    indir.mkdir()
    r = np.random.default_rng(0)
    for name, (h, w) in (("a", (24, 32)), ("b", (128, 192))):
        Image.fromarray(r.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(indir / f"{name}.png")
    written = script("superres").main(["--indir", str(indir), "--outdir", str(outdir), "--steps", "4", "--random_init",
                                       "--tiny"])
    assert sorted(os.path.basename(p) for p in written) == ["a.png", "b.png"]
    assert Image.open(outdir / "a.png").size == (128, 96) and Image.open(outdir / "b.png").size == (768, 512)


def test_every_plan_of_every_bsr_gemm_problem(cuda_dev):
    from test_gemm_plans_gpu import catalogue, run_sweep
    problems = catalogue(GEMM_MODEL_WORKLOADS["bsr_sr"], cuda_dev)
    print(f"\nbsr_sr UNet (9, 3+3, 128²) + tiled VQ-f4 decode: {len(problems)} distinct GEMM problems")
    assert problems
    run_sweep(problems, cuda_dev, "bsr_sr")
    torch.cuda.empty_cache()
