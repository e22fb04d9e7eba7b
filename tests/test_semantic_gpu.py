"""The LDM semantic-synthesis models on the H100: the float rescale kernel against torch's CUDA F.interpolate (bit for
bit) and fp64, the label kernel bit-identical to the float kernel on the one-hot, the cond stage / UNet eps / tiny
DDIM-10 against the unmodified reference (tests/golden/semantic.pt), graph replay against eager with the conditioning
refreshed, the full model at a larger-than-training size, scripts/semantic_synthesis.py end to end, and every GEMM
plan at the full UNet's GEMM problems."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers  # noqa: F401
import semantic_oracle as SO
from helpers import golden, rel_l2, script
from sdb200 import arch, ops, pipeline
from workloads import GEMM_MODEL_WORKLOADS

pytestmark = pytest.mark.gpu
UCFG = {"tiny": arch.TINY_SEMANTIC_UNET, "big": arch.SEMANTIC_SYNTHESIS_UNET}


def _gen(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def _max_ulp(a, b):
    ai = a.contiguous().view(torch.int32).long()
    bi = b.contiguous().view(torch.int32).long()
    ai = torch.where(ai < 0, -(ai & 0x7FFFFFFF), ai)
    bi = torch.where(bi < 0, -(bi & 0x7FFFFFFF), bi)
    return int((ai - bi).abs().max()) if ai.numel() else 0


@pytest.mark.parametrize("shape, n", [((2, 5, 32, 48), 2), ((1, 3, 30, 46), 2), ((2, 4, 17, 9), 1),
                                      ((1, 2, 64, 40), 3), ((1, 7, 13, 11), 0), ((1, 182, 36, 20), 2)])
def test_float_rescale_equals_cuda_interpolate(cuda_dev, shape, n):
    x = torch.randn(shape, device=cuda_dev)
    ref = x
    for _ in range(n):
        ref = F.interpolate(ref, scale_factor=0.5, mode="bilinear")
    out = ops.spatial_rescale(x, n)
    assert out.shape == ref.shape
    print(f"rescale {shape} n={n}: max ulp vs F.interpolate on CUDA {_max_ulp(out, ref)}")
    assert torch.equal(out, ref)


@pytest.mark.parametrize("shape, n, cout, bias", [((2, 182, 64, 64), 2, 3, False), ((1, 20, 30, 46), 1, 3, True),
                                                  ((1, 9, 24, 40), 3, 6, True), ((2, 5, 16, 16), 0, 5, False)])
def test_float_rescale_with_mapper_vs_fp64(cuda_dev, shape, n, cout, bias):
    g = torch.Generator(device=cuda_dev).manual_seed(3)
    x = torch.randn(shape, generator=g, device=cuda_dev)
    w = torch.randn((cout, shape[1]), generator=g, device=cuda_dev) / shape[1] ** 0.5
    b = torch.randn((cout,), generator=g, device=cuda_dev) if bias else None
    out = ops.spatial_rescale(x, n, w, b)
    ref = x.double()
    for _ in range(n):
        ref = F.interpolate(ref, scale_factor=0.5, mode="bilinear")
    ref = F.conv2d(ref, w.double()[:, :, None, None], None if b is None else b.double())
    err = rel_l2(out, ref)
    print(f"rescale + mapper {shape} n={n} -> {cout}: rel-L2 {err:.2e} vs fp64")
    assert err <= 1e-6
    assert torch.equal(out, ops.spatial_rescale(x, n, w, b))


def _label_cases():
    return [("voronoi64", SO.voronoi_labels(64, 64, 182, 21)[None], 182, 2),
            ("voronoi256", SO.voronoi_labels(256, 256, 182, 22)[None], 182, 2),
            ("voronoi30x46", SO.voronoi_labels(30, 46, 182, 23)[None], 182, 2),
            ("all_ids", SO.all_ids_labels(56, 64, 182, 24)[None], 182, 2),
            ("all_ids_n3", SO.all_ids_labels(64, 72, 182, 25)[None], 182, 3),
            ("batch2_odd", np.stack([SO.voronoi_labels(33, 70, 20, 26), SO.all_ids_labels(33, 70, 20, 27)]), 20, 1),
            ("n0", SO.all_ids_labels(12, 20, 182, 28)[None], 182, 0),
            ("256_classes", SO.all_ids_labels(64, 64, 256, 29)[None], 256, 2)]


@pytest.mark.parametrize("case", range(8))
@pytest.mark.parametrize("bias", [False, True])
def test_label_kernel_bit_identical_to_float_kernel_on_one_hot(cuda_dev, case, bias):
    tag, lab, n_classes, n = _label_cases()[case]
    g = torch.Generator(device=cuda_dev).manual_seed(case)
    w = torch.randn((3, n_classes), generator=g, device=cuda_dev) / n_classes ** 0.5
    b = torch.randn((3,), generator=g, device=cuda_dev) if bias else None
    ids = torch.from_numpy(lab).to(cuda_dev)
    fused = ops.seg_labels_rescale(ids, n_classes, n, w, b)
    dense = ops.spatial_rescale(SO.one_hot(ids, n_classes).to(cuda_dev), n, w, b)
    print(f"labels {tag} {tuple(lab.shape)} n={n} bias={bias}: bit-identical {torch.equal(fused, dense)}")
    assert torch.equal(fused, dense)


def _rescaler(cfg, seed, dev):
    import sdb200
    m = sdb200.SpatialRescaler(**cfg)
    return m.load_weights(arch.random_state_dict(arch.spatial_rescaler_param_shapes(cfg), seed), dev)


@pytest.mark.parametrize("idx", range(7))
def test_cond_stage_matches_reference(cuda_dev, idx):
    g = golden("semantic.pt")
    e = g["cond"][idx]
    cfg = {"full": arch.SEMANTIC_SYNTHESIS_COND, "tiny": arch.TINY_SEMANTIC_COND, "tiny_bias": g["tiny_bias_cond"]}[e["cfg"]]
    m = _rescaler(cfg, g["cond_seed"], cuda_dev)
    if e["kind"] == "soft":
        c = m.encode(SO.soft_map((1, cfg["in_channels"], e["h"], e["w"]), e["seed"]).to(cuda_dev))
    else:
        f = SO.voronoi_labels if e["kind"] == "voronoi" else SO.all_ids_labels
        lab = torch.from_numpy(f(e["h"], e["w"], cfg["in_channels"], e["seed"]))[None]
        c = m.encode(lab)
        assert torch.equal(c, m.encode(SO.one_hot(lab, cfg["in_channels"]).to(cuda_dev)))
    err = rel_l2(c, e["c"])
    print(f"cond {e['tag']}: rel-L2 {err:.2e} vs the reference, max abs {float((c.cpu() - e['c']).abs().max()):.2e}")
    assert tuple(c.shape) == tuple(e["c"].shape) and err <= 1e-6


def test_cond_stage_rejects_bad_ids_before_the_kernel(cuda_dev):
    m = _rescaler(arch.SEMANTIC_SYNTHESIS_COND, 13, cuda_dev)
    lab = torch.zeros(1, 16, 16, dtype=torch.int64, device=cuda_dev)
    lab[0, 2, 3] = 182
    n0 = ops.launch_count()
    with pytest.raises(IndexError):
        m(lab)
    lab[0, 2, 3] = -1
    with pytest.raises(IndexError):
        m(lab)
    assert ops.launch_count() == n0
    with pytest.raises(NotImplementedError):
        _rescaler(dict(n_stages=2, in_channels=182), 13, cuda_dev)(lab.clamp(0))


_UNETS = {}


def _unet(tag, dev):
    if tag not in _UNETS:
        import sdb200
        sd = arch.random_state_dict(arch.unet_param_shapes(UCFG[tag]), golden("semantic.pt")["unet_seed"])
        _UNETS[tag] = sdb200.UNetModel(**UCFG[tag]).load_weights(sd, dev)
    return _UNETS[tag]


@pytest.mark.parametrize("idx", range(3))
def test_unet_eps_matches_reference(cuda_dev, idx):
    case = golden("semantic.pt")["unet"][idx]
    u = _unet(case["cfg"], cuda_dev)
    x, t = _gen(case["shape"], case["x_seed"]).to(cuda_dev), case["t"].to(cuda_dev)
    eps = u(x[:, :3].contiguous(), t, concat=x[:, 3:].contiguous())
    err = rel_l2(eps, case["eps"])
    print(f"unet {case['cfg']} {tuple(x.shape)}: eps rel-L2 {err:.2e}")
    assert err < 1e-3, (case["cfg"], tuple(x.shape), err)
    assert torch.equal(eps, u(x, t))


def _tiny_model(dev):
    Sc = script("semantic_synthesis")
    g = golden("semantic.pt")
    m = Sc.load_model(random_init=True, tiny=True, device=dev)
    # load_model(random_init) draws on the device generator: load the CPU-drawn golden weights instead
    pipeline.load_random_weights(m, dev, seeds=(g["unet_seed"], g["vq_seed"], g["cond_seed"]))
    return Sc, m


def test_graph_equals_eager_and_conditioning_refreshes(cuda_dev):
    _, m = _tiny_model(cuda_dev)
    unet = m.model.diffusion_model
    n_cls = arch.TINY_SEMANTIC_COND["in_channels"]
    maps = [torch.from_numpy(np.stack([SO.voronoi_labels(64, 96, n_cls, s), SO.voronoi_labels(64, 96, n_cls, s + 1)]))
            for s in (40, 50)]
    conds = [m.get_learned_conditioning(lab) for lab in maps]
    assert not torch.equal(conds[0], conds[1])
    g = torch.Generator(device=cuda_dev).manual_seed(5)
    x = torch.randn(2, 3, 16, 24, generator=g, device=cuda_dev)
    t = torch.tensor([700, 20], device=cuda_dev)
    unet.autotune = False           # both routes on the default GEMM plans
    eager = [m.apply_model(x, t, c) for c in conds]
    try:
        unet.use_cuda_graph = True
        unet._graphs.clear()
        graph = [m.apply_model(x, t, c) for c in conds + conds]
    finally:
        unet.use_cuda_graph, unet.autotune = False, True
        unet._graphs.clear()
    for i, e in enumerate(graph):
        assert torch.equal(e, eager[i % 2]), i
    assert not torch.equal(eager[0], eager[1])


@pytest.mark.parametrize("eta", [0, 1])
@pytest.mark.parametrize("graph", [False, True])
def test_tiny_ddim10_matches_reference(cuda_dev, monkeypatch, eta, graph):
    from sdb200.samplers import DDIMSampler
    e = golden("semantic.pt")["e2e"]
    Sc, m = _tiny_model(cuda_dev)
    assert torch.equal(m.alphas_cumprod.cpu(), golden("semantic.pt")["alphas_cumprod"])
    m.model.diffusion_model.use_cuda_graph = graph
    r = e[f"eta{eta}"]
    x_T = _gen((1, 3, 16, 16), e["x_T_seed"]).to(cuda_dev)
    draws = [_gen((1, 3, 16, 16), e["noise_seed"] + i) for i in range(r["n_noise"])]
    if eta:
        monkeypatch.setattr(torch, "randn_like", lambda t, *a, **k: draws.pop(0).to(t.device))
    labels = torch.from_numpy(SO.voronoi_labels(e["h"], e["w"], arch.TINY_SEMANTIC_COND["in_channels"],
                                                e["labels_seed"]))[None]
    with m.ema_scope():
        x, c, s = Sc.synthesize(m, DDIMSampler(m), labels, steps=10, eta=float(eta), x_T=x_T, return_latents=True)
    monkeypatch.undo()
    m.model.diffusion_model.use_cuda_graph = False
    assert not eta or not draws
    e_c, e_s, e_x = rel_l2(c, e["c"]), rel_l2(s, r["sample"]), rel_l2(x, r["x_dec"])
    # the decode of the reference's own latent; the decode of ours matches too where the nearest-codebook search picks
    # the same codes (a near tie flips a code, and with it a whole 4x4 block of the image)
    e_d = rel_l2(m.decode_first_stage(r["sample"].to(cuda_dev)), r["x_dec"])
    q = m.first_stage_model.quantize
    same_codes = torch.equal(q(s)[2][2], q(r["sample"].to(cuda_dev))[2][2])
    print(f"tiny e2e eta {eta} graph {graph}: conditioning {e_c:.2e}, DDIM-10 latent rel-L2 {e_s:.2e}, decoded "
          f"{e_x:.2e} (same codes {same_codes}), decode of the reference latent {e_d:.2e}")
    assert e_c <= 1e-6 and e_s < 1e-3 and e_d < 1e-3 and (e_x < 1e-3 or not same_codes)


_FULL = {}


def _full(dev):
    if "m" not in _FULL:
        Sc = script("semantic_synthesis")
        _FULL["m"] = (Sc, Sc.load_model(random_init=True, device=dev, image_size=128))
    return _FULL["m"]


def test_full_model_landscape_beyond_training_size(cuda_dev, monkeypatch):
    """A 256x512 map with the 512 config: latent (1, 3, 64, 128), 4 DDIM steps at eta 1 through the graph path, and one
    graph evaluation bit-equal to eager at that size (both on the default GEMM plans)."""
    from sdb200.samplers import DDIMSampler
    Sc, m = _full(cuda_dev)
    unet = m.model.diffusion_model
    lab = torch.from_numpy(SO.voronoi_labels(256, 512, 182, 31))[None]
    g = torch.Generator(device=cuda_dev).manual_seed(6)
    xt = torch.randn(1, 3, 64, 128, generator=g, device=cuda_dev)
    t = torch.tensor([500], device=cuda_dev)
    try:
        unet.use_cuda_graph, unet.autotune = True, False
        unet._graphs.clear()
        with m.ema_scope():
            x, c, s = Sc.synthesize(m, DDIMSampler(m), lab, steps=4, eta=1.0, return_latents=True)
        eps_g = m.apply_model(xt, t, c)
        unet.use_cuda_graph = False
        eps_e = m.apply_model(xt, t, c)
    finally:
        unet.use_cuda_graph, unet.autotune = False, True
        unet._graphs.clear()
    assert tuple(c.shape) == (1, 3, 64, 128) and tuple(s.shape) == (1, 3, 64, 128)
    assert tuple(x.shape) == (1, 3, 256, 512) and bool(torch.isfinite(x).all()) and bool(torch.isfinite(s).all())
    assert torch.equal(eps_g, eps_e)
    with pytest.raises(ValueError, match="multiples of 16"):
        Sc.synthesize(m, DDIMSampler(m), torch.zeros(1, 256, 200, dtype=torch.uint8), steps=1)


def test_script_writes_pngs(cuda_dev, tmp_path):
    from PIL import Image
    indir, outdir = tmp_path / "in", tmp_path / "out"
    indir.mkdir()
    Image.fromarray(SO.voronoi_labels(64, 64, 20, 1), mode="L").save(indir / "a.png")
    p = Image.fromarray(SO.voronoi_labels(32, 48, 20, 2), mode="L").convert("P")
    p.putdata(SO.voronoi_labels(32, 48, 20, 2).reshape(-1).tolist())
    p.save(indir / "b.png")
    Sc = script("semantic_synthesis")
    written = Sc.main(["--indir", str(indir), "--outdir", str(outdir), "--steps", "4", "--n_samples", "2",
                       "--random_init", "--tiny"])
    assert sorted(os.path.basename(q) for q in written) == ["a_00.png", "a_01.png", "b_00.png", "b_01.png"]
    assert Image.open(outdir / "a_01.png").size == (64, 64) and Image.open(outdir / "b_00.png").size == (48, 32)
    # the full 256 model from random weights, one map
    Image.fromarray(SO.voronoi_labels(64, 128, 182, 3), mode="L").save(tmp_path / "map.png")
    written = Sc.main([str(tmp_path / "map.png"), "--outdir", str(outdir), "--steps", "2", "--random_init"])
    assert Image.open(written[0]).size == (128, 64)


def test_every_plan_of_every_ss_gemm_problem(cuda_dev):
    from test_gemm_plans_gpu import catalogue, run_sweep
    problems = catalogue(GEMM_MODEL_WORKLOADS["semantic"], cuda_dev)
    print(f"\nsemantic-synthesis UNet (8, 3+3, 64²) and (1, 3+3, 128²): {len(problems)} distinct GEMM problems")
    assert problems
    run_sweep(problems, cuda_dev, "semantic")
    torch.cuda.empty_cache()
