"""The class-conditional ImageNet LDM-VQ-8 (models/ldm/cin256; scripts/sample_imagenet.py --model cin256) on the H100.

Multi-head d = 32 attention at the UNet's head counts and token counts against fp64 (memory the kernel must not read
holds NaN), the UNet, the VQ-f8 first stage with its level attention and the quantizer against the unmodified reference
(tests/golden/cin_f8.pt) or fp64, graph replay and the C handle against eager, unguided DDIM trajectories on EMA
weights, every GEMM tile plan of the model's GEMM problems, and the sampling script."""

import pytest
import torch

import helpers  # noqa: F401
from helpers import golden, rel_l2, script
from sdb200 import arch, ops, pipeline
from workloads import GEMM_MODEL_WORKLOADS

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
UCFG = {"tiny": arch.TINY_CIN_F8_UNET, "cin256": arch.CIN256_F8_UNET}
CCFG = {"tiny": arch.TINY_CIN_F8_COND, "cin256": arch.CIN256_F8_COND}
VCFG = {"tiny": arch.TINY_VQ_F8, "vq_f8": arch.VQ_F8}
TOL = 1e-3
NAN = float("nan")
_models = {}


def _gen(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def _sub(x, g):
    """The pixels the golden stores of a decoded image: every g["image_stride"]-th in both directions."""
    k = g["image_stride"]
    return x[..., ::k, ::k]


def _unet(tag, dev):
    import sdb200
    if tag not in _models:
        g = golden("cin_f8.pt")
        _models[tag] = sdb200.UNetModel(**UCFG[tag]).load_weights(
            arch.random_state_dict(arch.unet_param_shapes(UCFG[tag]), g["unet_seed"]), dev)
    return _models[tag]


def _vq(tag, dev):
    import sdb200
    key = "vq_" + tag
    if key not in _models:
        g = golden("cin_f8.pt")
        _models[key] = sdb200.VQModelInterface(**VCFG[tag]).load_weights(
            arch.random_state_dict(arch.vq_param_shapes(VCFG[tag]), g["vq_seed"]), dev)
    return _models[key]


# ------------------------------------------------------------------------------------------------ d = 32 attention
@pytest.mark.parametrize("heads,n", [(8, 1024), (16, 256), (32, 64), (4, 48)])
def test_multihead_d32_attention_vs_fp64(cuda_dev, heads, n):
    """The spatial transformers' self-attention layout: Q | K side by side in one [B, n, 2 hd] buffer with heads at
    stride 32, V^T [B, hd, ld]. Rows past n, columns past 2 hd and V^T columns past n hold NaN."""
    B, d = 3, 32
    hd = heads * d
    g = torch.Generator(device=cuda_dev).manual_seed(heads * 1000 + n)
    rnd = lambda *s: torch.randn(*s, generator=g, device=cuda_dev).half()
    q, k, v = rnd(B, n, hd), rnd(B, n, hd), rnd(B, n, hd)
    qk = torch.full((B, n + 16, 2 * hd + 64), NAN, dtype=torch.float16, device=cuda_dev)
    qk[:, :n, :hd], qk[:, :n, hd:2 * hd] = q, k
    ld = (n + 7) // 8 * 8 + 8
    vt = torch.full((B, hd, ld), NAN, dtype=torch.float16, device=cuda_dev)
    vt[:, :, :n] = v.transpose(1, 2)
    wide = torch.full((B, n + 4, hd), NAN, dtype=torch.float16, device=cuda_dev)
    out = ops.attention(qk[:, :, :hd], qk[:, :, hd:2 * hd], vt, heads=heads, d=d, dpad=64, nq=n, nkv=n, scale=d ** -0.5,
                        head_stride=d, out=wide[:, :n])
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all()), "NaN the kernel must not read reached the output"
    assert bool(torch.isnan(wide[:, n:]).all()), "rows past nq were written"
    sp = lambda t: t.double().view(B, n, heads, d).transpose(1, 2)
    s = torch.einsum("bhid,bhjd->bhij", sp(q), sp(k)) * d ** -0.5
    ref = torch.einsum("bhij,bhjd->bhid", s.softmax(-1), sp(v)).transpose(1, 2).reshape(B, n, hd)
    err = rel_l2(out, ref)
    print(f"heads={heads} n={n} d=32: rel-L2 {err:.2e}")
    assert err < 2e-3, err


# ------------------------------------------------------------------------------------------------ UNet
def _case_inputs(case, dev):
    return _gen(case["shape"], case["x_seed"]).to(dev), case["t"].to(dev), case["c"].to(dev)


@pytest.mark.parametrize("idx", range(5))
def test_unet_vs_reference(cuda_dev, idx):
    case = golden("cin_f8.pt")["unet"][idx]
    net = _unet(case["cfg"], cuda_dev)
    x, t, c = _case_inputs(case, cuda_dev)
    eps = net(x, t, context=c)
    err = rel_l2(eps, case["eps"])
    print(f"unet {case['cfg']} {tuple(case['shape'])} rel-L2 {err:.3e}")
    assert eps.shape == case["eps"].shape and err < TOL


def test_cin256_graph_autotune_c_handle_and_class_switch(cuda_dev):
    """Graph replay (with autotuning) and the C handle equal the eager forward bit for bit; a new class batch refreshes
    the one-token vectors u in the captured graph's static buffers."""
    import sdb200
    g = golden("cin_f8.pt")
    case = g["unet"][2]
    assert case["cfg"] == "cin256" and tuple(case["shape"]) == (2, 4, 32, 32)
    net = sdb200.UNetModel(**arch.CIN256_F8_UNET).load_weights(
        arch.random_state_dict(arch.unet_param_shapes(arch.CIN256_F8_UNET), g["unet_seed"]), cuda_dev)
    emb = sdb200.ClassEmbedder(**arch.CIN256_F8_COND).load_weights(
        arch.random_state_dict(arch.class_embedder_param_shapes(arch.CIN256_F8_COND), g["cond_seed"]), cuda_dev)
    x, t, c = _case_inputs(case, cuda_dev)
    t = t.float()
    net.use_cuda_graph = True
    first = net(x, t, context=c).clone()
    replay = net(x, t, context=c)
    net.use_cuda_graph = False
    eager = net(x, t, context=c)
    h = net.c_handle(tuple(x.shape), c)
    try:
        out = h.forward(x, t)
        torch.cuda.synchronize()
        print(f"cin256 graph {rel_l2(replay, case['eps']):.3e} C handle {rel_l2(out, case['eps']):.3e}")
        assert torch.equal(first, replay) and torch.equal(replay, eager) and torch.equal(out, eager)
        assert rel_l2(replay, case["eps"]) < TOL
    finally:
        h.close()
    c2 = emb({"class_label": torch.tensor([3, 7], device=cuda_dev)})
    net.use_cuda_graph = True
    replay2 = net(x, t, context=c2).clone()
    net.use_cuda_graph = False
    eager2 = net(x, t, context=c2)
    assert torch.equal(replay2, eager2) and not torch.equal(eager2, eager)
    with pytest.raises(IndexError):          # n_classes 1000: there is no label 1000
        emb({"class_label": torch.tensor([1000], device=cuda_dev)})


# ------------------------------------------------------------------------------------------------ first stage
@pytest.mark.parametrize("idx", range(4))
def test_vq_f8_decode_vs_reference(cuda_dev, idx):
    """Quantize + post_quant_conv + decoder; the full stage runs its 32x32 level attention (1024 tokens, and 768 for the
    16x48 latent) in the d = 512 flash kernel, the tiny one both attention paths."""
    g = golden("cin_f8.pt")
    case = g["decode"][idx]
    m = _vq(case["cfg"], cuda_dev)
    h = _gen(case["shape"], case["seed"])
    x = m.decode(h.to(cuda_dev))
    err = rel_l2(_sub(x, g), case["x"])
    same = torch.equal(m.quantize(h.to(cuda_dev))[2][2].cpu(),
                       torch.cdist(h.permute(0, 2, 3, 1).reshape(-1, 4).double(),
                                   m._host_sd["quantize.embedding.weight"].double()).argmin(1))
    print(f"decode {case['cfg']} {tuple(case['shape'])}: rel-L2 {err:.2e} (codes equal the fp64 argmin: {same})")
    assert tuple(x.shape) == tuple(case["x_shape"]) and err < 2e-3


@pytest.mark.parametrize("idx", range(2))
def test_vq_f8_encode_vs_reference(cuda_dev, idx):
    case = golden("cin_f8.pt")["encode"][idx]
    m = _vq(case["cfg"], cuda_dev)
    h = m.encode(_gen(case["shape"], case["seed"]).clamp(-1, 1).to(cuda_dev))
    err = rel_l2(h, case["h"])
    print(f"encode {case['cfg']} {tuple(case['shape'])}: rel-L2 {err:.2e}")
    assert h.shape == case["h"].shape and err < 2e-3


def test_quantizer_indices_vs_fp64(cuda_dev):
    """16384 x 4 codebook: indices equal the fp64 argmin wherever the best distance leads the runner-up by more than
    fp32 rounding can swap."""
    m = _vq("vq_f8", cuda_dev)
    e = m._host_sd["quantize.embedding.weight"].double()
    z = _gen((4, 4, 32, 48), 77) * 1.5
    _, _, (_, _, idx) = m.quantize(z.to(cuda_dev))
    d = torch.cdist(z.permute(0, 2, 3, 1).reshape(-1, 4).double(), e) ** 2
    top = d.topk(2, dim=1, largest=False)
    clear = (top.values[:, 1] - top.values[:, 0]) > 1e-4 * (1 + top.values[:, 0])
    print(f"quantizer: {int(clear.sum())} of {clear.numel()} rows away from near-ties")
    assert int(clear.sum()) > 0.95 * clear.numel()
    assert torch.equal(idx.cpu()[clear], top.indices[clear, 0])


# ------------------------------------------------------------------------------------------------ sampling
def _tiny_model(dev):
    from sdb200.util import instantiate_from_config, remap_config
    g = golden("cin_f8.pt")
    node = script("sample_imagenet").cin256_f8_config(arch.TINY_CIN_F8_UNET, arch.TINY_VQ_F8, arch.TINY_CIN_F8_COND)
    m = pipeline.load_random_weights(instantiate_from_config(remap_config(node)), dev,
                                     seeds=(g["unet_seed"], g["vq_seed"], g["cond_seed"]))
    m.model.diffusion_model.set_weight_set("ema", arch.random_state_dict(arch.unet_param_shapes(arch.TINY_CIN_F8_UNET),
                                                                         g["ema_seed"]))
    return m.eval()


@pytest.mark.parametrize("eta", [0, 1])
@pytest.mark.parametrize("graph", [False, True])
def test_tiny_unguided_ddim10_matches_reference(cuda_dev, monkeypatch, eta, graph):
    """DDIM-10 without guidance inside ema_scope() (the EMA set differs from the raw weights), the reference's noise
    draws replayed at eta 1, then decode_first_stage."""
    from sdb200.samplers import DDIMSampler
    g = golden("cin_f8.pt")
    d = g["ddim"]
    r = d[f"eta{eta}"]
    m = _tiny_model(cuda_dev)
    assert torch.equal(m.alphas_cumprod.cpu(), g["alphas_cumprod"])
    m.model.diffusion_model.use_cuda_graph = graph
    x_T = _gen((2, 4, 16, 16), d["x_T_seed"]).to(cuda_dev)
    draws = [_gen((2, 4, 16, 16), d["noise_seed"] + i) for i in range(r["n_noise"])]
    if eta:
        monkeypatch.setattr(torch, "randn_like", lambda t, *a, **k: draws.pop(0).to(t.device))
    with m.ema_scope():
        c = m.get_learned_conditioning({m.cond_stage_key: d["classes"].to(cuda_dev)})
        s, _ = DDIMSampler(m).sample(10, batch_size=2, shape=[4, 16, 16], conditioning=c, eta=float(eta), verbose=False,
                                     x_T=x_T)
    monkeypatch.undo()
    m.model.diffusion_model.use_cuda_graph = False
    assert not eta or not draws
    e_s = rel_l2(s, r["sample"])
    e_d = rel_l2(_sub(m.decode_first_stage(r["sample"].to(cuda_dev)), g), r["x_dec"])
    print(f"tiny unguided DDIM-10 eta {eta} graph {graph}: latent rel-L2 {e_s:.2e}; decode of the reference latent {e_d:.2e}")
    assert e_s < 1e-3 and e_d < 2e-3


def test_sample_imagenet_script_cin256_tiny(cuda_dev, tmp_path):
    mod = script("sample_imagenet")
    path = mod.main(["--model", "cin256", "--random_init", "--tiny", "--outdir", str(tmp_path), "--classes", "25", "187",
                     "--n_samples_per_class", "2", "--ddim_steps", "4"])
    from PIL import Image
    assert Image.open(path).size == (2 * 130 + 2, 2 * 130 + 2)     # 16x16 latents -> 128x128 images through VQ-f8


# ------------------------------------------------------------------------------------------------ GEMM plans
def test_every_plan_of_every_cin256_gemm_problem(cuda_dev):
    """The cin256 UNet at (6, 4, 32, 32) (the unguided batch of bench_cin.py) and the VQ-f8 decoder at 256²."""
    from test_gemm_plans_gpu import catalogue, run_sweep
    problems = catalogue(GEMM_MODEL_WORKLOADS["cin256_f8"], cuda_dev)
    print(f"\ncin256 UNet (6, 4, 32²) and VQ-f8 decoder (1, 4, 32²): {len(problems)} distinct GEMM problems")
    assert problems
    run_sweep(problems, cuda_dev, "cin256")
    torch.cuda.empty_cache()
