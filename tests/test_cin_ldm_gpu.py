"""The class-conditional ImageNet LDM (cin256-v2; scripts/sample_imagenet.py) on the H100.

Single-head attention at d = 384 / 576 / 960 against fp64 (memory the kernel must not read holds NaN) and its
descriptor checks, the attn1 out-projection GEMM with FiLM and residual together (the one-token cross-attention fold)
against fp64, the ClassEmbedder, and the UNet, a guided DDIM trajectory and its VQ decode against the unmodified
reference (tests/golden/cin.pt)."""

import pytest
import torch

import helpers  # noqa: F401
from helpers import golden, rel_l2, script
from sdb200 import arch, pipeline

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
UCFG = {"tiny_cin": arch.TINY_CIN_UNET, "cin256": arch.CIN256_V2_UNET}
CCFG = {"tiny_cin": arch.TINY_CIN_COND, "cin256": arch.CIN256_V2_COND}
TOL = 1e-3
NAN = float("nan")
_models = {}


def _unet(tag, dev):
    import sdb200
    if tag not in _models:
        g = golden("cin.pt")
        _models[tag] = sdb200.UNetModel(**UCFG[tag]).load_weights(
            arch.random_state_dict(arch.unet_param_shapes(UCFG[tag]), g["unet_seed"]), dev)
    return _models[tag]


def _embedder(tag, dev):
    import sdb200
    key = "cond_" + tag
    if key not in _models:
        g = golden("cin.pt")
        cfg = CCFG[tag]
        _models[key] = sdb200.ClassEmbedder(**cfg).load_weights(
            arch.random_state_dict(arch.class_embedder_param_shapes(cfg), g["cond_seed"]), dev)
    return _models[key]


# ------------------------------------------------------------------------------------------------ wide attention
@pytest.mark.parametrize("nq,nkv", [(1024, 1024), (256, 256), (64, 64), (16, 16), (100, 37)])
@pytest.mark.parametrize("d", [384, 576, 960])
def test_single_head_attention_vs_fp64(cuda_dev, d, nq, nkv):
    from sdb200 import ops
    B = 3
    g = torch.Generator(device=cuda_dev).manual_seed(d + nq + nkv)
    rnd = lambda *s: torch.randn(*s, generator=g, device=cuda_dev).half()
    q, k, v = rnd(B, nq, d), rnd(B, nkv, d), rnd(B, nkv, d)
    # rows past nq / nkv and V^T columns past nkv hold NaN: the kernel must not let them reach the output
    qb = torch.full((B, nq + 16, d), NAN, dtype=torch.float16, device=cuda_dev)
    kb = torch.full((B, nkv + 16, d), NAN, dtype=torch.float16, device=cuda_dev)
    ld = (nkv + 7) // 8 * 8 + 8
    vt = torch.full((B, d, ld), NAN, dtype=torch.float16, device=cuda_dev)
    qb[:, :nq], kb[:, :nkv], vt[:, :, :nkv] = q, k, v.transpose(1, 2)
    wide = torch.full((B, nq + 4, d), NAN, dtype=torch.float16, device=cuda_dev)
    out = ops.attention(qb, kb, vt, heads=1, d=d, dpad=d, nq=nq, nkv=nkv, scale=d ** -0.5, out=wide[:, :nq])
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all()), "NaN the kernel must not read reached the output"
    assert bool(torch.isnan(wide[:, nq:]).all()), "rows past nq were written"
    s = torch.einsum("bid,bjd->bij", q.double(), k.double()) * d ** -0.5
    ref = torch.einsum("bij,bjd->bid", s.softmax(-1), v.double())
    err = rel_l2(out, ref)
    print(f"d={d} nq={nq} nkv={nkv}: rel-L2 {err:.2e}")
    assert err < 2e-3, err
    # head_stride = d (the packed layout) is the same kernel
    out2 = ops.attention(qb, kb, vt, heads=1, d=d, dpad=d, nq=nq, nkv=nkv, scale=d ** -0.5, head_stride=d)
    assert torch.equal(out2, out)


@pytest.mark.parametrize("bad", [dict(heads=2), dict(d=320), dict(causal=True), dict(d=448, dpad=448),
                                 dict(d=640, dpad=640), dict(head_stride=392)])
def test_single_head_attention_rejects_bad_descriptors(cuda_dev, bad):
    from sdb200 import lib, ops
    d = bad.get("dpad", 384)
    a = dict(heads=1, d=384, dpad=d, nq=64, nkv=64, scale=1.0, causal=False, head_stride=0)
    a.update(bad)
    h = a["heads"]
    q = torch.zeros(1, 64, h * d, dtype=torch.float16, device=cuda_dev)
    vt = torch.zeros(1, h * d, 64, dtype=torch.float16, device=cuda_dev)
    torch.cuda.synchronize()
    n0 = int(lib.load().sdb_launch_count())
    with pytest.raises(RuntimeError, match="sdb_attention"):
        ops.attention(q, q, vt, **a)
    assert int(lib.load().sdb_launch_count()) == n0, "a rejected descriptor launched a kernel"


# ------------------------------------------------------------------------------------------------ FiLM + residual GEMM
@pytest.mark.parametrize("ch", [384, 576, 960])
@pytest.mark.parametrize("nb,ntok", [(12, 1024), (12, 256), (12, 64), (4, 16), (2, 192), (2, 48), (2, 12)])
def test_out_projection_with_film_and_residual(cuda_dev, ch, nb, ntok):
    """t2 = o W^T + b + u[sample] + t0: the attn1 out-projection carrying the one-token cross-attention vector u (a
    column slice of the stacked [nb, sum ch] buffer) as FiLM, next to the residual, against fp64."""
    from sdb200 import ops
    g = torch.Generator().manual_seed(ch + nb + ntok)
    M = nb * ntok
    o = torch.randn(M, ch, generator=g).half().to(cuda_dev)
    w = (torch.randn(ch, ch, generator=g) * ch ** -0.5).half().to(cuda_dev)
    b = (0.1 * torch.randn(ch, generator=g)).to(cuda_dev)
    ubuf = torch.randn(nb, 10560, generator=g).to(cuda_dev)
    u = ubuf[:, 1344: 1344 + ch]
    t0 = torch.randn(M, ch, generator=g).to(cuda_dev)
    _, t2 = ops.gemm(o, w, bias=b, film=u, rows_per_sample=ntok, residual=t0, want_f32=True, splits=-1)
    ref = o.double() @ w.double().T + b.double() + u.double().repeat_interleave(ntok, 0) + t0.double()
    assert rel_l2(t2, ref) < 1e-5, rel_l2(t2, ref)


# ------------------------------------------------------------------------------------------------ ClassEmbedder
def test_class_embedder_rows_and_label_checks(cuda_dev):
    import sdb200
    m = _embedder("cin256", cuda_dev)
    labels = torch.tensor([25, 187, 448, 992, 1000, 0])
    c = m({"class_label": labels.to(cuda_dev)})
    table = arch.random_state_dict(arch.class_embedder_param_shapes(arch.CIN256_V2_COND), golden("cin.pt")["cond_seed"])
    assert c.shape == (6, 1, 512) and c.dtype == torch.float32
    assert torch.equal(c.cpu(), table["embedding.weight"][labels][:, None])
    assert torch.equal(m({"x": labels}, key="x").cpu(), c.cpu())          # host labels, explicit key
    for bad in (-1, 1001):
        with pytest.raises(IndexError):
            m({"class_label": torch.tensor([3, bad], device=cuda_dev)})
    assert isinstance(m, sdb200.ClassEmbedder)


# ------------------------------------------------------------------------------------------------ models vs reference
def _case_inputs(case, dev):
    return case["x"].to(dev), case["t"].to(dev), case["c"].to(dev)


@pytest.mark.parametrize("idx", range(5))
def test_unet_vs_reference(cuda_dev, idx):
    case = golden("cin.pt")["unet"][idx]
    net = _unet(case["cfg"], cuda_dev)
    x, t, c = _case_inputs(case, cuda_dev)
    eps = net(x, t, context=c)
    err = rel_l2(eps, case["eps"])
    print(f"unet {case['cfg']} {tuple(case['x'].shape)} rel-L2 {err:.3e}")
    assert eps.shape == case["eps"].shape and err < TOL


def test_cin256_graph_autotune_c_handle_and_class_switch(cuda_dev):
    """Graph replay (with autotuning) and the C handle equal the eager forward bit for bit; after switching to another
    class batch, replay equals eager on the new classes (the one-token vectors u live in static buffers)."""
    import sdb200
    g = golden("cin.pt")
    case = g["unet"][2]
    assert case["cfg"] == "cin256" and tuple(case["x"].shape) == (2, 3, 32, 32)
    net = sdb200.UNetModel(**arch.CIN256_V2_UNET).load_weights(
        arch.random_state_dict(arch.unet_param_shapes(arch.CIN256_V2_UNET), g["unet_seed"]), cuda_dev)
    emb = _embedder("cin256", cuda_dev)
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
    c2 = emb({"class_label": torch.tensor([1000, 7], device=cuda_dev)})
    net.use_cuda_graph = True
    replay2 = net(x, t, context=c2).clone()
    net.use_cuda_graph = False
    eager2 = net(x, t, context=c2)
    assert torch.equal(replay2, eager2) and not torch.equal(eager2, eager)


def _tiny_model(dev):
    from sdb200.util import instantiate_from_config, remap_config
    g = golden("cin.pt")
    node = script("sample_imagenet").cin_config(arch.TINY_CIN_UNET, arch.TINY_VQ, arch.TINY_CIN_COND)
    m = instantiate_from_config(remap_config(node))
    return pipeline.load_random_weights(m, dev, seeds=(g["unet_seed"], g["vq_seed"], g["cond_seed"])).eval()


def test_guided_ddim_trajectory_and_decode(cuda_dev):
    """DDIM-10, eta 0, scale 3.0 with the label-1000 unconditional conditioning (the notebook's sampling cell) on the
    tiny model, then decode_first_stage through the tiny VQ."""
    from sdb200.samplers import DDIMSampler
    d = golden("cin.pt")["ddim"]
    m = _tiny_model(cuda_dev)
    assert torch.equal(m.alphas_cumprod.cpu(), d["alphas_cumprod"])
    with m.ema_scope():
        c = m.get_learned_conditioning({m.cond_stage_key: d["classes"].to(cuda_dev)})
        uc = m.get_learned_conditioning({m.cond_stage_key: torch.full_like(d["classes"], 1000).to(cuda_dev)})
        s, _ = DDIMSampler(m).sample(10, batch_size=d["x_T"].shape[0], shape=list(d["x_T"].shape[1:]), conditioning=c,
                                     unconditional_guidance_scale=3.0, unconditional_conditioning=uc, eta=0.0,
                                     verbose=False, x_T=d["x_T"].to(cuda_dev))
    e_s = rel_l2(s, d["sample"])
    e_dec = rel_l2(m.decode_first_stage(d["sample"].to(cuda_dev)), d["x_dec"])
    print(f"guided ddim S=10 trajectory {e_s:.2e}; decode_first_stage {e_dec:.2e}")
    assert e_s < 5e-2 and e_dec < 2e-3


def test_sample_imagenet_script_random_init(cuda_dev, tmp_path):
    mod = script("sample_imagenet")
    path = mod.main(["--random_init", "--tiny", "--outdir", str(tmp_path), "--classes", "25", "187",
                     "--n_samples_per_class", "2", "--ddim_steps", "4"])
    from PIL import Image
    img = Image.open(path)
    assert img.size == (2 * 34 + 2, 2 * 34 + 2)
