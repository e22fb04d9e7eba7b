"""The VQ-f4 latent diffusion models (CelebA-HQ, FFHQ, LSUN-Bedrooms; scripts/sample_diffusion.py) on the H100.

GEMM A sources whose width is a multiple of 32 but not of 64 (224, 672, ...: the last 64-wide K step reads TMA's
out-of-bounds zeros, packed weights carry zero columns) against fp64 torch, GroupNorm at 7 / 21 / 49 channels per group,
the AttentionBlock at 14 / 21 / 28 heads of d = 32, the vector quantizer (sdb_vq_quantize) against the fp64 argmin, and
the UNet, VQ decode / encode and a DDIM trajectory against the unmodified reference (tests/golden/vq.pt)."""
import os

import pytest
import torch
import torch.nn.functional as F
import yaml

import helpers  # noqa: F401
from helpers import golden, rel_l2, script
from sdb200 import arch, pipeline

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
UCFG = {"tiny_vq": arch.TINY_VQ_UNET, "celebahq": arch.CELEBAHQ_UNET}
VCFG = {"tiny_vq": arch.TINY_VQ, "vq_f4": arch.VQ_F4}
TOL = 1e-3
_models = {}


def _r16(shape, dev, g, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).half().to(dev)


def _unet(tag, dev):
    import sdb200
    if tag not in _models:
        _models[tag] = sdb200.UNetModel(**UCFG[tag]).load_weights(
            arch.random_state_dict(arch.unet_param_shapes(UCFG[tag]), 11), dev)
    return _models[tag]


def _vq(tag, dev):
    import sdb200
    key = "vq_" + tag
    if key not in _models:
        _models[key] = sdb200.VQModelInterface(**VCFG[tag]).load_weights(
            arch.random_state_dict(arch.vq_param_shapes(VCFG[tag]), 12), dev)
    return _models[key]


# ------------------------------------------------------------------------------------------------ GEMM at 32-aligned K
@pytest.mark.parametrize("c", [32, 96, 224, 288, 672])
@pytest.mark.parametrize("nb,h,w,n", [(2, 16, 16, 224), (2, 8, 12, 96)])
def test_conv3x3_32_aligned_width(cuda_dev, c, nb, h, w, n):
    """3x3 conv with bias + FiLM + residual and fused statistics at sg = 1, weights packed per tap with zero tails."""
    from sdb200 import ops
    from sdb200.unet import _pack_conv3
    g = torch.Generator().manual_seed(c + h + n)
    x = _r16((nb, h, w, c), cuda_dev, g)
    wt = torch.randn(n, c, 3, 3, generator=g) * (9 * c) ** -0.5
    bias = torch.randn(n, generator=g).to(cuda_dev)
    film = torch.randn(nb, n, generator=g).to(cuda_dev)
    res = torch.randn(nb * h * w, n, generator=g).to(cuda_dev)
    wk = _pack_conv3(wt.to(cuda_dev))
    assert wk.shape == (n, 9 * ((c + 63) // 64 * 64))
    _, o32 = ops.gemm(x, wk, taps=9, bias=bias, film=film, residual=res, want_f32=True, splits=-1, want_stats=True,
                      stats_group=1)
    ref = F.conv2d(x.double().cpu().permute(0, 3, 1, 2), wt.half().double(), bias.double().cpu(), padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, n) + film.double().cpu().repeat_interleave(h * w, 0) + res.double().cpu()
    assert rel_l2(o32, ref) < 1e-5, rel_l2(o32, ref)
    gamma = (1 + 0.1 * torch.randn(n, generator=g)).to(cuda_dev)
    beta = (0.1 * torch.randn(n, generator=g)).to(cuda_dev)
    y, _ = ops.groupnorm(o32.view(nb, h, w, n), gamma, beta, eps=1e-5, silu=True)
    yr = F.silu(F.group_norm(ref.reshape(nb, h, w, n).permute(0, 3, 1, 2), 32, gamma.double().cpu(),
                             beta.double().cpu(), 1e-5)).permute(0, 2, 3, 1)
    assert rel_l2(y, yr) < 6e-4


@pytest.mark.parametrize("c", [224, 288, 672])
@pytest.mark.parametrize("shift", [0, 1])
def test_conv3x3_stride2_32_aligned_width(cuda_dev, c, shift):
    from sdb200 import ops
    from sdb200.unet import _pack_conv3
    g = torch.Generator().manual_seed(c + shift)
    nb, h, w, n = 2, 16, 12, c
    x = _r16((nb, h, w, c), cuda_dev, g)
    wt = torch.randn(n, c, 3, 3, generator=g) * (9 * c) ** -0.5
    bias = torch.randn(n, generator=g).to(cuda_dev)
    _, o32 = ops.gemm(x, _pack_conv3(wt.to(cuda_dev)), taps=9, conv_stride=2, conv_shift=shift, bias=bias,
                      want_f32=True, splits=-1)
    xin = x.double().cpu().permute(0, 3, 1, 2)
    wd = wt.half().double()
    ref = F.conv2d(F.pad(xin, (0, 1, 0, 1)), wd, bias.double().cpu(), stride=2) if shift else \
        F.conv2d(xin, wd, bias.double().cpu(), stride=2, padding=1)
    assert rel_l2(o32, ref.permute(0, 2, 3, 1).reshape(-1, n)) < 1e-5


@pytest.mark.parametrize("c", [32, 96, 224, 288, 672])
def test_1x1_and_hilo_32_aligned_width(cuda_dev, c):
    """Plain 1x1 (B exactly c wide) and the hi/lo triple [A_hi | A_lo | A_hi] . [W_hi | W_hi | W_lo] of the skip
    connections (each source padded to whole 64-wide K steps)."""
    from sdb200 import ops
    from sdb200.unet import _hilo, _pack_hilo_1x1
    g = torch.Generator().manual_seed(c)
    M, n = 700, 448
    a32 = torch.randn(M, c, generator=g).to(cuda_dev)
    w = (torch.randn(n, c, generator=g) * c ** -0.5).to(cuda_dev)
    bias = torch.randn(n, generator=g).to(cuda_dev)
    _, o = ops.gemm(a32.half(), w.half().contiguous(), bias=bias, want_f32=True, splits=-1)
    assert rel_l2(o, a32.half().double() @ w.half().double().T + bias.double()) < 1e-5
    hi, lo = _hilo(a32)
    _, o3 = ops.gemm(hi, _pack_hilo_1x1(w), a1=lo, a2=hi, bias=bias, want_f32=True, splits=-1)
    assert rel_l2(o3, a32.double() @ w.double().T + bias.double()) < 1e-5


@pytest.mark.parametrize("c0,c1", [(448, 224), (288, 192), (224, 224)])
def test_two_source_concat(cuda_dev, c0, c1):
    """3x3 conv over a two-source concat (a skip join read straight from both tensors)."""
    from sdb200 import ops
    from sdb200.unet import _pad64
    g = torch.Generator().manual_seed(c0 + c1)
    nb, h, w, n = 2, 8, 16, 224
    x0, x1 = _r16((nb, h, w, c0), cuda_dev, g), _r16((nb, h, w, c1), cuda_dev, g)
    wt = torch.randn(n, c0 + c1, 3, 3, generator=g) * (9 * (c0 + c1)) ** -0.5
    wk = wt.permute(0, 2, 3, 1)
    wk = torch.cat([_pad64(wk[..., :c0]), _pad64(wk[..., c0:])], -1).reshape(n, -1).half().contiguous().to(cuda_dev)
    _, o32 = ops.gemm(x0, wk, a1=x1, taps=9, want_f32=True)
    xin = torch.cat([x0, x1], -1).double().cpu().permute(0, 3, 1, 2)
    ref = F.conv2d(xin, wt.half().double(), padding=1).permute(0, 2, 3, 1).reshape(-1, n)
    assert rel_l2(o32, ref) < 1e-5


@pytest.mark.parametrize("bn,pair,sp,mode", [(128, 2, 1, 0), (128, 2, 2, 2), (160, 1, 4, 2), (0, 1, 3, 1),
                                              (0, 1, 2, 1)])
def test_pairs_and_splitk_at_672(cuda_dev, bn, pair, sp, mode):
    """CTA pairs, cluster split-K and workspace split-K with K = 9 x 704 (672 channels), fused statistics at sg = 1."""
    from sdb200 import ops
    from sdb200.unet import _pack_conv3
    g = torch.Generator().manual_seed(bn + pair + sp + mode)
    nb, h, w, c, n = 2, 16, 16, 672, 448
    x = _r16((nb, h, w, c), cuda_dev, g)
    wt = torch.randn(n, c, 3, 3, generator=g) * (9 * c) ** -0.5
    res = torch.randn(nb * h * w, n, generator=g).to(cuda_dev)
    _, o32 = ops.gemm(x, _pack_conv3(wt.to(cuda_dev)), taps=9, residual=res, want_f32=True, block_n=bn, pair=pair,
                      splits=sp, splitk_mode=mode, want_stats=True, stats_group=1)
    ref = F.conv2d(x.double().cpu().permute(0, 3, 1, 2), wt.half().double(), padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, n) + res.double().cpu()
    assert rel_l2(o32, ref) < 1e-5
    assert ops.channel_stats(o32) is not None
    y, _ = ops.groupnorm(o32.view(nb, h, w, n), torch.ones(n, device=cuda_dev), torch.zeros(n, device=cuda_dev))
    yr = F.group_norm(ref.reshape(nb, h, w, n).permute(0, 3, 1, 2), 32, eps=1e-5).permute(0, 2, 3, 1)
    assert rel_l2(y, yr) < 6e-4


def test_dynamic_b_vt_gemm_k672(cuda_dev):
    """The AttentionBlock's V^T = W_v . x^T with x as a dynamic B exactly 672 wide (tail zero-filled by TMA)."""
    from sdb200 import ops
    g = torch.Generator().manual_seed(672)
    M, c, hd = 2 * 256, 672, 21 * 64
    xm = _r16((M, c), cuda_dev, g)
    wv = _r16((hd, c), cuda_dev, g, c ** -0.5)
    vt, _ = ops.gemm(wv, xm, want_f16=True, b_dynamic=True)
    assert rel_l2(vt.float(), wv.double() @ xm.double().T) < 6e-4


@pytest.mark.parametrize("c0,c1", [(224, 0), (672, 0), (448, 224), (896, 672)])
@pytest.mark.parametrize("fused", [False, True])
def test_groupnorm_odd_channels_per_group(cuda_dev, c0, c1, fused):
    """GroupNorm(32) at 7, 21, 21 and 49 channels per group, statistics computed or taken from the producing GEMMs."""
    from sdb200 import ops
    from sdb200.unet import _pack_conv3
    g = torch.Generator().manual_seed(c0 + c1 + fused)
    nb, h, w = 2, 8, 8

    def make(c):
        if not fused:
            return (torch.randn(nb, h, w, c, generator=g) * 2 + 0.5).to(cuda_dev)
        x = _r16((nb, h, w, 64), cuda_dev, g)
        wt = (torch.randn(c, 64, 3, 3, generator=g) * 0.05).to(cuda_dev)
        _, o = ops.gemm(x, _pack_conv3(wt), taps=9, want_f32=True, want_stats=True, stats_group=1)
        assert ops.channel_stats(o) is not None
        return o.view(nb, h, w, c)
    x0 = make(c0)
    x1 = make(c1) if c1 else None
    C = c0 + c1
    gamma = (1 + 0.1 * torch.randn(C, generator=g)).to(cuda_dev)
    beta = (0.1 * torch.randn(C, generator=g)).to(cuda_dev)
    y, _ = ops.groupnorm(x0, gamma, beta, x1=x1, eps=1e-5, silu=True)
    cat = x0 if x1 is None else torch.cat([x0, x1], -1)
    yr = F.silu(F.group_norm(cat.double().permute(0, 3, 1, 2), 32, gamma.double(), beta.double(), 1e-5)).permute(0, 2, 3, 1)
    assert rel_l2(y, yr) < 6e-4


@pytest.mark.parametrize("heads,hw", [(14, (16, 16)), (21, (8, 8)), (28, (4, 4)), (21, (2, 6))])
def test_attention_block_heads_of_32(cuda_dev, heads, hw):
    """UNetModel._attn (qkv GEMM at K = ch, flash kernel with d = 32 in 64-wide head slots, proj_out) against the
    QKVAttentionLegacy formula in fp64."""
    import sdb200
    ch = heads * 32
    cfg = dict(arch.TINY_VQ_UNET)
    net = sdb200.UNetModel(**cfg)
    g = torch.Generator().manual_seed(heads)
    sd = {"norm.weight": 1 + 0.1 * torch.randn(ch, generator=g), "norm.bias": 0.1 * torch.randn(ch, generator=g),
          "qkv.weight": torch.randn(3 * ch, ch, 1, generator=g) * ch ** -0.5, "qkv.bias": 0.1 * torch.randn(3 * ch, generator=g),
          "proj_out.weight": torch.randn(ch, ch, 1, generator=g) * ch ** -0.5, "proj_out.bias": 0.1 * torch.randn(ch, generator=g)}
    net._host_sd = {**arch.random_state_dict(arch.unet_param_shapes(cfg), 11), **{"blk." + k: v for k, v in sd.items()}}
    net.plan = {**net.plan, "middle": [("attn", "blk", dict(ch=ch, heads=heads, dhead=32))]}
    net.pack_weights(cuda_dev)
    s = net.W["middle"][0][1]
    nb, (H, W) = 2, hw
    x = (torch.randn(nb, H, W, ch, generator=g)).to(cuda_dev)
    out = net._attn(s, x)
    import uncond_oracle as U
    sdd = {"blk." + k: v.double() for k, v in sd.items()}
    ref = U.attention_block(sdd, "blk", x.double().cpu().permute(0, 3, 1, 2), heads).permute(0, 2, 3, 1)
    assert rel_l2(out, ref) < 2e-3, rel_l2(out, ref)


# ------------------------------------------------------------------------------------------------ vector quantizer
def _vq_check(z, cb, scale, zq, idx):
    """Indices equal the fp64 argmin of the same formula wherever the runner-up is more than 1e-6 relative away; z_q is
    bit-equal to z + (e - z) in fp32 for the chosen index."""
    zs = (z.to(cb.device).float() * scale).reshape(-1, cb.shape[1])
    ed = cb.double()
    vals, inds = [], []
    for r in range(0, zs.shape[0], 2048):          # fp64 distances in row blocks, on the device
        zd = zs[r: r + 2048].double()
        top = ((zd ** 2).sum(1, keepdim=True) + (ed ** 2).sum(1) - 2 * zd @ ed.T).topk(2, dim=1, largest=False)
        vals.append(top.values.cpu())
        inds.append(top.indices[:, 0].cpu())
    vals, first = torch.cat(vals), torch.cat(inds)
    clear = (vals[:, 1] - vals[:, 0]) > 1e-6 * vals[:, 1].abs().clamp_min(1e-30)
    idx = idx.cpu()
    assert clear.float().mean() > 0.9
    assert torch.equal(idx[clear], first[clear])
    zs = zs.cpu()
    e = cb.cpu()[idx]
    assert torch.equal(zq.cpu().reshape(-1, cb.shape[1]), zs + (e - zs))


@pytest.mark.parametrize("n_e,e_dim,m", [(8192, 3, 10 * 64 * 64), (16384, 4, 3 * 32 * 32), (512, 3, 2 * 96), (700, 8, 333)])
def test_vq_quantize_vs_fp64_argmin(cuda_dev, n_e, e_dim, m):
    from sdb200 import ops
    g = torch.Generator().manual_seed(n_e + e_dim)
    cb = torch.randn(n_e, e_dim, generator=g).to(cuda_dev)
    z = (torch.randn(m, e_dim, generator=g) * 1.3).to(cuda_dev)
    code_sq = (cb.double() ** 2).sum(1).float()
    scale = 1.0 / 0.37
    zq, idx = ops.vq_quantize(z, cb, code_sq, scale=scale, want_indices=True)
    _vq_check(z, cb, scale, zq, idx)
    assert torch.equal(ops.vq_quantize(z, cb, code_sq, scale=scale), zq)


def test_vq_quantize_duplicate_codes_take_the_first_index(cuda_dev):
    from sdb200 import ops
    g = torch.Generator().manual_seed(3)
    cb = torch.randn(3000, 3, generator=g)
    cb[2500] = cb[17]
    cb[1200:2200] = cb[1100]          # a block of equal codes: the first of them wins
    cb = cb.to(cuda_dev)
    z = torch.cat([cb[17:18], cb[1100:1101], cb[1500:1501] + 1e-3]).to(cuda_dev)
    _, idx = ops.vq_quantize(z, cb, (cb.double() ** 2).sum(1).float(), want_indices=True)
    assert idx.tolist() == [17, 1100, 1100]


def test_vq_quantize_rejects_wide_codes(cuda_dev):
    from sdb200 import ops
    cb = torch.zeros(16, 9, device=cuda_dev)
    with pytest.raises(RuntimeError, match="e_dim"):
        ops.vq_quantize(torch.zeros(4, 9, device=cuda_dev), cb, torch.zeros(16, device=cuda_dev))


@pytest.mark.parametrize("idx", range(2))
def test_quantizer_vs_reference(cuda_dev, idx):
    case = golden("vq.pt")["quantize"][idx]
    m = _vq(case["cfg"], cuda_dev)
    zq, _, (_, _, ind) = m.quantize(case["z"].to(cuda_dev))
    cb = m.W["codebook"]
    z = case["z"].permute(0, 2, 3, 1).reshape(-1, cb.shape[1])
    _vq_check(z, cb, 1.0, zq.permute(0, 2, 3, 1).contiguous(), ind)
    near = ind.cpu() != case["indices"]
    assert near.float().mean() < 0.01, int(near.sum())          # only at near-ties
    ok = ~near.reshape(zq.shape[0], *zq.shape[2:]).unsqueeze(1).expand_as(zq)
    assert torch.equal(zq.cpu()[ok], case["z_q"][ok])


# ------------------------------------------------------------------------------------------------ models vs reference
@pytest.mark.parametrize("idx", range(4))
def test_unet_vs_reference(cuda_dev, idx):
    case = golden("vq.pt")["unet"][idx]
    net = _unet(case["cfg"], cuda_dev)
    eps = net(case["x"].to(cuda_dev), case["t"].to(cuda_dev))
    err = rel_l2(eps, case["eps"])
    print(f"unet {case['cfg']} {tuple(case['x'].shape)} rel-L2 {err:.3e}")
    assert eps.shape == case["eps"].shape and err < TOL


def test_celebahq_graph_autotune_and_c_handle(cuda_dev):
    import sdb200
    case = golden("vq.pt")["unet"][2]
    assert tuple(case["x"].shape) == (2, 3, 32, 32)
    graphed = sdb200.UNetModel(**arch.CELEBAHQ_UNET).load_weights(
        arch.random_state_dict(arch.unet_param_shapes(arch.CELEBAHQ_UNET), 11), cuda_dev)
    graphed.use_cuda_graph = True
    x, t = case["x"].to(cuda_dev), case["t"].to(cuda_dev).float()
    first = graphed(x, t).clone()
    replay = graphed(x, t)
    graphed.use_cuda_graph = False
    eager = graphed(x, t)
    h = graphed.c_handle(tuple(x.shape))
    try:
        out = h.forward(x, t)
        torch.cuda.synchronize()
        print(f"celebahq graph first {rel_l2(first, case['eps']):.3e} replay {rel_l2(replay, case['eps']):.3e} "
              f"C handle {rel_l2(out, case['eps']):.3e}")
        assert torch.equal(first, replay) and torch.equal(replay, eager) and torch.equal(out, eager)
        assert rel_l2(replay, case["eps"]) < TOL
    finally:
        h.close()


@pytest.mark.parametrize("idx", range(6))
def test_vq_decode_vs_reference(cuda_dev, idx):
    case = golden("vq.pt")["decode"][idx]
    m = _vq(case["cfg"], cuda_dev)
    x = m.decode(case["h"].to(cuda_dev), force_not_quantize=case["force_not_quantize"])
    err = rel_l2(x, case["x"])
    print(f"decode {case['cfg']} {tuple(case['h'].shape)} fnq={case['force_not_quantize']} rel-L2 {err:.3e}")
    assert x.shape == case["x"].shape and err < 2e-3


def test_vq_encode_vs_reference(cuda_dev):
    case = golden("vq.pt")["encode"]
    h = _vq(case["cfg"], cuda_dev).encode(case["x"].to(cuda_dev))
    err = rel_l2(h, case["h"])
    print(f"encode vq_f4 64x96 rel-L2 {err:.3e}")
    assert h.shape == case["h"].shape and err < 2e-3


def test_ddim_eta0_trajectory_with_ema(cuda_dev):
    """DDIM-10, eta 0, of the tiny VQ LDM (celebahq config values) inside ema_scope, then decode_first_stage."""
    from sdb200.samplers import DDIMSampler
    from sdb200.util import instantiate_from_config, remap_config
    g = golden("vq.pt")
    d = g["ddim"]
    node = script("sample_diffusion").celebahq_config(arch.TINY_VQ_UNET, arch.TINY_VQ)
    m = pipeline.load_random_weights(instantiate_from_config(remap_config(node)), cuda_dev,
                                     seeds=(g["unet_seed"], g["vq_seed"])).eval()
    m.model.diffusion_model.set_weight_set("ema", arch.random_state_dict(arch.unet_param_shapes(arch.TINY_VQ_UNET),
                                                                         g["ema_seed"]))
    assert m.use_ema and torch.equal(m.alphas_cumprod.cpu(), d["alphas_cumprod"])
    with m.ema_scope():
        s, _ = DDIMSampler(m).sample(10, batch_size=2, shape=[3, 16, 16], eta=0.0, verbose=False,
                                     x_T=d["x_T"].to(cuda_dev))
    e_s = rel_l2(s, d["sample"])
    e_dec = rel_l2(m.decode_first_stage(d["sample"].to(cuda_dev)), d["x_dec"])
    print(f"ddim eta=0 S=10 trajectory {e_s:.2e}; decode_first_stage {e_dec:.2e}")
    assert e_s < 5e-2 and e_dec < 2e-3
    with pytest.raises(NotImplementedError):
        m.decode_first_stage(d["sample"].to(cuda_dev), predict_cids=True)


def test_sample_diffusion_script_random_init_celebahq_config(cuda_dev, tmp_path):
    """The script with a CelebA-HQ-style config (VQ first stage, 3x64x64 latents shrunk to the tiny members)."""
    import glob
    import numpy as np
    mod = script("sample_diffusion")
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": mod.celebahq_config(arch.TINY_VQ_UNET, arch.TINY_VQ)}))
    logdir = mod.main(["--random_init", "--config", str(cfg), "-n", "2", "--batch_size", "2", "-c", "4", "-e", "0",
                       "-l", str(tmp_path / "out"), "--seed", "0"])
    pngs = sorted(glob.glob(os.path.join(logdir, "img", "*.png")))
    assert len(pngs) == 2
    npz = glob.glob(os.path.join(logdir, "numpy", "*.npz"))
    assert len(npz) == 1 and os.path.basename(npz[0]) == "2x32x32x3-samples.npz"     # tiny VQ: f = 2
    arr = np.load(npz[0])["arr_0"]
    assert arr.shape == (2, 32, 32, 3) and arr.dtype == np.uint8
