"""Tensor-level wrappers over the C ABI: PyTorch tensors in/out (device memory + current stream only).

Every function enqueues hand-written sm_90a kernels from libsdb200.so on the current CUDA stream; none of
them computes with torch. Shapes follow the engine's layouts: activations NHWC, fp32 residual stream,
fp16 tensor-core operands.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import lib as _l
from .lib import ACT_GEGLU, ACT_GELU, ACT_LEAKY_RELU, ACT_NONE, ACT_QUICK_GELU, ACT_RELU, ACT_SILU, AttnDesc, GemmDesc  # noqa: F401

LAUNCHES = 0        # op calls made through this module
_GRAPH_LAUNCHES = 0  # kernels replayed from CUDA graphs (counted at capture time, added per replay)
PROFILE = None      # when a list: gemm()/attention() append (kind, flops, start_event, end_event)
RECORD = None       # when a list: gemm() appends (desc, algorithmic_flops, keepalive) so bench.py can replay the launches
AUTOTUNE = False    # when True, gemm() times the (block_n, split-K) candidates of an unseen problem once and caches the best
TUNED = {}          # problem key -> (block_n, splits)


def launch_count():
    """Kernels launched from libsdb200.so: direct launches (counted in C) + kernels replayed inside CUDA graphs."""
    return int(_l.load().sdb_launch_count()) + _GRAPH_LAUNCHES


def add_graph_launches(n):
    global _GRAPH_LAUNCHES
    _GRAPH_LAUNCHES += int(n)



def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _count(n=1):
    global LAUNCHES
    LAUNCHES += n


def _chk16(t, name):
    assert t.dtype == torch.float16 and t.is_cuda and t.is_contiguous(), f"{name}: need contiguous cuda fp16"


def _chk32(t, name):
    assert t.dtype == torch.float32 and t.is_cuda and t.is_contiguous(), f"{name}: need contiguous cuda fp32"


def gemm(a0, b, *, a1=None, a2=None, a3=None, nb=None, h=None, w=None, taps=1, bias=None, film=None,
         rows_per_sample=0, residual=None, act=ACT_NONE, alpha=1.0, out_f16=None, out_f32=None, out_f16_lo=None,
         want_f16=False, want_f32=False, want_lo=False, n=None, block_n=0, splits=0, workspace=None,
         want_stats=False, stats_group=1, b_dynamic=False, conv_stride=1, conv_shift=0, pair=0, splitk_mode=0):
    """acc = A @ B^T with fused epilogue (see sdb_gemm in include/sdb200.h).

    a0 (, a1, a2, a3): fp16 [..., c_i] NHWC activations or plain [rows, c_i] matrices, concatenated along K.
    b: fp16 [n, taps*sum(c_i)].
    Returns (out_f16, out_f32), or (out_f16, out_f32, out_f16_lo) when the hi/lo pair is requested.
    block_n / pair / splits / splitk_mode: explicit tile width, CTA pairs (2) or single CTAs (1), split-K factor and how
    its partials meet (1 workspace + second kernel, 2 thread-block cluster); 0 = let the library (or the autotuner) pick.
    want_stats: the epilogue also stores per-tile GroupNorm partial sums of the fp32 output (entries of `stats_group`
    channels); they are attached to the output tensor (see channel_stats()) so the following groupnorm() skips its
    reduction pass.
    """
    _chk16(a0, "a0")
    _chk16(b, "b")
    srcs = [a0]
    for t_ in (a1, a2, a3):
        if t_ is None:
            break
        _chk16(t_, "a_i")
        assert t_.shape[:-1] == a0.shape[:-1]
        srcs.append(t_)
    chans = [t_.shape[-1] for t_ in srcs]
    c0 = chans[0]
    in_h = in_w = 0
    if taps == 9:
        assert a0.dim() == 4, "3x3 conv needs NHWC input"
        nb, h, w = a0.shape[0], a0.shape[1], a0.shape[2]
        if conv_stride == 2:      # output size of a 3x3 / stride-2 conv: symmetric pad 1 (shift 0) or pad right/bottom (shift 1)
            in_h, in_w = h, w
            h, w = (in_h + 1 - conv_shift) // 2, (in_w + 1 - conv_shift) // 2
    else:
        rows = a0.numel() // c0
        nb, h, w = 1, 1, rows
    n = b.shape[0] if n is None else n
    # B rows hold taps * sum(ceil64(c_i)) columns (zero tails pad a source whose width is a multiple of 32 only to whole
    # 64-wide K steps); one source of one tap may be exactly c wide
    kb = chans[0] if (len(srcs) == 1 and taps == 1) else taps * sum((c_ + 63) // 64 * 64 for c_ in chans)
    assert b.shape[1] == kb, (b.shape, taps, chans)
    M = nb * h * w
    n_out = n // 2 if act == ACT_GEGLU else n
    # the descriptor carries one row stride per operand and assumes unit column stride: check the layouts it implies
    if bias is not None:
        _chk32(bias, "bias")
        assert tuple(bias.shape) == (n,), f"bias: need fp32 [{n}], got {tuple(bias.shape)}"
    if film is not None:
        assert film.dtype == torch.float32 and film.is_cuda and film.dim() == 2, "film: need a 2-D cuda fp32 matrix"
        assert film.shape[1] == n and film.stride(1) == 1, f"film: need [samples, {n}] with unit column stride"
        rps_ = rows_per_sample if rows_per_sample else h * w
        assert film.shape[0] >= (M + rps_ - 1) // rps_, "film: fewer rows than samples"
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.is_cuda, "residual: need cuda fp32"
        residual = residual.view(-1, residual.shape[-1])     # raises when the rows are not one stride apart
        assert tuple(residual.shape) == (M, n_out) and residual.stride(1) == 1, \
            f"residual: need [{M}, {n_out}] rows with unit column stride, got {tuple(residual.shape)} {residual.stride()}"
    for t_, dt, name in ((out_f16, torch.float16, "out_f16"), (out_f32, torch.float32, "out_f32"),
                         (out_f16_lo, torch.float16, "out_f16_lo")):
        if t_ is not None:
            assert t_.dtype == dt and t_.is_cuda and t_.is_contiguous(), f"{name}: need contiguous cuda {dt}"
            assert t_.numel() == M * n_out and t_.shape[-1] == n_out, f"{name}: need [{M}, {n_out}], got {tuple(t_.shape)}"
    if out_f16 is None and (want_f16 or want_lo):
        out_f16 = torch.empty((M, n_out), dtype=torch.float16, device=a0.device)
    if out_f16_lo is None and want_lo:
        out_f16_lo = torch.empty((M, n_out), dtype=torch.float16, device=a0.device)
    if out_f32 is None and want_f32:
        out_f32 = torch.empty((M, n_out), dtype=torch.float32, device=a0.device)
    assert out_f16 is not None or out_f32 is not None
    lib = _l.load()
    d = GemmDesc()
    ptrs = [_ptr(t_) for t_ in srcs] + [None] * (4 - len(srcs))
    cs = chans + [0] * (4 - len(chans))
    d.a0, d.a1, d.a2, d.a3 = ptrs
    d.c0, d.c1, d.c2, d.c3 = cs
    d.nb, d.h, d.w, d.taps = nb, h, w, taps
    d.b, d.n, d.alpha = _ptr(b), n, alpha
    d.bias = _ptr(bias)
    d.film = _ptr(film)
    d.ldf = film.stride(0) if film is not None else 0
    d.rows_per_sample = rows_per_sample
    d.residual = _ptr(residual)
    d.ldr = residual.stride(0) if residual is not None else 0
    d.act = act
    d.out_f16, d.out_f32, d.out_f16_lo = _ptr(out_f16), _ptr(out_f32), _ptr(out_f16_lo)
    d.ldo = 0
    d.block_n, d.pair, d.splitk_mode = block_n, pair, splitk_mode
    d.b_dynamic = 1 if b_dynamic else 0   # b produced by the previous kernel: no early (pre-dependency) prefetch
    d.conv_stride, d.conv_shift, d.in_h, d.in_w = conv_stride, conv_shift, in_h, in_w
    d.splits = splits
    if splits and (splits > 1 or splits == -1) and splitk_mode != 2:
        if workspace is None:
            workspace = splitk_workspace(a0.device)
        d.workspace = _ptr(workspace)
        d.workspace_floats = workspace.numel()
    rps = rows_per_sample if rows_per_sample else h * w
    stats_ok = want_stats and out_f32 is not None and act != ACT_GEGLU and (taps == 9 or rows_per_sample) and \
        M % rps == 0 and n % stats_group == 0
    d.stats_group = stats_group
    if stats_ok:
        d.stats_out = C.c_void_p(16)     # placeholder: the plan only needs to know that statistics are wanted
    plan = (C.c_int32 * 5)()
    tunable = block_n == 0 and pair == 0 and splitk_mode == 0 and splits in (0, -1) and act != ACT_GEGLU
    if tunable:
        key = tune_key(d, b.shape[1], stats_ok)
        choice = TUNED.get(key)
        if choice is None and AUTOTUNE:
            choice = TUNED[key] = _tune_gemm(d, M, n, rps, stats_ok, stats_group)
        if choice is not None:
            d.block_n, d.pair, d.splits, d.splitk_mode = choice
    rc = lib.sdb_gemm_plan(C.byref(d), plan)
    if rc != 0 and stats_ok:             # this problem / tile shape cannot produce fused statistics: plain GEMM, the
        stats_ok = False                 # consumer falls back to its own reduction pass
        d.stats_out = None
        rc = lib.sdb_gemm_plan(C.byref(d), plan)
    _l.check(rc, "sdb_gemm_plan")
    d.block_n, d.pair, d.splits, d.splitk_mode = plan[0], plan[1], plan[2], plan[3]
    stats = None
    if stats_ok:
        shape = (M // rps, plan[4], n // stats_group, 2)
        stats = ARENA.take(shape) if ARENA is not None else None
        if stats is None:
            stats = torch.empty(shape, dtype=torch.float32, device=a0.device)
        d.stats_out = _ptr(stats)
        out_f32._sdb_stats = (stats, plan[4], stats_group)   # travels with the tensor object (and, through ._base, its views)
    if RECORD is not None:
        # operand-split passes ([A_hi|A_lo|A_hi]) are overhead, not algorithmic work: count K once
        k_alg = taps * sum(chans) // 3 if (len(srcs) == 3 and srcs[0] is srcs[2]) else taps * sum(chans)
        RECORD.append((d, 2.0 * M * n * k_alg, (srcs, b, bias, film, residual, out_f16, out_f32, out_f16_lo, workspace, stats)))
    if PROFILE is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _l.check(lib.sdb_gemm(C.byref(d), _stream()), "sdb_gemm")
    if PROFILE is not None:
        e1.record()
        PROFILE.append(("gemm", 2.0 * M * n * b.shape[1], e0, e1, (M, n, b.shape[1], taps)))
    _count(2 if plan[3] == 1 else 1)
    if out_f16_lo is not None:
        return out_f16, out_f32, out_f16_lo
    return out_f16, out_f32


class StatsArena:
    """One fp32 bump buffer per forward pass for all fused GroupNorm statistics. The GEMM epilogues STORE their per-tile
    partial sums (every slot has exactly one writer), so nothing is zeroed: reset() only rewinds the bump pointer;
    gemm(want_stats=True) carves its [samples, T, n / group, 2] slice."""

    def __init__(self, device, n_floats=4 * 1024 * 1024):
        self.buf = torch.empty(n_floats, dtype=torch.float32, device=device)
        self.off = 0

    def reset(self):
        self.off = 0

    def take(self, shape):
        n = 1
        for s_ in shape:
            n *= s_
        if self.off + n > self.buf.numel():
            return None
        v = self.buf[self.off: self.off + n].view(shape)
        self.off += (n + 3) // 4 * 4
        return v


ARENA = None   # set by the model around a forward pass (UNetModel._forward_impl)


def channel_stats(x):
    """Fused GroupNorm statistics (partials tensor, slots per sample, channels per entry) attached to `x` (or the tensor
    it is a view of) by the gemm() that produced it."""
    st = getattr(x, "_sdb_stats", None)
    if st is None and x._base is not None and x._base.numel() == x.numel():
        st = getattr(x._base, "_sdb_stats", None)
    return st


def tune_key(d, kb, stats_ok):
    """Key of the autotuner's cache (TUNED) for the descriptor gemm() built; kb = columns of B."""
    nsrc = sum(1 for p in (d.a0, d.a1, d.a2, d.a3) if p)
    return (d.nb * d.h * d.w, d.n, kb, d.taps, nsrc, bool(d.bias), bool(d.film), bool(d.residual), d.act,
            bool(d.out_f16), bool(d.out_f32), bool(d.out_f16_lo), stats_ok, d.stats_group, d.conv_stride)


def tune_candidates(d, M, n):
    """The (block_n, pair, splits, splitk_mode) candidates the autotuner times for descriptor `d`, in timing order, and
    the largest statistics slot count T among them. d.stats_out must already be set (a placeholder will do) when
    statistics are wanted; d's tile fields are left at the last candidate tried."""
    lib = _l.load()
    plan = (C.c_int32 * 5)()
    cands = []
    max_slots = 1
    import os
    bns = tuple(int(v) for v in os.environ.get("SDB_TUNE_BN", "64,128,160,256").split(","))
    cgs = tuple(int(v) for v in os.environ.get("SDB_TUNE_CG", "1,2").split(","))
    for bn in bns:
        pad = (n + bn - 1) // bn * bn - n
        if bn > 64 and pad >= bn // 2:
            continue
        for cg in cgs:
            for sp, mode in ((1, 0), (2, 2), (4, 2), (2, 1), (3, 1), (4, 1), (6, 1), (8, 1), (12, 1), (16, 1)):
                if mode == 1 and not d.workspace:
                    continue
                tiles = ((M + 127) // 128) * ((n + bn - 1) // bn) * sp
                if sp > 1 and tiles > 3 * lib.sdb_sm_count():
                    continue
                d.block_n, d.pair, d.splits, d.splitk_mode = bn, cg, sp, mode
                if lib.sdb_gemm_plan(C.byref(d), plan) != 0:
                    continue
                if (plan[0], plan[1], plan[2], plan[3]) != (bn, cg, sp, mode if sp > 1 else 0):
                    continue
                cands.append((bn, cg, sp, mode))
                max_slots = max(max_slots, int(plan[4]))
    return cands, max_slots


def _tune_gemm(d, M, n, rps, stats_ok, stats_group):
    """Time the (tile width, CTA pair, split-K) candidates of one GEMM problem on its real operands (CUDA events, GPU
    kept busy by a leading spin so host launch gaps do not enter) and return the fastest
    (block_n, pair, splits, splitk_mode)."""
    lib = _l.load()
    st = _stream()
    keep = (d.block_n, d.pair, d.splits, d.splitk_mode, d.stats_out)
    scratch = None
    if stats_ok:
        d.stats_out = C.c_void_p(16)     # placeholder while the candidates are planned (sized below)
    cands, max_slots = tune_candidates(d, M, n)
    if stats_ok:
        # the statistics slots per sample depend on the candidate (tiles x cluster splits, or one per 32 rows with the
        # workspace epilogue): size the scratch for the largest one - a smaller buffer is overrun by the epilogues
        scratch = torch.empty((M // rps) * max_slots * (n // stats_group) * 2 + 16, dtype=torch.float32,
                              device=torch.device("cuda", torch.cuda.current_device()))
        d.stats_out = _ptr(scratch)
    best, best_t = None, float("inf")
    for cand in cands:
        d.block_n, d.pair, d.splits, d.splitk_mode = cand
        if lib.sdb_gemm(C.byref(d), st) != 0:      # warm-up / validity
            continue
        t = float("inf")
        for _ in range(3):      # best of three short bursts: one noisy burst must not decide the captured tile shape
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(400_000)
            e0.record()
            for _ in range(4):
                lib.sdb_gemm(C.byref(d), st)
            e1.record()
            e1.synchronize()
            t = min(t, e0.elapsed_time(e1))
        if t < best_t:
            best, best_t = cand, t
    d.block_n, d.pair, d.splits, d.splitk_mode, d.stats_out = keep
    del scratch
    return best


_WS = {}
WS_FLOATS = 16 * 1024 * 1024


def splitk_workspace(device):
    """Persistent fp32 scratch for split-K partials (stream-ordered reuse: one GEMM at a time per stream)."""
    key = (device.type, device.index)
    if key not in _WS:
        _WS[key] = torch.empty(WS_FLOATS, dtype=torch.float32, device=device)
    return _WS[key]


def attention(q, k, vt, *, heads, d, dpad, nq, nkv, scale, causal=False, out=None, head_stride=0):
    """q [B, nq, heads*hs], k [B, nkv, heads*hs], vt [B, heads*hs, ldvt] fp16 -> out [B, nq, heads*d] fp16, where
    hs = head_stride (0: dpad) is the distance between heads; head_stride=d is the packed layout."""
    for name, t_ in (("q", q), ("k", k), ("vt", vt)):
        assert t_.dtype == torch.float16 and t_.is_cuda and t_.dim() == 3 and t_.stride(2) == 1, f"{name}: bad layout"
    B = q.shape[0]
    if out is None:
        out = torch.empty((B, nq, heads * d), dtype=torch.float16, device=q.device)
    a = AttnDesc()
    a.q, a.k, a.vt, a.out = _ptr(q), _ptr(k), _ptr(vt), _ptr(out)
    a.batch, a.heads, a.nq, a.nkv, a.d, a.dpad = B, heads, nq, nkv, d, dpad
    a.ldq, a.ldk, a.ldvt, a.ldo = q.stride(1), k.stride(1), vt.stride(1), out.stride(1)
    a.q_batch_stride, a.k_batch_stride = q.stride(0), k.stride(0)
    a.vt_batch_stride, a.o_batch_stride = vt.stride(0), out.stride(0)
    a.scale, a.causal, a.head_stride = scale, 1 if causal else 0, head_stride
    if PROFILE is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _l.check(_l.load().sdb_attention(C.byref(a), _stream()), "sdb_attention")
    if PROFILE is not None:
        e1.record()
        PROFILE.append(("attention", 4.0 * B * heads * nq * nkv * d, e0, e1, (B, heads, nq, nkv, d)))
    _count()
    return out


def groupnorm(x0, gamma, beta, *, x1=None, groups=32, eps=1e-5, silu=False, want_raw=False, want_lo=False,
              want_raw_lo=False):
    """x0 (, x1): fp32 NHWC [nb, h, w, c]; returns (normalised fp16 NHWC [nb,h,w,c0+c1], raw fp16 or None), plus the
    low halves (out_lo, raw_lo) of the hi/lo split when requested: (out, raw, out_lo, raw_lo)."""
    _chk32(x0, "x0")
    nb, h, w, c0 = x0.shape
    c1 = 0
    if x1 is not None:
        _chk32(x1, "x1")
        c1 = x1.shape[-1]
    out = torch.empty((nb, h, w, c0 + c1), dtype=torch.float16, device=x0.device)
    raw = torch.empty_like(out) if (want_raw or want_raw_lo) else None
    out_lo = torch.empty_like(out) if want_lo else None
    raw_lo = torch.empty_like(out) if want_raw_lo else None
    ws = torch.empty(nb * (128 * groups * 2 + groups * 2 + 1), dtype=torch.float32, device=x0.device)
    cs0 = channel_stats(x0)
    cs1 = channel_stats(x1) if x1 is not None else None
    sg = cs0[2] if cs0 is not None else 1
    cpg = (c0 + c1) // groups
    if cs0 is None or (x1 is not None and (cs1 is None or cs1[2] != sg)) or cpg % sg or c0 % sg or c1 % sg:
        cs0 = cs1 = None     # no (compatible) fused statistics: the kernel pair below computes them
    t0, t1 = (cs0[1] if cs0 else 0), (cs1[1] if cs1 else 0)
    _l.check(_l.load().sdb_groupnorm(_ptr(x0), _ptr(x1), c0, c1, nb, h * w, groups, _ptr(gamma), _ptr(beta),
                                     eps, 1 if silu else 0, _ptr(out), _ptr(raw), _ptr(out_lo), _ptr(raw_lo), _ptr(ws),
                                     _ptr(cs0[0]) if cs0 else None, _ptr(cs1[0]) if cs1 else None, t0, t1, sg,
                                     _stream()), "sdb_groupnorm")
    _count(1 if cs0 else 3)
    if want_lo or want_raw_lo:
        return out, raw, out_lo, raw_lo
    return out, raw


def groupnorm_mod(x, gamma, beta, *, scale=None, shift=None, resample=0, groups=32, eps=1e-5, silu=True):
    """x fp32 NHWC [nb, h, w, c] -> fp16 NHWC: SiLU(GN(x) [* (1 + scale) + shift]), optionally 2x2 average-pooled
    (resample=1) or nearest-2x upsampled (resample=2). scale / shift: fp32 [nb, c] views with unit column stride (the
    FiLM output's column slices). Uses the fused statistics attached to x by the producing gemm() when compatible."""
    _chk32(x, "x")
    nb, h, w, c = x.shape
    ldm = 0
    if scale is not None:
        for t_ in (scale, shift):
            assert t_.dtype == torch.float32 and t_.is_cuda and t_.shape == (nb, c) and t_.stride(1) == 1
        assert scale.stride(0) == shift.stride(0)
        ldm = scale.stride(0)
    ho, wo = (h // 2, w // 2) if resample == 1 else (2 * h, 2 * w) if resample == 2 else (h, w)
    out = torch.empty((nb, ho, wo, c), dtype=torch.float16, device=x.device)
    ws = torch.empty(nb * (128 * groups * 2 + groups * 2 + 1), dtype=torch.float32, device=x.device)
    cs = channel_stats(x)
    if cs is not None and ((c // groups) % cs[2] or c % cs[2]):
        cs = None
    _l.check(_l.load().sdb_groupnorm_mod(_ptr(x), c, nb, h, w, groups, _ptr(gamma), _ptr(beta), eps, 1 if silu else 0,
                                         _ptr(scale), _ptr(shift), ldm, resample, _ptr(out), _ptr(ws),
                                         _ptr(cs[0]) if cs else None, cs[1] if cs else 0, cs[2] if cs else 1,
                                         _stream()), "sdb_groupnorm_mod")
    _count(2)
    return out


def resample_f32(x, mode):
    """fp32 NHWC [nb, h, w, c] -> 2x2 average pool (mode 1) or nearest 2x (mode 2), fp32 NHWC."""
    _chk32(x, "x")
    nb, h, w, c = x.shape
    ho, wo = (h // 2, w // 2) if mode == 1 else (2 * h, 2 * w)
    out = torch.empty((nb, ho, wo, c), dtype=torch.float32, device=x.device)
    _l.check(_l.load().sdb_resample_f32(_ptr(x), nb, h, w, c, mode, _ptr(out), _stream()), "sdb_resample_f32")
    _count()
    return out


def ddpm_step(x, eps, noise, *, sqrt_recip_ac, sqrt_recipm1_ac, coef1, coef2, sigma, x_out=None, x0_out=None):
    """One ancestral DDPM update (sdb_ddpm_step); returns (x', x0)."""
    _chk32(x, "x")
    _chk32(eps, "eps")
    assert eps.numel() == x.numel()
    if noise is not None:
        _chk32(noise, "noise")
        assert noise.numel() == x.numel()
    if x_out is None:
        x_out = torch.empty_like(x)
    if x0_out is None:
        x0_out = torch.empty_like(x)
    _l.check(_l.load().sdb_ddpm_step(_ptr(x), _ptr(eps), _ptr(noise), sqrt_recip_ac, sqrt_recipm1_ac, coef1, coef2, sigma,
                                     x.numel(), _ptr(x_out), _ptr(x0_out), _stream()), "sdb_ddpm_step")
    _count()
    return x_out, x0_out


def vq_quantize(z, codebook, code_sq, scale=1.0, want_indices=False):
    """Nearest-codebook quantization (sdb_vq_quantize): z fp32 NHWC [..., e_dim] (times `scale` first), codebook fp32
    [n_e, e_dim], code_sq its squared row norms. Returns z_q (same shape), or (z_q, int64 indices [rows])."""
    _chk32(z, "z")
    _chk32(codebook, "codebook")
    _chk32(code_sq, "code_sq")
    n_e, e_dim = codebook.shape
    assert z.shape[-1] == e_dim and code_sq.shape == (n_e,)
    rows = z.numel() // e_dim
    z_q = torch.empty_like(z)
    idx = torch.empty(rows, dtype=torch.int64, device=z.device) if want_indices else None
    _l.check(_l.load().sdb_vq_quantize(_ptr(z), rows, e_dim, scale, _ptr(codebook), _ptr(code_sq), n_e, _ptr(z_q),
                                       _ptr(idx), _stream()), "sdb_vq_quantize")
    _count()
    return (z_q, idx) if want_indices else z_q


def layernorm(x, gamma, beta, eps=1e-5, want_f32=False):
    """x fp32 [rows, c] -> fp16 [rows, c]."""
    _chk32(x, "x")
    c = x.shape[-1]
    rows = x.numel() // c
    out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    out32 = torch.empty_like(x) if want_f32 else None
    _l.check(_l.load().sdb_layernorm(_ptr(x), rows, c, _ptr(gamma), _ptr(beta), eps, _ptr(out), _ptr(out32),
                                     _stream()), "sdb_layernorm")
    _count()
    return (out, out32) if want_f32 else out


def softmax_rows(x, scale):
    _chk32(x, "x")
    cols = x.shape[-1]
    rows = x.numel() // cols
    out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _l.check(_l.load().sdb_softmax_rows(_ptr(x), rows, cols, scale, _ptr(out), _stream()), "sdb_softmax_rows")
    _count()
    return out


def nchw_to_nhwc(x, want_f32=True, want_f16=False):
    _chk32(x, "x")
    nb, c, h, w = x.shape
    o32 = torch.empty((nb, h, w, c), dtype=torch.float32, device=x.device) if want_f32 else None
    o16 = torch.empty((nb, h, w, c), dtype=torch.float16, device=x.device) if want_f16 else None
    _l.check(_l.load().sdb_nchw_to_nhwc(_ptr(x), nb, c, h * w, _ptr(o32), _ptr(o16), _stream()), "sdb_nchw_to_nhwc")
    _count()
    return o32, o16


def nhwc_to_nchw(x, out=None):
    _chk32(x, "x")
    nb, h, w, c = x.shape
    if out is None:
        out = torch.empty((nb, c, h, w), dtype=torch.float32, device=x.device)
    _l.check(_l.load().sdb_nhwc_to_nchw(_ptr(x), nb, c, h * w, _ptr(out), _stream()), "sdb_nhwc_to_nchw")
    _count()
    return out


def im2col3x3(x, stride, pad_lo, ho, wo, kpad):
    _chk32(x, "x")
    nb, h, w, c = x.shape
    out = torch.empty((nb * ho * wo, kpad), dtype=torch.float16, device=x.device)
    _l.check(_l.load().sdb_im2col3x3(_ptr(x), nb, h, w, c, stride, pad_lo, ho, wo, kpad, _ptr(out), _stream()),
             "sdb_im2col3x3")
    _count()
    return out


def im2col3x3_concat(x, cond, kpad):
    """3x3 / pad 1 im2col of cat([x, cond], 1) from the two NCHW fp32 tensors -> fp16 [nb*h*w, kpad]."""
    _chk32(x, "x")
    _chk32(cond, "cond")
    nb, cx, h, w = x.shape
    out = torch.empty((nb * h * w, kpad), dtype=torch.float16, device=x.device)
    _l.check(_l.load().sdb_im2col3x3_concat(_ptr(x), nb, cx, h, w, _ptr(cond), cond.shape[0], cond.shape[1],
                                            cond.shape[2], cond.shape[3], kpad, _ptr(out), _stream()),
             "sdb_im2col3x3_concat")
    _count()
    return out


def inpaint_prepare(image_u8, mask_u8, cond, mask_channel):
    """image uint8 [nb, h, w, 3], mask uint8 [nb, h, w] -> the masked image fp32 NCHW [nb, 3, h, w]; writes the resized
    ±1 mask into channel `mask_channel` of cond fp32 [nb, c, hc, wc] (sdb_inpaint_prepare)."""
    _chk32(cond, "cond")
    nb, h, w, _ = image_u8.shape
    assert image_u8.dtype == torch.uint8 and mask_u8.dtype == torch.uint8 and image_u8.shape[3] == 3
    assert image_u8.is_contiguous() and mask_u8.is_contiguous() and tuple(mask_u8.shape) == (nb, h, w)
    assert cond.shape[0] == nb
    masked = torch.empty((nb, 3, h, w), dtype=torch.float32, device=image_u8.device)
    _l.check(_l.load().sdb_inpaint_prepare(_ptr(image_u8), _ptr(mask_u8), nb, h, w, _ptr(masked), _ptr(cond),
                                           cond.shape[1], cond.shape[2], cond.shape[3], mask_channel, _stream()),
             "sdb_inpaint_prepare")
    _count(2)
    return masked


def inpaint_composite(x_nhwc, image_u8, mask_u8):
    """Decoded image fp32 NHWC [nb, h, w, 3], original image uint8 [nb, h, w, 3], mask uint8 [nb, h, w] -> the inpainted
    uint8 image [nb, h, w, 3] (sdb_inpaint_composite)."""
    _chk32(x_nhwc, "x_nhwc")
    assert image_u8.dtype == torch.uint8 and mask_u8.dtype == torch.uint8
    assert image_u8.is_contiguous() and mask_u8.is_contiguous()
    assert tuple(image_u8.shape) == tuple(x_nhwc.shape) and x_nhwc.shape[-1] == 3
    assert tuple(mask_u8.shape) == tuple(x_nhwc.shape[:-1])
    out = torch.empty(image_u8.shape, dtype=torch.uint8, device=image_u8.device)
    _l.check(_l.load().sdb_inpaint_composite(_ptr(x_nhwc), _ptr(image_u8), _ptr(mask_u8), mask_u8.numel(), _ptr(out),
                                             _stream()), "sdb_inpaint_composite")
    _count()
    return out


def lr_prepare(image_u8):
    """Low-resolution image uint8 RGB [nb, h, w, 3] -> the super-resolution conditioning 2 * (u / 255) - 1, fp32 NCHW
    [nb, 3, h, w] (sdb_lr_prepare)."""
    assert image_u8.dtype == torch.uint8 and image_u8.is_cuda and image_u8.is_contiguous()
    assert image_u8.dim() == 4 and image_u8.shape[3] == 3, tuple(image_u8.shape)
    nb, h, w, _ = image_u8.shape
    out = torch.empty((nb, 3, h, w), dtype=torch.float32, device=image_u8.device)
    _l.check(_l.load().sdb_lr_prepare(_ptr(image_u8), nb, h, w, _ptr(out), _stream()), "sdb_lr_prepare")
    _count()
    return out


def patch_unfold(x, ks, stride, out=None):
    """nn.Unfold(ks, stride=stride) of x fp32 NCHW [nb, c, h, w] as tiles [L*nb, c, ks[0], ks[1]], tile l*nb + n
    (sdb_patch_unfold). `out` may be a preallocated contiguous buffer of that shape (a captured graph's input)."""
    _chk32(x, "x")
    nb, c, h, w = x.shape
    L = ((h - ks[0]) // stride[0] + 1) * ((w - ks[1]) // stride[1] + 1)
    shape = (L * nb, c, ks[0], ks[1])
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    _chk32(out, "out")
    assert tuple(out.shape) == shape, (tuple(out.shape), shape)
    _l.check(_l.load().sdb_patch_unfold(_ptr(x), nb, c, h, w, ks[0], ks[1], stride[0], stride[1], _ptr(out), _stream()),
             "sdb_patch_unfold")
    _count()
    return out


def patch_fold(tiles, weight, norm, grid, stride, nhwc=False):
    """fold(tiles * weight) / norm -> fp32 NCHW [nb, c, h, w] (sdb_patch_fold). tiles fp32 [ly*lx*nb, c, kh, kw] (or
    [.., kh, kw, c] with nhwc), weight fp32 [ly*lx, kh, kw], norm fp32 [h, w]; grid = (ly, lx)."""
    _chk32(tiles, "tiles")
    _chk32(weight, "weight")
    _chk32(norm, "norm")
    ly, lx = grid
    n, c, kh, kw = (tiles.shape[0], tiles.shape[3], tiles.shape[1], tiles.shape[2]) if nhwc else tiles.shape
    assert n % (ly * lx) == 0 and tuple(weight.shape) == (ly * lx, kh, kw), (tuple(tiles.shape), tuple(weight.shape))
    nb = n // (ly * lx)
    h, w = norm.shape
    out = torch.empty((nb, c, h, w), dtype=torch.float32, device=tiles.device)
    _l.check(_l.load().sdb_patch_fold(_ptr(tiles), int(nhwc), nb, c, kh, kw, ly, lx, stride[0], stride[1], _ptr(weight),
                                      _ptr(norm), h, w, _ptr(out), _stream()), "sdb_patch_fold")
    _count()
    return out


def spatial_rescale(x, n_stages, weight=None, bias=None):
    """SpatialRescaler (bilinear, multiplier 0.5) of x fp32 NCHW [nb, cin, h, w]: n_stages x0.5 interpolations, then the
    channel_mapper 1x1 conv when weight fp32 [cout, cin] is given (bias fp32 [cout] or None). Returns fp32 NCHW
    [nb, cout, h >> n_stages, w >> n_stages] (sdb_spatial_rescale)."""
    _chk32(x, "x")
    nb, cin, h, w = x.shape
    cout = cin
    if weight is not None:
        _chk32(weight, "weight")
        assert weight.dim() == 2 and weight.shape[1] == cin, (tuple(weight.shape), cin)
        cout = weight.shape[0]
    if bias is not None:
        assert weight is not None
        _chk32(bias, "bias")
        assert tuple(bias.shape) == (cout,)
    out = torch.empty((nb, cout, h >> n_stages, w >> n_stages), dtype=torch.float32, device=x.device)
    _l.check(_l.load().sdb_spatial_rescale(_ptr(x), nb, cin, h, w, n_stages, _ptr(weight), _ptr(bias), cout, _ptr(out),
                                           _stream()), "sdb_spatial_rescale")
    _count()
    return out


def seg_labels_rescale(labels_u8, cin, n_stages, weight, bias=None):
    """The SpatialRescaler of the one-hot of labels uint8 [nb, h, w] (ids < cin, checked by the caller) with the channel
    map weight fp32 [cout, cin] (+ bias), without materialising the one-hot: fp32 NCHW [nb, cout, h >> n_stages,
    w >> n_stages], bit-identical to spatial_rescale of the one-hot (sdb_seg_labels_rescale)."""
    assert labels_u8.dtype == torch.uint8 and labels_u8.is_cuda and labels_u8.is_contiguous() and labels_u8.dim() == 3
    _chk32(weight, "weight")
    assert weight.dim() == 2 and weight.shape[1] == cin, (tuple(weight.shape), cin)
    cout = weight.shape[0]
    if bias is not None:
        _chk32(bias, "bias")
        assert tuple(bias.shape) == (cout,)
    nb, h, w = labels_u8.shape
    out = torch.empty((nb, cout, h >> n_stages, w >> n_stages), dtype=torch.float32, device=labels_u8.device)
    _l.check(_l.load().sdb_seg_labels_rescale(_ptr(labels_u8), nb, cin, h, w, n_stages, _ptr(weight), _ptr(bias), cout,
                                              _ptr(out), _stream()), "sdb_seg_labels_rescale")
    _count()
    return out


KNN_MAX_QUERIES = 64   # queries per sdb_knn_topk launch


def knn_topk(db, queries, k):
    """Exact top-k by inner product (sdb_knn_topk): db fp16 [n, dim], queries fp16 [b <= 64, dim] -> (scores fp32
    [b, k], rows int64 [b, k]), score descending, the lower row first on equal scores."""
    _chk16(db, "db")
    _chk16(queries, "queries")
    n, dim = db.shape
    b = queries.shape[0]
    assert queries.shape == (b, dim), (tuple(queries.shape), dim)
    need = int(_l.load().sdb_knn_workspace(n, b, k))
    ws_s = torch.empty(max(need, 1), dtype=torch.float32, device=db.device)
    ws_i = torch.empty(max(need, 1), dtype=torch.int32, device=db.device)
    scores = torch.empty((b, k), dtype=torch.float32, device=db.device)
    rows = torch.empty((b, k), dtype=torch.int64, device=db.device)
    _l.check(_l.load().sdb_knn_topk(_ptr(db), n, dim, _ptr(queries), b, k, _ptr(ws_s), _ptr(ws_i), need, _ptr(scores),
                                    _ptr(rows), _stream()), "sdb_knn_topk")
    _count(2)
    return scores, rows


def rows_pool(x, ids=None, normalize=False):
    """x fp32 [rows, dim] -> fp32 [b, dim]: with ids (int64 [b, n_ctx]) the row at each sequence's largest id (CLIP's EOT
    token), else every row; normalize divides each row by its L2 norm (sdb_rows_pool)."""
    _chk32(x, "x")
    dim = x.shape[-1]
    if ids is not None:
        assert ids.dtype == torch.int64 and ids.is_cuda and ids.is_contiguous() and ids.dim() == 2
        b, n_ctx = ids.shape
        assert x.numel() == b * n_ctx * dim, (tuple(x.shape), tuple(ids.shape))
    else:
        b, n_ctx = x.numel() // dim, 0
    out = torch.empty((b, dim), dtype=torch.float32, device=x.device)
    _l.check(_l.load().sdb_rows_pool(_ptr(x), _ptr(ids), b, n_ctx, dim, int(normalize), _ptr(out), _stream()),
             "sdb_rows_pool")
    _count()
    return out


def clip_resize_patches(src, table, size, patch, kpad, mean, std, want_resized=False):
    """Ragged-batch CLIP image preprocessing (sdb_clip_resize_patches): src packed images, fp32 (NCHW each, in [-1, 1])
    or uint8 (HWC each), table int64 cuda [nb, 3] = (H, W, element offset) -> (fp16 patch rows [nb * (size/patch)^2,
    kpad], fp32 [nb, 3, size, size] resized values before (x + 1) / 2, or None)."""
    assert src.is_cuda and src.is_contiguous() and src.dtype in (torch.float32, torch.uint8), "src: contiguous cuda fp32 / uint8"
    assert table.dtype == torch.int64 and table.is_cuda and table.is_contiguous() and table.dim() == 2 and table.shape[1] == 3
    nb = table.shape[0]
    g = size // patch
    patches = torch.empty((nb * g * g, kpad), dtype=torch.float16, device=src.device)
    resized = torch.empty((nb, 3, size, size), dtype=torch.float32, device=src.device) if want_resized else None
    _l.check(_l.load().sdb_clip_resize_patches(_ptr(src), int(src.dtype == torch.uint8), _ptr(table), nb, size, patch,
                                               kpad, *mean, *std, _ptr(patches), _ptr(resized), _stream()),
             "sdb_clip_resize_patches")
    _count()
    return patches, resized


def vit_embed(pe, cls_pos, pos_patches, nb):
    """pe fp32 [nb * np, dim] (patch GEMM output) -> the token sequence fp32 [nb * (np + 1), dim] (sdb_vit_embed)."""
    _chk32(pe, "pe")
    _chk32(cls_pos, "cls_pos")
    _chk32(pos_patches, "pos_patches")
    np_, dim = pos_patches.shape
    assert pe.shape == (nb * np_, dim) and cls_pos.shape == (dim,)
    x = torch.empty((nb * (np_ + 1), dim), dtype=torch.float32, device=pe.device)
    _l.check(_l.load().sdb_vit_embed(_ptr(pe), _ptr(cls_pos), _ptr(pos_patches), nb, np_, dim, _ptr(x), _stream()),
             "sdb_vit_embed")
    _count()
    return x


def rows_gather(x, rows, row_stride):
    """x fp32 [>= (rows - 1) * row_stride + 1, dim] -> fp32 [rows, dim] of every row_stride-th row (sdb_rows_gather)."""
    _chk32(x, "x")
    dim = x.shape[-1]
    assert x.numel() // dim >= (rows - 1) * row_stride + 1
    out = torch.empty((rows, dim), dtype=torch.float32, device=x.device)
    _l.check(_l.load().sdb_rows_gather(_ptr(x), rows, row_stride, dim, _ptr(out), _stream()), "sdb_rows_gather")
    _count()
    return out


def upsample2x(x):
    _chk32(x, "x")
    nb, h, w, c = x.shape
    out = torch.empty((nb, 2 * h, 2 * w, c), dtype=torch.float16, device=x.device)
    _l.check(_l.load().sdb_upsample2x(_ptr(x), nb, h, w, c, _ptr(out), _stream()), "sdb_upsample2x")
    _count()
    return out


def cast_f16(x):
    _chk32(x, "x")
    out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _l.check(_l.load().sdb_cast_f16(_ptr(x), x.numel(), _ptr(out), _stream()), "sdb_cast_f16")
    _count()
    return out


def silu_f16(x):
    _chk32(x, "x")
    out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _l.check(_l.load().sdb_silu_f16(_ptr(x), x.numel(), _ptr(out), _stream()), "sdb_silu_f16")
    _count()
    return out


def transpose_f16(x, ldo=None, out=None):
    """x fp16 [B, rows, cols] -> [B, cols, ldo] (rows valid, ldo >= rows, multiple of 8 for TMA)."""
    _chk16(x, "x")
    B, rows, cols = x.shape
    if ldo is None:
        ldo = (rows + 7) // 8 * 8
    if out is None:
        out = torch.empty((B, cols, ldo), dtype=torch.float16, device=x.device)  # pad columns are never read
    assert out.shape == (B, cols, ldo) and out.is_contiguous()
    _l.check(_l.load().sdb_transpose_f16(_ptr(x), B, rows, cols, cols, _ptr(out), ldo, _stream()),
             "sdb_transpose_f16")
    _count()
    return out


def timestep_embedding(t, dim, max_period=10000.0):
    _chk32(t, "t")
    out = torch.empty((t.numel(), dim), dtype=torch.float16, device=t.device)
    _l.check(_l.load().sdb_timestep_embedding(_ptr(t), t.numel(), dim, max_period, _ptr(out), _stream()),
             "sdb_timestep_embedding")
    _count()
    return out


def timestep_embedding_f32(t, dim, max_period=10000.0):
    _chk32(t, "t")
    out = torch.empty((t.numel(), dim), dtype=torch.float32, device=t.device)
    _l.check(_l.load().sdb_timestep_embedding_f32(_ptr(t), t.numel(), dim, max_period, _ptr(out), _stream()),
             "sdb_timestep_embedding_f32")
    _count()
    return out


def linear_small(x, w, bias=None, act=ACT_NONE, want_f16=False, out=None):
    """x fp32 [m, k] (m small), w fp16 [n, k] -> fp32 [m, n] (fp32 activations end to end), into `out` if given."""
    _chk32(x, "x")
    _chk16(w, "w")
    m, k = x.shape
    n = w.shape[0]
    if out is None:
        out = torch.empty((m, n), dtype=torch.float32, device=x.device)
    _chk32(out, "out")
    assert out.shape == (m, n)
    out16 = torch.empty((m, n), dtype=torch.float16, device=x.device) if want_f16 else None
    _l.check(_l.load().sdb_linear_small(_ptr(x), m, k, _ptr(w), n, _ptr(bias), act, _ptr(out), _ptr(out16),
                                        _stream()), "sdb_linear_small")
    _count()
    return (out, out16) if want_f16 else out


def sampler_step(x, eps2, *, guided, scale, order, hist, noise, a_t, a_prev, sigma_t, sqrt_one_minus_a_t,
                 x_prev=None, pred_x0=None, e_out=None, dup=False, eps_cond=None):
    """One fused CFG + PLMS/DDIM update. x: [b,...] fp32; eps2: [2b,...] if guided else [b,...].
    dup: x_prev is a [2b,...] buffer and both halves receive the new latent (the next step's doubled batch)."""
    _chk32(x, "x")
    _chk32(eps2, "eps2")
    n = x.numel()
    if x_prev is None:
        x_prev = torch.empty((2,) + tuple(x.shape), dtype=torch.float32, device=x.device).flatten(0, 1) if dup \
            else torch.empty_like(x)
    if pred_x0 is None:
        pred_x0 = torch.empty_like(x)
    xp2 = None
    if dup:
        assert x_prev.numel() == 2 * n and x_prev.is_contiguous()
        xp2 = C.c_void_p(x_prev.data_ptr() + 4 * n)
    h = list(hist) + [None] * (3 - len(hist))
    _l.check(_l.load().sdb_sampler_step(_ptr(x), _ptr(eps2), _ptr(eps_cond), 1 if guided else 0, scale, order, _ptr(h[0]),
                                        _ptr(h[1]), _ptr(h[2]), _ptr(noise), a_t, a_prev, sigma_t,
                                        sqrt_one_minus_a_t, n, _ptr(x_prev), xp2, _ptr(pred_x0), _ptr(e_out),
                                        _stream()), "sdb_sampler_step")
    _count()
    return x_prev, pred_x0, e_out


def dpm_solver_step(x, eps2, *, guided, scale, sigma_s, alpha_s, order, m_prev, c_x, c_m, inv_r0, x_out, dup=False,
                    eps_cond=None):
    """One fused CFG + data-prediction + DPM-Solver++ (2M) update; returns (x_out, m0). dup as in sampler_step."""
    _chk32(x, "x")
    _chk32(eps2, "eps2")
    n = x.numel()
    m_out = torch.empty_like(x)
    xo2 = None
    if dup:
        assert x_out.numel() == 2 * n and x_out.is_contiguous()
        xo2 = C.c_void_p(x_out.data_ptr() + 4 * n)
    _l.check(_l.load().sdb_dpm_solver_step(_ptr(x), _ptr(eps2), _ptr(eps_cond), 1 if guided else 0, scale, sigma_s, alpha_s, order,
                                           _ptr(m_prev), c_x, c_m, inv_r0, n, _ptr(m_out), _ptr(x_out), xo2,
                                           _stream()), "sdb_dpm_solver_step")
    _count()
    return x_out, m_out


def mask_blend(img_orig, mask, img, b, dup=False):
    """img[:b] = img_orig * mask + (1 - mask) * img[:b], in place; dup also writes the result to img[b:2b]."""
    _chk32(img_orig, "img_orig")
    _chk32(mask, "mask")
    _chk32(img, "img")
    nb, c = img_orig.shape[0], img_orig.shape[1]
    hw = img_orig[0, 0].numel()
    assert nb == b and mask.shape[0] == nb and mask[0, 0].numel() == hw, (img_orig.shape, mask.shape)
    i2 = C.c_void_p(img.data_ptr() + 4 * img_orig.numel()) if dup else None
    _l.check(_l.load().sdb_mask_blend(_ptr(img_orig), _ptr(mask), mask.shape[1], nb, c, hw, _ptr(img), i2, _stream()),
             "sdb_mask_blend")
    _count()
    return img


LOSS_KINDS = {"l1": 1, "l2": 2}


def _check_t(t, nb, num_timesteps):
    assert t.dtype == torch.int64 and t.is_cuda and t.is_contiguous() and t.shape == (nb,), \
        f"t: need contiguous cuda int64 [{nb}], got {t.dtype} {tuple(t.shape)} on {t.device}"
    lo, hi = (int(v) for v in torch.stack([t.min(), t.max()]).cpu())
    if lo < 0 or hi >= num_timesteps:
        raise IndexError(f"timesteps must lie in [0, {num_timesteps}), got min {lo} and max {hi}")


def q_sample_t(x0, noise, t, sqrt_ac, sqrt_1m_ac):
    """sqrt_ac[t_b] * x0 + sqrt_1m_ac[t_b] * noise with one int64 timestep per sample (sdb_q_sample_t). Raises
    IndexError, before any launch, when a t lies outside the schedule."""
    _chk32(x0, "x0")
    _chk32(noise, "noise")
    _chk32(sqrt_ac, "sqrt_ac")
    _chk32(sqrt_1m_ac, "sqrt_1m_ac")
    assert noise.shape == x0.shape and sqrt_ac.shape == sqrt_1m_ac.shape and sqrt_ac.dim() == 1
    nb = x0.shape[0]
    _check_t(t, nb, sqrt_ac.numel())
    out = torch.empty_like(x0)
    _l.check(_l.load().sdb_q_sample_t(_ptr(x0), _ptr(noise), _ptr(t), _ptr(sqrt_ac), _ptr(sqrt_1m_ac), nb,
                                      x0[0].numel(), _ptr(out), _stream()), "sdb_q_sample_t")
    _count()
    return out


def diffusion_loss(pred, target, kind, t, logvar, lvlb_weights):
    """Per-sample (loss_simple, loss, loss_vlb) of p_losses before the batch means (sdb_diffusion_loss): fp32 [3, nb].
    kind is "l1" or "l2". Raises IndexError, before any launch, when a t lies outside the tables."""
    _chk32(pred, "pred")
    _chk32(target, "target")
    _chk32(logvar, "logvar")
    _chk32(lvlb_weights, "lvlb_weights")
    assert pred.shape == target.shape and logvar.shape == lvlb_weights.shape and logvar.dim() == 1
    if kind not in LOSS_KINDS:
        raise NotImplementedError(f"unknown loss type '{kind}'")
    nb = pred.shape[0]
    _check_t(t, nb, logvar.numel())
    out = torch.empty((3, nb), dtype=torch.float32, device=pred.device)
    _l.check(_l.load().sdb_diffusion_loss(_ptr(pred), _ptr(target), LOSS_KINDS[kind], _ptr(t), _ptr(logvar),
                                          _ptr(lvlb_weights), nb, pred[0].numel(), _ptr(out), _stream()),
             "sdb_diffusion_loss")
    _count()
    return out


def axpby2(x, y, a, b):
    _chk32(x, "x")
    _chk32(y, "y")
    out = torch.empty_like(x)
    _l.check(_l.load().sdb_axpby2(_ptr(x), _ptr(y), a, b, x.numel(), _ptr(out), _stream()), "sdb_axpby2")
    _count()
    return out


def vae_sample(moments, noise, nb, hw, scale_factor):
    _chk32(moments, "moments")
    z = torch.empty((nb, 4, hw), dtype=torch.float32, device=moments.device)
    _l.check(_l.load().sdb_vae_sample(_ptr(moments), _ptr(noise), nb, hw, scale_factor, _ptr(z), _stream()),
             "sdb_vae_sample")
    _count()
    return z


def to_uint8(x):
    _chk32(x, "x")
    out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    _l.check(_l.load().sdb_to_uint8(_ptr(x), x.numel(), _ptr(out), _stream()), "sdb_to_uint8")
    _count()
    return out


def axpby(x, a, b=0.0, out=None):
    _chk32(x, "x")
    if out is None:
        out = torch.empty_like(x)
    else:
        _chk32(out, "out")
        assert out.numel() == x.numel()
    _l.check(_l.load().sdb_axpby(_ptr(x), a, b, x.numel(), _ptr(out), _stream()), "sdb_axpby")
    _count()
    return out


def pointwise_small(x, w, b=None, alpha=1.0):
    """x fp32 [..., cin] NHWC, w fp32 [cout, cin] -> fp32 [..., cout]."""
    _chk32(x, "x")
    _chk32(w, "w")
    cout, cin = w.shape
    assert x.shape[-1] == cin
    out = torch.empty(tuple(x.shape[:-1]) + (cout,), dtype=torch.float32, device=x.device)
    _l.check(_l.load().sdb_pointwise_small(_ptr(x), x.numel() // cin, cin, cout, _ptr(w), _ptr(b), alpha, _ptr(out),
                                           _stream()), "sdb_pointwise_small")
    _count()
    return out


def embed_tokens(ids, tok, pos):
    """ids int64 [B, n] -> fp32 [B*n, dim]: tok[ids] + pos[:n]. Ids outside [0, vocab) are clamped by the kernel, so
    callers validate them on the host."""
    assert ids.dtype == torch.int64 and ids.is_cuda and ids.is_contiguous()
    B, n = ids.shape
    dim = tok.shape[1]
    assert pos.dim() == 2 and pos.shape[0] >= n and pos.shape[1] == dim, (tuple(ids.shape), tuple(tok.shape),
                                                                         tuple(pos.shape))
    out = torch.empty((B * n, dim), dtype=torch.float32, device=ids.device)
    _l.check(_l.load().sdb_embed_tokens(_ptr(ids), B * n, n, dim, tok.shape[0], _ptr(tok), _ptr(pos), _ptr(out),
                                        _stream()), "sdb_embed_tokens")
    _count()
    return out


# ---- first-stage loss (include/sdb200_ae_loss.h) ----
def lpips_scale(in0, in1, shift, scale):
    """LPIPS ScalingLayer of both NCHW fp32 [nb, 3, h, w] inputs -> NHWC fp32 [2 * nb, h, w, 3] (in0's images first)."""
    _chk32(in0, "in0")
    _chk32(in1, "in1")
    _chk32(shift, "shift")
    _chk32(scale, "scale")
    assert in0.dim() == 4 and in0.shape[1] == 3 and in1.shape == in0.shape, (tuple(in0.shape), tuple(in1.shape))
    assert shift.numel() == 3 and scale.numel() == 3
    nb, _, h, w = in0.shape
    out = torch.empty((2 * nb, h, w, 3), dtype=torch.float32, device=in0.device)
    _l.check(_l.load().sdb_lpips_scale(_ptr(in0), _ptr(in1), nb, h, w, _ptr(shift), _ptr(scale), _ptr(out), _stream()),
             "sdb_lpips_scale")
    _count()
    return out


def maxpool2x2(x):
    """MaxPool2d(2, 2) of NHWC fp16 [nb, h, w, c] -> [nb, h // 2, w // 2, c]."""
    _chk16(x, "x")
    nb, h, w, c = x.shape
    out = torch.empty((nb, h // 2, w // 2, c), dtype=torch.float16, device=x.device)
    _l.check(_l.load().sdb_maxpool2x2(_ptr(x), nb, h, w, c, _ptr(out), _stream()), "sdb_maxpool2x2")
    _count()
    return out


def lpips_head(f, lin_w, acc, first, out=None):
    """One LPIPS layer of the feature pair f fp16 [2 * nb, h, w, c] (in0's samples first), accumulated into the fp64
    per-sample acc [nb] (overwritten when first); out fp32 [nb], when given, receives acc rounded to fp32."""
    _chk16(f, "f")
    _chk32(lin_w, "lin_w")
    n2, h, w, c = f.shape
    nb = n2 // 2
    assert n2 == 2 * nb and lin_w.numel() == c and acc.dtype == torch.float64 and acc.shape == (nb,) and acc.is_cuda
    if out is not None:
        _chk32(out, "out")
        assert out.numel() == nb
    lib = _l.load()
    work = torch.empty(int(lib.sdb_lpips_head_work(nb, h * w)), dtype=torch.float64, device=f.device)
    _l.check(lib.sdb_lpips_head(_ptr(f), nb, h * w, c, _ptr(lin_w), 1 if first else 0, _ptr(work), _ptr(acc),
                                _ptr(out), _stream()), "sdb_lpips_head")
    _count(2)
    return acc


def im2col(x, k, stride, pad, kpad):
    """k x k patches of NHWC fp16 [nb, h, w, c] -> fp16 [nb * ho * wo, kpad], column (ky * k + kx) * c + ch."""
    _chk16(x, "x")
    nb, h, w, c = x.shape
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    assert ho > 0 and wo > 0, f"im2col: a {k}x{k} / stride {stride} / pad {pad} conv leaves no pixel of {h}x{w}"
    out = torch.empty((nb * ho * wo, kpad), dtype=torch.float16, device=x.device)
    _l.check(_l.load().sdb_im2col(_ptr(x), nb, h, w, c, k, stride, pad, ho, wo, kpad, _ptr(out), _stream()),
             "sdb_im2col")
    _count()
    return out, ho, wo


AE_TERM_KINDS = {"abs": 1, "kl": 2, "logits": 3}


def ae_loss_terms(a, kind, b=None, n=None, cc=1):
    """Per-sample fp64 sums of sdb_ae_loss_terms: "abs" sum |a - b| of fp32 [nb, ...] pairs -> [1, nb]; "kl" the
    posterior KL of NHWC moments a fp32 [nb, h, w, 2 * cc] -> [1, nb]; "logits" the five logit sums of column 0 of a
    fp32 [nb * n, cc] -> [5, nb]."""
    _chk32(a, "a")
    k = AE_TERM_KINDS[kind]
    if k == 1:
        _chk32(b, "b")
        assert b.shape == a.shape
        nb, n = a.shape[0], a[0].numel()
    elif k == 2:
        nb, n = a.shape[0], a[0].numel() // 2
        assert a.shape[-1] == 2 * cc
    else:
        nb = a.shape[0] // n
        assert a.dim() == 2 and a.shape == (nb * n, cc)
    out = torch.empty((5 if k == 3 else 1, nb), dtype=torch.float64, device=a.device)
    _l.check(_l.load().sdb_ae_loss_terms(_ptr(a), _ptr(b), k, nb, n, cc, _ptr(out), _stream()), "sdb_ae_loss_terms")
    _count()
    return out
