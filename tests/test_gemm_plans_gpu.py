"""Every GEMM tile plan the planner or the autotuner can pick, at every GEMM problem the models issue, against fp64.

Which code runs for one sdb_gemm call depends on its plan (block_n, single CTAs or CTA pairs, no / workspace / cluster
split-K) and on the problem (epilogue kind, TMA-store or scalar path, FiLM column table, statistics). With splits = -1
the planner's cost model picks the plan, and in graph mode the autotuner keeps whichever candidate was fastest in that
run. So any accepted plan can end up behind an image, and each one has to be exact.

The sweep:
  1. records the sdb200.ops.gemm calls of one eager forward of each model (random weights) and deduplicates them by
     everything that reaches the plan or the kernel (geometry, sources, layouts, epilogue, outputs, alignment);
  2. regenerates seeded operands per problem (recorded buffers are overwritten later in the pass) and computes the
     fp64 restatement of the sdb_gemm contract (include/sdb200.h) once, with an abs-value twin for elementwise bounds;
  3. launches the default plan, every autotuner candidate (ops.tune_candidates) and every other explicit plan
     sdb_gemm_plan accepts, into NaN-filled outputs, workspace and statistics, and checks each element, the hi/lo
     pair, the statistics slots and bit-reproducibility.
Failures are collected per model and reported as one table.

Bounds (calibrated on the default plans; the largest observed ratio is printed per model):
  fp32 output      |out - ref| <= TAU * absref everywhere, absref = |alpha||A||B|^T + |bias| + |film| + |res|, and
                   rel-L2 < REL_L2 * max(1, sqrt(K / 4608)): the unsplit plans of the 3x3 convs over the widest skip
                   concats (K = 9 x 2560 = 23040) reach 1.5e-5, default plans included
  fp16 output      |out - ref| <= ulp16(ref) + TAU * absref
  SILU/QUICK_GELU/GELU  |out - ref| <= 1.2 TAU * absref + ACT_REL * |v| (+ one fp16 ulp for fp16 outputs)
  RELU / LEAKY_RELU     |out - ref| <= TAU * absref (+ LRELU_ULPS u |v| for the fp32 slope 0.2f x): both are
                        1-Lipschitz; they run in epilogue kind 4, which never splits K
  GEGLU            |out - ref| <= ulp16 + TAU (|gelu(g)| absref_x + 1.2 |x| absref_g) + ACT_REL |x| (|g| + 1)
  hi/lo            hi == fp16(f32); |hi + lo - f32| <= 2e-6 |f32| + 6e-8
  statistics       every slot finite, T as sdb_gemm_plan reports it, and the slots summed over T within 1e-5 of the
                   fp64 sum of |x| (sum of x^2) of the kernel's own fp32 output
"""
import ctypes as C
import math
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

import helpers  # noqa: F401  (puts the repository on sys.path)
from helpers import rel_l2
from sdb200 import arch, ops
from sdb200 import lib as _l
from sdb200.lib import ACT_GEGLU, ACT_GELU, ACT_LEAKY_RELU, ACT_NONE, ACT_QUICK_GELU, ACT_RELU, ACT_SILU
from sweeps import NAN, Tally, check_coverage, eoff, record, ulp16
from workloads import GEMM_WORKLOADS, _unet

TAU = 1e-5        # elementwise bound of the fp32 accumulation, relative to the abs-value reference
REL_L2 = 1e-5     # rel-L2 of fp32 outputs for K <= 4608, growing as sqrt(K) beyond (one 64-deep wgmma K step after another)
ACT_REL = 4e-6    # __expf / rcp.approx / erf polynomial inside the epilogue activations, relative to |v|
LRELU_ULPS = 4 * 2.0 ** -24   # LeakyReLU's 0.2f * x: 0.2f is 0.2 (1 + 1.5e-8), and the product rounds once
RELU_FAMILY = (ACT_RELU, ACT_LEAKY_RELU)
BNS = (32, 64, 128, 160, 256)
MODES = [(1, 0), (2, 2), (4, 2)] + [(s, 1) for s in (2, 3, 4, 6, 8, 12, 16, 24, 32)]


# ------------------------------------------------------------------------------------------------ fp64 reference
def gemm_ref(srcs, b, *, taps=1, conv_stride=1, conv_shift=0, alpha=1.0, bias=None, film=None, rows_per_sample=0,
             residual=None):
    """fp64 restatement of sdb_gemm before the activation: v = alpha * A B^T + bias + film[m / rps] + residual, and its
    abs-value twin |alpha| |A| |B|^T + |bias| + |film| + |residual|. srcs are concatenated along K; B holds
    taps * sum(ceil64(c_i)) columns (one source of one tap: exactly c0), k = tap * sum(ceil64(c_i)) + offset_i + c.
    taps = 9: 3x3 conv over NHWC sources, input pixel = stride * o + tap - 1 + shift per axis."""
    chans = [s.shape[-1] for s in srcs]
    n = b.shape[0]
    C_ = sum(chans)
    bd = b.double()
    if len(srcs) == 1 and taps == 1:
        wk = bd[:, None, :]
    else:
        pads = [(c + 63) // 64 * 64 for c in chans]
        bt = bd.view(n, taps, sum(pads))
        parts, off = [], 0
        for c, pc in zip(chans, pads):
            parts.append(bt[:, :, off: off + c])
            off += pc
        wk = torch.cat(parts, -1)
    a = torch.cat([s.double() for s in srcs], -1)
    if taps == 1:
        A = a.reshape(-1, C_)
        acc = A @ wk[:, 0].t()
        aacc = A.abs() @ wk[:, 0].abs().t()
        hw = A.shape[0]
    else:
        x = a.permute(0, 3, 1, 2)
        w = wk.view(n, 3, 3, C_).permute(0, 3, 1, 2)
        pad = 1
        if conv_shift:
            x = F.pad(x, (0, 1, 0, 1))
            pad = 0
        conv = lambda xx, ww: F.conv2d(xx, ww, stride=conv_stride, padding=pad)
        o = conv(x, w)
        ao = conv(x.abs(), w.abs())
        hw = o.shape[2] * o.shape[3]
        acc = o.permute(0, 2, 3, 1).reshape(-1, n)
        aacc = ao.permute(0, 2, 3, 1).reshape(-1, n)
    v = alpha * acc
    av = abs(alpha) * aacc
    if bias is not None:
        v = v + bias.double()
        av = av + bias.double().abs()
    if film is not None:
        rps = rows_per_sample or hw
        idx = torch.arange(v.shape[0], device=v.device) // rps
        f = film.double()[idx]
        v = v + f
        av = av + f.abs()
    if residual is not None:
        v = v + residual.double()
        av = av + residual.double().abs()
    return v, av


def _gelu64(g):
    return 0.5 * g * (1.0 + torch.erf(g * 0.5 ** 0.5))


def act_ref(v, av, act, bn):
    """(out, bound without the fp16 rounding term, n_out columns) of the epilogue activation in fp64."""
    if act == ACT_NONE:
        return v, TAU * av
    if act in (ACT_SILU, ACT_QUICK_GELU):
        s = 1.702 if act == ACT_QUICK_GELU else 1.0
        return v * torch.sigmoid(s * v), 1.2 * TAU * av + ACT_REL * v.abs()
    if act == ACT_GELU:     # exact GELU; its slope is within [-0.17, 1.13], bound as SILU's
        return _gelu64(v), 1.2 * TAU * av + ACT_REL * v.abs()
    if act == ACT_RELU:
        return torch.where(v < 0, torch.zeros_like(v), v), TAU * av
    if act == ACT_LEAKY_RELU:
        return torch.where(v > 0, v, 0.2 * v), TAU * av + LRELU_ULPS * v.abs()
    if act != ACT_GEGLU:
        raise ValueError(f"act_ref: no reference for activation {act}")
    M, n = v.shape      # GEGLU: each accumulator tile of bn columns is [bn/2 values | bn/2 gates]
    vv, aa = v.view(M, n // bn, 2, bn // 2), av.view(M, n // bn, 2, bn // 2)
    x, g, ax, ag = vv[:, :, 0], vv[:, :, 1], aa[:, :, 0], aa[:, :, 1]
    out = (x * _gelu64(g)).reshape(M, n // 2)
    bound = TAU * (_gelu64(g).abs() * ax + 1.2 * x.abs() * ag) + ACT_REL * x.abs() * (g.abs() + 1.0)
    return out, bound.reshape(M, n // 2)


# ------------------------------------------------------------------------------------------------ problem catalogue
def signature(a0, b, kw):
    """Everything of one ops.gemm call that reaches the plan or the kernel, as a hashable tuple of items."""
    srcs = [a0] + [kw[k] for k in ("a1", "a2", "a3") if kw.get(k) is not None]
    taps = kw.get("taps", 1)
    geo = tuple(a0.shape[:3]) if taps == 9 else (a0.numel() // a0.shape[-1],)
    film, res = kw.get("film"), kw.get("residual")
    act = kw.get("act", ACT_NONE)
    f16 = kw.get("out_f16") is not None or kw.get("want_f16", False) or kw.get("want_lo", False)
    lo = kw.get("out_f16_lo") is not None or kw.get("want_lo", False)
    f32 = kw.get("out_f32") is not None or kw.get("want_f32", False)
    if res is not None:
        res = res.view(-1, res.shape[-1])
    p = dict(
        geo=geo, taps=taps, conv_stride=kw.get("conv_stride", 1), conv_shift=kw.get("conv_shift", 0),
        chans=tuple(s.shape[-1] for s in srcs), hilo=len(srcs) == 3 and srcs[2] is srcs[0],
        n=kw.get("n") or b.shape[0], b_dynamic=bool(kw.get("b_dynamic", False)),
        bias=kw.get("bias") is not None,
        film=None if film is None else (film.stride(0), film.storage_offset() % film.stride(0), film.shape[0]),
        rps=kw.get("rows_per_sample", 0),
        res=None if res is None else (res.stride(0), eoff(res)),
        act=act, f16=f16, f32=f32, lo=lo,
        out_off=tuple(eoff(kw[k]) if kw.get(k) is not None else 0 for k in ("out_f16", "out_f32", "out_f16_lo")),
        alpha=float(kw.get("alpha", 1.0)), stats=bool(kw.get("want_stats", False)), sg=kw.get("stats_group", 1),
        splits=kw.get("splits", 0), block_n=kw.get("block_n", 0), pair=kw.get("pair", 0),
        splitk_mode=kw.get("splitk_mode", 0))
    return tuple(sorted(p.items()))


def catalogue(workload, dev):
    """The distinct ops.gemm problems of one run of workload(dev), in first-call order."""
    return record(workload, dev, {"gemm": lambda a0, b, **kw: dict(signature(a0, b, kw))})[1]


def label(p):
    g = "x".join(str(v) for v in p["geo"])
    bits = [f"{'conv' if p['taps'] == 9 else 'mm'}[{g}]", f"c={'+'.join(map(str, p['chans']))}", f"n={p['n']}"]
    if p["conv_stride"] == 2:
        bits.append(f"s2/shift{p['conv_shift']}")
    bits += [k for k in ("hilo", "bias", "b_dynamic") if p[k]]
    if p["film"]:
        bits.append("film(ld%d,off%d)" % p["film"][:2])
    if p["res"]:
        bits.append("res(ld%d)" % p["res"][0])
    if p["rps"]:
        bits.append(f"rps={p['rps']}")
    if p["act"]:
        bits.append({1: "geglu", 2: "qgelu", 3: "silu", 4: "gelu", 6: "relu", 7: "lrelu"}[p["act"]])
    if p["alpha"] != 1.0:
        bits.append(f"alpha={p['alpha']:g}")
    bits.append("out=" + "".join(k for k in ("f16", "f32", "lo") if p[k]))
    if p["stats"]:
        bits.append(f"stats/{p['sg']}")
    bits.append(f"splits={p['splits']}")
    return " ".join(bits)


# ------------------------------------------------------------------------------------------------ operands
def _buf(shape, dtype, off, dev, fill=NAN):
    n = 1
    for s in shape:
        n *= s
    return torch.full((n + off + 8,), fill, dtype=dtype, device=dev)[off: off + n].view(shape)


class Operands:
    """Seeded fresh operands at a problem's recorded shapes, strides and alignments."""

    def __init__(self, p, dev, seed):
        g = torch.Generator(device=dev).manual_seed(seed)
        rn = lambda *s: torch.randn(*s, generator=g, device=dev)
        self.p = p
        taps, chans, n = p["taps"], p["chans"], p["n"]
        shape = p["geo"]
        srcs = []
        for i, c in enumerate(chans):
            if p["hilo"] and i == 2:
                srcs.append(srcs[0])                                  # [A_hi | A_lo | A_hi]
            else:
                srcs.append((rn(*shape, c) * (1e-3 if p["hilo"] and i == 1 else 1.0)).half())
        self.srcs = srcs
        K = taps * sum(chans)
        if len(chans) == 1 and taps == 1:
            self.b = (rn(n, chans[0]) * K ** -0.5).half()
        else:   # zero tails: a source of width c % 64 == 32 is padded to whole 64-wide K steps in B
            pads = [(c + 63) // 64 * 64 for c in chans]
            bt = torch.zeros(n, taps, sum(pads), device=dev)
            off = 0
            for c, pc in zip(chans, pads):
                bt[:, :, off: off + c] = rn(n, taps, c) * K ** -0.5
                off += pc
            self.b = bt.reshape(n, -1).half()
        if taps == 9:
            nb, ih, iw = shape
            if p["conv_stride"] == 2:
                h, w = (ih + 1 - p["conv_shift"]) // 2, (iw + 1 - p["conv_shift"]) // 2
            else:
                h, w = ih, iw
            self.M, self.hw = nb * h * w, h * w
        else:
            self.M = self.hw = shape[0]
        self.n_out = n // 2 if p["act"] == ACT_GEGLU else n
        self.bias = rn(n) if p["bias"] else None
        self.film = None
        if p["film"]:
            ldf, off, rows = p["film"]
            self.film = rn(rows, ldf)[:, off: off + n]               # a column slice of a wider matrix (UNetModel._res)
        self.residual = None
        if p["res"]:
            ldr, off = p["res"]
            self.residual = _buf((self.M, ldr), torch.float32, off, dev)
            self.residual.copy_(rn(self.M, ldr))
            self.residual = self.residual[:, :self.n_out]
        self.dev = dev

    def kwargs(self):
        p = self.p
        kw = dict(taps=p["taps"], bias=self.bias, film=self.film, rows_per_sample=p["rps"], residual=self.residual,
                  act=p["act"], alpha=p["alpha"], want_stats=p["stats"], stats_group=p["sg"],
                  b_dynamic=p["b_dynamic"], conv_stride=p["conv_stride"], conv_shift=p["conv_shift"])
        for i, k in enumerate(("a1", "a2", "a3")[: len(self.srcs) - 1]):
            kw[k] = self.srcs[i + 1]
        return kw

    def outputs(self):
        p = self.p
        o16, o32, olo = p["out_off"]
        mk = lambda want, dt, off: _buf((self.M, self.n_out), dt, off, self.dev) if want else None
        return dict(out_f16=mk(p["f16"], torch.float16, o16), out_f32=mk(p["f32"], torch.float32, o32),
                    out_f16_lo=mk(p["lo"], torch.float16, olo))

    def reference(self, bn):
        p = self.p
        v, av = gemm_ref(self.srcs, self.b, taps=p["taps"], conv_stride=p["conv_stride"], conv_shift=p["conv_shift"],
                         alpha=p["alpha"], bias=self.bias, film=self.film, rows_per_sample=p["rps"],
                         residual=self.residual)
        out, bound = act_ref(v, av, p["act"], bn)
        return v, out, bound


# ------------------------------------------------------------------------------------------------ plans
def _plan(d):
    plan = (C.c_int32 * 5)()
    rc = _l.load().sdb_gemm_plan(C.byref(d), plan)
    return None if rc else tuple(plan)


def _copy(d):
    return ops.GemmDesc.from_buffer_copy(d)


def explicit_plans(d, geglu_bn):
    """Every (block_n, pair, splits, mode) that sdb_gemm_plan accepts as an explicit request and honours, with the
    split-K workspace attached; GEGLU keeps its packed tile width."""
    out = {}
    dd = _copy(d)
    dd.workspace = ops.splitk_workspace(torch.device("cuda", torch.cuda.current_device())).data_ptr()
    dd.workspace_floats = ops.WS_FLOATS
    for bn in ((geglu_bn,) if geglu_bn else BNS):
        for cg in (1, 2):
            for sp, mode in MODES:
                dd.block_n, dd.pair, dd.splits, dd.splitk_mode = bn, cg, sp, mode
                pl = _plan(dd)
                if pl and pl[:4] == (bn, cg, sp, mode if sp > 1 else 0):
                    out[(bn, cg, sp, mode if sp > 1 else 0)] = pl[4]
    return out


def split_requests_not_unsplit(d):
    """The split-K requests (splits -1, 2, 8; workspace or cluster mode) of a ReLU-family problem that sdb_gemm_plan
    does not resolve to one split, with the plan it chose: kind 4 has no split-K second pass and no cluster split-K."""
    bad = []
    dd = _copy(d)
    dd.workspace = ops.splitk_workspace(torch.device("cuda", torch.cuda.current_device())).data_ptr()
    dd.workspace_floats = ops.WS_FLOATS
    dd.block_n, dd.pair = 0, 0
    for sp in (-1, 2, 8):
        for mode in (0, 2):
            dd.splits, dd.splitk_mode = sp, mode
            pl = _plan(dd)
            if pl is None or pl[2:4] != (1, 0):
                bad.append(((sp, mode), pl))
    return bad


def tuner_view(d, p, stats_ok):
    """The descriptor gemm() hands to the autotuner for this request: nothing explicit, statistics placeholder."""
    dd = _copy(d)
    dd.block_n, dd.pair, dd.splitk_mode, dd.splits = 0, 0, 0, p["splits"]
    if p["splits"] != -1:
        dd.workspace, dd.workspace_floats = None, 0
    dd.stats_out = 16 if stats_ok else None
    return dd


def _pow2_divisor(v, cap):
    q = 1
    while q * 2 <= cap and v % (q * 2) == 0:
        q *= 2
    return q


def classify(d, plan, sms):
    """Branch classes of gemm_tc.cu's sdb_gemm for this launch (restated from its host code)."""
    bn, cg, sp, mode = plan[:4]
    geglu = d.act == ACT_GEGLU
    n_out = d.n // 2 if geglu else d.n
    ldo, ldf, ldr = d.ldo or n_out, d.ldf or d.n, d.ldr or d.n
    al = lambda q: not q or q % 16 == 0
    fast_possible = (n_out % 32 == 0 and ldo % 8 == 0 and al(d.bias) and (not d.film or (al(d.film) and ldf % 4 == 0))
                     and (not d.residual or (al(d.residual) and ldr % 4 == 0)) and al(d.out_f32) and al(d.out_f16)
                     and al(d.out_f16_lo))
    ws = sp > 1 and mode == 1
    fast = fast_possible and (not ws or d.n % 32 == 0)
    csk = sp > 1 and mode == 2
    M = d.nb * d.h * d.w
    rps = d.rows_per_sample or d.h * d.w
    if d.taps == 9:
        tw = _pow2_divisor(d.w, 128)
        th = _pow2_divisor(d.h, 128 // tw)
        tn = 128 // (tw * th)
    else:
        tw, th, tn = 128, 1, 1
    film_table = 0
    if d.film:
        film_table = int(rps % 64 == 0) if d.taps == 1 else int(tw * th >= 64 and rps == d.h * d.w)
    kind = 4 if d.act in RELU_FAMILY else 2      # the ReLU family never splits K (no cluster split-K: kind 3)
    if fast and geglu and not d.out_f32 and not d.out_f16_lo and not ws:
        kind = 1
    elif fast and d.act == ACT_NONE and (not d.film or film_table) and not (d.out_f32 and d.out_f16 and d.out_f16_lo):
        kind = 0
    if kind == 0 and csk:
        kind = 3
    cls = {f"kind{kind}", "fast" if fast else "scalar", f"cg{cg}"}
    if d.film:
        cls.add(f"film_table{film_table}")
    if ws:
        sg = d.stats_group or 1
        vec = d.n % 4 == 0 and ldo % 4 == 0 and (not d.residual or ldr % 4 == 0) and (not d.film or ldf % 4 == 0)
        wide = d.n % 160 == 0 and 160 % sg == 0
        narrow = wide and 40 % sg == 0 and (d.n // 160) * ((M + 31) // 32) < 2 * sms
        cls.add("splitk<10>" if vec and narrow else "splitk<40>" if vec and wide else "splitk<32>" if vec
                else "splitk_scalar")
    if csk:
        cls.add(f"cluster{sp}")
    if d.conv_stride == 2:
        cls.add(f"stride2_shift{d.conv_shift}")
    chans = [c for c in (d.c0, d.c1, d.c2, d.c3) if c]
    cls.add(f"nsrc{len(chans)}")
    if any(c % 64 == 32 for c in chans):
        cls.add("tail32")
    if tn > 1:
        cls.add("TN>1")
    return cls


REQUIRED = ({f"kind{k}" for k in range(5)} | {"fast", "scalar", "film_table0", "film_table1", "splitk<10>", "splitk<40>",
            "splitk<32>", "splitk_scalar", "cg1", "cg2", "cluster2", "cluster4", "stride2_shift0", "stride2_shift1",
            "nsrc1", "nsrc2", "nsrc3", "nsrc4", "tail32", "TN>1"})
COVER = defaultdict(int)
TUNER_KEYS = {}     # key -> (candidate set, problem label), over every model of the session
SHARED_KEYS = set()  # keys that more than one problem maps to


# ------------------------------------------------------------------------------------------------ one problem
def _launch(X, outs, plan, ws, arena):
    """One ops.gemm launch of problem X with an explicit plan (or the recorded request when plan is None) into
    NaN-filled outputs, workspace and statistics. Returns (channel_stats of the fp32 output or None, descriptor)."""
    p = X.p
    for t in outs.values():
        if t is not None:
            t.fill_(NAN)
            if hasattr(t, "_sdb_stats"):
                del t._sdb_stats
    ws.fill_(NAN)
    arena.buf.fill_(NAN)
    arena.reset()
    kw = X.kwargs()
    kw.update(outs)
    kw["workspace"] = ws
    if plan is None:
        kw.update(block_n=p["block_n"], pair=p["pair"], splits=p["splits"], splitk_mode=p["splitk_mode"])
    else:
        bn, cg, sp, mode = plan
        kw.update(block_n=bn, pair=cg, splits=sp, splitk_mode=mode)
    rec = []
    ops.RECORD = rec
    try:
        ops.gemm(X.srcs[0], X.b, **kw)
    finally:
        ops.RECORD = None
    d = rec[0][0]
    st = ops.channel_stats(outs["out_f32"]) if outs["out_f32"] is not None else None
    return st, d


def _checks(X, outs, st, v, ref, bound):
    """Scalar results (as 0-d device tensors) of every per-plan check; True / small = pass."""
    p = X.p
    r = {}
    o16, o32, olo = outs["out_f16"], outs["out_f32"], outs["out_f16_lo"]
    if o32 is not None:
        e = (o32.double() - ref).abs()
        r["finite_f32"] = torch.isfinite(o32).all()
        r["elem_f32"] = (e / bound.clamp_min(1e-300)).max()
        r["rel_l2_f32"] = (o32.double() - ref).norm() / ref.norm().clamp_min(1e-30)
    if o16 is not None:
        h = o16.double()
        r["finite_f16"] = torch.isfinite(o16).all()
        r["elem_f16"] = ((h - ref).abs() / (torch.maximum(ulp16(ref), ulp16(h)) + bound)).max()
    if olo is not None:
        s = o16.double() + olo.double()
        r["finite_lo"] = torch.isfinite(olo).all()
        if o32 is not None:
            r["hi_eq_f32"] = torch.equal(o16, o32.half())
            r["hilo_vs_f32"] = ((s - o32.double()).abs() / (2e-6 * o32.double().abs() + 6e-8)).max()
        else:
            r["hilo_vs_ref"] = ((s - ref).abs() / (bound + 2e-6 * ref.abs() + 6e-8)).max()
    if st is not None:
        stats, T, sg = st
        ns = X.M // (p["rps"] or X.hw)
        x = o32.double().view(ns, -1, p["n"] // sg, sg)
        got = stats.double().sum(1)
        r["stats_finite"] = torch.isfinite(stats).all()
        ref_s = torch.stack([x.sum((1, 3)), (x * x).sum((1, 3))], -1)
        abs_s = torch.stack([x.abs().sum((1, 3)), (x * x).sum((1, 3))], -1)
        r["stats_sum"] = ((got - ref_s).abs() / (1e-5 * abs_s + 1e-30)).max()
    return r


def _limits(K):
    return dict(finite_f32=True, elem_f32=1.0, rel_l2_f32=REL_L2 * max(1.0, math.sqrt(K / 4608)), finite_f16=True, elem_f16=1.0, finite_lo=True,
                hi_eq_f32=True, hilo_vs_f32=1.0, hilo_vs_ref=1.0, stats_finite=True, stats_sum=1.0)


def sweep_problem(X, failures, calib, sms, ws, arena):
    """Launch the default plan, every autotuner candidate and every other accepted explicit plan of problem X and
    check each; returns the number of launches."""
    p = X.p
    lim = _limits(p["taps"] * sum(p["chans"]))
    outs = X.outputs()
    outs2 = X.outputs()
    lab = label(p)
    # default plan (the recorded request): also yields the descriptor for enumerating the others
    try:
        st, d = _launch(X, outs, None, ws, arena)
    except AssertionError as e:
        failures.append((lab, "default", "launch", repr(e)[:200]))
        return 0
    default = _plan(d)[:4]
    geglu = p["act"] == ACT_GEGLU
    geglu_bn = default[0] if geglu else 0
    v, ref, bound = X.reference(geglu_bn or 128)
    n_launch = 0
    M = X.M
    rps = p["rps"] or X.hw
    stats_ok = (p["stats"] and p["f32"] and not geglu and (p["taps"] == 9 or p["rps"]) and M % rps == 0
                and p["n"] % p["sg"] == 0)
    plans = [None] + [pl for pl in explicit_plans(d, geglu_bn) if pl != default]
    if p["act"] in RELU_FAMILY:
        for req, pl in split_requests_not_unsplit(d):
            failures.append((lab, f"request splits/mode {req}", "ReLU family split", str(pl)))
        for pl in [default] + plans[1:]:
            if pl[2] > 1:
                failures.append((lab, str(pl), "ReLU family split", "explicit plan accepted"))
    tunable = p["block_n"] == 0 and p["pair"] == 0 and p["splitk_mode"] == 0 and p["splits"] in (0, -1) and not geglu
    cands = []
    if tunable:
        dt = tuner_view(d, p, stats_ok)
        cands, _ = ops.tune_candidates(dt, M, p["n"])
        key = ops.tune_key(tuner_view(d, p, stats_ok), X.b.shape[1], stats_ok)
        prev = TUNER_KEYS.get(key)
        if prev is None:
            TUNER_KEYS[key] = (frozenset(cands), lab)
        else:
            SHARED_KEYS.add(key)
            if prev[0] != frozenset(cands):
                failures.append((lab, "tuner key", "candidates differ from", prev[1]))
        swept = set(plans[1:]) | {default}
        missing = [c for c in cands if c not in swept]
        if missing:
            failures.append((lab, str(missing), "tuner candidate not swept", ""))
    for plan in plans:
        pl_lab = f"default {default}" if plan is None else str(plan)
        try:
            if plan is not None:
                st, d = _launch(X, outs, plan, ws, arena)
            n_launch += 1
            T = st[1] if st is not None else 0
            want_T = _plan(d)[4] if st is not None else 0
            r = _checks(X, outs, st, v, ref, bound)
            keep = {k: t.clone() for k, t in outs.items() if t is not None}
            keep_st = st[0].clone() if st is not None else None
            st2, _ = _launch(X, outs2, plan, ws, arena)
            n_launch += 1
            same = all(torch.equal(keep[k], outs2[k]) for k in keep)
            if keep_st is not None:
                same = same and st2 is not None and torch.equal(keep_st, st2[0])
            vals = {k: (t if isinstance(t, bool) else t.item()) for k, t in r.items()}
        except Exception as e:  # noqa: BLE001 - a fault must name its problem and plan
            raise RuntimeError(f"{lab} plan {pl_lab}: {e}") from e
        if st is not None and T != want_T:
            failures.append((lab, pl_lab, "stats slots T", f"{T} != plan {want_T}"))
        if not same:
            failures.append((lab, pl_lab, "bit-reproducible", "second launch differs"))
        for k, val in vals.items():
            L = lim[k]
            bad = (val is not True) if isinstance(L, bool) else not (val <= L)
            if bad:
                failures.append((lab, pl_lab, k, f"{val:.3e}" if isinstance(val, float) else str(val)))
            elif not isinstance(L, bool):
                key = k if plan is None else k + " (all plans)"
                calib[key] = max(calib.get(key, 0.0), val / L)
        for c in classify(d, _plan(d), sms):
            COVER[c] += 1
    return n_launch


def run_sweep(problems, dev, title):
    sms = _l.load().sdb_sm_count()
    ws = torch.empty(ops.WS_FLOATS, dtype=torch.float32, device=dev)
    arena = ops.StatsArena(dev, 8 * 1024 * 1024)
    tally, calib = Tally(title, "problem, plan, check, value"), {}
    saved = (ops.AUTOTUNE, ops.TUNED, ops.ARENA)
    ops.AUTOTUNE, ops.TUNED, ops.ARENA = False, {}, arena
    try:
        for i, p in enumerate(problems):
            X = Operands(p, dev, 1000 + i)
            tally.launches += sweep_problem(X, tally.failures, calib, sms, ws, arena)
            del X
    finally:
        ops.AUTOTUNE, ops.TUNED, ops.ARENA = saved
    tally.finish(len(problems), "largest share of each bound used (default plans / all plans): "
                 + ", ".join(f"{k} {v:.2f}" for k, v in sorted(calib.items())))


# ------------------------------------------------------------------------------------------------ model workloads
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", list(GEMM_WORKLOADS))
def test_every_plan_of_every_model_problem(cuda_dev, name):
    problems = catalogue(GEMM_WORKLOADS[name], cuda_dev)
    print(f"\n{name}: {len(problems)} distinct GEMM problems")
    assert problems
    run_sweep(problems, cuda_dev, name)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ synthetic problems
def _synthetic(**kw):
    p = dict(geo=(300,), taps=1, conv_stride=1, conv_shift=0, chans=(640,), hilo=False, n=128, b_dynamic=False,
             bias=True, film=None, rps=0, res=None, act=ACT_NONE, f16=False, f32=True, lo=False, out_off=(0, 0, 0),
             alpha=1.0, stats=False, sg=1, splits=-1, block_n=0, pair=0, splitk_mode=0)
    p.update(kw)
    if p["res"] is True:
        p["res"] = (p["n"] // (2 if p["act"] == ACT_GEGLU else 1), 0)
    return p


# contract features no model uses but the C ABI offers, and branches the models may not reach
SYNTHETIC = {
    "n6_workspace_scalar_pass": _synthetic(n=6, res=True, f16=True),                      # N % 4 != 0: scalar second pass
    "n36_scalar_epilogue": _synthetic(geo=(2, 16, 16), taps=9, chans=(128,), n=36, res=True, film=(40, 4, 2)),
    "alpha_split": _synthetic(geo=(512,), chans=(1280,), n=320, alpha=0.37, res=True, f16=True),
    "alpha_conv": _synthetic(geo=(2, 16, 16), taps=9, chans=(320,), n=320, alpha=-1.75, film=(640, 320, 2), res=True),
    "two_sources": _synthetic(geo=(200,), chans=(128, 96), n=192, res=True, f16=True),
    "two_sources_conv": _synthetic(geo=(2, 16, 16), taps=9, chans=(320, 640), n=320, film=(320, 0, 2), res=True,
                                   stats=True, sg=10),
    "four_sources": _synthetic(geo=(384,), chans=(64, 128, 96, 64), n=160, res=True, f16=True),
    "four_sources_conv": _synthetic(geo=(2, 8, 8), taps=9, chans=(64, 32, 64, 128), n=128, film=(128, 0, 2)),
    "silu_split": _synthetic(geo=(256,), chans=(1280,), n=640, act=ACT_SILU, res=True),
    "qgelu_split": _synthetic(geo=(640,), chans=(1024,), n=320, act=ACT_QUICK_GELU, f16=True, f32=False),
    "silu_conv_split": _synthetic(geo=(2, 8, 8), taps=9, chans=(640,), n=640, act=ACT_SILU, f16=True),
    "hilo_film_rows": _synthetic(geo=(2 * 80,), chans=(320, 320, 320), hilo=True, n=320, film=(960, 320, 2), rps=80,
                                 res=True, f16=True, lo=True),
    # epilogue kind 4 (ReLU / LeakyReLU): TMA-store and scalar stores, each output set, FiLM per row and as a column
    # table, residual, statistics and a stride-2 conv; every split-K request resolves to one split
    "relu_conv_f16": _synthetic(geo=(2, 16, 16), taps=9, chans=(128,), n=128, act=ACT_RELU, f16=True, f32=False),
    "lrelu_scalar_n36": _synthetic(n=36, act=ACT_LEAKY_RELU, res=True),
    "relu_f16_f32_lo": _synthetic(geo=(512,), chans=(256,), n=256, act=ACT_RELU, f16=True, lo=True),
    "lrelu_film_rows": _synthetic(geo=(2 * 80,), chans=(320,), n=320, act=ACT_LEAKY_RELU, film=(640, 320, 2), rps=80,
                                  res=True),
    "relu_film_table": _synthetic(geo=(2 * 128,), chans=(512,), n=256, act=ACT_RELU, film=(256, 0, 2), rps=128,
                                  res=True, f16=True),
    "lrelu_conv_stats": _synthetic(geo=(2, 16, 16), taps=9, chans=(64,), n=128, act=ACT_LEAKY_RELU, res=True, stats=True,
                                   sg=4),
    "relu_conv_s2": _synthetic(geo=(2, 32, 32), taps=9, chans=(64,), conv_stride=2, n=128, act=ACT_RELU, f16=True),
    "lrelu_conv_s2_shift": _synthetic(geo=(2, 16, 24), taps=9, chans=(128,), conv_stride=2, conv_shift=1, n=64,
                                      act=ACT_LEAKY_RELU, f16=True, f32=False),
}


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_every_plan_of_synthetic_problems(cuda_dev):
    run_sweep(list(SYNTHETIC.values()), cuda_dev, "synthetic")


@pytest.mark.gpu
def test_row_stride_beyond_output_width_keeps_guard_columns(cuda_dev):
    """ldo > n_out through the descriptor: every plan writes exactly the n_out valid columns of each row; the guard
    columns between rows keep their NaN."""
    g = torch.Generator(device=cuda_dev).manual_seed(7)
    M, K, n, ldo = 640, 1280, 320, 360
    a = torch.randn(M, K, generator=g, device=cuda_dev).half()
    b = (torch.randn(n, K, generator=g, device=cuda_dev) * K ** -0.5).half()
    bias = torch.randn(n, generator=g, device=cuda_dev)
    res = torch.randn(M, n, generator=g, device=cuda_dev)
    v, av = gemm_ref([a], b, bias=bias, residual=res)
    rec = []
    ops.RECORD = rec
    try:
        ops.gemm(a, b, bias=bias, residual=res, want_f32=True, want_f16=True, splits=-1)
    finally:
        ops.RECORD = None
    d = _copy(rec[0][0])
    o32 = torch.empty(M, ldo, device=cuda_dev)
    o16 = torch.empty(M, ldo, dtype=torch.float16, device=cuda_dev)
    ws = torch.empty(ops.WS_FLOATS, device=cuda_dev)
    d.out_f32, d.out_f16, d.ldo, d.stats_out = o32.data_ptr(), o16.data_ptr(), ldo, None
    d.workspace, d.workspace_floats = ws.data_ptr(), ws.numel()
    lib = _l.load()
    bad = []
    plans = explicit_plans(d, 0)
    assert len(plans) > 20
    for plan in plans:
        o32.fill_(NAN)
        o16.fill_(NAN)
        ws.fill_(NAN)
        d.block_n, d.pair, d.splits, d.splitk_mode = plan
        _l.check(lib.sdb_gemm(C.byref(d), ops._stream()), f"sdb_gemm {plan}")
        e32 = float(((o32[:, :n].double() - v).abs() / (TAU * av)).max())
        e16 = float(((o16[:, :n].double() - v).abs() / (ulp16(v) + TAU * av)).max())
        guard = bool(o32[:, n:].isnan().all()) and bool(o16[:, n:].isnan().all())
        if not (e32 <= 1 and e16 <= 1 and guard):
            bad.append((plan, e32, e16, guard))
    assert not bad, bad


@pytest.mark.gpu
def test_branch_coverage_and_tuner_key():
    """Every branch class of sdb_gemm was launched by the sweeps above, and problems that share an autotuner cache key
    accept the same candidates (checked while sweeping; a collision is reported there)."""
    check_coverage(COVER, REQUIRED, "plan")
    print(f"tuner keys: {len(TUNER_KEYS)}, shared by two or more problems: {len(SHARED_KEYS)}")


# ------------------------------------------------------------------------------------------------ ops.gemm layouts
@pytest.mark.gpu
def test_gemm_column_sliced_residual_and_film(cuda_dev):
    g = torch.Generator(device=cuda_dev).manual_seed(9)
    M, K, n = 512, 320, 320
    a = torch.randn(M, K, generator=g, device=cuda_dev).half()
    b = (torch.randn(n, K, generator=g, device=cuda_dev) * K ** -0.5).half()
    wide = torch.randn(M, n + 96, generator=g, device=cuda_dev)
    res = wide[:, 32: 32 + n]                                       # row stride n + 96
    fw = torch.randn(4, 3 * n, generator=g, device=cuda_dev)
    film = fw[:, n: 2 * n]
    for sp in (0, 4):
        _, o32 = ops.gemm(a, b, residual=res, film=film, rows_per_sample=128, want_f32=True, splits=sp)
        v, av = gemm_ref([a], b, residual=res, film=film, rows_per_sample=128)
        assert float(((o32.double() - v).abs() / (TAU * av)).max()) <= 1.0
        assert rel_l2(o32, v) < 1e-5


@pytest.mark.gpu
def test_gemm_rejects_layouts_it_cannot_address(cuda_dev):
    M, K, n = 256, 64, 64
    a = torch.randn(M, K, device=cuda_dev).half()
    b = torch.randn(n, K, device=cuda_dev).half()
    with pytest.raises(AssertionError):
        ops.gemm(a, b, out_f32=torch.empty(M, n + 1, device=cuda_dev))
    with pytest.raises(AssertionError):
        ops.gemm(a, b, out_f32=torch.empty(n, M, device=cuda_dev).t())       # right shape, column-major
    with pytest.raises(AssertionError):
        ops.gemm(a, b, out_f16=torch.empty(M, n, device=cuda_dev), want_f32=True)   # wrong dtype
    with pytest.raises(AssertionError):
        ops.gemm(a, b, residual=torch.randn(n, M, device=cuda_dev).t(), want_f32=True)
    with pytest.raises(AssertionError):
        ops.gemm(a, b, residual=torch.randn(M, n + 1, device=cuda_dev), want_f32=True)
    with pytest.raises(AssertionError):
        ops.gemm(a, b, film=torch.randn(n, 2, device=cuda_dev).t(), rows_per_sample=128, want_f32=True)
    with pytest.raises(AssertionError):
        ops.gemm(a, b, bias=torch.randn(2 * n, device=cuda_dev)[::2], want_f32=True)
    with pytest.raises(AssertionError):
        ops.gemm(a, b, bias=torch.randn(n + 4, device=cuda_dev), want_f32=True)


# ------------------------------------------------------------------------------------------------ small-M kernels
@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 40, 192, 224, 256, 320, 512, 768, 896, 1024, 1280])
@pytest.mark.parametrize("M", [1, 2, 8, 9, 12, 16, 17])
def test_linear_small_vs_fp64(cuda_dev, M, K):
    """out = act(x W^T + b) with fp32 activations; M > 8 takes the kernel's second pass over samples. N is a
    multiple of neither a warp's 4 nor a block's 32 output features."""
    g = torch.Generator(device=cuda_dev).manual_seed(M * 1000 + K)
    for N in (37, 1283):
        x = torch.randn(M, K, generator=g, device=cuda_dev)
        w = (torch.randn(N, K, generator=g, device=cuda_dev) * K ** -0.5).half()
        bias = torch.randn(N, generator=g, device=cuda_dev)
        acc = x.double() @ w.double().t()
        absref = x.double().abs() @ w.double().abs().t() + bias.double().abs()
        v = acc + bias.double()
        for act in (ACT_NONE, ACT_SILU):
            ref = v * torch.sigmoid(v) if act == ACT_SILU else v
            out = torch.full((M, N), NAN, device=cuda_dev)
            o32, o16 = ops.linear_small(x, w, bias, act=act, want_f16=True, out=out)
            bound = 1e-5 * absref * (1.2 if act else 1.0) + ACT_REL * v.abs()
            e32 = float(((o32.double() - ref).abs() / bound).max())
            e16 = float(((o16.double() - ref).abs() / (ulp16(ref) + bound)).max())
            assert bool(torch.isfinite(o32).all()) and bool(torch.isfinite(o16).all()), (M, K, N, act)
            assert e32 <= 1.0 and e16 <= 1.0, (M, K, N, act, e32, e16)
            assert rel_l2(o32, ref) < 2e-6
        o = ops.linear_small(x, w)                          # no bias, fp32 only
        assert float(((o.double() - acc).abs() / (1e-5 * absref + 1e-30)).max()) <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout", [(4, 4), (8, 8), (3, 3), (3, 8)])
@pytest.mark.parametrize("alpha", [1.0, 1 / 0.18215, -0.5])
def test_pointwise_small_alpha_vs_fp64(cuda_dev, cin, cout, alpha):
    """post_quant_conv with 1 / scale_factor folded in as alpha: out = (alpha x) W^T + b."""
    g = torch.Generator(device=cuda_dev).manual_seed(cin * 10 + cout)
    x = torch.randn(2, 64, 61, cin, generator=g, device=cuda_dev)
    w = torch.randn(cout, cin, generator=g, device=cuda_dev)
    bias = torch.randn(cout, generator=g, device=cuda_dev)
    out = ops.pointwise_small(x, w, bias, alpha=alpha)
    ref = (alpha * x.double()) @ w.double().t() + bias.double()
    absref = (abs(alpha) * x.double().abs()) @ w.double().abs().t() + bias.double().abs()
    assert float(((out.double() - ref).abs() / (1e-5 * absref)).max()) <= 1.0


# ------------------------------------------------------------------------------------------------ batch independence
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("tag", ["sdv1_b16", "cin256_b12"])
def test_unet_benchmarked_batch_equals_batches_of_two(cuda_dev, tag):
    """The full benchmarked batch and the same samples evaluated two at a time agree per sample (different tile
    shapes, same arithmetic per sample): FiLM rows, per-sample statistics, linear_small's second pass over samples and
    the attention grid all index samples beyond the batch sizes the reference tests use."""
    cfg, shape, ctx = {"sdv1_b16": (arch.SD_V1_UNET, (16, 4, 64, 64), (77, 768)),
                       "cin256_b12": (arch.CIN256_V2_UNET, (12, 3, 64, 64), (1, 512))}[tag]
    net = _unet(cfg, cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(4)
    x = torch.randn(*shape, generator=g, device=cuda_dev)
    t = torch.linspace(1, 981, shape[0], device=cuda_dev).round()
    c = torch.randn(shape[0], *ctx, generator=g, device=cuda_dev)
    full = net(x, t, context=c).clone()
    assert bool(torch.isfinite(full).all())
    errs = []
    for i in range(0, shape[0], 2):
        part = net(x[i: i + 2].contiguous(), t[i: i + 2].contiguous(), context=c[i: i + 2].contiguous())
        assert bool(torch.isfinite(part).all())
        errs += [rel_l2(full[i + j], part[j]) for j in range(2)]
    print(f"{tag}: per-sample rel-L2 max {max(errs):.2e}")
    assert max(errs) < 1.5e-3, errs


# ------------------------------------------------------------------------------------------------ CPU: the reference
def _naive_conv(srcs, b, stride, shift):
    """Direct 3x3 tap loop over the B layout (k = tap * sum(ceil64) + offset + c), independent of F.conv2d."""
    nb, ih, iw, _ = srcs[0].shape
    chans = [s.shape[-1] for s in srcs]
    pads = [(c + 63) // 64 * 64 for c in chans]
    n = b.shape[0]
    bt = b.double().view(n, 9, sum(pads))
    oh, ow = ((ih + 1 - shift) // 2, (iw + 1 - shift) // 2) if stride == 2 else (ih, iw)
    out = torch.zeros(nb, oh, ow, n, dtype=torch.float64)
    for oy in range(oh):
        for ox in range(ow):
            for ky in range(3):
                for kx in range(3):
                    iy, ix = stride * oy + ky - 1 + shift, stride * ox + kx - 1 + shift
                    if not (0 <= iy < ih and 0 <= ix < iw):
                        continue
                    off = 0
                    for s, c, pc in zip(srcs, chans, pads):
                        out[:, oy, ox] += s[:, iy, ix].double() @ bt[:, ky * 3 + kx, off: off + c].t()
                        off += pc
    return out.reshape(-1, n)


@pytest.mark.parametrize("stride,shift,hw", [(1, 0, (5, 6)), (2, 0, (7, 6)), (2, 1, (6, 7))])
def test_reference_conv_layout_cpu(stride, shift, hw):
    g = torch.Generator().manual_seed(stride * 10 + shift)
    srcs = [torch.randn(2, *hw, c, generator=g).half() for c in (64, 32)]
    n = 8
    b = torch.randn(n, 9 * 128, generator=g).half()
    v, av = gemm_ref(srcs, b, taps=9, conv_stride=stride, conv_shift=shift)
    ref = _naive_conv(srcs, b, stride, shift)
    assert torch.allclose(v, ref, rtol=1e-12, atol=1e-12)
    assert bool((av >= v.abs() - 1e-12).all())


def test_reference_epilogue_cpu():
    g = torch.Generator().manual_seed(1)
    hi = torch.randn(6, 64, generator=g).half()
    lo = (torch.randn(6, 64, generator=g) * 1e-3).half()
    b = torch.randn(256, 3 * 64, generator=g).half()
    bias, res = torch.randn(256, generator=g), torch.randn(6, 256, generator=g)
    film = torch.randn(2, 512, generator=g)[:, 100: 356]
    v, av = gemm_ref([hi, lo, hi], b, alpha=0.5, bias=bias, film=film, rows_per_sample=3, residual=res)
    A = torch.cat([hi, lo, hi], -1).double()
    ref = 0.5 * A @ b.double().t() + bias.double() + film.double().repeat_interleave(3, 0) + res.double()
    assert torch.allclose(v, ref, rtol=1e-12, atol=1e-12)
    out, _ = act_ref(v, av, ACT_GEGLU, 128)
    x, gate = v[:, :64], v[:, 64:128]
    assert torch.allclose(out[:, :64], x * 0.5 * gate * (1 + torch.erf(gate / math.sqrt(2))), rtol=1e-12)
    assert torch.allclose(out[:, 64:], v[:, 128:192] * _gelu64(v[:, 192:]), rtol=1e-12)
    assert float(ulp16(torch.tensor([1.0, 1.5, 2.0, 1e-6]))[0]) == 2.0 ** -10
    assert float(ulp16(torch.tensor([1e-6]))[0]) == 2.0 ** -24


def test_relu_family_reference_cpu():
    """ReLU and LeakyReLU(0.2) in fp64 with the accumulation bound alone (plus the slope's ulps for LeakyReLU); an
    activation without a reference raises instead of being checked against another one."""
    v = torch.tensor([[-2.0, -0.5, 0.0, 3.0]], dtype=torch.float64)
    av = v.abs() + 1.0
    out, bound = act_ref(v, av, ACT_RELU, 128)
    assert out.tolist() == [[0.0, 0.0, 0.0, 3.0]] and torch.equal(bound, TAU * av)
    out, bound = act_ref(v, av, ACT_LEAKY_RELU, 128)
    assert torch.allclose(out, torch.tensor([[-0.4, -0.1, 0.0, 3.0]], dtype=torch.float64), rtol=1e-15)
    assert torch.equal(bound, TAU * av + LRELU_ULPS * v.abs())
    for bad in (5, 8):
        with pytest.raises(ValueError):
            act_ref(v, av, bad, 128)
    assert " relu " in label(_synthetic(act=ACT_RELU)) and " lrelu " in label(_synthetic(act=ACT_LEAKY_RELU))


def test_signature_dedups_and_keeps_layouts_cpu():
    a = torch.zeros(4, 8, 8, 64, dtype=torch.float16)
    b = torch.zeros(32, 9 * 64, dtype=torch.float16)
    film = torch.zeros(4, 96)
    s1 = signature(a, b, dict(taps=9, film=film[:, 32:64], want_f32=True, splits=-1))
    s2 = signature(a.clone(), b.clone(), dict(taps=9, film=film[:, 32:64], want_f32=True, splits=-1))
    s3 = signature(a, b, dict(taps=9, film=film[:, 33:65], want_f32=True, splits=-1))
    s4 = signature(a, b, dict(taps=9, film=film[:, 32:64], want_f32=True, splits=0))
    assert s1 == s2 and len({s1, s3, s4}) == 3
    p = dict(s1)
    assert p["film"] == (96, 32, 4) and p["geo"] == (4, 8, 8) and "film(ld96,off32)" in label(p)
