"""Every normalisation launch the models make (GroupNorm, modulated GroupNorm, LayerNorm, row softmax), elementwise
against fp64.

Which code runs for one norm.cu call depends on the problem: the statistics pass (12 or 14 channels per thread, the
channel-lane width and so how many row lanes meet per channel, the slab count and its 128 cap), where fused statistics
are folded (inside the apply kernel or in gn_fold_kernel), the concatenated source and where a group straddles it, the
LayerNorm template instance, its vector or scalar variant and its warps per block. The sweep:
  1. records the sdb200.ops.groupnorm / groupnorm_mod / layernorm / softmax_rows calls of one eager forward of each
     model (random weights) and deduplicates them by everything that reaches a kernel or a dispatch decision;
  2. regenerates seeded operands at each recorded shape and alignment (recorded buffers are overwritten later in the
     pass); fused statistics are synthesized here from the fp64 sums of row chunks, so the fold is tested on its own;
  3. launches through the C entry points into NaN-filled outputs (with NaN guards around them) and a NaN-filled
     workspace, checks every element against the fp64 reference, the guards, and a bit-equal second launch;
then a synthetic grid covers the edges no model reaches, and a Python mirror of the host dispatch records which
branches ran (test_norm_branch_coverage).

Bounds (z = (x - mean) rstd in fp64, g = gamma (1 + scale), b = beta (1 + scale) + shift, v = z g + b):
  GroupNorm fp16   |out - ref| <= ulp16(ref) + TAU_N (|z||g| + |b|) + APPLY_REL (|x| + |mean|) rstd |g|
                   (x 1.1 + ACT_REL |v| through SiLU; the mean of the four taps' bounds under 2x2 pooling). The
                   APPLY_REL term is the fp32 rounding of the one-FMA apply x a + b, which grows with |mean| / std.
  hi/lo            raw == fp16(x), raw_lo == fp16(x - raw) bit-exact; |out + out_lo - ref| <= the bound above - ulp16
                   + 6e-8
  LayerNorm        |out32 - ref| <= TAU_L (|z||gamma| + |beta|) + APPLY_REL (|x| + |mean|) rstd |gamma|;
                   out16 == fp16(out32) bit-exact when both are written, else ulp16 + the same term
  softmax          |p - ref| <= ulp16(ref) + ref (1e-6 + 1.2e-7 |s x - m| + 6e-8 (|s x| + |m|)), m the row max of s x
The largest share of each bound used is printed per workload.
"""
import ctypes as C
import math
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

import helpers  # noqa: F401  (puts the repository on sys.path)
from sdb200 import ops
from sdb200 import lib as _l
from sweeps import GUARD, NAN, Tally, check_coverage, eoff, record, signature, ulp16
from workloads import WORKLOADS

TAU_N = 8e-6       # GroupNorm: statistics and apply, relative to |z||g| + |b|
TAU_L = 4e-6       # LayerNorm: fp32 two-pass statistics in one warp
APPLY_REL = 3e-7   # fp32 rounding of a = rstd g, b = beta - mean a and x a + b, relative to (|x| + |mean|) rstd |g|
ACT_REL = 4e-6     # __expf / __fdividef inside SiLU, relative to |v|
GN_MAX_SLABS = 128
LN_V2 = {320: 5, 512: 8, 640: 10, 768: 12, 1280: 20}
LN_NPL = (2, 4, 10, 20, 24, 40, 48, 56)


# ------------------------------------------------------------------------------------------------ host dispatch mirror
def gn_branches(p, sms):
    """Branch classes of sdb_groupnorm / sdb_groupnorm_mod for problem p (restated from norm.cu's host code)."""
    C_ = p["c0"] + p["c1"]
    nb, hw, groups = p["nb"], p["h"] * p["w"], p["groups"]
    cpg = C_ // groups
    st = p["stats"]
    mod = p["kind"] == "gnmod"
    fused = st is not None and (mod or groups <= 32)
    cls = {p["kind"]}
    if not fused:
        cw = 256
        while cw > 32 and cw // 2 >= C_:
            cw //= 2
        rstep = 256 // cw
        slabs = max(1, min(min((hw + rstep - 1) // rstep, GN_MAX_SLABS), (sms * 4 + nb - 1) // nb))
        rpb = (hw + slabs - 1) // slabs
        slabs = (hw + rpb - 1) // rpb
        cls |= {"fold:none", f"cpt{14 if C_ > 3072 else 12}", f"rstep{rstep}"}
        if slabs == GN_MAX_SLABS:
            cls.add("slab_cap")
        if hw % rpb:
            cls.add("ragged_slab")
    elif mod or max(st[0], st[1]) * (cpg // st[2]) > 512:
        cls.add("fold:kernel")
    else:
        cls.add("fold:in_apply")
    if hw == 1:
        cls.add("hw1")
    if groups > 32:
        cls.add("groups64")
    if p["c1"]:
        cls.add("x1")
        if p["c0"] % cpg:
            cls.add("x1_straddle" + ("_fused" if fused else ""))
    if not mod:
        cls |= {k for k in ("raw", "lo", "raw_lo") if p[k]}
    else:
        cls.add(f"resample{p['resample']}")
        if p["ldm"]:
            cls.add("modulated")
    return cls


def ln_branches(p, sms):
    c, rows = p["c"], p["rows"]
    wpb = 8 if rows >= 16 * sms else 4 if rows >= 8 * sms else 2 if rows >= 4 * sms else 1
    al8 = all(o % 2 == 0 for o in p["align"])    # x, gamma, beta, out32 8-byte aligned (fp16 out: 4-byte, always)
    cls = {"ln", f"wpb{wpb}"}
    if c % 64 == 0 and al8 and c in LN_V2:
        cls.add(f"ln_v2<{LN_V2[c]}>")
    else:
        npl = (c + 31) // 32
        cls.add(f"ln_npl<{next(n for n in LN_NPL if npl <= n)}>")
    cls |= {k for k in ("ln_f16", "ln_f32") if p[k[3:]]}
    return cls


REQUIRED = ({"cpt12", "cpt14", "rstep1", "rstep2", "rstep4", "rstep8", "slab_cap", "ragged_slab", "hw1", "groups64",
             "fold:none", "fold:in_apply", "fold:kernel", "x1", "x1_straddle", "x1_straddle_fused", "raw", "lo",
             "raw_lo", "gnmod", "resample0", "resample1", "resample2", "modulated", "ln_f16", "ln_f32", "softmax",
             "wpb1", "wpb2", "wpb4", "wpb8"}
            | {f"ln_v2<{n}>" for n in LN_V2.values()} | {f"ln_npl<{n}>" for n in LN_NPL})
COVER = defaultdict(int)


# ------------------------------------------------------------------------------------------------ problem catalogue
def _gn(**kw):
    """A GroupNorm problem (kind 'gn': sdb_groupnorm, 'gnmod': sdb_groupnorm_mod) with defaults for what is not given.
    stats: None (computed by the statistics pass) or (T0, T1, sg) fused partials; a0 / a1: element offsets of the
    sources from a 16-byte boundary; oo: element offset of the outputs; mean / std: operand distribution."""
    p = dict(kind="gn", nb=2, h=8, w=8, c0=320, c1=0, groups=32, eps=1e-5, silu=False, raw=False, lo=False,
             raw_lo=False, stats=None, ldm=0, resample=0, a0=0, a1=0, oo=0, mean=0.5, std=2.0)
    p.update(kw)
    return p


def _ln(**kw):
    p = dict(kind="ln", rows=77, c=768, eps=1e-5, f16=True, f32=False, align=(0, 0, 0, 0), mean=0.5, std=2.0)
    p.update(kw)
    return p


def _sm(**kw):
    p = dict(kind="softmax", rows=4, cols=256, scale=1.0, align=0, mag=3.0, const=False)
    p.update(kw)
    return p


def _gn_sig(x0, gamma, beta, *, x1=None, groups=32, eps=1e-5, silu=False, want_raw=False, want_lo=False,
            want_raw_lo=False):
    nb, h, w, c0 = x0.shape
    c1 = 0 if x1 is None else x1.shape[-1]
    cs0 = ops.channel_stats(x0)
    cs1 = ops.channel_stats(x1) if x1 is not None else None
    sg = cs0[2] if cs0 is not None else 1
    cpg = (c0 + c1) // groups
    stats = None         # the same compatibility test as ops.groupnorm
    if not (cs0 is None or (x1 is not None and (cs1 is None or cs1[2] != sg)) or cpg % sg or c0 % sg or c1 % sg):
        stats = (cs0[1], cs1[1] if cs1 else 0, sg)
    return _gn(nb=nb, h=h, w=w, c0=c0, c1=c1, groups=groups, eps=eps, silu=bool(silu), raw=want_raw or want_raw_lo,
               lo=want_lo, raw_lo=want_raw_lo, stats=stats, a0=eoff(x0), a1=eoff(x1) if x1 is not None else 0)


def _gnmod_sig(x, gamma, beta, *, scale=None, shift=None, resample=0, groups=32, eps=1e-5, silu=True):
    nb, h, w, c = x.shape
    cs = ops.channel_stats(x)
    stats = None
    if cs is not None and not ((c // groups) % cs[2] or c % cs[2]):
        stats = (cs[1], 0, cs[2])
    return _gn(kind="gnmod", nb=nb, h=h, w=w, c0=c, groups=groups, eps=eps, silu=bool(silu), stats=stats,
               ldm=scale.stride(0) if scale is not None else 0, resample=resample, a0=eoff(x))


def _ln_sig(x, gamma, beta, eps=1e-5, want_f32=False):
    c = x.shape[-1]
    return _ln(rows=x.numel() // c, c=c, eps=eps, f32=bool(want_f32), align=(eoff(x), eoff(gamma), eoff(beta), 0))


def _sm_sig(x, scale):
    cols = x.shape[-1]
    return _sm(rows=x.numel() // cols, cols=cols, scale=float(scale), align=eoff(x))


SIGS = {"groupnorm": _gn_sig, "groupnorm_mod": _gnmod_sig, "layernorm": _ln_sig, "softmax_rows": _sm_sig}


def label(p):
    if p["kind"] == "ln":
        return f"ln[{p['rows']}x{p['c']}] align{p['align']} out={'f16' * p['f16']}{'f32' * p['f32']}"
    if p["kind"] == "softmax":
        return f"softmax[{p['rows']}x{p['cols']}] scale={p['scale']:g} align{p['align']}"
    bits = [f"{p['kind']}[{p['nb']}x{p['h']}x{p['w']}]", f"c={p['c0']}" + (f"+{p['c1']}" if p["c1"] else ""),
            f"g{p['groups']}"]
    bits += [k for k in ("silu", "raw", "lo", "raw_lo") if p[k]]
    if p["stats"]:
        bits.append("stats(T%d,%d,sg%d)" % p["stats"])
    if p["ldm"]:
        bits.append(f"mod(ld{p['ldm']})")
    if p["resample"]:
        bits.append(("", "down", "up")[p["resample"]])
    if p["a0"] or p["a1"] or p["oo"]:
        bits.append(f"off({p['a0']},{p['a1']},{p['oo']})")
    if (p["mean"], p["std"]) != (0.5, 2.0):
        bits.append(f"mean/std {p['mean']:g}/{p['std']:g}")
    return " ".join(bits)


# ------------------------------------------------------------------------------------------------ operands
def _input(shape, off, gen, mean, std, chan_mean=True):
    """Seeded fp32 operand at element offset `off` of its allocation: mean + std randn, plus a per-channel offset of
    std / 2 randn so the channels of a group differ."""
    n = math.prod(shape)
    buf = torch.empty(n + off + 4, device=gen.device)
    x = buf[off: off + n].view(shape)
    v = torch.randn(shape, generator=gen, device=gen.device, dtype=torch.float64) * std + mean
    if chan_mean:
        v = v + torch.randn(shape[-1], generator=gen, device=gen.device, dtype=torch.float64) * (std / 2)
    x.copy_(v)
    return x


def _out(shape, dtype, off, dev):
    """(whole NaN buffer, view of `shape` at element offset GUARD + off): the rest of the buffer is the guard."""
    n = math.prod(shape)
    buf = torch.full((n + off + 2 * GUARD,), NAN, dtype=dtype, device=dev)
    return buf, buf[GUARD + off: GUARD + off + n].view(shape)


def _guard_ok(buf, view):
    lo = view.storage_offset() - buf.storage_offset()
    return bool(buf[:lo].isnan().all()) and bool(buf[lo + view.numel():].isnan().all())


def partials(x, T, sg):
    """Fused GroupNorm statistics as a producing GEMM stores them: fp32 [nb, T, c / sg, 2] {sum x, sum x^2} per chunk of
    rows (the rows of each sample split into T contiguous chunks) and entry of sg channels, summed in fp64."""
    nb, hw, c = x.shape
    xd = x.double().view(nb, hw, c // sg, sg)
    s = torch.stack([xd.sum(3), (xd * xd).sum(3)], -1)                 # [nb, hw, E, 2]
    cs = torch.cat([torch.zeros_like(s[:, :1]), s.cumsum(1)], 1)       # prefix sums over rows
    edges = torch.tensor([hw * t // T for t in range(T + 1)], device=x.device)
    return (cs[:, edges[1:]] - cs[:, edges[:-1]]).float().contiguous()


class GNOperands:
    def __init__(self, p, dev, seed):
        g = torch.Generator(device=dev).manual_seed(seed)
        nb, h, w, c0, c1 = p["nb"], p["h"], p["w"], p["c0"], p["c1"]
        C_ = c0 + c1
        self.p, self.dev = p, dev
        self.x0 = _input((nb, h, w, c0), p["a0"], g, p["mean"], p["std"])
        self.x1 = _input((nb, h, w, c1), p["a1"], g, p["mean"], p["std"]) if c1 else None
        if p.get("flat_group") is not None:         # one near-constant group: variance far below eps
            k = p["flat_group"]
            cpg = C_ // p["groups"]
            x = self.x0 if (k + 1) * cpg <= c0 else None
            if x is not None:
                x[..., k * cpg: (k + 1) * cpg] = 3.0 + 1e-6 * torch.randn(nb, h, w, cpg, generator=g, device=dev)
        self.gamma = torch.randn(C_, generator=g, device=dev)
        self.beta = torch.randn(C_, generator=g, device=dev) * 0.5
        self.scale = self.shift = None
        if p["ldm"]:          # column slices of row stride ldm: of one FiLM output when it holds both, else of two
            film = torch.randn(nb, p["ldm"], generator=g, device=dev) * 0.5
            self.scale = film[:, :C_]
            self.shift = (film[:, C_: 2 * C_] if p["ldm"] >= 2 * C_ else
                          (torch.randn(nb, p["ldm"], generator=g, device=dev) * 0.5)[:, :C_])
        self.cs0 = self.cs1 = None
        if p["stats"]:
            T0, T1, sg = p["stats"]
            self.cs0 = partials(self.x0.view(nb, h * w, c0), T0, sg)
            self.cs1 = partials(self.x1.view(nb, h * w, c1), T1, sg) if c1 else None
        ho, wo = (h // 2, w // 2) if p["resample"] == 1 else (2 * h, 2 * w) if p["resample"] == 2 else (h, w)
        self.oshape = (nb, ho, wo, C_)
        self.ws = torch.empty(nb * (GN_MAX_SLABS * p["groups"] * 2 + p["groups"] * 2 + 1), device=dev)

    def outputs(self):
        p = self.p
        names = ("out",) if p["kind"] == "gnmod" else ("out",) + tuple(k for k in ("raw", "lo", "raw_lo") if p[k])
        return {k: _out(self.oshape, torch.float16, p["oo"], self.dev) for k in names}

    def launch(self, outs):
        p = self.p
        for buf, _ in outs.values():
            buf.fill_(NAN)
        self.ws.fill_(NAN)
        v = lambda k: outs[k][1] if k in outs else None
        P = ops._ptr
        lib = _l.load()
        nb, h, w = p["nb"], p["h"], p["w"]
        T0, T1, sg = p["stats"] or (0, 0, 1)
        if p["kind"] == "gn":
            rc = lib.sdb_groupnorm(P(self.x0), P(self.x1), p["c0"], p["c1"], nb, h * w, p["groups"], P(self.gamma),
                                   P(self.beta), p["eps"], int(p["silu"]), P(v("out")), P(v("raw")), P(v("lo")),
                                   P(v("raw_lo")), P(self.ws), P(self.cs0), P(self.cs1), T0, T1, sg, ops._stream())
        else:
            rc = lib.sdb_groupnorm_mod(P(self.x0), p["c0"], nb, h, w, p["groups"], P(self.gamma), P(self.beta),
                                       p["eps"], int(p["silu"]), P(self.scale), P(self.shift), p["ldm"],
                                       p["resample"], P(v("out")), P(self.ws), P(self.cs0), T0, sg, ops._stream())
        _l.check(rc, p["kind"])

    def reference(self):
        p = self.p
        return gn_ref(self.x0, self.x1, self.gamma, self.beta, p["groups"], p["eps"], p["silu"], self.scale,
                      self.shift, p["resample"])


def gn_ref(x0, x1, gamma, beta, groups, eps, silu, scale=None, shift=None, resample=0):
    """fp64 GroupNorm -> (1 + scale), + shift -> SiLU -> resample, NHWC; returns (ref, bound without the fp16 term, v,
    the pre-activation value at the output resolution or None under pooling)."""
    x = x0.double() if x1 is None else torch.cat([x0.double(), x1.double()], -1)
    nb, h, w, C_ = x.shape
    xn = x.permute(0, 3, 1, 2)
    z = F.group_norm(xn, groups, eps=eps)
    xg = xn.reshape(nb, groups, -1)
    mean = xg.mean(-1)
    rstd = 1.0 / torch.sqrt(xg.var(-1, unbiased=False) + eps)
    col = lambda t: t.repeat_interleave(C_ // groups, 1)[:, :, None, None]
    ge = gamma.double()[None, :, None, None].expand(nb, C_, 1, 1)
    be = beta.double()[None, :, None, None].expand(nb, C_, 1, 1)
    if scale is not None:
        s1 = 1.0 + scale.double()[:, :, None, None]
        ge, be = ge * s1, be * s1 + shift.double()[:, :, None, None]
    v = z * ge + be
    bound = TAU_N * (z.abs() * ge.abs() + be.abs()) + APPLY_REL * (xn.abs() + col(mean).abs()) * col(rstd) * ge.abs()
    y = v
    if silu:
        y = v * torch.sigmoid(v)
        bound = 1.1 * bound + ACT_REL * v.abs()
    if resample == 1:
        bound = F.avg_pool2d(bound + 2.4e-7 * y.abs(), 2)
        y = F.avg_pool2d(y, 2)
        v = None
    elif resample == 2:
        y, bound, v = (F.interpolate(t, scale_factor=2, mode="nearest") for t in (y, bound, v))
    nhwc = lambda t: None if t is None else t.permute(0, 2, 3, 1).contiguous()
    return nhwc(y), nhwc(bound), nhwc(v)


def ln_ref(x, gamma, beta, eps):
    xd = x.double()
    z = F.layer_norm(xd, (x.shape[-1],), eps=eps)
    mean = xd.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + eps)
    g, b = gamma.double(), beta.double()
    ref = z * g + b
    bound = TAU_L * (z.abs() * g.abs() + b.abs()) + APPLY_REL * (xd.abs() + mean.abs()) * rstd * g.abs()
    return ref, bound


def softmax_ref(x, scale):
    sx = x.double() * scale
    m = sx.max(-1, keepdim=True).values
    ref = sx.softmax(-1)
    bound = ref * (1e-6 + 1.2e-7 * (sx - m).abs() + 6e-8 * (sx.abs() + m.abs()))
    return ref, bound


# ------------------------------------------------------------------------------------------------ one problem
def _share(err, bound):
    return float((err / bound.clamp_min(1e-300)).max())


def check_gn(X, outs):
    p = X.p
    ref, bound, v = X.reference()
    r = {}
    out = outs["out"][1]
    r["finite"] = bool(torch.isfinite(out).all())
    r["guards"] = all(_guard_ok(*o) for o in outs.values())
    h = out.double()
    r["gn_elem"] = _share((h - ref).abs(), torch.maximum(ulp16(ref), ulp16(h)) + bound)
    if "lo" in outs:
        s = h + outs["lo"][1].double()
        r["finite"] = r["finite"] and bool(torch.isfinite(outs["lo"][1]).all())
        r["gn_hilo"] = _share((s - ref).abs(), bound + 6e-8)
    if "raw" in outs:
        x = X.x0 if X.x1 is None else torch.cat([X.x0, X.x1], -1)
        raw = x.half()
        r["raw_exact"] = torch.equal(outs["raw"][1], raw)
        if "raw_lo" in outs:
            r["raw_lo_exact"] = torch.equal(outs["raw_lo"][1], (x - raw.float()).half())
    return r


def check_ln(p, x, gamma, beta, o16, o32):
    ref, bound = ln_ref(x, gamma, beta, p["eps"])
    r = {"finite": True, "guards": True}
    if o32 is not None:
        r["finite"] = bool(torch.isfinite(o32[1]).all())
        r["guards"] = _guard_ok(*o32)
        r["ln_elem_f32"] = _share((o32[1].double() - ref).abs(), bound)
    if o16 is not None:
        r["finite"] = r["finite"] and bool(torch.isfinite(o16[1]).all())
        r["guards"] = r["guards"] and _guard_ok(*o16)
        if o32 is not None:
            r["ln_f16_eq_f32"] = torch.equal(o16[1], o32[1].half())
        else:
            h = o16[1].double()
            r["ln_elem_f16"] = _share((h - ref).abs(), torch.maximum(ulp16(ref), ulp16(h)) + bound)
    return r


class Sweep(Tally):
    """Failures and calibration of one title (workload or synthetic group)."""

    def __init__(self, title):
        super().__init__(title)
        self.calib, self.sms = {}, _l.load().sdb_sm_count()

    def record(self, lab, r, same):
        if not same:
            self.failures.append((lab, "bit-reproducible", "second launch differs"))
        for k, val in r.items():
            if isinstance(val, bool):
                if not val:
                    self.failures.append((lab, k, "False"))
            elif not val <= 1.0:
                self.failures.append((lab, k, f"{val:.3e}"))
            else:
                self.calib[k] = max(self.calib.get(k, 0.0), val)

    def gn(self, p, seed):
        X = GNOperands(p, torch.device("cuda", torch.cuda.current_device()), seed)
        lab = label(p)
        try:
            outs = X.outputs()
            X.launch(outs)
            keep = {k: v[1].clone() for k, v in outs.items()}
            r = check_gn(X, outs)
            X.launch(outs)
            same = all(torch.equal(keep[k], outs[k][1]) for k in keep)
        except Exception as e:  # noqa: BLE001 - a fault must name its problem
            raise RuntimeError(f"{lab}: {e}") from e
        self.launches += 2
        self.record(lab, r, same)
        for c in gn_branches(p, self.sms):
            COVER[c] += 1
        return r

    def ln(self, p, seed):
        dev = torch.device("cuda", torch.cuda.current_device())
        g = torch.Generator(device=dev).manual_seed(seed)
        ax, ag, ab, ao = p["align"]
        x = _input((p["rows"], p["c"]), ax, g, p["mean"], p["std"])
        gamma = _input((p["c"],), ag, g, 1.0, 0.5, chan_mean=False)
        beta = _input((p["c"],), ab, g, 0.0, 0.5, chan_mean=False)
        o16 = _out((p["rows"], p["c"]), torch.float16, 0, dev) if p["f16"] else None
        o32 = _out((p["rows"], p["c"]), torch.float32, ao, dev) if p["f32"] else None
        lab = label(p)

        def launch():
            for o in (o16, o32):
                if o is not None:
                    o[0].fill_(NAN)
            _l.check(_l.load().sdb_layernorm(ops._ptr(x), p["rows"], p["c"], ops._ptr(gamma), ops._ptr(beta), p["eps"],
                                             ops._ptr(o16[1]) if o16 else None, ops._ptr(o32[1]) if o32 else None,
                                             ops._stream()), "sdb_layernorm")
            return [o[1].clone() for o in (o16, o32) if o is not None]
        try:
            first = launch()
            r = check_ln(p, x, gamma, beta, o16, o32)
            same = all(torch.equal(a, b) for a, b in zip(first, launch()))
        except Exception as e:  # noqa: BLE001
            raise RuntimeError(f"{lab}: {e}") from e
        self.launches += 2
        self.record(lab, r, same)
        for c in ln_branches(dict(p, align=(ax, ag, ab, ao)), self.sms):
            COVER[c] += 1
        return r

    def softmax(self, p, seed):
        dev = torch.device("cuda", torch.cuda.current_device())
        g = torch.Generator(device=dev).manual_seed(seed)
        x = _input((p["rows"], p["cols"]), p["align"], g, 0.0, p["mag"], chan_mean=False)
        if p["const"]:
            x.copy_(x[:, :1].expand_as(x))
        o = _out((p["rows"], p["cols"]), torch.float16, 0, dev)
        lab = label(p)

        def launch():
            o[0].fill_(NAN)
            _l.check(_l.load().sdb_softmax_rows(ops._ptr(x), p["rows"], p["cols"], p["scale"], ops._ptr(o[1]),
                                                ops._stream()), "sdb_softmax_rows")
            return o[1].clone()
        try:
            first = launch()
            ref, bound = softmax_ref(x, p["scale"])
            h = first.double()
            r = {"finite": bool(torch.isfinite(first).all()), "guards": _guard_ok(*o),
                 "softmax_elem": _share((h - ref).abs(), torch.maximum(ulp16(ref), ulp16(h)) + bound)}
            same = torch.equal(first, launch())
        except Exception as e:  # noqa: BLE001
            raise RuntimeError(f"{lab}: {e}") from e
        self.launches += 2
        self.record(lab, r, same)
        COVER["softmax"] += 1
        return r

    def run(self, p, seed):
        return {"gn": self.gn, "gnmod": self.gn, "ln": self.ln, "softmax": self.softmax}[p["kind"]](p, seed)

    def calibration(self):
        return "largest share of each bound used: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(self.calib.items()))


def run_sweep(problems, title):
    sw = Sweep(title)
    for i, p in enumerate(problems):
        sw.run(p, 1000 + i)
    sw.finish(len(problems), sw.calibration())


# ------------------------------------------------------------------------------------------------ model workloads
@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(WORKLOADS))
def test_every_norm_launch_of_every_model(cuda_dev, name):
    calls, problems = record(WORKLOADS[name], cuda_dev, SIGS)
    kinds = defaultdict(int)
    for p in problems:
        kinds[p["kind"]] += 1
    print(f"\n{name}: {calls} calls, {len(problems)} distinct problems ({dict(kinds)})")
    assert problems
    run_sweep(problems, name)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ synthetic grid
def _gn_grid():
    ps = []
    # every width class, straddling concats included; 3072 / 3104 sit on the 12 / 14 channels-per-thread boundary
    for c in (32, 64, 96, 128, 192, 320, 448, 960, 1920, 3072, 3104, 3584):
        ps.append(_gn(nb=3, h=1, w=129, c0=c, silu=True))
    ps += [_gn(nb=3, h=3, w=43, c0=c, groups=16) for c in (64, 448, 3584)]
    ps += [_gn(nb=3, h=1, w=127, c0=c, groups=64) for c in (64, 128, 320, 1920)]        # standalone only
    ps += [_gn(nb=1, h=1, w=127, c0=128, groups=64, stats=(2, 0, 1))]                  # fused ignored above 32 groups
    # rows per sample: hw 1, 3, ragged slabs, the 128-slab cap, batches that lower the slab count
    for hw in (1, 3, 127, 129, 4095):
        for nb in (1, 3, 16):
            ps.append(_gn(nb=nb, h=1, w=hw, c0=320, silu=nb == 3))
    ps += [_gn(nb=1, h=512, w=512, c0=128, silu=True), _gn(nb=1, h=512, w=512, c0=32, groups=16),
           _gn(nb=3, h=61, w=67, c0=64, raw=True)]
    # concatenated sources: groups straddling c0, standalone and fused (sg divides c0, c1 and the group)
    ps += [_gn(nb=2, h=5, w=12, c0=196, c1=124, silu=True), _gn(nb=2, h=8, w=9, c0=640, c1=320, raw=True, lo=True),
           _gn(nb=2, h=8, w=9, c0=640, c1=320, stats=(3, 5, 10)), _gn(nb=2, h=4, w=6, c0=20, c1=44, groups=16),
           _gn(nb=1, h=4, w=4, c0=1280, c1=1280, stats=(1, 1, 20), silu=True),
           _gn(nb=2, h=16, w=8, c0=640, c1=320, stats=(600, 600, 10)), _gn(nb=2, h=3, w=7, c0=1920, c1=1280, a1=0)]
    # fused partials on each side of the fold threshold max(T0, T1) (cpg / sg) > 512
    ps += [_gn(nb=2, h=32, w=32, c0=320, stats=(T, 0, sg), silu=True) for T, sg in ((512, 10), (513, 10), (51, 1),
                                                                                   (52, 1), (1, 1), (1024, 2))]
    # operand outputs, unaligned outputs (8-byte, not 16), a near-constant group
    ps += [_gn(nb=2, h=7, w=10, c0=320, raw=True, lo=True, raw_lo=True, silu=True),
           _gn(nb=2, h=7, w=10, c0=320, raw=True, raw_lo=True, stats=(4, 0, 10)),
           _gn(nb=2, h=7, w=10, c0=448, raw=True, lo=True, raw_lo=True, oo=4),
           _gn(nb=2, h=9, w=9, c0=320, flat_group=3), _gn(nb=2, h=9, w=9, c0=64, flat_group=0, eps=1e-6, silu=True)]
    # modulated GroupNorm: resample x modulation x computed / fused statistics, odd-by-even non-square sizes
    for rs in (0, 1, 2):
        h, w = (6, 10) if rs == 1 else (7, 10)
        for ldm in (0, 3 * 320):
            for stats in (None, (5, 0, 10)):
                ps.append(_gn(kind="gnmod", nb=3, h=h, w=w, c0=320, silu=True, ldm=ldm, resample=rs, stats=stats))
    ps += [_gn(kind="gnmod", nb=2, h=14, w=10, c0=64, ldm=64, resample=1, silu=True),
           _gn(kind="gnmod", nb=1, h=1, w=1, c0=3584, ldm=3584, resample=2),
           _gn(kind="gnmod", nb=2, h=5, w=8, c0=192, silu=False, stats=(600, 0, 1))]
    return ps


def _ln_grid(sms):
    ps = [_ln(rows=77, c=c) for c in LN_V2]                                   # the vector instances
    ps += [_ln(rows=77, c=c) for c in (48, 64, 77, 100, 128, 192, 448, 576, 704, 896, 1024, 1344, 1792)]
    ps += [_ln(rows=77, c=768, align=(1, 0, 0, 0)), _ln(rows=77, c=320, align=(0, 2, 0, 0)),
           _ln(rows=77, c=1280, align=(0, 0, 0, 2), f32=True)]                  # a v2 width falls back to scalar
    for rows in (1, 4 * sms + 1, 8 * sms + 3, 16 * sms + 5):                   # warps per block 1, 2, 4, 8
        ps += [_ln(rows=rows, c=768, f32=True), _ln(rows=rows, c=1024)]
    ps += [_ln(rows=257, c=c, f16=False, f32=True) for c in (768, 1024)]       # fp32 only
    ps += [_ln(rows=257, c=c, f32=True, mean=100.0, std=1.0) for c in (768, 1024, 1280, 77)]
    return ps


def _sm_grid():
    ps = [_sm(rows=3, cols=c, scale=s) for c in (1, 7, 96, 255, 256, 257, 6144) for s in (1.0, 0.125)]
    ps += [_sm(rows=5, cols=c, mag=1e3) for c in (7, 257, 6144)]
    ps += [_sm(rows=2, cols=c, const=True) for c in (1, 257, 6144)]
    ps += [_sm(rows=2, cols=255, align=1, scale=0.0625)]
    return ps


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_norm_synthetic_grid(cuda_dev):
    sms = _l.load().sdb_sm_count()
    ps = _gn_grid() + _ln_grid(sms) + _sm_grid()
    run_sweep(ps, "synthetic")


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_groupnorm_conditioning(cuda_dev):
    """Inputs with mean / std up to 256 at 4096 and 262144 rows per sample. The statistics pass takes its sums around
    a pivot and meets the main bound throughout. Fused partials carry sum x^2 in fp32, so (mean / std)^2 of the
    variance is lost to their rounding: they meet the bound up to mean / std 64 (asserted); the share at 256 is
    printed."""
    sw = Sweep("conditioning")
    fused_beyond = {}
    for hw in (4096, 262144):
        for ratio in (0.0, 4.0, 16.0, 64.0, 256.0):
            p = _gn(nb=1, h=hw // 64, w=64, c0=128, mean=ratio, std=1.0)
            sw.gn(p, 7)
            T = hw // 128                   # one partial slot per 128 rows, as the GEMM epilogues store them
            q = dict(p, stats=(T, 0, 1))
            if ratio <= 64:
                sw.gn(q, 7)
            else:
                X = GNOperands(q, cuda_dev, 7)
                outs = X.outputs()
                X.launch(outs)
                fused_beyond[(hw, ratio)] = check_gn(X, outs)["gn_elem"]
    sw.finish(20, sw.calibration())
    print("fused statistics at mean/std 256 (not asserted), share of the bound: "
          + ", ".join(f"hw {k[0]} ratio {k[1]:g}: {v:.2f}" for k, v in sorted(fused_beyond.items())))


@pytest.mark.gpu
def test_norm_branch_coverage():
    """Every dispatch branch of norm.cu was launched by the sweeps above."""
    check_coverage(COVER, REQUIRED, "norm")


# ------------------------------------------------------------------------------------------------ host guards
def _off(shape, k, dev):
    """A contiguous fp32 view at a k-float offset of its allocation."""
    return torch.randn(math.prod(shape) + k, device=dev)[k:].view(shape)


@pytest.mark.gpu
def test_norm_rejects_what_it_cannot_address(cuda_dev):
    """Checked on the host before anything launches."""
    g = torch.ones(320, device=cuda_dev)
    b = torch.zeros(320, device=cuda_dev)
    x = torch.randn(2, 4, 4, 320, device=cuda_dev)
    for bad in (_off((2, 4, 4, 320), 1, cuda_dev), _off((2, 4, 4, 320), 2, cuda_dev)):
        with pytest.raises(RuntimeError, match="aligned"):
            ops.groupnorm(bad, g, b)
        with pytest.raises(RuntimeError, match="aligned"):
            ops.groupnorm(x[..., :160].contiguous(), g, b, x1=_off((2, 4, 4, 160), 1, cuda_dev))
        with pytest.raises(RuntimeError, match="aligned"):
            ops.groupnorm_mod(bad, g, b)
    P, lib = ops._ptr, _l.load()
    ws = torch.empty(2 * (GN_MAX_SLABS * 64 + 65), device=cuda_dev)
    out = torch.empty(2 * 16 * 320 + 2, dtype=torch.float16, device=cuda_dev)[2:]     # 4-byte aligned only
    assert lib.sdb_groupnorm(P(x), None, 320, 0, 2, 16, 32, P(g), P(b), 1e-5, 0, P(out), None, None, None, P(ws),
                             None, None, 0, 0, 1, ops._stream()) != 0
    assert b"aligned" in lib.sdb_last_error()
    assert lib.sdb_groupnorm_mod(P(x), 320, 2, 4, 4, 32, P(g), P(b), 1e-5, 1, None, None, 0, 0, P(out), P(ws), None,
                                 0, 1, ops._stream()) != 0
    assert b"aligned" in lib.sdb_last_error()
    big = torch.randn(1, 2, 2, 3616, device=cuda_dev)
    with pytest.raises(RuntimeError, match="too large"):
        ops.groupnorm(big, torch.ones(3616, device=cuda_dev), torch.zeros(3616, device=cuda_dev))
    with pytest.raises(RuntimeError, match="multiple of 4"):
        ops.groupnorm_mod(big, torch.ones(3616, device=cuda_dev), torch.zeros(3616, device=cuda_dev))
    with pytest.raises(RuntimeError, match="multiples of 4"):
        ops.groupnorm(torch.randn(1, 2, 2, 66, device=cuda_dev), g[:66].contiguous(), b[:66].contiguous(), groups=33)
    with pytest.raises(RuntimeError, match="divisible"):
        ops.groupnorm(torch.randn(1, 2, 2, 256, device=cuda_dev), g[:256].contiguous(), b[:256].contiguous(),
                      groups=128)
    with pytest.raises(RuntimeError, match="even sides"):
        ops.groupnorm_mod(torch.randn(1, 3, 4, 320, device=cuda_dev), g, b, resample=1)
    with pytest.raises(RuntimeError, match="too large"):
        ops.layernorm(torch.randn(4, 1824, device=cuda_dev), torch.ones(1824, device=cuda_dev),
                      torch.zeros(1824, device=cuda_dev))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ CPU: the harness
def test_dispatch_mirror_cpu():
    sms = 132
    # SD-v1 VAE top level at 512²: 128 channels -> cw 128, two row lanes; 528 target blocks cap the slabs at 128
    c = gn_branches(_gn(nb=1, h=512, w=512, c0=128), sms)
    assert {"cpt12", "rstep2", "slab_cap", "fold:none"} <= c and "ragged_slab" not in c
    c = gn_branches(_gn(nb=16, h=1, w=129, c0=32), sms)        # 8 row lanes; 17 slabs of 8 rows, the last ragged
    assert {"rstep8", "ragged_slab"} <= c and "slab_cap" not in c
    assert "cpt14" in gn_branches(_gn(c0=3104), sms) and "cpt12" in gn_branches(_gn(c0=3072), sms)
    assert "rstep4" in gn_branches(_gn(c0=64), sms) and "rstep1" in gn_branches(_gn(c0=320), sms)
    assert "fold:in_apply" in gn_branches(_gn(stats=(512, 0, 10)), sms)
    assert "fold:kernel" in gn_branches(_gn(stats=(513, 0, 10)), sms)
    assert "fold:kernel" in gn_branches(_gn(stats=(52, 0, 1)), sms) and "fold:in_apply" in gn_branches(
        _gn(stats=(51, 0, 1)), sms)
    assert "fold:kernel" in gn_branches(_gn(kind="gnmod", stats=(1, 0, 1)), sms)
    assert "fold:none" in gn_branches(_gn(c0=128, groups=64, stats=(1, 0, 1)), sms)     # > 32 groups: not fused
    c = gn_branches(_gn(c0=640, c1=320, stats=(3, 5, 10)), sms)                            # cpg 30, 640 % 30 = 10
    assert {"x1", "x1_straddle_fused", "fold:in_apply"} <= c
    assert "x1_straddle" not in gn_branches(_gn(c0=640, c1=640), sms)
    assert "hw1" in gn_branches(_gn(h=1, w=1), sms)
    wp = lambda rows: {k for k in ln_branches(_ln(rows=rows), sms) if k.startswith("wpb")}
    assert [wp(r) for r in (527, 528, 1056, 2112)] == [{"wpb1"}, {"wpb2"}, {"wpb4"}, {"wpb8"}]
    assert "ln_v2<12>" in ln_branches(_ln(c=768), sms)
    assert "ln_npl<24>" in ln_branches(_ln(c=768, align=(1, 0, 0, 0)), sms)
    assert "ln_npl<40>" in ln_branches(_ln(c=1024), sms) and "ln_npl<56>" in ln_branches(_ln(c=1792), sms)
    assert "ln_npl<4>" in ln_branches(_ln(c=77), sms) and "ln_npl<20>" in ln_branches(_ln(c=448), sms)


def test_references_against_torch_fp32_cpu():
    g = torch.Generator().manual_seed(0)
    x0, x1 = torch.randn(2, 6, 4, 12, generator=g) + 0.5, torch.randn(2, 6, 4, 20, generator=g) * 2
    gamma, beta = torch.randn(32, generator=g), torch.randn(32, generator=g)
    scale, shift = torch.randn(2, 32, generator=g) * 0.3, torch.randn(2, 32, generator=g)
    x = torch.cat([x0, x1], -1).permute(0, 3, 1, 2)
    for silu, rs in ((False, 0), (True, 1), (True, 2)):
        y = F.group_norm(x, 8, gamma, beta, eps=1e-5) * (1 + scale[:, :, None, None]) + shift[:, :, None, None]
        if silu:
            y = F.silu(y)
        y = F.avg_pool2d(y, 2) if rs == 1 else F.interpolate(y, scale_factor=2) if rs == 2 else y
        ref, bound, _ = gn_ref(x0, x1, gamma, beta, 8, 1e-5, silu, scale, shift, rs)
        assert torch.allclose(ref, y.permute(0, 2, 3, 1).double(), rtol=1e-5, atol=1e-5)
        assert bool((bound > 0).all())
    ref, _, _ = gn_ref(x0, x1, gamma, beta, 8, 1e-5, False)
    assert torch.allclose(ref, F.group_norm(x, 8, gamma, beta).permute(0, 2, 3, 1).double(), atol=1e-5)
    xl = torch.randn(5, 77, generator=g) * 3 + 100
    ref, _ = ln_ref(xl, gamma[:1].expand(77), beta[:1].expand(77), 1e-5)
    assert torch.allclose(ref, F.layer_norm(xl.double(), (77,), gamma[:1].expand(77).double(),
                                            beta[:1].expand(77).double()), atol=1e-12)
    assert torch.allclose(ref.float(), F.layer_norm(xl, (77,), gamma[:1].expand(77), beta[:1].expand(77)), atol=1e-4)
    xs = torch.randn(3, 257, generator=g) * 30
    ref, bound = softmax_ref(xs, 0.125)
    assert torch.allclose(ref.float(), (xs * 0.125).softmax(-1), atol=1e-6) and bool((bound > 0).all())
    assert float(ulp16(torch.tensor([1.0]))[0]) == 2.0 ** -10 and float(ulp16(torch.tensor([1e-7]))[0]) == 2.0 ** -24


def test_partials_builder_cpu():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(3, 37, 40, generator=g) + 2.0
    for T, sg in ((1, 1), (5, 4), (37, 10), (50, 2)):
        st = partials(x, T, sg)
        assert st.shape == (3, T, 40 // sg, 2) and st.dtype == torch.float32
        xd = x.double().view(3, 37, 40 // sg, sg)
        assert torch.allclose(st.double().sum(1)[..., 0], xd.sum((1, 3)), rtol=1e-6)
        assert torch.allclose(st.double().sum(1)[..., 1], (xd * xd).sum((1, 3)), rtol=1e-6)
    st = partials(x, 4, 1)       # chunk t holds rows [37 t / 4, 37 (t + 1) / 4)
    assert torch.allclose(st[:, 1, :, 0].double(), x[:, 9:18].double().sum(1), rtol=1e-6)


def test_signature_dedups_cpu():
    x = torch.zeros(2, 4, 4, 320)
    gm = torch.ones(320)
    s = lambda **kw: signature(_gn_sig(x, gm, gm, **kw))
    assert s() == s() and s(silu=True) != s() and s(want_raw_lo=True) != s(want_raw=True)
    assert signature(_gn_sig(torch.zeros(2, 4, 4, 321)[..., 1:].contiguous(), gm, gm)) == s()
    base = torch.zeros(2 * 16 * 320 + 4)
    off = base[1:1 + 2 * 16 * 320].view(2, 4, 4, 320)
    assert _gn_sig(off, gm, gm)["a0"] == (eoff(base) + 1) % 4 and signature(_gn_sig(off, gm, gm)) != s()
    x._sdb_stats = (torch.zeros(1), 7, 10)
    p = _gn_sig(x, gm, gm)
    assert p["stats"] == (7, 0, 10) and "stats(T7,0,sg10)" in label(p)
    x._sdb_stats = (torch.zeros(1), 7, 3)                 # 3 does not divide the 10-channel groups
    assert _gn_sig(x, gm, gm)["stats"] is None
    m = torch.zeros(2, 960)
    p = _gnmod_sig(torch.zeros(2, 6, 10, 320), gm, gm, scale=m[:, :320], shift=m[:, 320:640], resample=1)
    assert p["ldm"] == 960 and p["resample"] == 1 and p["kind"] == "gnmod"
    a = _ln_sig(torch.zeros(7, 11, 768), gm, gm, eps=1e-6, want_f32=True)
    assert (a["rows"], a["c"], a["eps"], a["f32"]) == (77, 768, 1e-6, True)
    assert _sm_sig(torch.zeros(4, 2, 96), 0.5) == _sm(rows=8, cols=96, scale=0.5)
