"""Every attention launch the models make, and the softmax edges none of them reach, elementwise against fp64.

attention_tc_kernel<DPAD, DV> (15 instances behind sdb_attention) is a software-pipelined S / PV loop over 64-key tiles
with two mbarrier rings, an online softmax whose running maximum rescales O, a polynomial exp on a quarter of the
columns, streamed Q at d = 960 and zero-filled head padding through the tensor maps. The sweep:
  1. records the sdb200.ops.attention calls of one eager forward of each model (random weights) and deduplicates them
     by everything that reaches the kernel or the host dispatch (sizes, leading dimensions, batch strides, pointer
     offsets, whether K is a column slice of Q's buffer);
  2. regenerates seeded operands at each recorded geometry inside NaN-filled buffers (every element the kernel must
     not read is NaN, every element it must not write is NaN), under each operand family below;
  3. launches through the C entry point, checks every element against the fp64 reference, the signed bias of the
     launch, the exact answers two families have, NaN containment, a bit-equal second launch, and (randn only) that a
     sample, a 128-row query block and a head computed alone are bit-equal to their part of the full launch;
then a synthetic grid covers the edges no model reaches, and a Python mirror of the host dispatch records which
classes ran (test_attention_branch_coverage).

Operand families (scale s, logits in natural units after s; columns 0 / 1 of q and k are reserved where a pattern is
built: q = (a_i, 1, noise..), k = (b_j, c_j, noise..), so the logit is s (a_i b_j + c_j + noise)):
  randn1 / randn4  q, k, v ~ N(0, 1) amp, amp 1 / 4: logit std sqrt(d) s amp^2 (1 / 16 at s = d^-1/2).
  posv             randn1 with v = |N(0, 1)|: ref = A, so an error of P with a sign shows undiluted in the bias.
  uniform          q = 0: every logit 0, P = 1.0 exactly. v[j, c] = 1 where c mod G == j mod G, G = min(d, 8): the
                   output is (number of admitted keys of the class) / (number admitted), an exact count.
  peaked           up to 7 key positions per head (0, nkv-1, 63 / 64 / 127 / 128, 24 / 31 / 56 / 88 / 95 inside the
                   polynomial column blocks, ..) carry b = m, c = -m^2 L / 2 (m = 0, 1, ..), a_i = L m*(i): logit
                   s L (m* m - m^2 / 2), largest at m = m*(i) by s L / 2 >= 40 (L = the power of two >= 80 / s; every
                   value is exact in fp16 and the fp32 sums are exact); all other keys sit at -60. Causal rows pick
                   among the positions <= i, and i itself when it is one. out row = v[j*] to one fp16 ulp.
  rising           a = 3 / s, b_j = the key's tile index: the row maximum rises by 3 every 64 keys (+ N(0, ~1)
                   noise), so the O rescale is ~e^-3 on every tile. Range [0, 3 tiles].
  falling          b_j reversed: the first tile holds the maximum, later tiles contribute at e^-3k.
  jump             randn-like logits, but a = 100 / s and b = 1 on the last-but-one tile: the maximum jumps by 100
                   (144 in log2 units, beyond fp32's exponent range): earlier O and l underflow to 0, no NaN / inf.
  bigv             randn1 logits, v ~ N(0, 2e4) clamped to 6e4, every fourth channel +-6e4 alternating by key.

Bound per element (ref = P v in fp64 from the fp16 operands, A = P |v|, L_i = sum_j exp(s_ij - max_j s_ij) >= 1,
smag_i = s max_j |q_i| . |k_j|):
  |out - ref| <= 0.5 ulp16 (1 + 2^-10) + (TAU_P + TAU_S smag_i) A[i, c] + 2^-25 (sum_j |v[j, c]|) / L_i
    0.5 ulp16       the fp16 rounding of the output (ulp at the larger of |ref|, |out|), 2^-10 for the fp32 O / l
    TAU_P A         relative error of one P: fp16 rounding 2^-11, poly_exp2 1.02e-4, MUFU 2^-22, together 6e-4. The
                    errors of different keys are independent, so rows of many keys use a small part of it (0.1 at
                    16384 keys), but a row carried by one or two keys can meet it: the 3- and 11-token contexts of the
                    retrieval-augmented UNet reach 3.5e-4 A, so the provable value stays
    TAU_S smag A    fp32 accumulation of the logits and of s q.k - max, entering through exp
    2^-25 sum|v|/L  P below 2^-14 is an fp16 subnormal: absolute error up to 2^-25 per key before the 1 / l
Bias per launch: the mean of (out - ref) sign(ref) / A over the elements with A > 16 ulp16 stays within
BIAS + ACC_RZ nkv + 5 std / sqrt(n) (n >= 256 elements): a P that is systematically small (packed by truncation), a
biased exp polynomial or an l that sees other values than PV moves this by 1e-4 and moves no single element past its
bound. ACC_RZ: the tensor cores truncate their fp32 accumulator where the row sum l is added with rounding to nearest,
so with v of one sign O falls behind l by 6.3e-9 per key (posv: -2.5e-5 at 4096 keys, -3.8e-5 at 6144, -1.0e-4 at
16384, measured; signed v cancels it). uniform and peaked are left out: their outputs are the same few values in every
row, whose fp16 rounding does not average out, and they are checked exactly instead.
The largest share of the bound used and the largest bias are printed per workload and family.
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
from sweeps import GUARD, NAN, Tally, check_coverage, eoff, record, ulp16
from workloads import ATTENTION_WORKLOADS

TAU_P = 6e-4       # relative error of P (fp16 rounding + exp), relative to A = P |v|
TAU_S = 4e-6       # fp32 logit accumulation, relative to smag A
BIAS = 1.5e-5      # |mean signed relative error| of one launch
ACC_RZ = 1.2e-8    # ... plus this per key: the truncating fp32 accumulation of O (measured 6.3e-9 with v > 0)
CHUNK = 1 << 26    # fp64 logits per reference chunk (512 MiB; a few temporaries of that size are alive at once)
HEAVY = 1 << 28    # logits per launch above which only LIGHT_FAMILIES run
AQ, AKV = 128, 64
FAMILIES = ("randn1", "randn4", "posv", "uniform", "peaked", "rising", "falling", "jump", "bigv")
LIGHT_FAMILIES = ("randn1", "posv", "uniform", "rising")
WIDE_DV = {384: 128, 512: 128, 576: 96, 960: 160}


def _c8(n):
    return (n + 7) // 8 * 8


# ------------------------------------------------------------------------------------------------ host dispatch mirror
def attn_dv(dpad, d):
    """PV width of the instance sdb_attention picks (0: none), restated from attention_tc.cu."""
    if dpad in WIDE_DV:
        return WIDE_DV[dpad]
    dv = _c8(d)
    if dpad == 64:
        return dv if dv <= 48 else 64
    if dpad == 128:
        return dv if dv in (80, 96) else 128
    return 160 if dv <= 160 else 0


def ring(dpad):
    """(K panels per tile, K ring depth in panels, V ring depth in tiles, class name)."""
    panels = dpad // 64
    if dpad > 192:
        return panels, 4, 2, "960" if dpad == 960 else "wide"
    return panels, max(4, 2 * panels), 4, str(dpad)


def n_iters(p):
    """Key tiles walked by each 128-row query block (the causal clamp skips tiles above the diagonal)."""
    out = []
    for q0 in range(0, p["nq"], AQ):
        eff = min(p["nkv"], q0 + AQ) if p["causal"] else p["nkv"]
        out.append((eff + AKV - 1) // AKV)
    return out


def attn_branches(p):
    """Classes of the host dispatch and of the kernel's control flow that problem p reaches."""
    d, dpad, nq, nkv = p["d"], p["dpad"], p["nq"], p["nkv"]
    panels, kst, vst, cl = ring(dpad)
    its = n_iters(p)
    top = max(its)
    cls = {f"<{dpad},{attn_dv(dpad, d)}>"}
    if 1 in its:
        cls.add(f"tiles:1@{cl}")
    if 2 in its:
        cls.add(f"tiles:2@{cl}")
    if top > vst:
        cls.add(f"tiles:v_wrap@{cl}")
    if top * panels > 2 * kst:
        cls.add(f"tiles:k_phase2@{cl}")
    if top > 2 * vst:
        cls.add(f"tiles:v_phase2@{cl}")
    if nkv % AKV:
        cls.add("ragged_kv")
    if nq % AQ:
        cls.add("ragged_q")
    if 0 < nq % AQ <= 64:
        cls.add("wg1_empty")
    if p["causal"]:
        cls.add("causal")
        if min(its) < (nkv + AKV - 1) // AKV:
            cls.add("causal_skip")
        if nq != nkv:
            cls.add("causal_nq_ne_nkv")
    if dpad <= 192:
        hs = p["hs"] or dpad
        cls |= {k for k, v in (("hs:packed", hs == _c8(d)), ("hs:padded", hs == dpad)) if v}
        if hs not in (_c8(d), dpad):
            cls.add("hs:mid")
        if d % 16:
            cls.add("zero_fill_k16")
        if d % 8:
            cls.add("zero_fill_v8")
    if dpad == 960 and top > 1:
        cls.add("stream_q_multi")
        if nkv % AKV:
            cls.add("stream_q_ragged")
    if p["B"] > 1 and p["vbs"] < p["ldvt"]:
        cls.add("vt_permuted")
    if p["k_rel"] is not None and p["ldq"] == p["ldk"] and 0 < p["k_rel"] < p["ldq"]:
        cls.add("qk_fused_slices")
    if p["ldo"] > p["heads"] * d:
        cls.add("ldo_wide")
    if min((p["B"] - 1) * p["qbs"] + (nq - 1) * p["ldq"], (p["B"] - 1) * p["obs"] + (nq - 1) * p["ldo"]) >= 2 ** 31:
        cls.add("offset_gt_2^31")
    return cls


INSTANCES = ({f"<64,{w}>" for w in (8, 16, 24, 32, 40, 48, 64)} | {f"<128,{w}>" for w in (80, 96, 128)}
             | {"<192,160>"} | {f"<{k},{v}>" for k, v in WIDE_DV.items()})
REQUIRED = (INSTANCES
            | {f"tiles:{t}@{c}" for t in ("1", "2", "v_wrap", "k_phase2", "v_phase2")
               for c in ("64", "128", "192", "wide", "960")}
            | {"ragged_kv", "ragged_q", "wg1_empty", "causal", "causal_skip", "causal_nq_ne_nkv", "hs:packed", "hs:mid",
               "hs:padded", "stream_q_multi", "stream_q_ragged", "zero_fill_k16", "zero_fill_v8", "vt_permuted",
               "qk_fused_slices", "ldo_wide", "offset_gt_2^31"})
COVER = defaultdict(int)


# ------------------------------------------------------------------------------------------------ problem catalogue
def _ap(**kw):
    """An attention problem with defaults for what is not given. hs: head_stride as passed (0 = dpad); ld* / *bs:
    leading dimensions and batch strides in elements; oq / ok / ov / oo: element offsets of the pointers from a
    16-byte boundary; k_rel: element offset of k from q when both are views of one buffer, else None; fam: the operand
    families to run (not part of what reaches the kernel)."""
    p = dict(B=1, heads=2, nq=129, nkv=257, d=40, dpad=None, hs=None, causal=False, scale=None, ldq=None, ldk=None,
             ldvt=None, ldo=None, qbs=None, kbs=None, vbs=None, obs=None, oq=0, ok=0, ov=0, oo=0, k_rel=None, fam=None)
    p.update(kw)
    d = p["d"]
    if p["dpad"] is None:
        p["dpad"] = d if d > 192 else (d + 63) // 64 * 64
    if p["hs"] is None:
        p["hs"] = 0 if p["dpad"] > 192 else _c8(d)
    hs = p["hs"] or p["dpad"]
    width = (p["heads"] - 1) * hs + d
    for k_, v in (("ldq", _c8(width)), ("ldk", _c8(width)), ("ldvt", _c8(p["nkv"])), ("ldo", p["heads"] * d)):
        if p[k_] is None:
            p[k_] = v
    for k_, v in (("qbs", p["nq"] * p["ldq"]), ("kbs", p["nkv"] * p["ldk"]), ("vbs", p["heads"] * hs * p["ldvt"]),
                  ("obs", p["nq"] * p["ldo"])):
        if p[k_] is None:
            p[k_] = v
    if p["scale"] is None:
        p["scale"] = d ** -0.5
    return p


def _attn_sig(q, k, vt, *, heads, d, dpad, nq, nkv, scale, causal=False, out=None, head_stride=0):
    B = q.shape[0]
    shared = q.untyped_storage().data_ptr() == k.untyped_storage().data_ptr()
    ldo, obs, oo = (heads * d, nq * heads * d, 0) if out is None else (out.stride(1), out.stride(0), eoff(out))
    return _ap(B=B, heads=heads, nq=nq, nkv=nkv, d=d, dpad=dpad, hs=head_stride, causal=bool(causal),
               scale=float(scale), ldq=q.stride(1), ldk=k.stride(1), ldvt=vt.stride(1), ldo=ldo, qbs=q.stride(0),
               kbs=k.stride(0), vbs=vt.stride(0), obs=obs, oq=eoff(q), ok=eoff(k), ov=eoff(vt), oo=oo,
               k_rel=(k.data_ptr() - q.data_ptr()) // 2 if shared else None)


def signature(p):
    return tuple(sorted((k, v) for k, v in p.items() if k != "fam"))


def label(p):
    bits = [f"attn[{p['B']}x{p['heads']}h {p['nq']}x{p['nkv']}] d={p['d']}/{p['dpad']} hs={p['hs']}",
            f"ld({p['ldq']},{p['ldk']},{p['ldvt']},{p['ldo']})"]
    if p["causal"]:
        bits.append("causal")
    if p["k_rel"] is not None:
        bits.append(f"k=q+{p['k_rel']}")
    if p["B"] > 1:
        bits.append(f"bs({p['qbs']},{p['kbs']},{p['vbs']},{p['obs']})")
    if p["oq"] or p["ok"] or p["ov"] or p["oo"]:
        bits.append(f"off({p['oq']},{p['ok']},{p['ov']},{p['oo']})")
    if p["scale"] != p["d"] ** -0.5:
        bits.append(f"scale={p['scale']:g}")
    return " ".join(bits)


def families(p):
    if p["fam"]:
        return p["fam"]
    return LIGHT_FAMILIES if p["B"] * p["heads"] * p["nq"] * p["nkv"] > HEAVY else FAMILIES


# ------------------------------------------------------------------------------------------------ operands
PEAK_SETS = (lambda n: (0, n - 1, 63, 64, 127, 128), lambda n: (24, 31, 56, 88, 95, n - 2),
             lambda n: (1, 29, 62, 65, 120, n // 2))


def _randn16(shape, gen):
    return torch.randn(shape, generator=gen, device=gen.device, dtype=torch.float16)


def _peaked(nq, nkv, d, scale, causal, which, dev):
    """q [nq, d], k [nkv, d] (fp32, exact in fp16) and j* [nq] of the peaked family for position set `which`."""
    pos = sorted({x % nkv for x in PEAK_SETS[which](nkv)} | ({0} if causal else set()))
    lam = 2.0 ** math.ceil(math.log2(80.0 / scale))
    M = len(pos)
    assert (M - 1) ** 2 * lam / 2 <= 65504 and lam * (M - 1) <= 65504, "peaked family leaves fp16 range"
    q = torch.zeros(nq, d, device=dev)
    k = torch.zeros(nkv, d, device=dev)
    q[:, 1] = 1.0
    k[:, 1] = -float(torch.tensor(60.0 / scale).half())
    post = torch.tensor(pos, device=dev)
    m = torch.arange(M, device=dev, dtype=torch.float32)
    k[post, 0] = m
    k[post, 1] = -m * m * lam / 2
    i = torch.arange(nq, device=dev)
    if causal:      # among the positions <= i; the diagonal when i is a position
        cnt = torch.searchsorted(post, i, right=True)
        ms = i % cnt
        ms = torch.where(post[cnt - 1] == i, cnt - 1, ms)
    else:
        ms = i % M
    q[:, 0] = lam * ms.float()
    return q, k, post[ms]


def make_operands(p, fam, gen):
    """Dense fp16 q [B, H, nq, d], k, v [B, H, nkv, d] of family `fam` and what the family knows exactly."""
    B, H, nq, nkv, d, scale = p["B"], p["heads"], p["nq"], p["nkv"], p["d"], p["scale"]
    dev = gen.device
    info = {}
    if fam in ("randn1", "randn4", "posv"):
        amp = 4.0 if fam == "randn4" else 1.0
        q, k, v = (_randn16((B, H, n, d), gen) * amp for n in (nq, nkv, nkv))
        if fam == "posv":
            v = v.abs()
    elif fam == "bigv":
        q, k = _randn16((B, H, nq, d), gen), _randn16((B, H, nkv, d), gen)
        v = (torch.randn((B, H, nkv, d), generator=gen, device=dev) * 2e4).clamp(-6e4, 6e4)
        sign = 1.0 - 2.0 * (torch.arange(nkv, device=dev) % 2).float()
        v[..., ::4] = (6e4 * sign)[:, None]
        v = v.half()
    elif fam == "uniform":
        G = min(d, 8)
        q = torch.zeros((B, H, nq, d), dtype=torch.float16, device=dev)
        k = _randn16((B, H, nkv, d), gen)
        hot = (torch.arange(d, device=dev)[None, :] % G) == (torch.arange(nkv, device=dev)[:, None] % G)
        v = hot.half().expand(B, H, nkv, d)
    elif fam == "peaked":
        qs, ks, js = zip(*(_peaked(nq, nkv, d, scale, p["causal"], w, dev) for w in range(3)))
        g = torch.arange(B * H, device=dev) % 3
        q = torch.stack(qs)[g].view(B, H, nq, d).half()
        k = torch.stack(ks)[g].view(B, H, nkv, d).half()
        info["jstar"] = torch.stack(js)[g].view(B, H, nq)
        v = _randn16((B, H, nkv, d), gen)
    else:
        q = torch.zeros((B, H, nq, d), device=dev)
        k = torch.zeros((B, H, nkv, d), device=dev)
        q[..., 1] = 1.0
        k[..., 1] = torch.randn((B, H, nkv), generator=gen, device=dev)
        if d > 2:
            q[..., 2:] = torch.randn((B, H, nq, d - 2), generator=gen, device=dev)
            k[..., 2:] = torch.randn((B, H, nkv, d - 2), generator=gen, device=dev)
        tile = (torch.arange(nkv, device=dev) // AKV).float()
        T = (nkv + AKV - 1) // AKV
        if fam == "rising":
            q[..., 0], k[..., 0] = 3.0 / scale, tile
        elif fam == "falling":
            q[..., 0], k[..., 0] = 3.0 / scale, T - 1 - tile
        else:
            assert fam == "jump", fam
            q[..., 0] = 100.0 / scale
            k[..., 0] = (tile == max(T - 2, 0)).float() if T > 1 else (torch.arange(nkv, device=dev) >= nkv // 2).float()
        q, k = q.half(), k.half()
        v = _randn16((B, H, nkv, d), gen)
    return q, k, v, info


def uniform_expected(p, dev):
    """(count [nq, d], admitted [nq, 1]) of the uniform family: keys j < admitted_i with j mod G == c mod G."""
    G = min(p["d"], 8)
    i = torch.arange(p["nq"], device=dev)
    n = torch.clamp(i + 1, max=p["nkv"]) if p["causal"] else torch.full_like(i, p["nkv"])
    g = torch.arange(p["d"], device=dev) % G
    cnt = torch.clamp((n[:, None] - 1 - g[None, :]) // G + 1, min=0)
    return cnt, n[:, None]


# ------------------------------------------------------------------------------------------------ fp64 reference
def attn_ref_chunks(q, k, v, scale, causal, max_elems=CHUNK):
    """Yields (b, h0, h1, r0, r1, ref, A, smag, L) over chunks of heads and query rows of at most max_elems logits:
    ref = softmax(scale q k^T) v, A = softmax(..) |v| [h, r, d], smag = scale max_j |q_i|.|k_j|, L = the row sum of
    exp(s - max s) [h, r], all fp64 from the fp16 operands."""
    B, H, nq, d = q.shape
    nkv = k.shape[2]
    hc = max(1, min(H, max_elems // max(1, min(nq, AQ) * nkv)))
    rc = max(1, min(nq, max_elems // (hc * nkv)))
    for b in range(B):
        for h0 in range(0, H, hc):
            h1 = min(H, h0 + hc)
            kd = k[b, h0:h1].double()
            vd = v[b, h0:h1].double()
            vv = torch.cat([vd, vd.abs()], -1)
            for r0 in range(0, nq, rc):
                r1 = min(nq, r0 + rc)
                qd = q[b, h0:h1, r0:r1].double()
                s = torch.matmul(qd, kd.transpose(1, 2)) * scale
                if causal:
                    i = torch.arange(r0, r1, device=q.device)[:, None]
                    s.masked_fill_(torch.arange(nkv, device=q.device)[None, :] > i, float("-inf"))
                s -= s.amax(-1, keepdim=True)
                s.exp_()
                L = s.sum(-1)
                s /= L[..., None]
                o = torch.matmul(s, vv)
                del s
                smag = torch.matmul(qd.abs(), kd.abs().transpose(1, 2)).amax(-1) * scale
                yield b, h0, h1, r0, r1, o[..., :d], o[..., d:], smag, L


def check(q, k, v, out4, p, max_elems=CHUNK):
    """Largest share of the elementwise bound used by out4 [B, H, nq, d] and the bias statistics of the launch."""
    dev = q.device
    share = torch.zeros((), dtype=torch.float64, device=dev)
    s1, s2, n = (torch.zeros((), dtype=torch.float64, device=dev) for _ in range(3))
    sv = v.double().abs().sum(2)                                    # [B, H, d]
    for b, h0, h1, r0, r1, ref, A, smag, L in attn_ref_chunks(q, k, v, p["scale"], p["causal"], max_elems):
        o = out4[b, h0:h1, r0:r1].double()
        u = torch.maximum(ulp16(ref), ulp16(o))
        bound = (0.5 * (1 + 2.0 ** -10) * u + (TAU_P + TAU_S * smag[..., None]) * A
                 + 2.0 ** -25 * sv[b, h0:h1, None, :] / L[..., None])
        err = o - ref
        share = torch.maximum(share, (err.abs() / bound).max())
        m = A > 16 * u
        r = torch.where(m, err * torch.sign(ref) / A.clamp_min(1e-300), torch.zeros_like(err))
        s1 += r.sum()
        s2 += (r * r).sum()
        n += m.sum()
    n_ = float(n)
    mean = float(s1) / n_ if n_ else 0.0
    std = math.sqrt(max(float(s2) / n_ - mean * mean, 0.0)) if n_ else 0.0
    return float(share), mean, std, int(n_)


# ------------------------------------------------------------------------------------------------ one problem
def _span(sizes, strides):
    return 1 + sum((n - 1) * s for n, s in zip(sizes, strides))


class Placed:
    """NaN-filled buffers holding q, k, V^T and out as strided views at problem p's geometry."""

    def __init__(self, p, dev):
        self.p, self.dev = p, dev
        B, H, nq, nkv, d = p["B"], p["heads"], p["nq"], p["nkv"], p["d"]
        hs = p["hs"] or p["dpad"]
        qst, kst = (p["qbs"], hs, p["ldq"], 1), (p["kbs"], hs, p["ldk"], 1)
        vst = (p["vbs"], hs * p["ldvt"], p["ldvt"], 1)
        new = lambda n: torch.full((n + 8,), NAN, dtype=torch.float16, device=dev)
        sq, sk = _span((B, H, nq, d), qst), _span((B, H, nkv, d), kst)
        if p["k_rel"] is not None:      # column slices of one buffer
            lo = min(0, p["k_rel"])
            self.qbuf = self.kbuf = new(max(sq, p["k_rel"] + sk) - lo + p["oq"])
            qo, ko = p["oq"] - lo, p["oq"] - lo + p["k_rel"]
        else:
            self.qbuf, self.kbuf = new(sq + p["oq"]), new(sk + p["ok"])
            qo, ko = p["oq"], p["ok"]
        self.vbuf = new(_span((B, H, d, nkv), vst) + p["ov"])
        self.q4 = self.qbuf.as_strided((B, H, nq, d), qst, qo)
        self.k4 = self.kbuf.as_strided((B, H, nkv, d), kst, ko)
        self.vt4 = self.vbuf.as_strided((B, H, d, nkv), vst, p["ov"])
        n_out = _span((B, nq, H * d), (p["obs"], p["ldo"], 1))
        self.obuf = torch.full((n_out + p["oo"] + 2 * GUARD,), NAN, dtype=torch.float16, device=dev)
        self.out3 = self.obuf.as_strided((B, nq, H * d), (p["obs"], p["ldo"], 1), GUARD + p["oo"])
        self.out4 = self.obuf.as_strided((B, H, nq, d), (p["obs"], d, p["ldo"], 1), GUARD + p["oo"])
        self.written = torch.zeros(self.obuf.numel(), dtype=torch.bool, device=dev)
        self.written.as_strided(self.out3.shape, self.out3.stride(), GUARD + p["oo"]).fill_(True)

    def fill(self, q, k, v):
        self.q4.copy_(q)
        self.k4.copy_(k)
        self.vt4.copy_(v.transpose(2, 3))

    def launch(self, out=None, b=None, rows=None, head=None):
        """The full problem into its own output, or one sample / row range / head of it into the dense `out`."""
        p = self.p
        hs = p["hs"] or p["dpad"]
        a = _l.AttnDesc()
        qp, kp, vp = self.q4.data_ptr(), self.k4.data_ptr(), self.vt4.data_ptr()
        B, H, nq = p["B"], p["heads"], p["nq"]
        if b is not None:
            qp, kp, vp, B = qp + 2 * b * p["qbs"], kp + 2 * b * p["kbs"], vp + 2 * b * p["vbs"], 1
        if rows is not None:
            qp, nq = qp + 2 * rows[0] * p["ldq"], rows[1] - rows[0]
        if head is not None:
            qp, kp, vp, H = qp + 2 * head * hs, kp + 2 * head * hs, vp + 2 * head * hs * p["ldvt"], 1
        o = self.out3 if out is None else out
        a.q, a.k, a.vt, a.out = qp, kp, vp, o.data_ptr()
        a.batch, a.heads, a.nq, a.nkv, a.d, a.dpad = B, H, nq, p["nkv"], p["d"], p["dpad"]
        a.ldq, a.ldk, a.ldvt, a.ldo = p["ldq"], p["ldk"], p["ldvt"], o.stride(1)
        a.q_batch_stride, a.k_batch_stride, a.vt_batch_stride = p["qbs"], p["kbs"], p["vbs"]
        a.o_batch_stride = o.stride(0)
        a.scale, a.causal, a.head_stride = p["scale"], int(p["causal"]), p["hs"]
        _l.check(_l.load().sdb_attention(C.byref(a), ops._stream()), "sdb_attention")

    def contained(self):
        """Every element of the output view is finite and nothing outside it (guards, columns heads d .. ldo - 1, the
        rows between samples) was written."""
        return torch.equal(self.obuf.isnan(), ~self.written) and not bool(torch.isinf(self.obuf).any())

    def part(self, **kw):
        p = self.p
        B = 1 if "b" in kw else p["B"]
        nq = kw["rows"][1] - kw["rows"][0] if "rows" in kw else p["nq"]
        w = p["d"] if "head" in kw else p["heads"] * p["d"]
        out = torch.full((B, nq, w), NAN, dtype=torch.float16, device=self.dev)
        self.launch(out=out, **kw)
        return out


def exact_checks(fam, p, X, v, info):
    """The answers a family knows exactly; {} for the others."""
    o = X.out4.double()
    if fam == "uniform":
        cnt, n = uniform_expected(p, X.dev)
        exp = (cnt.double() / n.double()).half().double()
        r = {"uniform_1ulp": bool(((o - exp).abs() <= ulp16(exp)).all())}
        ok = (n.double() * ulp16(exp) < 0.5).expand_as(exp)
        r["uniform_counts"] = bool((torch.round(o * n.double())[..., ok] == cnt.double()[ok]).all())
        return r
    if fam == "peaked":
        vj = torch.gather(v.double(), 2, info["jstar"][..., None].expand(-1, -1, -1, p["d"]))
        return {"peaked_1ulp": bool(((o - vj).abs() <= ulp16(vj) + 1e-12).all())}
    return {}


class Sweep(Tally):
    """Failures and calibration of one title (workload or synthetic group)."""

    def __init__(self, title):
        super().__init__(title)
        self.share, self.bias = defaultdict(float), defaultdict(float)

    def fail(self, lab, chk, val):
        self.failures.append((lab, chk, val))

    def run(self, p, seed):
        dev = torch.device("cuda", torch.cuda.current_device())
        X = Placed(p, dev)
        for fi, fam in enumerate(families(p)):
            lab = f"{label(p)} {fam}"
            try:
                gen = torch.Generator(device=dev).manual_seed(seed * 16 + fi)
                q, k, v, info = make_operands(p, fam, gen)
                X.fill(q, k, v)
                X.obuf.fill_(NAN)
                X.launch()
                if not X.contained():
                    self.fail(lab, "containment", "non-finite output or a write outside it")
                share, mean, std, n = check(q, k, v, X.out4, p)
                for key, ok in exact_checks(fam, p, X, v, info).items():
                    if not ok:
                        self.fail(lab, key, "False")
                first = X.out3.clone()
                X.launch()
                self.launches += 2
                if not torch.equal(first, X.out3):
                    self.fail(lab, "bit-reproducible", "second launch differs")
                if fam == "randn1" and p["nq"] < 1 << 20:
                    self.parts(X, p, first, lab)
                del first
            except Exception as e:  # noqa: BLE001 - a fault must name its problem
                raise RuntimeError(f"{lab}: {e}") from e
            if not share <= 1.0:
                self.fail(lab, "elementwise", f"{share:.3e}")
            self.share[fam] = max(self.share[fam], share)
            if n >= 256 and fam not in ("uniform", "peaked"):
                if not abs(mean) <= BIAS + ACC_RZ * p["nkv"] + 5 * std / math.sqrt(n):
                    self.fail(lab, "bias", f"{mean:.3e} (std {std:.2e}, n {n})")
                if n >= 65536:
                    self.bias[fam] = max(self.bias[fam], abs(mean))
        for c in attn_branches(p):
            COVER[c] += 1

    def parts(self, X, p, full, lab):
        """A sample, up to three 128-row query blocks and a head, each launched alone, are bit-equal to the full
        launch (a causal launch keeps its row indices only for the first block)."""
        if p["B"] > 1:
            b = p["B"] - 1
            if not torch.equal(X.part(b=b)[0], full[b]):
                self.fail(lab, "sample alone", f"b={b}")
            self.launches += 1
        nb = (p["nq"] + AQ - 1) // AQ
        for r in sorted({0} if p["causal"] else {0, nb // 2, nb - 1}):
            if nb > 1:
                rows = (AQ * r, min(p["nq"], AQ * r + AQ))
                if not torch.equal(X.part(rows=rows), full[:, rows[0]:rows[1]]):
                    self.fail(lab, "row block alone", f"rows {rows}")
                self.launches += 1
        if p["heads"] > 1:
            h, d = p["heads"] - 1, p["d"]
            if not torch.equal(X.part(head=h), full[:, :, h * d:(h + 1) * d]):
                self.fail(lab, "head alone", f"h={h}")
            self.launches += 1

    def calibration(self):
        return "largest share of the bound / largest |bias| per family: " + ", ".join(
            f"{f} {self.share[f]:.3f} / {self.bias[f]:.1e}" for f in FAMILIES if f in self.share)


def run_sweep(problems, title):
    sw = Sweep(title)
    for i, p in enumerate(problems):
        sw.run(p, 1000 + i)
        torch.cuda.empty_cache()
    sw.finish(len(problems), sw.calibration())


# ------------------------------------------------------------------------------------------------ model workloads
@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(ATTENTION_WORKLOADS))
def test_every_attention_launch_of_every_model(cuda_dev, name):
    calls, problems = record(ATTENTION_WORKLOADS[name], cuda_dev, {"attention": _attn_sig})
    print(f"\n{name}: {calls} calls, {len(problems)} distinct problems")
    assert problems
    if name == "rdm_one_token_context":     # the one-token context is folded into the out-projection: self-attention only
        assert all(p["nq"] == p["nkv"] and p["k_rel"] is not None for p in problems), [label(p) for p in problems]
    run_sweep(problems, name)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ synthetic grid
NKV_WALK = (1, 7, 63, 64, 65, 128, 129, 257, 320, 513, 577, 1025, 1100)
NQ_WALK = (1, 8, 63, 64, 65, 127, 129, 300)
D_GRID = (2, 6, 8, 10, 16, 24, 32, 34, 40, 48, 56, 64, 66, 80, 96, 98, 112, 128, 130, 144, 160)
FEW = ("randn1", "posv", "uniform", "peaked")


def _grid_heads():
    """Every multi-head instance by its d, at head_stride ceil8(d), an in-between multiple of 8 and dpad."""
    ps = []
    for d in D_GRID:
        dpad = (d + 63) // 64 * 64
        lo = _c8(d)
        for hs in sorted({lo, (lo + dpad) // 16 * 8, dpad}):
            for heads in (1, 3):
                ps.append(_ap(d=d, hs=hs, heads=heads, nq=129, nkv=257, fam=None if heads == 3 and hs == lo else FEW))
    return ps


def _grid_tiles():
    ps = [_ap(d=d, heads=2, nq=65, nkv=n) for d in (40, 80, 160) for n in NKV_WALK]
    ps += [_ap(d=d, heads=2, nq=n, nkv=129) for d in (40, 80, 160) for n in NQ_WALK]
    return ps


def _grid_causal():
    ps = []
    for d, hs in ((64, 0), (40, 40), (80, 128)):
        for nq, nkv in ((77, 77), (128, 128), (129, 129), (300, 300), (77, 200), (300, 97)):
            ps.append(_ap(d=d, hs=hs, heads=3, nq=nq, nkv=nkv, causal=True))
    return ps


def _grid_wide():
    ps = []
    for dp in (384, 512, 576, 960):
        for nq, nkv in ((1, 1), (16, 16), (64, 64), (65, 65), (100, 37), (129, 130), (256, 1100), (1024, 1024)):
            ps.append(_ap(d=dp, heads=1, nq=nq, nkv=nkv, B=1, hs=0))
            ps.append(_ap(d=dp, heads=1, nq=nq, nkv=nkv, B=3, hs=dp, fam=FEW + ("rising", "jump")))
    ps.append(_ap(d=960, heads=1, nq=130, nkv=200, B=2))            # streamed Q, the 4-deep ring wrapping inside a tile
    ps.append(_ap(d=512, heads=1, nq=16384, nkv=16384, fam=("randn1", "uniform")))
    return ps


def _grid_strides():
    ps = []
    for d, heads in ((40, 8), (64, 3), (80, 2), (160, 2)):
        hd = heads * d
        ps.append(_ap(d=d, heads=heads, B=2, nq=130, nkv=200, ldo=hd + 6, oo=2))         # out 4-byte aligned, ldo even
        ps.append(_ap(d=d, heads=heads, B=2, nq=130, nkv=200, ldq=hd + 24, ldk=hd + 8, qbs=131 * (hd + 24) + 64,
                      kbs=203 * (hd + 8), obs=130 * hd + 10, vbs=hd * 200 + 4096))        # ldq != ldk, slack strides
        ps.append(_ap(d=d, heads=heads, B=2, nq=136, nkv=136, ldq=2 * hd, ldk=2 * hd, k_rel=hd))   # fused q | k
    for B in (2, 3, 5):                  # V^T [hd, B * ntok] viewed per sample: ldvt = B ntok, batch stride ntok
        ps.append(_ap(d=40, heads=8, B=B, nq=144, nkv=144, ldvt=B * 144, vbs=144))
        ps.append(_ap(d=512, heads=1, B=B, nq=72, nkv=72, ldvt=B * 72, vbs=72))
    ps.append(_ap(d=64, heads=2, nq=100, nkv=300, scale=0.5))
    ps.append(_ap(d=32, heads=2, nq=100, nkv=300, scale=0.03125))
    return ps


def _grid_extents():
    return [_ap(d=32, heads=56, B=2, nq=576, nkv=576), _ap(d=32, heads=56, B=2, nq=2304, nkv=11),
            _ap(d=64, heads=16, B=256, nq=257, nkv=257, hs=0, ldq=2048, ldk=2048, k_rel=1024, fam=FEW)]


GRIDS = {"heads": _grid_heads, "tiles": _grid_tiles, "causal": _grid_causal, "wide": _grid_wide,
         "strides": _grid_strides, "extents": _grid_extents}


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(GRIDS))
def test_attention_synthetic_grid(cuda_dev, name):
    run_sweep(GRIDS[name](), f"synthetic/{name}")


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_attention_beyond_2g_elements(cuda_dev):
    """Q and the output each hold more than 2^31 elements (8 heads of d = 64 over 4,194,432 query rows, 77 keys): row
    offsets must be 64-bit everywhere."""
    free = torch.cuda.mem_get_info()[0]
    if free < 24 << 30:
        pytest.skip(f"needs 24 GiB of free device memory, {free >> 30} GiB are free")
    run_sweep([_ap(d=64, heads=8, nq=(1 << 22) + 128, nkv=77, fam=("randn1",))], "beyond 2^31 elements")


@pytest.mark.gpu
def test_attention_branch_coverage():
    """Every instance and every control-flow class of attention_tc.cu was launched by the sweeps above."""
    check_coverage(COVER, REQUIRED, "attention")


# ------------------------------------------------------------------------------------------------ host guards
BAD = [  # (what, base problem: "m" multi-head d = 40 / "w" single-head d = 512, descriptor fields to overwrite)
    ("null q", "m", dict(q=None)), ("null k", "m", dict(k=None)), ("null vt", "m", dict(vt=None)),
    ("null out", "m", dict(out=None)),
    ("odd d", "m", dict(d=39)), ("d = 0", "m", dict(d=0)), ("d > dpad", "m", dict(d=66, head_stride=72)),
    ("d > 160 at dpad 192", "m", dict(d=162, dpad=192, head_stride=168)), ("dpad 256", "m", dict(dpad=256)),
    ("dpad 0", "m", dict(dpad=0)), ("head_stride < d", "m", dict(head_stride=32)),
    ("head_stride % 8", "m", dict(head_stride=44)),
    ("ldq % 8", "m", dict(ldq=84)), ("ldk % 8", "m", dict(ldk=84)), ("ldvt % 8", "m", dict(ldvt=68)),
    ("odd ldo", "m", dict(ldo=81)), ("odd o_batch_stride", "m", dict(o_batch_stride=80 * 64 + 1)),
    ("batch 0", "m", dict(batch=0)), ("heads 0", "m", dict(heads=0)), ("nq 0", "m", dict(nq=0)),
    ("nkv 0", "m", dict(nkv=0)),
    ("scale 0", "m", dict(scale=0.0)), ("scale < 0", "m", dict(scale=-0.125)), ("scale NaN", "m", dict(scale=NAN)),
    ("scale inf", "m", dict(scale=float("inf"))),
    ("wide: scale < 0", "w", dict(scale=-1.0)), ("wide: scale NaN", "w", dict(scale=NAN)),
    ("wide: heads 2", "w", dict(heads=2)), ("wide: d != dpad", "w", dict(d=384)), ("wide: causal", "w", dict(causal=1)),
    ("wide: head_stride 256", "w", dict(head_stride=256)), ("wide: ldo % 8", "w", dict(ldo=516)),
    ("wide: o_batch_stride % 8", "w", dict(o_batch_stride=512 * 64 + 2)), ("wide: ldq % 8", "w", dict(ldq=516)),
    ("wide: ldvt % 8", "w", dict(ldvt=68)), ("wide: nkv 0", "w", dict(nkv=0)), ("wide: batch 0", "w", dict(batch=0)),
]


@pytest.mark.gpu
def test_attention_rejects_bad_descriptors(cuda_dev):
    """Checked on the host: nonzero, a message naming sdb_attention, nothing launched. The unmodified descriptors
    launch."""
    lib = _l.load()
    buf = torch.zeros(4 * 64 * 512, dtype=torch.float16, device=cuda_dev)

    def desc(base, **kw):
        a = _l.AttnDesc()
        a.q = a.k = a.vt = a.out = buf.data_ptr()
        a.batch, a.nq, a.nkv, a.ldvt, a.causal, a.scale = 1, 64, 64, 64, 0, 0.125
        if base == "m":
            a.heads, a.d, a.dpad, a.head_stride = 2, 40, 64, 40
            a.ldq = a.ldk = a.ldo = 80
        else:
            a.heads, a.d, a.dpad, a.head_stride = 1, 512, 512, 0
            a.ldq = a.ldk = a.ldo = 512
        a.q_batch_stride = a.k_batch_stride = a.o_batch_stride = 64 * a.ldq
        a.vt_batch_stride = a.heads * a.d * 64
        for k_, v in kw.items():
            setattr(a, k_, v)
        return a
    for base in ("m", "w"):
        n0 = lib.sdb_launch_count()
        assert lib.sdb_attention(C.byref(desc(base)), ops._stream()) == 0, lib.sdb_last_error()
        assert lib.sdb_launch_count() == n0 + 1
    torch.cuda.synchronize()
    wrong = []
    for what, base, kw in BAD:
        n0 = lib.sdb_launch_count()
        rc = lib.sdb_attention(C.byref(desc(base, **kw)), ops._stream())
        msg = lib.sdb_last_error() or b""
        if rc == 0 or b"sdb_attention" not in msg or lib.sdb_launch_count() != n0:
            wrong.append((what, rc, msg, lib.sdb_launch_count() - n0))
    torch.cuda.synchronize()
    assert not wrong, wrong


# ------------------------------------------------------------------------------------------------ CPU: the harness
def test_dispatch_mirror_cpu():
    table = [  # (problem, labels it must have, labels it must not have)
        (_ap(d=40, nq=4096, nkv=4096), {"<64,40>", "tiles:v_wrap@64", "tiles:k_phase2@64", "tiles:v_phase2@64",
                                        "hs:packed", "zero_fill_k16"}, {"ragged_kv", "ragged_q", "zero_fill_v8"}),
        (_ap(d=34, hs=48, nq=65, nkv=65), {"<64,40>", "hs:mid", "zero_fill_v8", "tiles:2@64", "ragged_q"},
         {"wg1_empty", "tiles:v_wrap@64"}),
        (_ap(d=56, hs=0), {"<64,64>", "hs:padded"}, {"hs:packed"}), (_ap(d=64), {"<64,64>", "hs:packed", "hs:padded"}, set()),
        (_ap(d=66, nkv=129), {"<128,128>", "hs:packed"}, {"hs:padded", "tiles:k_phase2@128", "tiles:v_wrap@128"}),
        (_ap(d=80, nkv=320), {"<128,80>", "tiles:v_wrap@128", "tiles:k_phase2@128"}, {"tiles:v_phase2@128"}),
        (_ap(d=96), {"<128,96>"}, set()), (_ap(d=112), {"<128,128>"}, set()), (_ap(d=130), {"<192,160>"}, set()),
        (_ap(d=16), {"<64,16>"}, {"zero_fill_k16"}), (_ap(d=48), {"<64,48>"}, set()),
        (_ap(d=160, nkv=257), {"<192,160>", "tiles:k_phase2@192", "tiles:v_wrap@192"}, {"tiles:v_phase2@192"}),
        (_ap(d=960, heads=1, nq=130, nkv=200), {"<960,160>", "stream_q_multi", "stream_q_ragged", "tiles:k_phase2@960",
                                                "tiles:v_wrap@960"}, {"hs:packed"}),
        (_ap(d=960, heads=1, nq=64, nkv=64), {"tiles:1@960", "tiles:k_phase2@960", "wg1_empty"}, {"stream_q_multi"}),
        (_ap(d=512, heads=1, nq=16, nkv=16), {"<512,128>", "tiles:1@wide"}, {"tiles:k_phase2@wide"}),
        (_ap(d=576, heads=1, nkv=128), {"<576,96>", "tiles:2@wide", "tiles:k_phase2@wide"}, {"tiles:v_wrap@wide"}),
        # causal: block 0 walks 2 tiles, block 1 min(300, 256) -> 4, block 2 all 5
        (_ap(d=64, nq=300, nkv=300, causal=True), {"causal", "causal_skip", "tiles:2@64", "tiles:v_wrap@64"},
         {"causal_nq_ne_nkv"}),
        (_ap(d=64, nq=300, nkv=97, causal=True), {"causal", "causal_nq_ne_nkv"}, {"causal_skip"}),
        (_ap(d=64, nq=77, nkv=200, causal=True), {"causal_skip", "tiles:2@64"}, {"tiles:v_wrap@64", "wg1_empty"}),
        (_ap(d=40, heads=8, B=2, nq=144, nkv=144, ldvt=288, vbs=144), {"vt_permuted"}, {"qk_fused_slices"}),
        (_ap(d=40, heads=8, ldq=640, ldk=640, k_rel=320), {"qk_fused_slices"}, {"vt_permuted", "ldo_wide"}),
        (_ap(d=40, heads=8, ldo=326), {"ldo_wide"}, {"offset_gt_2^31"}),
        (_ap(d=64, heads=8, nq=(1 << 22) + 128, nkv=77), {"offset_gt_2^31", "tiles:2@64"}, set()),
    ]
    for p, has, lacks in table:
        c = attn_branches(p)
        assert has <= c and not (lacks & c), (label(p), sorted(has - c), sorted(lacks & c))
    assert n_iters(_ap(nq=300, nkv=300, causal=True)) == [2, 4, 5] and n_iters(_ap(nq=300, nkv=300)) == [5, 5, 5]
    assert [attn_dv(192, d) for d in (130, 160, 162)] == [160, 160, 0] and attn_dv(128, 66) == 128
    assert len(INSTANCES) == 15
    grid = sum((g() for g in GRIDS.values()), []) + [_ap(d=64, heads=8, nq=(1 << 22) + 128, nkv=77)]
    got = set().union(*(attn_branches(p) for p in grid))
    # the synthetic grid alone reaches every required class
    assert REQUIRED <= got, sorted(REQUIRED - got)


def _sdpa(q, k, v, scale, causal):
    mask = None
    if causal:
        mask = ~torch.ones(q.shape[2], k.shape[2], dtype=torch.bool).triu(1)
    return F.scaled_dot_product_attention(q.float(), k.float(), v.float(), attn_mask=mask, scale=scale)


def test_references_against_torch_fp32_cpu():
    g = torch.Generator().manual_seed(0)
    for B, H, nq, nkv, d, causal in ((2, 3, 37, 50, 8, False), (1, 2, 70, 70, 16, True), (1, 2, 20, 45, 6, True),
                                     (1, 1, 45, 20, 10, True)):
        q, k, v = (_randn16((B, H, n, d), g) for n in (nq, nkv, nkv))
        want = _sdpa(q, k, v, 0.3, causal)
        whole = {(b, h0): (ref, A, smag, L) for b, h0, _, _, _, ref, A, smag, L in
                 attn_ref_chunks(q, k, v, 0.3, causal, 1 << 40)}
        assert len(whole) == B
        got = torch.empty(B, H, nq, d, dtype=torch.float64)
        for b, h0, h1, r0, r1, ref, A, smag, L in attn_ref_chunks(q, k, v, 0.3, causal, 7 * nkv):
            got[b, h0:h1, r0:r1] = ref
            w = whole[(b, 0)]
            assert torch.allclose(ref, w[0][h0:h1, r0:r1], rtol=1e-13, atol=1e-14)            # chunked equals unchunked
            assert torch.allclose(A, w[1][h0:h1, r0:r1], rtol=1e-13) and torch.allclose(L, w[3][h0:h1, r0:r1], rtol=1e-13)
            assert bool((A >= ref.abs() - 1e-15).all()) and bool((L >= 1).all())
            s = torch.matmul(q[b, h0:h1, r0:r1].double().abs(), k[b, h0:h1].double().abs().transpose(1, 2)) * 0.3
            assert torch.equal(smag, s.amax(-1))
        assert torch.allclose(got.float(), want, atol=2e-6, rtol=1e-5)
        # the reference passes its own check; a 2^-11 relative bias on P v does not
        p = _ap(B=B, heads=H, nq=nq, nkv=nkv, d=d, causal=causal, scale=0.3)
        share, mean, std, n = check(q, k, v, got.half(), p, 7 * nkv)
        assert share < 1.0 and n > 0
        share, _, _, _ = check(q, k, v, (got * (1 + 2.0 ** -9)).half(), p)
        assert share > 1.0
    assert float(ulp16(torch.tensor([1.0]))[0]) == 2.0 ** -10 and float(ulp16(torch.tensor([1e-7]))[0]) == 2.0 ** -24


def test_bias_statistic_sees_truncated_p_cpu():
    """P packed by truncation moves the signed mean of a launch by a few 1e-4 (downwards); P rounded to nearest stays
    within BIAS and within every elementwise bound."""
    g = torch.Generator().manual_seed(1)
    p = _ap(B=1, heads=4, nq=128, nkv=128, d=64)
    q, k, v, _ = make_operands(p, "posv", g)
    e = torch.softmax(torch.matmul(q.double(), k.double().transpose(2, 3)) * p["scale"], -1)
    e = e / e.amax(-1, keepdim=True)

    def out(rz):
        h = e.half().double()
        if rz:
            h = torch.where(h > e, h - ulp16(e), h)
        return (torch.matmul(h, v.double()) / e.sum(-1, keepdim=True)).half()
    share, mean, std, n = check(q, k, v, out(False), p)
    assert share <= 1.0 and n >= 4096 and abs(mean) <= BIAS + 5 * std / math.sqrt(n)
    share, mean, std, n = check(q, k, v, out(True), p)
    assert mean < -(BIAS + 5 * std / math.sqrt(n)) and mean < -1e-4, (share, mean, std, n)


@pytest.mark.parametrize("d,nq,nkv,causal", [(2, 9, 200, False), (8, 70, 130, False), (40, 130, 321, False),
                                             (64, 200, 200, True), (40, 77, 200, True), (512, 7, 190, False),
                                             (960, 7, 130, False)])
def test_operand_families_cpu(d, nq, nkv, causal):
    p = _ap(B=2, heads=3 if d <= 192 else 1, nq=nq, nkv=nkv, d=d, causal=causal)
    H, scale = p["heads"], p["scale"]
    T = (nkv + AKV - 1) // AKV
    tiles = torch.arange(nkv) // AKV
    for fi, fam in enumerate(FAMILIES):
        q, k, v, info = make_operands(p, fam, torch.Generator().manual_seed(fi))
        assert q.shape == (2, H, nq, d) and k.shape == v.shape == (2, H, nkv, d)
        assert all(t.dtype == torch.float16 and bool(torch.isfinite(t).all()) for t in (q, k, v)), fam
        s = torch.matmul(q.double(), k.double().transpose(2, 3)) * scale
        if causal:
            s = s.masked_fill(torch.arange(nkv)[None, :] > torch.arange(nq)[:, None], float("-inf"))
        tmax = torch.stack([s[..., tiles == t].amax(-1) for t in range(T)], -1)        # [B, H, nq, T]
        full = slice(nkv - 1, None) if causal else slice(None)                       # rows that see every tile
        seen = not causal or nq >= nkv
        Tf = nkv // AKV                                                               # whole tiles
        if fam == "uniform":
            assert bool((s[torch.isfinite(s)] == 0).all())
            cnt, n = uniform_expected(p, torch.device("cpu"))
            brute = torch.stack([(v[0, 0, :int(n[i]), :] == 1).sum(0) for i in range(nq)])
            assert torch.equal(cnt, brute)
        elif fam == "peaked":
            top2 = s.topk(min(2, nkv), -1)
            assert torch.equal(top2.indices[..., 0], info["jstar"])
            assert bool((top2.values[..., 0] - top2.values[..., 1] >= 40).all())
            if causal:
                i = torch.arange(nq)
                assert bool((info["jstar"] <= i).all()) and bool((info["jstar"][0, 0, 63:65] == i[63:65]).all())
            assert {0, nkv - 1, 63, 64, 127, 128} <= set(info["jstar"][0, 0].tolist()) or causal
            assert len(set(info["jstar"].flatten().tolist())) >= (8 if not causal else 4)
        elif fam in ("rising", "falling") and Tf > 1 and seen:
            step = (tmax[..., full, 1:Tf] - tmax[..., full, :Tf - 1]) * (1 if fam == "rising" else -1)
            assert float(step.min()) > 0 and float(step.max()) < 6.5 and 2.5 < float(step.mean()) < 3.5, fam
        elif fam == "jump" and T > 1 and seen:
            j = max(T - 2, 0)
            rest = torch.cat([tmax[..., full, :j], tmax[..., full, j + 1:]], -1).amax(-1)
            assert bool((tmax[..., full, j] - rest > 127 * math.log(2)).all())
        elif fam == "bigv":
            assert float(v.abs().max()) == 60000.0 and bool((v[0, 0, 0, ::4] == -v[0, 0, 1, ::4]).all())
        elif fam == "randn4":
            assert 8 < float(s[torch.isfinite(s)].std()) < 24


def test_signature_dedups_cpu():
    qk = torch.zeros(2, 64, 640, dtype=torch.float16)
    vt = torch.zeros(2, 320, 64, dtype=torch.float16)
    kw = dict(heads=8, d=40, dpad=64, nq=64, nkv=64, scale=40 ** -0.5, head_stride=40)
    s = lambda q=qk[:, :, :320], k=qk[:, :, 320:], v=vt, **o: signature(_attn_sig(q, k, v, **{**kw, **o}))
    assert s() == s() and s(causal=True) != s() and s(head_stride=0) != s() and s(scale=0.2) != s()
    p = _attn_sig(qk[:, :, :320], qk[:, :, 320:], vt, **kw)
    assert (p["k_rel"], p["ldq"], p["ldk"], p["qbs"], p["ldo"], p["obs"]) == (320, 640, 640, 64 * 640, 320, 64 * 320)
    assert "qk_fused_slices" in attn_branches(p) and "k=q+320" in label(p)
    assert s(k=torch.zeros(2, 64, 640, dtype=torch.float16)[:, :, 320:]) != s()          # K in a buffer of its own
    wide = torch.zeros(3, 64, 640, dtype=torch.float16)
    assert s(q=wide[::2, :, :320], k=wide[::2, :, 320:]) != s()                          # a batch stride
    perm = torch.zeros(320, 2, 64, dtype=torch.float16).permute(1, 0, 2)
    pp = _attn_sig(qk[:, :, :320], qk[:, :, 320:], perm, **kw)
    assert (pp["ldvt"], pp["vbs"]) == (128, 64) and "vt_permuted" in attn_branches(pp) and signature(pp) != s()
    base = torch.zeros(2 * 64 * 320 + 8, dtype=torch.float16)
    o0 = base[:2 * 64 * 320].view(2, 64, 320)
    o2 = base[2:2 + 2 * 64 * 320].view(2, 64, 320)
    assert s(out=o2) != s(out=o0) and _attn_sig(qk[:, :, :320], qk[:, :, 320:], vt, out=o2, **kw)["oo"] == (eoff(base) + 2) % 8
    ow = torch.zeros(2, 64, 326, dtype=torch.float16)[:, :, :320]
    assert _attn_sig(qk[:, :, :320], qk[:, :, 320:], vt, out=ow, **kw)["ldo"] == 326
    assert signature(dict(p, fam=("randn1",))) == signature(p)
