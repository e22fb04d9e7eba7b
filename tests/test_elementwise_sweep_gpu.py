"""Every layout, embedding and small-layer launch the models make, elementwise against an exact or fp64 reference; the
grid-stride wrap and the edges no model reaches; and the map from every kernel-launching C entry point to the tests
that check it.

The sweep:
  1. records the calls of one eager forward of each model (ELEMENTWISE_WORKLOADS) to the sdb200.ops functions in SIGS
     and deduplicates them by everything that reaches the kernel or its host code: sizes, flags, which optional
     outputs are requested and the element offset of every pointer;
  2. regenerates seeded operands per problem, each at its recorded element offset inside a NaN-filled buffer; what
     the kernel must not read is NaN as well: the rows rows_gather skips, the rows rows_pool does not select, the
     columns past `cols` of a transpose source with ldx > cols, the token and position rows no id selects;
  3. launches through the C entry point into outputs filled with NaN (uint8: a fill byte), with GUARD fill elements on
     both sides, checks every element, the guards, and a second launch into refilled outputs (uint8: another fill
     byte) for bit equality;
then a synthetic grid covers what no model reaches, and a Python mirror of the launch geometry records which classes
ran (test_elementwise_branch_coverage).

References and bounds (u = 2^-24, the fp32 unit roundoff):
  bit-exact     nchw_to_nhwc / nhwc_to_nchw (fp32 and fp16 out), transpose_f16 (pad columns [rows, ldo) untouched),
                cast_f16 (= torch .half(), round to nearest even), im2col3x3 (= .half() of the zero-padded F.unfold
                gather; the kpad tail exactly 0), upsample2x, resample_f32 mode 2 and mode 1 (= (((x00 + x01) + x10)
                + x11) / 4 in fp32: avg_pool2d's order), rows_gather, vit_embed, embed_tokens (fp32 tok + pos),
                axpby at a = 1, b = 0, rows_pool without normalisation (ties select the first maximum, as
                torch.argmax), and the sampler_step / dpm_solver_step / ddpm_step / mask_blend / axpby2 updates
                against their fp32 restatement in the kernels' operation order.
  byte-exact    to_uint8 against clamp((x + 1) / 2, 0, 1), then 255. * v in fp32, then truncation (txt2img.py:322-323)
                on the CPU, at every 2k/255 - 1 and one fp32 ulp either side, +-1, beyond +-1 and -0.0.
  linear_small  |out - ref| <= LS_REL (|x| |W|^T + |b|) (x 1.2 under SiLU) + ACT_REL |v|: fp32 FMA chains of K
                terms in 8-wide pieces and a 32-lane shuffle tree stay far below K u, so 1e-5 bounds K <= 6400
                with margin; __expf / the division inside SiLU are ACT_REL. The fp16 output adds half an fp16 ulp.
  pointwise     |out - ref| <= LS_REL (|alpha| |x| |W|^T + |b|): one rounding of alpha x per term, a chain of cin <= 128
                FMAs and the bias add stay below (cin + 2) u = 7.8e-6 relative to that sum.
  vq_quantize   z_q bit-exact against the fp32 restatement zv = fl(scale z), then fl(zv + fl(e[idx] - zv)). The index:
                the kernel compares d(j) = fl(fl(zz + q_j) - 2 dot_j) over codes j, where zz sums the D rounded squares
                fl(zv_k^2) with rounded adds (error <= D u sum zv^2), dot_j is an fma chain of length D (<= D u
                sum |zv e_j|, doubled exactly), q_j = code_sq is the fp64 sum of e_j^2 rounded once (<= u sum e_j^2),
                and the add and the subtract round once each (<= u (zz + q_j) and u |d|). With A_j = sum (|zv| +
                |e_j|)^2 >= sum zv^2 + sum e_j^2 + 2 sum |zv e_j|, every piece fits in (D + 2) u A_j, and (D + 3) u A_j
                covers the second-order terms. The kernel's choice beats the fp64 argmin j* in its own arithmetic, so
                d64(idx) - d64(j*) <= VQ_REL(D) (A_idx + A_j*), VQ_REL(D) = (D + 3) u, with d64 the fp64 distance from
                zv. Bit-identical codes have bit-identical distances, so idx is never a code with an identical twin of
                lower index (the lowest index wins a tie, as torch.argmin). Without indices, z_q equals that of the
                same launch with them.
  timestep      the frequency exp(-ln(P) j / half) is formed from three fp32 roundings of an exponent of magnitude
                e_j = ln(P) j / half and one expf (2 ulp): relative error <= (3 e_j + 3) u; the product t f adds u;
                cosf / sinf add 2 ulp of a value <= 1. So |out - ref| <= u ((3 e_j + 4) |t f| + TS_ABS) with
                TS_ABS = 6. t reaches 999, so the argument does: a frequency index off by one, or cos and sin
                swapped, is orders of magnitude past this. The fp16 variant adds an fp16 ulp of the value.
  vae_sample    |z - ref| <= VS_REL (|mean| + std |noise|) |scale| (expf 2 ulp, product, sum, scale: 5 u; VS_REL =
                8 u), with logvar drawn past both clamps (-30, 20) and without noise.
  rows_pool     normalised: |out - ref| <= (dim + 2) u |ref| (an fp32 sum of dim squares, sqrtf, one division).
  silu_f16      |out - ref| <= an fp16 ulp + ACT_REL |x|.
The largest share of each bound used is printed per workload.
"""
import ctypes as C
import math
import os
import re
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

import helpers  # noqa: F401  (puts the repository on sys.path)
from sdb200 import ops
from sdb200 import lib as _l
from sweeps import GUARD, NAN, Tally, check_coverage, eoff, record, signature, ulp16
from workloads import ELEMENTWISE_WORKLOADS

U = 2.0 ** -24
LS_REL = 1e-5
ACT_REL = 4e-6
TS_ABS = 6.0
VS_REL = 8 * U
LS_ROWS = 8                        # linear_small: samples per pass
LS_SMEM_FLOATS = 200 * 1024 // 4   # linear_small: activations of one pass in shared memory
FILL_U8 = (0x5A, 0xA5)             # the two fills of a uint8 output: equal results mean every byte was written
FILL_I64 = (-7, -9)                # the two fills of an int64 output (it has no NaN): code indices are never negative
FILLS = {torch.uint8: FILL_U8, torch.int64: FILL_I64}
VQ_CHUNK = 1024                    # vq_quantize: codes per shared-memory chunk
VQ_THREADS = 256                   # vq_quantize: latent pixels per block
PW_NARROW = 32                     # pointwise_small: the widest head before KL-f32 (SD-v1's VAE: 8 -> 8, 4 -> 4)
ACT_SILU = _l.ACT_SILU


# ------------------------------------------------------------------------------------------------ signatures
def _ao(t):
    return 0 if t is None else eoff(t)


def _nchw_to_nhwc_sig(x, want_f32=True, want_f16=False):
    nb, c, h, w = x.shape
    return dict(op="nchw_to_nhwc", nb=nb, c=c, h=h, w=w, f32=bool(want_f32), f16=bool(want_f16), ax=eoff(x))


def _nhwc_to_nchw_sig(x, out=None):
    nb, h, w, c = x.shape
    return dict(op="nhwc_to_nchw", nb=nb, c=c, h=h, w=w, ax=eoff(x), ao=_ao(out))


def _transpose_f16_sig(x, ldo=None, out=None):
    B, rows, cols = x.shape
    return dict(op="transpose_f16", B=B, rows=rows, cols=cols, ldx=cols, ldo=ldo or (rows + 7) // 8 * 8, ax=eoff(x),
                ao=_ao(out))


def _im2col3x3_sig(x, stride, pad_lo, ho, wo, kpad):
    nb, h, w, c = x.shape
    return dict(op="im2col3x3", nb=nb, h=h, w=w, c=c, stride=stride, pad_lo=pad_lo, ho=ho, wo=wo, kpad=kpad,
                ax=eoff(x))


def _upsample2x_sig(x):
    nb, h, w, c = x.shape
    return dict(op="upsample2x", nb=nb, h=h, w=w, c=c, ax=eoff(x))


def _resample_f32_sig(x, mode):
    nb, h, w, c = x.shape
    return dict(op="resample_f32", nb=nb, h=h, w=w, c=c, mode=mode, ax=eoff(x))


def _cast_f16_sig(x):
    return dict(op="cast_f16", n=x.numel(), ax=eoff(x))


def _timestep_embedding_f32_sig(t, dim, max_period=10000.0):
    return dict(op="timestep_embedding_f32", n=t.numel(), dim=dim, max_period=float(max_period), ax=eoff(t))


def _embed_tokens_sig(ids, tok, pos):
    B, n = ids.shape
    return dict(op="embed_tokens", B=B, n=n, dim=tok.shape[1], vocab=tok.shape[0], npos=pos.shape[0], ai=eoff(ids),
                at=eoff(tok), ap=eoff(pos))


def _vit_embed_sig(pe, cls_pos, pos_patches, nb):
    np_, dim = pos_patches.shape
    return dict(op="vit_embed", nb=nb, np=np_, dim=dim, ax=eoff(pe), ac=eoff(cls_pos), ap=eoff(pos_patches))


def _rows_gather_sig(x, rows, row_stride):
    dim = x.shape[-1]
    return dict(op="rows_gather", rows=rows, stride=row_stride, dim=dim, xrows=x.numel() // dim, ax=eoff(x))


def _rows_pool_sig(x, ids=None, normalize=False):
    dim = x.shape[-1]
    b, n_ctx = ids.shape if ids is not None else (x.numel() // dim, 0)
    return dict(op="rows_pool", b=b, n_ctx=n_ctx, dim=dim, ids=ids is not None, normalize=bool(normalize),
                ax=eoff(x))


def _linear_small_sig(x, w, bias=None, act=_l.ACT_NONE, want_f16=False, out=None):
    m, k = x.shape
    return dict(op="linear_small", M=m, K=k, N=w.shape[0], bias=bias is not None, act=int(act), f16=bool(want_f16),
                ax=eoff(x), aw=eoff(w), ab=_ao(bias), ao=_ao(out))


def _pointwise_small_sig(x, w, b=None, alpha=1.0):
    cout, cin = w.shape
    return dict(op="pointwise_small", npix=x.numel() // cin, cin=cin, cout=cout, alpha=float(alpha), bias=b is not None,
                ax=eoff(x), aw=eoff(w), ab=_ao(b))


def _vae_sample_sig(moments, noise, nb, hw, scale_factor):
    return dict(op="vae_sample", nb=nb, hw=hw, scale=float(scale_factor), noise=noise is not None, ax=eoff(moments),
                an=_ao(noise))


def _to_uint8_sig(x):
    return dict(op="to_uint8", n=x.numel(), ax=eoff(x))


def _axpby_sig(x, a, b=0.0, out=None):
    return dict(op="axpby", n=x.numel(), a=float(a), b=float(b), ax=eoff(x), ao=_ao(out))


def _vq_quantize_sig(z, codebook, code_sq, scale=1.0, want_indices=False):
    n_e, e_dim = codebook.shape
    # z_q and the indices are allocated by ops.vq_quantize: offset 0
    return dict(op="vq_quantize", m=z.numel() // e_dim, e_dim=e_dim, n_e=n_e, scale=float(scale),
                idx=bool(want_indices), az=eoff(z), aq=0, ae=eoff(codebook), asq=eoff(code_sq))


SIGS = {"nchw_to_nhwc": _nchw_to_nhwc_sig, "nhwc_to_nchw": _nhwc_to_nchw_sig, "transpose_f16": _transpose_f16_sig,
        "im2col3x3": _im2col3x3_sig, "upsample2x": _upsample2x_sig, "resample_f32": _resample_f32_sig,
        "cast_f16": _cast_f16_sig, "timestep_embedding_f32": _timestep_embedding_f32_sig,
        "embed_tokens": _embed_tokens_sig, "vit_embed": _vit_embed_sig, "rows_gather": _rows_gather_sig,
        "rows_pool": _rows_pool_sig, "linear_small": _linear_small_sig, "pointwise_small": _pointwise_small_sig,
        "vae_sample": _vae_sample_sig, "to_uint8": _to_uint8_sig, "axpby": _axpby_sig, "vq_quantize": _vq_quantize_sig}


def label(p):
    return p["op"] + "[" + " ".join(f"{k}={v}" for k, v in p.items() if k != "op") + "]"


# ------------------------------------------------------------------------------------------------ launch geometry
def grid_threads(sms):
    """Threads of a capped grid-stride launch (grid_for in elementwise.cu, cgrid in clip_image.cu)."""
    return sms * 16 * 256


def work_items(p):
    """Loop iterations of the grid-stride kernels (None: not a capped grid-stride launch)."""
    op = p["op"]
    if op == "im2col3x3":
        return p["nb"] * p["ho"] * p["wo"] * p["kpad"]
    if op == "upsample2x":
        return p["nb"] * 4 * p["h"] * p["w"] * (p["c"] // 4)
    if op == "resample_f32":
        return p["nb"] * p["h"] * p["w"] * (p["c"] // 4) * (4 if p["mode"] == 2 else 1) // (1 if p["mode"] == 2 else 4)
    if op in ("cast_f16", "silu_f16", "to_uint8", "axpby", "axpby2", "sampler_step", "dpm_solver_step", "ddpm_step",
              "mask_blend"):
        return p["n"]
    if op == "timestep_embedding":
        return p["n"] * (p["dim"] // 2)
    if op == "vae_sample":
        return p["nb"] * 4 * p["hw"]
    if op == "pointwise_small":
        return p["npix"] * p["cout"]
    if op == "embed_tokens":
        return p["B"] * p["n"] * p["dim"]
    if op == "vit_embed":
        return p["nb"] * (p["np"] + 1) * (p["dim"] // 4)
    if op == "rows_gather":
        return p["rows"] * p["dim"]
    return None


def classes(p, sms):
    """The classes of problem p that the coverage test requires (restated from the kernels' launch code)."""
    op = p["op"]
    cls = {op}
    n = work_items(p)
    if n is not None and n > grid_threads(sms):
        cls.add(f"wrap:{op}")
    if op == "linear_small":
        cls.add("ls:passes" if p["M"] > LS_ROWS else "ls:one_pass")
        if (p["K"] // 8) % 32:
            cls.add("ls:partial_u")          # a k-sweep where only some lanes have a u step
        if p["N"] % 32:
            cls.add("ls:n_tail")             # a block with features past N
        cls |= {k for k, on in (("ls:bias", p["bias"]), ("ls:silu", p["act"] == ACT_SILU), ("ls:f16", p["f16"])) if on}
    elif op == "im2col3x3":
        cls.add(f"im2col:s{p['stride']}p{p['pad_lo']}")
    elif op == "resample_f32":
        cls.add(f"resample:{p['mode']}")
    elif op == "rows_pool":
        cls |= {k for k, on in (("pool:ids", p["ids"]), ("pool:normalize", p["normalize"])) if on}
    elif op == "nchw_to_nhwc":
        cls.add("nhwc:" + ("both" if p["f32"] and p["f16"] else "f32" if p["f32"] else "f16"))
    elif op == "pointwise_small":
        cls |= {k for k, on in (("pw:wide_in", p["cin"] > PW_NARROW), ("pw:wide_out", p["cout"] > PW_NARROW)) if on}
    elif op == "vq_quantize":
        cls.add(f"vq:e{p['e_dim']}")
        if p["n_e"] > VQ_CHUNK:
            cls.add("vq:multi_chunk")
            if p["n_e"] % VQ_CHUNK:
                cls.add("vq:partial_chunk")      # a last chunk shorter than the full ones before it
        if p["m"] % VQ_THREADS:
            cls.add("vq:tail_block")             # a block with threads past the last pixel
        if not p["idx"]:
            cls.add("vq:no_indices")
    return cls


GRID_STRIDE_OPS = ("im2col3x3", "upsample2x", "resample_f32", "cast_f16", "silu_f16", "to_uint8", "axpby", "axpby2",
                   "sampler_step", "dpm_solver_step", "ddpm_step", "mask_blend", "timestep_embedding", "vae_sample",
                   "pointwise_small", "embed_tokens", "vit_embed", "rows_gather")
REQUIRED = ({"ls:one_pass", "ls:passes", "ls:partial_u", "ls:n_tail", "ls:bias", "ls:silu", "ls:f16",
             "im2col:s1p1", "im2col:s2p0", "im2col:s2p1", "resample:1", "resample:2", "pool:ids", "pool:normalize",
             "nhwc:f32", "nhwc:f16", "nhwc:both", "nhwc_to_nchw", "transpose_f16", "timestep_embedding_f32",
             "rows_pool", "to_uint8", "silu_f16", "timestep_embedding", "pw:wide_in", "pw:wide_out",
             "vq:multi_chunk", "vq:partial_chunk", "vq:tail_block", "vq:no_indices"}
            | {f"vq:e{d}" for d in range(1, 9)} | {f"wrap:{op}" for op in GRID_STRIDE_OPS})
COVER = defaultdict(int)


# ------------------------------------------------------------------------------------------------ buffers
def _inp(values, off, fill=NAN):
    """values placed at element offset `off` (from a 16-byte boundary) of a buffer filled with `fill` before and after."""
    n = values.numel()
    buf = torch.full((n + off + GUARD,), fill, dtype=values.dtype, device=values.device)
    v = buf[off: off + n].view(values.shape)
    v.copy_(values)
    return v


class Out:
    """An output view at element offset `off` inside GUARD fill elements on both sides (NaN; uint8 and int64: FILLS)."""

    def __init__(self, shape, dtype, dev, off=0):
        n = math.prod(shape)
        self.buf = torch.empty(n + off + 2 * GUARD, dtype=dtype, device=dev)
        self.v = self.buf[GUARD + off: GUARD + off + n].view(shape)
        self.lo, self.n = GUARD + off, n

    def fill(self, k):
        self.buf.fill_(FILLS[self.buf.dtype][k] if self.buf.dtype in FILLS else NAN)

    def guards_ok(self, k):
        out = torch.cat([self.buf[:self.lo], self.buf[self.lo + self.n:]])
        return bool((out == FILLS[out.dtype][k]).all()) if out.dtype in FILLS else bool(out.isnan().all())


def _bits(t):
    return t.contiguous().view(torch.uint8)


def launch2(outs, call, what, before=None):
    """Two launches into freshly filled outputs: (the first results, bit-equal second results, guards intact)."""
    first, same, guards = None, True, True
    for k in (0, 1):
        for o in outs.values():
            o.fill(k)
        if before is not None:
            before()
        _l.check(call(), what)
        torch.cuda.synchronize()
        guards = guards and all(o.guards_ok(k) for o in outs.values())
        if first is None:
            first = {name: o.v.clone() for name, o in outs.items()}
        else:
            same = all(torch.equal(_bits(first[name]), _bits(o.v)) for name, o in outs.items())
    return first, same, guards


def _share(err, bound):
    return float((err / bound.clamp_min(1e-300)).max()) if err.numel() else 0.0


def _eq(a, b):
    """Bit-equal, NaN patterns included."""
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


P = ops._ptr


def S():
    return ops._stream()


def L():
    return _l.load()


# ------------------------------------------------------------------------------------------------ references
def im2col_ref(x, stride, pad_lo, ho, wo, kpad):
    """fp16 [nb * ho * wo, kpad]: column k = tap * c + ch, tap = 3 ky + kx, of the zero-padded input; tail 0."""
    nb, h, w, c = x.shape
    pad_hi_y = max(0, (ho - 1) * stride + 3 - pad_lo - h)
    pad_hi_x = max(0, (wo - 1) * stride + 3 - pad_lo - w)
    xp = F.pad(x.permute(0, 3, 1, 2), (pad_lo, pad_hi_x, pad_lo, pad_hi_y))
    u = F.unfold(xp, 3, stride=stride)                                          # [nb, c * 9, L'] in (ch, ky, kx) order
    hu = (h + pad_lo + pad_hi_y - 3) // stride + 1
    wu = (w + pad_lo + pad_hi_x - 3) // stride + 1
    u = u.view(nb, c, 9, hu, wu)[:, :, :, :ho, :wo]
    cols = u.permute(0, 3, 4, 2, 1).reshape(nb * ho * wo, 9 * c)
    out = torch.zeros(nb * ho * wo, kpad, dtype=torch.float16, device=x.device)
    out[:, :9 * c] = cols.half()
    return out


def pool_ref(x):
    """2x2 average pool in avg_pool2d's order, fp32 NHWC."""
    return (((x[:, 0::2, 0::2] + x[:, 0::2, 1::2]) + x[:, 1::2, 0::2]) + x[:, 1::2, 1::2]) / 4.0


def to_uint8_ref(x):
    """txt2img.py:320-323 on the CPU: clamp((x + 1) / 2, 0, 1), 255. * v in fp32, truncation to uint8."""
    v = torch.clamp((x.cpu() + 1.0) / 2.0, min=0.0, max=1.0)
    return (torch.tensor(255.0, dtype=torch.float32) * v).to(torch.uint8)


def to_uint8_edges():
    """2k/255 - 1 for every k, one fp32 ulp either side, +-1, beyond +-1, +-0."""
    t = (torch.arange(256, dtype=torch.float64) * 2 / 255 - 1).float()
    up, dn = torch.nextafter(t, torch.tensor(2.0)), torch.nextafter(t, torch.tensor(-2.0))
    extra = torch.tensor([1.0, -1.0, 1.0000001, -1.0000001, 1.5, -1.5, 7.0, -7.0, 1e30, -1e30, 0.0, -0.0])
    return torch.cat([t, up, dn, extra])


def first_max(ids):
    """Index of the first largest id of each row (torch.argmax's choice among ties)."""
    n = ids.shape[1]
    mx = ids.max(1, keepdim=True).values
    idx = torch.arange(n, device=ids.device).expand_as(ids)
    return torch.where(ids == mx, idx, n).min(1).values


def timestep_ref(t, dim, max_period):
    """(fp64 [n, dim] reference, the bound of the docstring)."""
    half = dim // 2
    e = math.log(max_period) * torch.arange(half, dtype=torch.float64, device=t.device) / half
    arg = t.double()[:, None] * torch.exp(-e)[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    b = U * ((3 * e[None] + 4) * arg.abs() + TS_ABS)
    return ref, torch.cat([b, b], 1)


def f32(v):
    return torch.tensor(v, dtype=torch.float32)


def sampler_ref(x, eu, ec, h1, h2, h3, noise, scale, a_t, a_prev, sigma_t, sq1m):
    """sdb_sampler_step at order 3, guided, with noise: fp32 in the kernel's operation order (CPU)."""
    e = eu + f32(scale) * (ec - eu)
    ep = (((f32(55.0) * e - f32(59.0) * h1) + f32(37.0) * h2) - f32(9.0) * h3) / f32(24.0)
    sa, sp = torch.sqrt(f32(a_t)), torch.sqrt(f32(a_prev))
    dc = torch.sqrt((f32(1.0) - f32(a_prev)) - f32(sigma_t) * f32(sigma_t))
    p0 = (x - f32(sq1m) * ep) / sa
    xp = (sp * p0 + dc * ep) + f32(sigma_t) * noise
    return xp, p0, e


def dpm_ref(x, eu, ec, m_prev, scale, sigma_s, alpha_s, c_x, c_m, inv_r0):
    e = eu + f32(scale) * (ec - eu)
    m0 = (x - f32(sigma_s) * e) / f32(alpha_s)
    xt = f32(c_x) * x - f32(c_m) * m0
    xt = xt - (f32(0.5) * f32(c_m)) * (f32(inv_r0) * (m0 - m_prev))
    return xt, m0


def ddpm_ref(x, eps, noise, sra, srm1, c1, c2, sigma):
    x0 = f32(sra) * x - f32(srm1) * eps
    return (f32(c1) * x0 + f32(c2) * x) + f32(sigma) * noise, x0


# ------------------------------------------------------------------------------------------------ one problem per op
def _randn(shape, g, scale=1.0):
    return torch.randn(shape, generator=g, device=g.device) * scale


def run_nchw_to_nhwc(p, g, dev):
    nb, c, h, w = p["nb"], p["c"], p["h"], p["w"]
    x = _inp(_randn((nb, c, h, w), g, 3.0), p["ax"])
    outs = {}
    if p["f32"]:
        outs["o32"] = Out((nb, h, w, c), torch.float32, dev)
    if p["f16"]:
        outs["o16"] = Out((nb, h, w, c), torch.float16, dev)
    o = lambda k: P(outs[k].v) if k in outs else None
    res, same, guards = launch2(outs, lambda: L().sdb_nchw_to_nhwc(P(x), nb, c, h * w, o("o32"), o("o16"), S()),
                                "sdb_nchw_to_nhwc")
    ref = x.permute(0, 2, 3, 1)
    r = {}
    if "o32" in res:
        r["exact_f32"] = _eq(res["o32"], ref.contiguous())
    if "o16" in res:
        r["exact_f16"] = _eq(res["o16"], ref.half().contiguous())
    return r, same, guards


def run_nhwc_to_nchw(p, g, dev):
    nb, c, h, w = p["nb"], p["c"], p["h"], p["w"]
    x = _inp(_randn((nb, h, w, c), g, 3.0), p["ax"])
    outs = {"o": Out((nb, c, h, w), torch.float32, dev, p["ao"])}
    res, same, guards = launch2(outs, lambda: L().sdb_nhwc_to_nchw(P(x), nb, c, h * w, P(outs["o"].v), S()),
                                "sdb_nhwc_to_nchw")
    return {"exact": _eq(res["o"], x.permute(0, 3, 1, 2).contiguous())}, same, guards


def run_transpose_f16(p, g, dev):
    B, rows, cols, ldx, ldo = p["B"], p["rows"], p["cols"], p["ldx"], p["ldo"]
    src = torch.full((B, rows, ldx), NAN, dtype=torch.float16, device=dev)   # columns past cols: never read
    src[..., :cols] = _randn((B, rows, cols), g, 2.0).half()
    x = _inp(src, p["ax"])
    outs = {"o": Out((B, cols, ldo), torch.float16, dev, p["ao"])}
    res, same, guards = launch2(outs, lambda: L().sdb_transpose_f16(P(x), B, rows, cols, ldx, P(outs["o"].v), ldo,
                                                                    S()), "sdb_transpose_f16")
    o = res["o"]
    return {"exact": _eq(o[..., :rows].contiguous(), src[..., :cols].transpose(1, 2).contiguous()),
            "pad_untouched": bool(o[..., rows:].isnan().all())}, same, guards


def run_im2col3x3(p, g, dev):
    nb, h, w, c = p["nb"], p["h"], p["w"], p["c"]
    x = _inp(_randn((nb, h, w, c), g, 2.0), p["ax"])
    outs = {"o": Out((nb * p["ho"] * p["wo"], p["kpad"]), torch.float16, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_im2col3x3(P(x), nb, h, w, c, p["stride"], p["pad_lo"], p["ho"],
                                                                p["wo"], p["kpad"], P(outs["o"].v), S()),
                                "sdb_im2col3x3")
    ref = im2col_ref(x, p["stride"], p["pad_lo"], p["ho"], p["wo"], p["kpad"])
    return {"exact": _eq(res["o"], ref), "tail_zero": bool((res["o"][:, 9 * c:] == 0).all())}, same, guards


def run_upsample2x(p, g, dev):
    nb, h, w, c = p["nb"], p["h"], p["w"], p["c"]
    x = _inp(_randn((nb, h, w, c), g, 2.0), p["ax"])
    outs = {"o": Out((nb, 2 * h, 2 * w, c), torch.float16, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_upsample2x(P(x), nb, h, w, c, P(outs["o"].v), S()),
                                "sdb_upsample2x")
    ref = x.repeat_interleave(2, 1).repeat_interleave(2, 2).half()
    return {"exact": _eq(res["o"], ref)}, same, guards


def run_resample_f32(p, g, dev):
    nb, h, w, c, mode = p["nb"], p["h"], p["w"], p["c"], p["mode"]
    x = _inp(_randn((nb, h, w, c), g, 2.0) + 0.3, p["ax"])
    oshape = (nb, h // 2, w // 2, c) if mode == 1 else (nb, 2 * h, 2 * w, c)
    outs = {"o": Out(oshape, torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_resample_f32(P(x), nb, h, w, c, mode, P(outs["o"].v), S()),
                                "sdb_resample_f32")
    ref = pool_ref(x) if mode == 1 else x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    return {"exact": _eq(res["o"], ref.contiguous())}, same, guards


def _wide(n, g):
    """fp32 values over fp16's whole range and past it: subnormals, overflow to inf, round-half-even cases."""
    v = _randn((n,), g) * torch.exp2(torch.randint(-30, 18, (n,), generator=g, device=g.device).float())
    k = min(n, 64)
    v[:k] = torch.tensor([1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 65504.0, 65520.0, -65520.0, 2.0 ** -25, 2.0 ** -24,
                          -(2.0 ** -26), 0.0, -0.0] * 7, device=g.device)[:k]
    return v


def run_cast_f16(p, g, dev):
    x = _inp(_wide(p["n"], g), p["ax"])
    outs = {"o": Out((p["n"],), torch.float16, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_cast_f16(P(x), p["n"], P(outs["o"].v), S()), "sdb_cast_f16")
    return {"exact": _eq(res["o"], x.half())}, same, guards


def run_silu_f16(p, g, dev):
    x = _inp(_randn((p["n"],), g, 6.0), p["ax"])
    outs = {"o": Out((p["n"],), torch.float16, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_silu_f16(P(x), p["n"], P(outs["o"].v), S()), "sdb_silu_f16")
    xd = x.double()
    ref = xd * torch.sigmoid(xd)
    h = res["o"].double()
    return {"finite": bool(torch.isfinite(res["o"]).all()),
            "silu_elem": _share((h - ref).abs(), torch.maximum(ulp16(ref), ulp16(h)) + ACT_REL * xd.abs())}, same, guards


def _timesteps(p, g):
    t = p.get("t")
    if t is not None:
        return torch.tensor(t, dtype=torch.float32, device=g.device)
    t = torch.randint(0, 1000, (p["n"],), generator=g, device=g.device).float()
    t[0] = 999.0
    return t


def run_timestep_embedding_f32(p, g, dev):
    t = _inp(_timesteps(p, g), p["ax"])
    n, dim = t.numel(), p["dim"]
    outs = {"o": Out((n, dim), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_timestep_embedding_f32(P(t), n, dim, p["max_period"],
                                                                             P(outs["o"].v), S()),
                                "sdb_timestep_embedding_f32")
    ref, bound = timestep_ref(t, dim, p["max_period"])
    return {"finite": bool(torch.isfinite(res["o"]).all()),
            "timestep_elem": _share((res["o"].double() - ref).abs(), bound)}, same, guards


def run_timestep_embedding(p, g, dev):
    t = _inp(_timesteps(p, g), p["ax"])
    n, dim = t.numel(), p["dim"]
    outs = {"o": Out((n, dim), torch.float16, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_timestep_embedding(P(t), n, dim, p["max_period"],
                                                                         P(outs["o"].v), S()),
                                "sdb_timestep_embedding")
    ref, bound = timestep_ref(t, dim, p["max_period"])
    h = res["o"].double()
    return {"finite": bool(torch.isfinite(res["o"]).all()),
            "timestep16_elem": _share((h - ref).abs(), torch.maximum(ulp16(ref), ulp16(h)) + bound)}, same, guards


def run_embed_tokens(p, g, dev):
    B, n, dim, vocab, npos = p["B"], p["n"], p["dim"], p["vocab"], p["npos"]
    ids = torch.randint(0, vocab, (B, n), generator=g, device=dev)
    if B * n >= vocab:
        ids.view(-1)[:vocab] = torch.randperm(vocab, generator=g, device=dev)     # every row of the table
    ids.view(-1)[0], ids.view(-1)[-1] = 0, vocab - 1
    ids = _inp(ids, p["ai"], fill=-1)
    tok_v = torch.full((vocab, dim), NAN, device=dev)                # rows no id selects: NaN
    used = ids.unique()
    tok_v[used] = _randn((used.numel(), dim), g)
    pos_v = torch.full((npos, dim), NAN, device=dev)                 # position rows past n: NaN
    pos_v[:n] = _randn((n, dim), g, 0.5)
    tok, pos = _inp(tok_v, p["at"]), _inp(pos_v, p["ap"])
    outs = {"o": Out((B * n, dim), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_embed_tokens(P(ids), B * n, n, dim, vocab, P(tok), P(pos),
                                                                   P(outs["o"].v), S()), "sdb_embed_tokens")
    ref = tok[ids.view(-1)] + pos[:n].repeat(B, 1)
    return {"exact": _eq(res["o"], ref)}, same, guards


def run_vit_embed(p, g, dev):
    nb, np_, dim = p["nb"], p["np"], p["dim"]
    pe = _inp(_randn((nb * np_, dim), g), p["ax"])
    cls_pos = _inp(_randn((dim,), g), p["ac"])
    pos = _inp(_randn((np_, dim), g, 0.5), p["ap"])
    outs = {"o": Out((nb * (np_ + 1), dim), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_vit_embed(P(pe), P(cls_pos), P(pos), nb, np_, dim,
                                                                P(outs["o"].v), S()), "sdb_vit_embed")
    ref = torch.cat([cls_pos.expand(nb, 1, dim), pe.view(nb, np_, dim) + pos[None]], 1).view(-1, dim)
    return {"exact": _eq(res["o"], ref)}, same, guards


def run_rows_gather(p, g, dev):
    rows, stride, dim, xrows = p["rows"], p["stride"], p["dim"], p["xrows"]
    xv = torch.full((xrows, dim), NAN, device=dev)                   # rows the gather skips: NaN
    sel = torch.arange(rows, device=dev) * stride
    xv[sel] = _randn((rows, dim), g)
    x = _inp(xv, p["ax"])
    outs = {"o": Out((rows, dim), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_rows_gather(P(x), rows, stride, dim, P(outs["o"].v), S()),
                                "sdb_rows_gather")
    return {"exact": _eq(res["o"], x[sel])}, same, guards


def _eot_ids(b, n_ctx, g):
    """CLIP-like ids: BOS, tokens, EOT (the largest id), then padding; odd rows pad with EOT, so the maximum repeats."""
    eot = 49407
    ids = torch.randint(1, eot - 1, (b, n_ctx), generator=g, device=g.device)
    if n_ctx == 1:
        return ids
    ends = torch.randint(1, n_ctx, (b,), generator=g, device=g.device)
    ids[:, 0] = eot - 1
    for i in range(b):
        e = int(ends[i])
        ids[i, e] = eot
        ids[i, e + 1:] = eot if i % 2 else 0
    ids[0, -1] = eot
    return ids


def run_rows_pool(p, g, dev):
    b, n_ctx, dim = p["b"], p["n_ctx"], p["dim"]
    ids = _eot_ids(b, n_ctx, g) if p["ids"] else None
    rows = b * n_ctx if ids is not None else b
    xv = _randn((rows, dim), g, 2.0)
    src = torch.arange(b, device=dev)
    if ids is not None:
        src = src * n_ctx + first_max(ids)
        keep = torch.full((rows, dim), NAN, device=dev)              # rows other than the first EOT: NaN
        keep[src] = xv[src]
        xv = keep
        ids = _inp(ids, 0, fill=-1)
    x = _inp(xv, p["ax"])
    outs = {"o": Out((b, dim), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_rows_pool(P(x), P(ids), b, n_ctx, dim, int(p["normalize"]),
                                                                P(outs["o"].v), S()), "sdb_rows_pool")
    sel = x[src]
    if not p["normalize"]:
        return {"exact": _eq(res["o"], sel)}, same, guards
    sd = sel.double()
    ref = sd / sd.norm(dim=1, keepdim=True)
    return {"finite": bool(torch.isfinite(res["o"]).all()),
            "pool_norm_elem": _share((res["o"].double() - ref).abs(), (dim + 2) * U * ref.abs() + 1e-300)}, same, guards


def run_linear_small(p, g, dev):
    M, K, N = p["M"], p["K"], p["N"]
    x = _inp(_randn((M, K), g), p["ax"])
    w = _inp((_randn((N, K), g) * K ** -0.5).half(), p["aw"])
    bias = _inp(_randn((N,), g), p["ab"]) if p["bias"] else None
    outs = {"o32": Out((M, N), torch.float32, dev, p["ao"])}
    if p["f16"]:
        outs["o16"] = Out((M, N), torch.float16, dev)
    res, same, guards = launch2(outs, lambda: L().sdb_linear_small(
        P(x), M, K, P(w), N, P(bias), p["act"], P(outs["o32"].v), P(outs["o16"].v) if "o16" in outs else None, S()),
        "sdb_linear_small")
    bd = bias.double() if bias is not None else torch.zeros(N, dtype=torch.float64, device=dev)
    v = x.double() @ w.double().t() + bd
    absref = x.double().abs() @ w.double().abs().t() + bd.abs()
    silu = p["act"] == ACT_SILU
    ref = v * torch.sigmoid(v) if silu else v
    bound = LS_REL * absref * (1.2 if silu else 1.0) + (ACT_REL * v.abs() if silu else 0.0)
    o = res["o32"]
    r = {"finite": bool(torch.isfinite(o).all()), "ls_elem": _share((o.double() - ref).abs(), bound)}
    if "o16" in res:
        h = res["o16"].double()
        r["finite"] = r["finite"] and bool(torch.isfinite(res["o16"]).all())
        r["ls_elem_f16"] = _share((h - ref).abs(), 0.5 * torch.maximum(ulp16(ref), ulp16(h)) + bound)
    return r, same, guards


def run_pointwise_small(p, g, dev):
    npix, cin, cout, alpha = p["npix"], p["cin"], p["cout"], p["alpha"]
    x = _inp(_randn((npix, cin), g, 2.0), p["ax"])
    w = _inp(_randn((cout, cin), g) * cin ** -0.5, p["aw"])
    b = _inp(_randn((cout,), g), p["ab"]) if p["bias"] else None
    outs = {"o": Out((npix, cout), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_pointwise_small(P(x), npix, cin, cout, P(w), P(b), alpha,
                                                                      P(outs["o"].v), S()), "sdb_pointwise_small")
    bd = b.double() if b is not None else torch.zeros(cout, dtype=torch.float64, device=dev)
    ref = (alpha * x.double()) @ w.double().t() + bd
    absref = (abs(alpha) * x.double().abs()) @ w.double().abs().t() + bd.abs()
    return {"finite": bool(torch.isfinite(res["o"]).all()),
            "pointwise_elem": _share((res["o"].double() - ref).abs(), LS_REL * absref)}, same, guards


def run_vae_sample(p, g, dev):
    nb, hw, scale = p["nb"], p["hw"], p["scale"]
    m = _randn((nb * hw, 8), g, 2.0)
    m[:, 4:] = _randn((nb * hw, 4), g, 20.0)                       # logvar: past both clamps (-30, 20)
    m = _inp(m, p["ax"])
    noise = _inp(_randn((nb, 4, hw), g), p["an"]) if p["noise"] else None
    outs = {"o": Out((nb, 4, hw), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_vae_sample(P(m), P(noise), nb, hw, scale, P(outs["o"].v), S()),
                                "sdb_vae_sample")
    md = m.double().view(nb, hw, 8).permute(0, 2, 1)
    mean, std = md[:, :4], torch.exp(0.5 * md[:, 4:].clamp(-30.0, 20.0))
    nd = noise.double() if noise is not None else torch.zeros_like(mean)
    ref = (mean + std * nd) * scale
    bound = VS_REL * (mean.abs() + std * nd.abs()) * abs(scale) + 1e-300
    return {"finite": bool(torch.isfinite(res["o"]).all()),
            "vae_sample_elem": _share((res["o"].double() - ref).abs(), bound)}, same, guards


def run_to_uint8(p, g, dev):
    n = p["n"]
    v = torch.rand(n, generator=g, device=dev) * 2.4 - 1.2
    e = to_uint8_edges().to(dev)
    k = min(n, e.numel())
    v[:k] = e[:k]
    x = _inp(v, p["ax"])
    outs = {"o": Out((n,), torch.uint8, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_to_uint8(P(x), n, P(outs["o"].v), S()), "sdb_to_uint8")
    return {"exact": torch.equal(res["o"].cpu(), to_uint8_ref(x))}, same, guards


def run_axpby(p, g, dev):
    n, a, b = p["n"], p["a"], p["b"]
    x = _inp(_randn((n,), g, 3.0), p["ax"])
    outs = {"o": Out((n,), torch.float32, dev, p["ao"])}
    res, same, guards = launch2(outs, lambda: L().sdb_axpby(P(x), a, b, n, P(outs["o"].v), S()), "sdb_axpby")
    if (a, b) == (1.0, 0.0):
        return {"exact": _eq(res["o"], x.clone())}, same, guards
    ref = float(f32(a)) * x.double() + float(f32(b))
    return {"axpby_elem": _share((res["o"].double() - ref).abs(), U * (ref.abs() + (float(f32(a)) * x.double()).abs())
                                 + 1e-300)}, same, guards


def run_axpby2(p, g, dev):
    n, a, b = p["n"], p["a"], p["b"]
    x, y = _inp(_randn((n,), g), 0), _inp(_randn((n,), g), 0)
    outs = {"o": Out((n,), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_axpby2(P(x), P(y), a, b, n, P(outs["o"].v), S()), "sdb_axpby2")
    ref = f32(a) * x.cpu() + f32(b) * y.cpu()
    return {"exact": _eq(res["o"].cpu(), ref)}, same, guards


SAMPLER_K = dict(scale=7.5, a_t=0.3, a_prev=0.45, sigma_t=0.2, sq1m=0.8366600265340756)


def run_sampler_step(p, g, dev):
    n = p["n"]
    x, eps2, h1, h2, h3, noise = (_inp(_randn((m,), g), 0) for m in (n, 2 * n, n, n, n, n))
    outs = {k: Out((n,), torch.float32, dev) for k in ("x_prev", "x_prev2", "pred_x0", "e_out")}
    k = SAMPLER_K
    res, same, guards = launch2(outs, lambda: L().sdb_sampler_step(
        P(x), P(eps2), None, 1, k["scale"], 3, P(h1), P(h2), P(h3), P(noise), k["a_t"], k["a_prev"], k["sigma_t"],
        k["sq1m"], n, P(outs["x_prev"].v), P(outs["x_prev2"].v), P(outs["pred_x0"].v), P(outs["e_out"].v), S()),
        "sdb_sampler_step")
    c = lambda t: t.cpu()
    xp, p0, e = sampler_ref(c(x), c(eps2[:n]), c(eps2[n:]), c(h1), c(h2), c(h3), c(noise), k["scale"], k["a_t"],
                            k["a_prev"], k["sigma_t"], k["sq1m"])
    return {"exact_x": _eq(c(res["x_prev"]), xp), "exact_x2": _eq(c(res["x_prev2"]), xp),
            "exact_pred_x0": _eq(c(res["pred_x0"]), p0), "exact_e": _eq(c(res["e_out"]), e)}, same, guards


DPM_K = dict(scale=5.0, sigma_s=0.6, alpha_s=0.8, c_x=0.9, c_m=-0.35, inv_r0=1.7)


def run_dpm_solver_step(p, g, dev):
    n = p["n"]
    x, eps2, m_prev = (_inp(_randn((m,), g), 0) for m in (n, 2 * n, n))
    outs = {k: Out((n,), torch.float32, dev) for k in ("m_out", "x_out", "x_out2")}
    k = DPM_K
    res, same, guards = launch2(outs, lambda: L().sdb_dpm_solver_step(
        P(x), P(eps2), None, 1, k["scale"], k["sigma_s"], k["alpha_s"], 2, P(m_prev), k["c_x"], k["c_m"], k["inv_r0"],
        n, P(outs["m_out"].v), P(outs["x_out"].v), P(outs["x_out2"].v), S()), "sdb_dpm_solver_step")
    c = lambda t: t.cpu()
    xt, m0 = dpm_ref(c(x), c(eps2[:n]), c(eps2[n:]), c(m_prev), k["scale"], k["sigma_s"], k["alpha_s"], k["c_x"],
                     k["c_m"], k["inv_r0"])
    return {"exact_x": _eq(c(res["x_out"]), xt), "exact_x2": _eq(c(res["x_out2"]), xt),
            "exact_m": _eq(c(res["m_out"]), m0)}, same, guards


DDPM_K = dict(sra=1.3, srm1=0.83, c1=0.21, c2=0.77, sigma=0.11)


def run_ddpm_step(p, g, dev):
    n = p["n"]
    x, eps, noise = (_inp(_randn((n,), g), 0) for _ in range(3))
    outs = {k: Out((n,), torch.float32, dev) for k in ("x_out", "x0_out")}
    k = DDPM_K
    res, same, guards = launch2(outs, lambda: L().sdb_ddpm_step(
        P(x), P(eps), P(noise), k["sra"], k["srm1"], k["c1"], k["c2"], k["sigma"], n, P(outs["x_out"].v),
        P(outs["x0_out"].v), S()), "sdb_ddpm_step")
    c = lambda t: t.cpu()
    xo, x0 = ddpm_ref(c(x), c(eps), c(noise), k["sra"], k["srm1"], k["c1"], k["c2"], k["sigma"])
    return {"exact_x": _eq(c(res["x_out"]), xo), "exact_x0": _eq(c(res["x0_out"]), x0)}, same, guards


def run_mask_blend(p, g, dev):
    nb, c, hw = p["nb"], p["c"], p["hw"]
    orig = _inp(_randn((nb, c, hw), g), 0)
    mask = _inp(torch.rand(nb, 1, hw, generator=g, device=dev).round(), 0)
    mask.view(-1)[::7] = 0.375                                       # soft values too
    img0 = _randn((nb, c, hw), g)
    outs = {"img": Out((nb, c, hw), torch.float32, dev), "img2": Out((nb, c, hw), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_mask_blend(P(orig), P(mask), 1, nb, c, hw, P(outs["img"].v),
                                                                 P(outs["img2"].v), S()), "sdb_mask_blend",
                                before=lambda: outs["img"].v.copy_(img0))
    m = mask.cpu()
    ref = orig.cpu() * m + (f32(1.0) - m) * img0.cpu()
    return {"exact": _eq(res["img"].cpu(), ref), "exact_dup": _eq(res["img2"].cpu(), ref)}, same, guards


def vq_operands(p, g):
    """(z, codebook, zv = fl(scale z)) of a vq_quantize problem on g's device: zv and the codes N(0, 1), with two
    planted decisions. Code n_e - 1 equals zv of row 0 (distance 0; when n_e % 1024 == 1 it is the only code of the
    last chunk). When n_e > 1025 and m > 1, codes 1023 and 1024 both equal zv of row m - 1: an exact tie across a chunk
    boundary, which the lower index must win."""
    m, n_e = p["m"], p["n_e"]
    s = f32(p["scale"]).to(g.device)
    z = _randn((m, p["e_dim"]), g) / s
    zv = z * s
    cb = _randn((n_e, p["e_dim"]), g)
    cb[n_e - 1] = zv[0]
    if n_e > VQ_CHUNK + 1 and m > 1:
        cb[VQ_CHUNK - 1] = zv[m - 1]
        cb[VQ_CHUNK] = zv[m - 1]
    return z, cb, zv


def vq_check(zv, cb, idx, zq):
    """The vq_quantize checks of the module docstring for the indices idx and the output zq of zv = fl(scale z)."""
    m, D = zv.shape
    n_e = cb.shape[0]
    r = {"idx_range": bool(((idx >= 0) & (idx < n_e)).all())}
    if not r["idx_range"]:
        return r
    r["exact_zq"] = _eq(zq, zv + (cb[idx] - zv))
    zd, ed = zv.double(), cb.double()
    e2 = (ed * ed).sum(1)
    best = torch.empty(m, dtype=torch.int64, device=zv.device)     # the fp64 argmin, in chunks of <= 2^25 distances
    step = max(1, (1 << 25) // n_e)
    for r0 in range(0, m, step):
        zc = zd[r0:r0 + step]
        best[r0:r0 + step] = ((zc * zc).sum(1, keepdim=True) + e2[None] - 2 * zc @ ed.t()).argmin(1)
    dist = lambda j: ((zd - ed[j]) ** 2).sum(1)
    amag = lambda j: ((zd.abs() + ed[j].abs()) ** 2).sum(1)
    r["vq_decision"] = _share((dist(idx) - dist(best)).clamp_min(0), (D + 3) * U * (amag(idx) + amag(best)))
    _, inv = torch.unique(cb, dim=0, return_inverse=True)
    first = torch.full((int(inv.max()) + 1,), n_e, device=cb.device).scatter_reduce(
        0, inv, torch.arange(n_e, device=cb.device), "amin")                 # lowest index of each distinct code
    r["lowest_of_equal"] = bool((first[inv[idx]] == idx).all())
    return r


def run_vq_quantize(p, g, dev):
    m, D, n_e = p["m"], p["e_dim"], p["n_e"]
    z, cb, zv = vq_operands(p, g)
    z, cb = _inp(z, p["az"]), _inp(cb, p["ae"])
    code_sq = _inp((cb.double() ** 2).sum(1).float(), p["asq"])                # as VQModel.pack_weights
    outs = {"zq": Out((m, D), torch.float32, dev, p["aq"])}
    if p["idx"]:
        outs["idx"] = Out((m,), torch.int64, dev)
    launch = lambda zq, idx: L().sdb_vq_quantize(P(z), m, D, p["scale"], P(cb), P(code_sq), n_e, P(zq), P(idx), S())
    res, same, guards = launch2(outs, lambda: launch(outs["zq"].v, outs["idx"].v if p["idx"] else None),
                                "sdb_vq_quantize")
    if p["idx"]:
        return vq_check(zv, cb, res["idx"], res["zq"]), same, guards
    zq, idx = torch.empty_like(zv), torch.empty(m, dtype=torch.int64, device=dev)   # the same launch with indices
    _l.check(launch(zq, idx), "sdb_vq_quantize")
    torch.cuda.synchronize()
    r = vq_check(zv, cb, idx, zq)
    r["same_as_indexed"] = _eq(res["zq"], zq)
    return r, same, guards


RUN ={k[4:]: v for k, v in globals().items() if k.startswith("run_")}


# ------------------------------------------------------------------------------------------------ the sweep
class Sweep(Tally):
    def __init__(self, title):
        super().__init__(title)
        self.calib, self.sms = {}, _l.load().sdb_sm_count()

    def run(self, p, seed):
        dev = torch.device("cuda", torch.cuda.current_device())
        g = torch.Generator(device=dev).manual_seed(seed)
        lab = label(p)
        try:
            r, same, guards = RUN[p["op"]](p, g, dev)
        except Exception as e:  # noqa: BLE001 - a fault must name its problem
            raise RuntimeError(f"{lab}: {e}") from e
        self.launches += 2
        if not same:
            self.failures.append((lab, "bit-reproducible", "second launch differs"))
        if not guards:
            self.failures.append((lab, "guards", "written"))
        for k, val in r.items():
            if isinstance(val, bool):
                if not val:
                    self.failures.append((lab, k, "False"))
            elif not val <= 1.0:
                self.failures.append((lab, k, f"{val:.3e}"))
            else:
                self.calib[k] = max(self.calib.get(k, 0.0), val)
        for c in classes(p, self.sms):
            COVER[c] += 1

    def calibration(self):
        return "largest share of each bound used: " + (", ".join(f"{k} {v:.3f}" for k, v in sorted(self.calib.items()))
                                                       or "none (every check exact)")


def run_sweep(problems, title):
    sw = Sweep(title)
    for i, p in enumerate(problems):
        sw.run(p, 1000 + i)
    sw.finish(len(problems), sw.calibration())


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(ELEMENTWISE_WORKLOADS))
def test_every_elementwise_launch_of_every_model(cuda_dev, name):
    calls, problems = record(ELEMENTWISE_WORKLOADS[name], cuda_dev, SIGS)
    ops_ = defaultdict(int)
    for p in problems:
        ops_[p["op"]] += 1
    print(f"\n{name}: {calls} calls, {len(problems)} distinct problems ({dict(ops_)})")
    assert problems
    run_sweep(problems, name)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ synthetic grid
def _p(op, **kw):
    base = {"nchw_to_nhwc": dict(f32=True, f16=False, ax=0), "nhwc_to_nchw": dict(ax=0, ao=0),
            "transpose_f16": dict(ax=0, ao=0), "im2col3x3": dict(ax=0), "upsample2x": dict(ax=0),
            "resample_f32": dict(ax=0), "cast_f16": dict(ax=0), "silu_f16": dict(ax=0),
            "timestep_embedding_f32": dict(max_period=10000.0, ax=0), "timestep_embedding": dict(max_period=10000.0, ax=0),
            "embed_tokens": dict(ai=0, at=0, ap=0), "vit_embed": dict(ax=0, ac=0, ap=0), "rows_gather": dict(ax=0),
            "rows_pool": dict(ax=0), "linear_small": dict(bias=True, act=0, f16=False, ax=0, aw=0, ab=0, ao=0),
            "pointwise_small": dict(alpha=1.0, bias=True, ax=0, aw=0, ab=0), "vae_sample": dict(ax=0, an=0),
            "to_uint8": dict(ax=0), "axpby": dict(ax=0, ao=0),
            "vq_quantize": dict(scale=1.0, idx=True, az=0, aq=0, ae=0, asq=0)}.get(op, {})
    return dict(dict(op=op, **base), **kw)


def wrap_grid(sms):
    """Every capped grid-stride kernel at a size one grid past its cap, so the stride loop runs more than once."""
    cap = grid_threads(sms)
    n = 2 * cap + 37
    side = math.isqrt(2 * cap // 64) + 2
    ps = [_p("im2col3x3", nb=1, h=side, w=side, c=4, stride=1, pad_lo=1, ho=side, wo=side, kpad=64),
          _p("upsample2x", nb=1, h=3, w=cap // 6 + 5, c=4),
          _p("resample_f32", nb=1, h=3, w=cap // 6 + 5, c=4, mode=2),
          _p("resample_f32", nb=1, h=2 * 4, w=2 * (cap // 2 + 3), c=4, mode=1),
          _p("cast_f16", n=n), _p("silu_f16", n=n), _p("to_uint8", n=n), _p("axpby", n=n, a=1.0, b=0.0),
          _p("axpby", n=n, a=1.5, b=-0.25), _p("axpby2", n=n, a=0.7, b=-1.3),
          _p("sampler_step", n=n), _p("dpm_solver_step", n=n), _p("ddpm_step", n=n),
          _p("mask_blend", nb=1, c=4, hw=cap // 2 + 11, n=4 * (cap // 2 + 11)),
          _p("timestep_embedding", n=2 * cap // 160 + 3, dim=320),
          _p("vae_sample", nb=1, hw=cap // 2 + 5, scale=0.18215, noise=True),
          _p("pointwise_small", npix=cap // 2 + 3, cin=4, cout=4),
          _p("embed_tokens", B=2 * cap // (64 * 77) + 1, n=77, dim=64, vocab=1000, npos=77),
          _p("vit_embed", nb=2 * cap // (16 * 257) + 1, np=256, dim=64),
          _p("rows_gather", rows=2 * cap // 1024 + 3, stride=3, dim=1024, xrows=3 * (2 * cap // 1024 + 2) + 1)]
    return ps


def edge_grid():
    ps = []
    # transposes with C and HW not multiples of 32
    for f32_, f16_ in ((True, False), (False, True), (True, True)):
        ps.append(_p("nchw_to_nhwc", nb=2, c=37, h=5, w=13, f32=f32_, f16=f16_))
    ps += [_p("nhwc_to_nchw", nb=2, c=37, h=5, w=13), _p("nhwc_to_nchw", nb=1, c=70, h=3, w=33, ao=2),
           _p("transpose_f16", B=3, rows=45, cols=70, ldx=77, ldo=64),
           _p("transpose_f16", B=2, rows=77, cols=33, ldx=40, ldo=96)]
    # im2col: every (stride, pad_lo) pair a conv can take, odd sizes
    ps += [_p("im2col3x3", nb=2, h=7, w=10, c=12, stride=1, pad_lo=1, ho=7, wo=10, kpad=128),
           _p("im2col3x3", nb=2, h=8, w=10, c=12, stride=2, pad_lo=0, ho=4, wo=5, kpad=128),
           _p("im2col3x3", nb=2, h=7, w=10, c=12, stride=2, pad_lo=1, ho=4, wo=5, kpad=128)]
    # linear_small: passes of 8 rows, a k-sweep where only lane 0 has a u step (K = 264), K at the shared-memory
    # limit, N tails, no bias, SiLU and fp16 out
    kmax = LS_SMEM_FLOATS // LS_ROWS
    for M in (1, 7, 8, 9, 64, 129):
        ps.append(_p("linear_small", M=M, K=320, N=37, act=ACT_SILU if M % 2 else 0, f16=M > 8))
    ps += [_p("linear_small", M=9, K=264, N=70), _p("linear_small", M=8, K=kmax, N=33, f16=True),
           _p("linear_small", M=9, K=kmax, N=31, act=ACT_SILU), _p("linear_small", M=3, K=1280, N=1),
           _p("linear_small", M=17, K=128, N=33, bias=False), _p("linear_small", M=2, K=64, N=31, bias=False, f16=True)]
    # embed_tokens at ids 0 and vocab - 1 (every operand does), a one-row context, a position table longer than n
    ps += [_p("embed_tokens", B=3, n=77, dim=64, vocab=1000, npos=77), _p("embed_tokens", B=1001, n=1, dim=512,
                                                                          vocab=1001, npos=1),
           _p("embed_tokens", B=2, n=13, dim=128, vocab=1000, npos=77)]
    ps += [_p("pointwise_small", npix=1000, cin=32, cout=32), _p("pointwise_small", npix=777, cin=3, cout=8,
                                                                 alpha=1 / 0.18215, bias=False)]
    ps += [_p("resample_f32", nb=2, h=7, w=10, c=12, mode=2), _p("resample_f32", nb=2, h=6, w=10, c=12, mode=1),
           _p("upsample2x", nb=2, h=7, w=10, c=4)]
    ps += [_p("timestep_embedding_f32", n=5, dim=d, t=[0.0, 0.5, 1.0, 500.5, 999.0]) for d in (2, 320, 1280)]
    ps += [_p("timestep_embedding", n=5, dim=d, t=[0.0, 0.5, 1.0, 500.5, 999.0]) for d in (2, 320)]
    ps += [_p("silu_f16", n=4099)]
    ps += [_p("vae_sample", nb=2, hw=77, scale=0.18215, noise=False), _p("vae_sample", nb=1, hw=64, scale=-2.0,
                                                                         noise=True, an=3)]
    for ids in (True, False):
        for norm in (True, False):
            ps.append(_p("rows_pool", b=5, n_ctx=77 if ids else 0, dim=768, ids=ids, normalize=norm))
    ps += [_p("rows_pool", b=3, n_ctx=1, dim=64, ids=True, normalize=False)]
    ps += [_p("rows_gather", rows=5, stride=257, dim=1024, xrows=4 * 257 + 1), _p("vit_embed", nb=3, np=7, dim=12)]
    ps += [_p("to_uint8", n=3 * 17 * 13), _p("axpby", n=1000, a=1.0, b=0.0, ax=1, ao=3)]
    # the wide 1x1 heads (KL-f32: 128 -> 128, 64 -> 64): past 32 channels in, out or both, with and without bias
    for cin in (33, 64, 127, 128):
        for cout in (33, 64, 127, 128):
            for bias in (True, False):
                ps.append(_p("pointwise_small", npix=257, cin=cin, cout=cout, bias=bias,
                             alpha=1 / 0.18215 if bias else -0.5, ax=cin % 4, aw=cout % 4, ab=1))
    ps += [_p("pointwise_small", npix=300, cin=4, cout=128), _p("pointwise_small", npix=300, cin=128, cout=3,
                                                                bias=False, alpha=1.3)]
    return ps


def vq_grid():
    """vq_quantize at every compiled e_dim; codebooks of one code, of one chunk, one code short of and past a chunk
    (1025: a last chunk of one code), two chunks and one code (2049) and VQ-f16's 16384; 1 pixel, one short of a block,
    one block (VQ-f16's 16² latent) and one past it; indices on and off; scale 1 and not; operands off 16-byte
    boundaries. vq_operands plants a code at distance 0 and, past 1025 codes, an exact tie across a chunk boundary."""
    ps = []
    for D in range(1, 9):
        for n_e in (1, 256, 1023, 1024, 1025, 2049, 16384):
            for m, idx in ((1, True), (255, True), (256, True), (257, True), (257, False)):
                ps.append(_p("vq_quantize", m=m, e_dim=D, n_e=n_e, scale=1.0 if (m + D) % 2 else 1.3, idx=idx,
                             az=D % 4, aq=m % 4, ae=n_e % 4, asq=(m + D) % 4))
    return ps


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_elementwise_synthetic_grid(cuda_dev):
    sms = _l.load().sdb_sm_count()
    run_sweep(wrap_grid(sms) + edge_grid() + vq_grid(), "synthetic")


@pytest.mark.gpu
def test_elementwise_branch_coverage():
    """Every class of REQUIRED was launched by the sweeps above."""
    check_coverage(COVER, REQUIRED, "elementwise")


# ------------------------------------------------------------------------------------------------ host guards
def _at(shape, k, dev, dtype=torch.float32):
    """A contiguous view k elements into its allocation."""
    return torch.randn(math.prod(shape) + k, device=dev).to(dtype)[k:].view(shape)


@pytest.mark.gpu
def test_vector_kernels_reject_misaligned_pointers(cuda_dev):
    """sdb_upsample2x reads x as float4 and writes out as 8-byte pieces; sdb_resample_f32 reads and writes float4. A
    pointer they cannot address so is an error returned before anything launches."""
    lib, before = _l.load(), _l.load().sdb_launch_count()
    x = torch.randn(2, 4, 6, 8, device=cuda_dev)
    for k in (1, 2):
        with pytest.raises(RuntimeError, match="aligned"):
            ops.upsample2x(_at((2, 4, 6, 8), k, cuda_dev))
        with pytest.raises(RuntimeError, match="aligned"):
            ops.resample_f32(_at((2, 4, 6, 8), k, cuda_dev), 1)
        with pytest.raises(RuntimeError, match="aligned"):
            ops.resample_f32(_at((2, 4, 6, 8), k, cuda_dev), 2)
    o16 = torch.empty(2 * 8 * 12 * 8 + 2, dtype=torch.float16, device=cuda_dev)
    for k in (1, 2):                                     # 2 and 4 bytes into an 8-byte piece
        assert lib.sdb_upsample2x(P(x), 2, 4, 6, 8, P(o16[k:]), S()) != 0
        assert b"aligned" in lib.sdb_last_error()
    o32 = torch.empty(2 * 8 * 12 * 8 + 3, device=cuda_dev)
    for k in (1, 2, 3):
        assert lib.sdb_resample_f32(P(x), 2, 4, 6, 8, 2, P(o32[k:]), S()) != 0
        assert b"aligned" in lib.sdb_last_error()
    assert lib.sdb_launch_count() == before
    assert lib.sdb_upsample2x(P(x), 2, 4, 6, 8, P(o16), S()) == 0     # aligned: accepted
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_token_embedding_rejects_what_it_cannot_read(cuda_dev):
    """embed_tokens needs a position row of the same width per token. FrozenCLIPEmbedder and the projected variant
    check ids before any launch, as BERTEmbedder does: shape, type and length always, the id range of host ids (GPU ids
    are not read back; the kernel clamps them)."""
    import sdb200
    from sdb200 import arch
    tok, pos = torch.randn(100, 64, device=cuda_dev), torch.randn(77, 64, device=cuda_dev)
    ids = torch.zeros(2, 78, dtype=torch.int64, device=cuda_dev)
    with pytest.raises(AssertionError):
        ops.embed_tokens(ids, tok, pos)
    with pytest.raises(AssertionError):
        ops.embed_tokens(ids[:, :77].contiguous(), tok, pos[:, :32].contiguous())
    for cls, cfg, shapes in ((sdb200.FrozenCLIPEmbedder, arch.TINY_CLIP, arch.clip_param_shapes),
                             (sdb200.FrozenCLIPTextEmbedder, arch.TINY_CLIP_TEXT_PROJ, arch.clip_text_proj_param_shapes)):
        enc = cls(config=cfg).load_weights(arch.random_state_dict(shapes(cfg), 13, device=cuda_dev), cuda_dev)
        v = cfg["vocab_size"]
        ok = torch.randint(0, v, (2, 77), generator=torch.Generator().manual_seed(1))
        torch.cuda.synchronize()
        before = ops.launch_count()
        for dev in ("cpu", cuda_dev):
            with pytest.raises(ValueError):
                enc.encode_ids(torch.zeros(2, 78, dtype=torch.int64, device=dev))
            with pytest.raises(ValueError):
                enc.encode_ids(torch.zeros(2, 0, dtype=torch.int64, device=dev))
            with pytest.raises(TypeError):
                enc.encode_ids(ok.float().to(dev))
            with pytest.raises(TypeError):
                enc.encode_ids(ok[0].to(dev))
        for bad in (v, -1):
            b = ok.clone()
            b[1, 5] = bad
            with pytest.raises(IndexError):
                enc.encode_ids(b)
            with pytest.raises(IndexError):
                enc(b)
        assert ops.launch_count() == before
        ref = enc.encode_ids(ok.to(cuda_dev))
        for same in (enc.encode_ids(ok), enc.encode_ids(ok.int().to(cuda_dev)), enc(ok)):
            torch.cuda.synchronize()
            assert torch.equal(same, ref)                # host ids and int32 ids take the path of int64 GPU ids


# ------------------------------------------------------------------------------------------------ entry-point map
HERE = os.path.basename(__file__)

# kernel-launching C entry point -> the test files that check what it computes elementwise or bit for bit
ENTRY_POINT_TESTS = {
    "sdb_gemm": ("test_gemm_plans_gpu.py",),
    "sdb_attention": ("test_attention_sweep_gpu.py",),
    "sdb_groupnorm": ("test_norm_sweep_gpu.py",),
    "sdb_groupnorm_mod": ("test_norm_sweep_gpu.py",),
    "sdb_layernorm": ("test_norm_sweep_gpu.py",),
    "sdb_softmax_rows": ("test_norm_sweep_gpu.py",),
    "sdb_resample_f32": (HERE, "test_uncond_ldm_gpu.py"),
    "sdb_ddpm_step": (HERE, "test_uncond_ldm_gpu.py"),
    "sdb_vq_quantize": (HERE, "test_vq_ldm_gpu.py"),
    "sdb_nchw_to_nhwc": (HERE,),
    "sdb_nhwc_to_nchw": (HERE,),
    "sdb_im2col3x3": (HERE,),
    "sdb_im2col3x3_concat": ("test_inpaint_gpu.py",),
    "sdb_upsample2x": (HERE,),
    "sdb_cast_f16": (HERE,),
    "sdb_transpose_f16": (HERE,),
    "sdb_timestep_embedding": (HERE,),
    "sdb_timestep_embedding_f32": (HERE,),
    "sdb_linear_small": (HERE, "test_gemm_plans_gpu.py"),
    "sdb_silu_f16": (HERE,),
    "sdb_sampler_step": (HERE, "test_pipeline_gpu.py"),
    "sdb_vae_sample": (HERE,),
    "sdb_to_uint8": (HERE,),
    "sdb_axpby": (HERE,),
    "sdb_pointwise_small": (HERE, "test_gemm_plans_gpu.py"),
    "sdb_embed_tokens": (HERE,),
    "sdb_dpm_solver_step": (HERE, "test_samplers_ext_gpu.py"),
    "sdb_mask_blend": (HERE, "test_samplers_ext_gpu.py"),
    "sdb_axpby2": (HERE,),
    "sdb_inpaint_prepare": ("test_inpaint_gpu.py",),
    "sdb_inpaint_composite": ("test_inpaint_gpu.py",),
    "sdb_lr_prepare": ("test_superres_gpu.py",),
    "sdb_patch_unfold": ("test_superres_gpu.py",),
    "sdb_patch_fold": ("test_superres_gpu.py",),
    "sdb_spatial_rescale": ("test_semantic_gpu.py",),
    "sdb_seg_labels_rescale": ("test_semantic_gpu.py",),
    "sdb_knn_topk": ("test_rdm_gpu.py",),
    "sdb_rows_pool": (HERE,),
    "sdb_clip_resize_patches": ("test_clip_image_gpu.py",),
    "sdb_vit_embed": (HERE,),
    "sdb_rows_gather": (HERE,),
    "sdb_resample_u8": ("test_safety_gpu.py",),
    "sdb_clip_normalize": ("test_safety_gpu.py",),
    "sdb_patchify": ("test_safety_gpu.py",),
    "sdb_safety_scores": ("test_safety_gpu.py",),
    "sdb_blank_flagged": ("test_safety_gpu.py",),
    "sdb_watermark_dwtdct": ("test_safety_gpu.py",),
    "sdb_fill_f32": ("test_handle_gpu.py",),
    "sdb_sample_plms": ("test_handle_gpu.py",),
    # evaluation (include/sdb200_eval.h, include/sdb200_ae_loss.h)
    "sdb_q_sample_t": ("test_losses_gpu.py",),
    "sdb_diffusion_loss": ("test_losses_gpu.py",),
    "sdb_lpips_scale": ("test_ae_loss_sweep_gpu.py", "test_ae_loss_gpu.py"),
    "sdb_maxpool2x2": ("test_ae_loss_sweep_gpu.py", "test_ae_loss_gpu.py"),
    "sdb_lpips_head": ("test_ae_loss_sweep_gpu.py", "test_ae_loss_gpu.py"),
    "sdb_im2col": ("test_ae_loss_sweep_gpu.py", "test_ae_loss_gpu.py"),
    "sdb_ae_loss_terms": ("test_ae_loss_sweep_gpu.py", "test_ae_loss_gpu.py"),
}
# entry points whose Python caller is not ops.<name without sdb_>: the call a test file makes to reach them
CALLED_AS = {
    "sdb_sampler_step": ("PLMSSampler",),
    "sdb_dpm_solver_step": ("DPMSolverSampler",),
    "sdb_resample_u8": ("CLIPImagePreprocessor",),
    "sdb_clip_normalize": ("CLIPImagePreprocessor",),
    "sdb_patchify": ("image_embeds",),
    "sdb_safety_scores": ("forward",),
    "sdb_blank_flagged": ("forward",),
    "sdb_watermark_dwtdct": ("put_watermark",),
    "sdb_fill_f32": ("sample_plms",),            # writes the timestep of each UNet evaluation of sdb_sample_plms
    "sdb_sample_plms": ("sample_plms",),
}
HOST_ONLY = ("sdb_last_error", "sdb_version", "sdb_sm_count", "sdb_launch_count", "sdb_debug_trace", "sdb_knn_workspace",
             "sdb_gemm_plan", "sdb_plan_begin", "sdb_plan_end", "sdb_plan_size", "sdb_plan_run", "sdb_plan_launch",
             "sdb_plan_destroy", "sdb_unet_create", "sdb_unet_forward", "sdb_unet_destroy", "sdb_lpips_head_work")
ALL_SIGNATURES = {**_l.SIGNATURES, **_l.EVAL_SIGNATURES, **_l.AE_LOSS_SIGNATURES}


def _calls(src, sym):
    """Whether source text calls entry point sym: directly (lib.sdb_x(...)), through ops.x(...), or as CALLED_AS."""
    names = [re.escape(sym), r"ops\." + re.escape(sym[4:])] + [re.escape(n) for n in CALLED_AS.get(sym, ())]
    return re.search(r"\b(?:%s)\s*\(" % "|".join(names), src) is not None


def test_every_entry_point_maps_to_its_tests():
    assert set(ENTRY_POINT_TESTS).isdisjoint(HOST_ONLY)
    assert set(ENTRY_POINT_TESTS) | set(HOST_ONLY) == set(ALL_SIGNATURES), (
        "unmapped: " + str(sorted(set(ALL_SIGNATURES) - set(ENTRY_POINT_TESTS) - set(HOST_ONLY)))
        + ", in no signature table: " + str(sorted((set(ENTRY_POINT_TESTS) | set(HOST_ONLY)) - set(ALL_SIGNATURES))))
    here = os.path.dirname(os.path.abspath(__file__))
    missing, silent = [], []
    for sym, files in ENTRY_POINT_TESTS.items():
        assert files, sym
        for f in files:
            path = os.path.join(here, f)
            if not os.path.isfile(path):
                missing.append((sym, f))
                continue
            with open(path) as fh:
                if not _calls(fh.read(), sym):
                    silent.append((sym, f))
    assert not missing, missing
    assert not silent, silent


def test_sweep_calls_each_entry_point_it_claims_cpu():
    """Every entry point mapped to this file has a launch here through ctypes (lib.sdb_x(...))."""
    with open(os.path.abspath(__file__)) as fh:
        src = fh.read()
    for sym, files in ENTRY_POINT_TESTS.items():
        if HERE in files:
            assert re.search(r"L\(\)\.%s\(" % re.escape(sym), src), sym


# ------------------------------------------------------------------------------------------------ CPU: the harness
def test_references_cpu():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 7, 10, 5, generator=g)
    wt = torch.randn(3, 5, 3, 3, generator=g).half().float()
    for stride, pad_lo, ho, wo in ((1, 1, 7, 10), (2, 0, 3, 4), (2, 1, 4, 5)):
        col = im2col_ref(x, stride, pad_lo, ho, wo, 64)
        assert col.shape == (2 * ho * wo, 64) and bool((col[:, 45:] == 0).all())
        wm = wt.permute(0, 2, 3, 1).reshape(3, 45)                    # [n, (ky, kx, c)]
        y = (col[:, :45].float() @ wm.t()).view(2, ho, wo, 3)
        xp = F.pad(x.half().float().permute(0, 3, 1, 2), (pad_lo, 3, pad_lo, 3))
        ref = F.conv2d(xp, wt, stride=stride)[:, :, :ho, :wo].permute(0, 2, 3, 1)
        assert torch.allclose(y, ref, atol=1e-4)
    xs = torch.randn(2, 6, 10, 4, generator=g)
    assert torch.allclose(pool_ref(xs).permute(0, 3, 1, 2), F.avg_pool2d(xs.permute(0, 3, 1, 2), 2), atol=1e-7)
    e = to_uint8_edges()
    u = to_uint8_ref(e)
    assert int(u[255]) == 255 and int(u[0]) == 0 and int(u[256]) == 0   # -1 + ulp stays 0
    assert int(u[-1]) == int(u[-2]) == 127 and int(u[-3]) == 0 and int(u[-4]) == 255
    assert (u[:256].int() - torch.arange(256)).abs().max() <= 1
    ids = torch.tensor([[3, 9, 9, 1], [9, 0, 0, 9], [1, 2, 3, 4]])
    assert first_max(ids).tolist() == [1, 0, 3] and first_max(ids).tolist() == ids.argmax(1).tolist()
    t = torch.tensor([0.0, 999.0])
    ref, b = timestep_ref(t, 320, 10000.0)
    assert torch.allclose(ref[0], torch.cat([torch.ones(160), torch.zeros(160)]).double())
    assert float(b.max()) < 1e-3 and float(b.min()) > 0


def test_signatures_and_classes_cpu():
    x = torch.zeros(2, 8, 6, 320)
    w = torch.zeros(1280, 320, dtype=torch.float16)
    p = _linear_small_sig(torch.zeros(9, 320), w, torch.zeros(1280), act=ACT_SILU)
    assert (p["M"], p["K"], p["N"], p["bias"], p["act"]) == (9, 320, 1280, True, ACT_SILU)
    assert classes(p, 132) >= {"ls:passes", "ls:bias", "ls:silu", "ls:partial_u"} and "ls:n_tail" not in classes(p, 132)
    assert "ls:partial_u" in classes(_p("linear_small", M=1, K=264, N=31), 132)
    assert "ls:partial_u" not in classes(_p("linear_small", M=1, K=512, N=32), 132)
    assert signature(_resample_f32_sig(x, 1)) != signature(_resample_f32_sig(x, 2))
    assert _rows_pool_sig(torch.zeros(154, 768), torch.zeros(2, 77, dtype=torch.int64))["b"] == 2
    assert _embed_tokens_sig(torch.zeros(3, 1, dtype=torch.int64), torch.zeros(1001, 512), torch.zeros(1, 512))["npos"] == 1
    cap = grid_threads(132)
    for q in wrap_grid(132):
        assert work_items(q) > cap, q
    assert {f"wrap:{q['op']}" for q in wrap_grid(132)} == {f"wrap:{op}" for op in GRID_STRIDE_OPS}
    assert set(RUN) >= {q["op"] for q in wrap_grid(132) + edge_grid()} and set(RUN) >= set(SIGS)


def test_vq_and_pointwise_signatures_and_classes_cpu():
    book = torch.zeros(16384, 8)
    p = _vq_quantize_sig(torch.zeros(1, 16, 16, 8), book, torch.zeros(16384), scale=1.3, want_indices=True)
    assert (p["m"], p["e_dim"], p["n_e"], p["scale"], p["idx"]) == (256, 8, 16384, 1.3, True)
    assert classes(p, 132) == {"vq_quantize", "vq:e8", "vq:multi_chunk"}               # VQ-f16 at 256²
    assert signature(p) != signature(_vq_quantize_sig(torch.zeros(1, 16, 16, 8), book, torch.zeros(16384), 1.3))
    q = _vq_quantize_sig(torch.zeros(2, 8, 12, 4), torch.zeros(256, 4), torch.zeros(256))
    assert classes(q, 132) == {"vq_quantize", "vq:e4", "vq:tail_block", "vq:no_indices"}  # VQ-f8-n256, 64x96, batch 2
    assert "vq:partial_chunk" in classes(_p("vq_quantize", m=1, e_dim=1, n_e=1025), 132)
    assert not classes(_p("vq_quantize", m=256, e_dim=3, n_e=1023), 132) & {"vq:partial_chunk", "vq:multi_chunk"}
    w = _pointwise_small_sig(torch.zeros(2, 4, 4, 128), torch.zeros(128, 128), torch.zeros(128), alpha=1.3)
    assert (w["npix"], w["cin"], w["cout"], w["alpha"]) == (32, 128, 128, 1.3)
    assert classes(w, 132) >= {"pw:wide_in", "pw:wide_out"}
    assert classes(_pointwise_small_sig(torch.zeros(10, 32), torch.zeros(32, 32)), 132) == {"pointwise_small"}
    assert classes(_p("pointwise_small", npix=9, cin=4, cout=64), 132) == {"pointwise_small", "pw:wide_out"}
    grid = {c for q in edge_grid() + vq_grid() for c in classes(q, 132)}
    assert {c for c in REQUIRED if c.startswith(("vq:", "pw:"))} <= grid
    assert {c for c in REQUIRED if c.startswith(("vq:", "pw:"))} == {f"vq:e{d}" for d in range(1, 9)} | {
        "vq:multi_chunk", "vq:partial_chunk", "vq:tail_block", "vq:no_indices", "pw:wide_in", "pw:wide_out"}


@pytest.mark.parametrize("n_e", [1025, 2049])
def test_vq_checks_cpu(n_e):
    """vq_check passes the fp64 nearest codes (lowest index first) and fails each value mutant of the kernel: the
    highest index of a tie, the last partial chunk skipped, z_q = e without the straight-through rounding, and
    distances from the unscaled z."""
    z, cb, zv = vq_operands(_p("vq_quantize", m=257, e_dim=3, n_e=n_e, scale=1.3), torch.Generator().manual_seed(5))
    nearest = lambda x, codes: torch.cdist(x.double(), codes.double()).argmin(1)       # the first of equal minima
    st = lambda i: zv + (cb[i] - zv)
    idx = nearest(zv, cb)
    assert int(idx[0]) == n_e - 1 and (n_e < 2049 or int(idx[-1]) == VQ_CHUNK - 1)
    ok = vq_check(zv, cb, idx, st(idx))
    assert ok["idx_range"] and ok["exact_zq"] and ok["lowest_of_equal"] and ok["vq_decision"] == 0.0
    if n_e == 2049:
        tie = torch.where(idx == VQ_CHUNK - 1, VQ_CHUNK, idx)
        assert not vq_check(zv, cb, tie, st(tie))["lowest_of_equal"]
    skip = nearest(zv, cb[:(n_e - 1) // VQ_CHUNK * VQ_CHUNK])
    assert vq_check(zv, cb, skip, st(skip))["vq_decision"] > 1
    assert not vq_check(zv, cb, idx, cb[idx])["exact_zq"]
    unscaled = nearest(z, cb)
    assert vq_check(zv, cb, unscaled, st(unscaled))["vq_decision"] > 1
    assert not vq_check(zv, cb, torch.full_like(idx, FILL_I64[0]), zv)["idx_range"]


def test_clip_check_ids_cpu():
    import sdb200
    from sdb200 import arch
    enc = sdb200.FrozenCLIPEmbedder(config=arch.TINY_CLIP)
    enc.check_ids(torch.zeros(2, 77, dtype=torch.int64))
    enc.check_ids(torch.full((1, 1), 999, dtype=torch.int32))
    with pytest.raises(ValueError):
        enc.check_ids(torch.zeros(1, 78, dtype=torch.int64))
    with pytest.raises(IndexError):
        enc.check_ids(torch.full((1, 3), 1000))
    with pytest.raises(IndexError):
        enc.check_ids(torch.full((1, 3), -1))
    with pytest.raises(TypeError):
        enc.check_ids(torch.zeros(2, 77))
    with pytest.raises(TypeError):
        enc.check_ids(torch.zeros(77, dtype=torch.int64))
