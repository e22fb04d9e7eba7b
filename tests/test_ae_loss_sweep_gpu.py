"""The fp64 kernel sweeps over the KL autoencoders' validation loss (workloads.AE_LOSS_WORKLOADS: both
LPIPSWithDiscriminator calls at 256² batch 4 and at 72x104 batch 2, and LPIPS at its smallest side), the edges of the
five include/sdb200_ae_loss.h kernels that no model reaches, and NaN propagation against torch. Like
test_first_stage_sweep_gpu.py, it reuses the sweeps of the other files:
  - every GEMM problem with every tile plan (test_gemm_plans_gpu.py): the VGG16 trunk's ReLU convs, conv1_1 through
    im2col, the discriminator's LeakyReLU convs and its one-logit head;
  - every layout launch (test_elementwise_sweep_gpu.py): the discriminator's nchw_to_nhwc, LPIPS's im2col3x3;
  - every operand read before griddepcontrol.wait lies in packed weights (test_pdl_order_gpu.py);
and adds one for the kernels of include/sdb200_ae_loss.h. It records the calls of ops.lpips_scale, maxpool2x2,
lpips_head, im2col and ae_loss_terms, regenerates seeded operands per problem at the recorded element offsets, and
launches through the C entry points into NaN-filled outputs with GUARD NaN elements on both sides, twice (bit equality).

References and bounds (u = 2^-24, the fp32 unit roundoff):
  bit-exact     lpips_scale (= torch fp32 (x - shift) / scale, both IEEE-rounded), im2col (= the fp16 values of F.unfold
                in (ky, kx, c) column order, the tail up to kpad +0), maxpool2x2 (= F.max_pool2d's values and NaN
                positions: a max is one of its inputs).
  lpips_head    |acc - ref| <= 2^-20 absref, as test_ae_loss_gpu.py: the normalised features and their difference
                carry a few fp32 roundings, squared and summed with non-negative weights in fp64. Checked after the
                first tap (out NULL: untouched) and after five accumulated taps (out = (float) acc).
  ae_loss_terms the exact fp64 sum of the reference's fp32 element values (torch fp32 ops in the reference's order)
                within n 2^-52 sum |v|: two fp64 sums of n terms. KL adds 8u e + 6u (m^2 + e + 1 + |lv|) per element
                (e = exp(lv)): expf and torch.exp are each within 2 ulp (4u) of exp, and a different e can flip the
                three fp32 roundings after it (2u of each partial, every one <= the abs-value sum). The two softplus
                sums add SP_REL sp per element: an implementation within 2 ulp of exp (4u, times t / (1 + t) <= sp)
                and 1 ulp of log1p (2u) is within 6u sp of softplus; kernel and torch are two of them.
The largest share of each bound used is printed per workload.
"""
import os
import sys
import time
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

import helpers
import test_elementwise_sweep_gpu as ES
import test_gemm_plans_gpu as GP
from sweeps import NAN, Tally, eoff, record
from test_ae_loss_gpu import _head_ref
from test_pdl_order_gpu import audit_workload
from workloads import AE_LOSS_WORKLOADS
import sdb200
from sdb200 import ae_loss, ops
from sdb200 import lib as _l
from sdb200.lib import ACT_LEAKY_RELU, ACT_NONE, ACT_RELU

NAMES = list(AE_LOSS_WORKLOADS)
# one H100 80GB HBM3 (700 W) runs the whole file in about 30 s, no sweep test in more than 3 s: 120 s leaves room for a
# slower card or a cold start without letting a hang run on
TIMEOUT = 120
U = 2.0 ** -24
HEAD_REL = 2.0 ** -20
SP_REL = 12 * U
KIND = ops.AE_TERM_KINDS
Out, launch2, P = ES.Out, ES.launch2, ops._ptr


def S():
    return ops._stream()


def L():
    return _l.load()


# ------------------------------------------------------------------------------------------------ signatures
def _lpips_scale_sig(in0, in1, shift, scale):
    nb, _, h, w = in0.shape
    return dict(op="lpips_scale", nb=nb, h=h, w=w, a0=eoff(in0), a1=eoff(in1))


def _maxpool2x2_sig(x):
    nb, h, w, c = x.shape
    return dict(op="maxpool2x2", nb=nb, h=h, w=w, c=c, ax=eoff(x))


def _lpips_head_sig(f, lin_w, acc, first, out=None):
    n2, h, w, c = f.shape
    # every problem runs the first tap (out NULL) and five accumulated taps (out given): first / out are not keys
    return dict(op="lpips_head", nb=n2 // 2, hw=h * w, c=c, af=eoff(f), zeros=False)


def _im2col_sig(x, k, stride, pad, kpad):
    nb, h, w, c = x.shape
    return dict(op="im2col", nb=nb, h=h, w=w, c=c, k=k, stride=stride, pad=pad, kpad=kpad, ax=eoff(x))


def _ae_loss_terms_sig(a, kind, b=None, n=None, cc=1):
    k = KIND[kind]
    if k == 1:
        nb, n = a.shape[0], a[0].numel()
    elif k == 2:
        nb, n = a.shape[0], a[0].numel() // 2
    else:
        nb = a.shape[0] // n
    return dict(op="ae_loss_terms", kind=k, nb=nb, n=n, cc=cc if k != 1 else 1, aa=eoff(a),
                ab=0 if b is None else eoff(b), plant=False)


SIGS = {"lpips_scale": _lpips_scale_sig, "maxpool2x2": _maxpool2x2_sig, "lpips_head": _lpips_head_sig,
        "im2col": _im2col_sig, "ae_loss_terms": _ae_loss_terms_sig}


def label(p):
    return p["op"] + "[" + " ".join(f"{k}={v}" for k, v in p.items() if k != "op") + "]"


# ------------------------------------------------------------------------------------------------ one problem per op
def _randn(shape, g, scale=1.0):
    return torch.randn(shape, generator=g, device=g.device) * scale


def _same_values(a, b):
    """Equal values and NaN positions (a max may pick either of +0 / -0)."""
    return (a.shape == b.shape and torch.equal(a.isnan(), b.isnan())
            and torch.equal(a.float().nan_to_num(0.0), b.float().nan_to_num(0.0)))


def _terms_share(got, ref_v, extra, n):
    """Largest |got - sum v| / (n 2^-52 sum |v| + sum extra) over the samples: ref_v, extra fp64 [nb, n]."""
    err = (got - ref_v.sum(1)).abs()
    bound = n * 2.0 ** -52 * ref_v.abs().sum(1) + extra.sum(1)
    return ES._share(err, bound)


def run_lpips_scale(p, g, dev):
    nb, h, w = p["nb"], p["h"], p["w"]
    in0 = ES._inp(torch.rand((nb, 3, h, w), generator=g, device=dev) * 2 - 1, p["a0"])
    in1 = ES._inp(_randn((nb, 3, h, w), g, 2.0), p["a1"])
    shift = torch.tensor(ae_loss.LPIPS_SHIFT, device=dev)
    scale = torch.tensor(ae_loss.LPIPS_SCALE, device=dev)
    outs = {"o": Out((2 * nb, h, w, 3), torch.float32, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_lpips_scale(P(in0), P(in1), nb, h, w, P(shift), P(scale),
                                                                  P(outs["o"].v), S()), "sdb_lpips_scale")
    x = torch.cat([in0, in1])
    ref = ((x - shift.view(1, 3, 1, 1)) / scale.view(1, 3, 1, 1)).permute(0, 2, 3, 1).contiguous()
    return {"exact": ES._eq(res["o"], ref)}, same, guards


def maxpool_operand(p, g):
    nb, h, w, c = p["nb"], p["h"], p["w"], p["c"]
    x = _randn((nb, h, w, c), g, 2.0)
    if p.get("special"):
        # window j of row pair 0 holds one NaN at position j % 4 in channel j // 4; row pair 1 holds +inf, -inf and
        # an all -inf window; the rest stays finite
        for j in range(min(4 * c, w // 2)):
            x[0, (j % 4) // 2, 2 * j + (j % 2), j // 4] = NAN
        if h >= 4:
            x[0, 2, 0, :] = float("inf")
            x[0, 3, 3, :] = float("-inf")
            x[0, 2:4, 4:6, :] = float("-inf")
    return x.half()


def run_maxpool2x2(p, g, dev):
    nb, h, w, c = p["nb"], p["h"], p["w"], p["c"]
    x = ES._inp(maxpool_operand(p, g), p["ax"])
    outs = {"o": Out((nb, h // 2, w // 2, c), torch.float16, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_maxpool2x2(P(x), nb, h, w, c, P(outs["o"].v), S()),
                                "sdb_maxpool2x2")
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 2, 2).permute(0, 2, 3, 1).half()
    r = {"exact": _same_values(res["o"], ref)}
    if p.get("special"):
        r["nan_windows"] = int(res["o"].isnan().sum()) == min(4 * c, w // 2)
    return r, same, guards


def head_features(p, g):
    """fp16 [2 nb, hw, c] non-negative features (VGG's ReLU outputs); with zeros, every third pixel of the first map
    and every fifth of the second is all zero (the 1e-10 norm path), both at pixels 0, 15, 30, ..."""
    nb, hw, c = p["nb"], p["hw"], p["c"]
    f = _randn((2 * nb, hw, c), g).abs()
    if p["zeros"]:
        f[:nb, ::3] = 0
        f[nb:, ::5] = 0
    return ES._inp(f.half(), p["af"])


def run_lpips_head(p, g, dev):
    nb, hw, c = p["nb"], p["hw"], p["c"]
    feats = [head_features(p, g) for _ in range(5)]
    lin_w = torch.rand(c, generator=g, device=dev)
    work_n = int(L().sdb_lpips_head_work(nb, hw))
    assert work_n == nb * ((hw + 255) // 256)
    outs = {"acc": Out((nb,), torch.float64, dev), "out": Out((nb,), torch.float32, dev),
            "work": Out((work_n,), torch.float64, dev)}

    def taps(k):
        def call():
            for t in range(k):
                rc = L().sdb_lpips_head(P(feats[t]), nb, hw, c, P(lin_w), int(t == 0), P(outs["work"].v),
                                        P(outs["acc"].v), P(outs["out"].v) if t == 4 else None, S())
                if rc:
                    return rc
            return 0
        return call

    refs = [_head_ref(f.view(2 * nb, hw, 1, c), lin_w, nb) for f in feats]
    one, same1, guards1 = launch2(outs, taps(1), "sdb_lpips_head")
    five, same5, guards5 = launch2(outs, taps(5), "sdb_lpips_head")
    ref5 = sum(r[0] for r in refs)
    abs5 = sum(r[1] for r in refs)
    r = {"head_first": ES._share((one["acc"] - refs[0][0]).abs(), HEAD_REL * refs[0][1]),
         "out_null_untouched": bool(one["out"].isnan().all()),
         "head_5_taps": ES._share((five["acc"] - ref5).abs(), HEAD_REL * abs5),
         "out_is_acc": torch.equal(five["out"], five["acc"].float()),
         "finite": bool(torch.isfinite(five["acc"]).all())}
    return r, same1 and same5, guards1 and guards5


def im2col_ref(x, k, stride, pad, kpad):
    nb, h, w, c = x.shape
    u = F.unfold(x.float().permute(0, 3, 1, 2), k, padding=pad, stride=stride)        # [nb, c*k*k, L], (c, ky, kx)
    L_ = u.shape[-1]
    u = u.view(nb, c, k * k, L_).permute(0, 3, 2, 1).reshape(nb * L_, k * k * c)
    return F.pad(u, (0, kpad - k * k * c)).half()


def run_im2col(p, g, dev):
    nb, h, w, c, k, s, pad, kpad = (p[q] for q in ("nb", "h", "w", "c", "k", "stride", "pad", "kpad"))
    ho, wo = (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1
    x = ES._inp(_randn((nb, h, w, c), g, 2.0).half(), p["ax"])
    outs = {"o": Out((nb * ho * wo, kpad), torch.float16, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_im2col(P(x), nb, h, w, c, k, s, pad, ho, wo, kpad,
                                                             P(outs["o"].v), S()), "sdb_im2col")
    return {"exact": ES._eq(res["o"], im2col_ref(x, k, s, pad, kpad))}, same, guards


def _after(v, toward):
    return torch.nextafter(torch.tensor(v, dtype=torch.float32), torch.tensor(toward, dtype=torch.float32)).item()


LOGVAR_EDGES = [-30.0, 20.0, _after(-30.0, -1e9), _after(-30.0, 0.0), _after(20.0, 1e9), _after(20.0, 0.0), -31.0,
                21.0, -1e30, 1e30, float("-inf"), float("inf")]
LOGIT_EDGES = [s * v for s in (1.0, -1.0) for v in (20.0, _after(20.0, 1e9), _after(20.0, 0.0), 1.0,
                                                    _after(1.0, 1e9), _after(1.0, 0.0), 0.0, 88.0, 100.0)]


def terms_operands(p, g):
    """(a, b) of one problem; with plant, the edge values sit at the first elements each sample reads."""
    dev = g.device
    k, nb, n, cc = p["kind"], p["nb"], p["n"], p["cc"]
    if k == 1:
        return ES._inp(_randn((nb, n), g), p["aa"]), ES._inp(_randn((nb, n), g), p["ab"])
    if k == 2:      # [nb * pixels, 2 cc]: cc means, then cc logvars per pixel
        pix = n // cc
        mu, lv = _randn((nb, pix, cc), g, 2.0), _randn((nb, pix * cc), g, 8.0)
        if p["plant"]:
            e = torch.tensor(LOGVAR_EDGES, device=dev)[: pix * cc]
            lv[:, : e.numel()] = e
        return ES._inp(torch.cat([mu, lv.view(nb, pix, cc)], 2).view(nb * pix, 2 * cc), p["aa"]), None
    a = _randn((nb * n, cc), g, 8.0)
    if p["plant"]:
        e = torch.tensor(LOGIT_EDGES, device=dev)[:n]
        a.view(nb, n, cc)[:, : e.numel(), 0] = e
    return ES._inp(a, p["aa"]), None


def terms_reference(p, a, b):
    """(element values fp64 [R, nb, n] as the reference computes them in fp32, extra tolerance fp64 [R, nb, n])."""
    k, nb, n, cc = p["kind"], p["nb"], p["n"], p["cc"]
    if k == 1:
        v = (a - b).abs().double()
        return v[None], torch.zeros_like(v)[None]
    if k == 2:
        m = a.view(nb, n // cc, 2 * cc)
        mu, lv = m[..., :cc].reshape(nb, n), torch.clamp(m[..., cc:].reshape(nb, n), -30.0, 20.0)
        e = torch.exp(lv)
        v = (mu * mu + e - 1.0 - lv).double()
        extra = 8 * U * e.double() + 6 * U * (mu.double() ** 2 + e.double() + 1 + lv.double().abs())
        return 0.5 * v[None], 0.5 * extra[None]
    lg = a.view(nb, n, cc)[..., 0]
    sp_m, sp_p = F.softplus(-lg), F.softplus(lg)
    v = torch.stack([lg, F.relu(1.0 - lg), F.relu(1.0 + lg), sp_m, sp_p]).double()
    z = torch.zeros_like(lg, dtype=torch.float64)
    extra = torch.stack([z, z, z, SP_REL * sp_m.double(), SP_REL * sp_p.double()])
    return v, extra


def run_ae_loss_terms(p, g, dev):
    k, nb, n, cc = p["kind"], p["nb"], p["n"], p["cc"]
    a, b = terms_operands(p, g)
    R = 5 if k == 3 else 1
    outs = {"o": Out((R, nb), torch.float64, dev)}
    res, same, guards = launch2(outs, lambda: L().sdb_ae_loss_terms(P(a), P(b), k, nb, n, cc, P(outs["o"].v), S()),
                                "sdb_ae_loss_terms")
    v, extra = terms_reference(p, a, b)
    r = {"finite": bool(torch.isfinite(res["o"]).all())}
    for i in range(R):
        r[f"terms{k}.{i}"] = _terms_share(res["o"][i], v[i], extra[i], n)
    return r, same, guards


RUN = {"lpips_scale": run_lpips_scale, "maxpool2x2": run_maxpool2x2, "lpips_head": run_lpips_head,
       "im2col": run_im2col, "ae_loss_terms": run_ae_loss_terms}


def run_sweep(problems, title):
    tally, calib = Tally(title), {}
    dev = torch.device("cuda", torch.cuda.current_device())
    for i, p in enumerate(problems):
        g = torch.Generator(device=dev).manual_seed(1000 + i)
        lab = label(p)
        try:
            r, same, guards = RUN[p["op"]](p, g, dev)
        except Exception as e:  # noqa: BLE001 - a fault must name its problem
            raise RuntimeError(f"{lab}: {e}") from e
        tally.launches += 2
        if not same:
            tally.failures.append((lab, "bit-reproducible", "second launch differs"))
        if not guards:
            tally.failures.append((lab, "guards", "written"))
        for k, val in r.items():
            if isinstance(val, bool):
                if not val:
                    tally.failures.append((lab, k, "False"))
            elif not val <= 1.0:
                tally.failures.append((lab, k, f"{val:.3e}"))
            else:
                calib[k] = max(calib.get(k, 0.0), val)
    tally.finish(len(problems), "largest share of each bound used: "
                 + (", ".join(f"{k} {v:.3f}" for k, v in sorted(calib.items())) or "none (every check exact)"))


# ------------------------------------------------------------------------------------------------ model workloads
@pytest.mark.gpu
@pytest.mark.timeout(TIMEOUT)
@pytest.mark.parametrize("name", NAMES)
def test_every_plan_of_every_ae_loss_gemm_problem(cuda_dev, name):
    """The VGG16 trunk's ReLU convs (conv1_1 as an im2col'd GEMM, the rest implicit 3x3), and for the full loss the
    discriminator's LeakyReLU convs and its one-logit head (padded to 32 columns, no activation, fp32 out)."""
    problems = GP.catalogue(AE_LOSS_WORKLOADS[name], cuda_dev)
    relu = [p for p in problems if p["act"] == ACT_RELU]
    assert any(p["taps"] == 1 and p["chans"] == (64,) and p["n"] == 64 for p in relu), "conv1_1 through im2col"
    assert any(p["taps"] == 9 and p["chans"] == (512,) for p in relu)
    if name != "lpips_min_side":
        lrelu = [p for p in problems if p["act"] == ACT_LEAKY_RELU]
        assert {p["n"] for p in lrelu} == {64, 128, 256, 512}, lrelu
        assert any(p["act"] == ACT_NONE and p["n"] == 32 and p["chans"] == (16 * 512,) and p["f32"] for p in problems)
    print(f"\n{name}: {len(problems)} distinct GEMM problems")
    GP.run_sweep(problems, cuda_dev, name)
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.timeout(TIMEOUT)
@pytest.mark.parametrize("name", NAMES)
def test_every_layout_launch_of_every_ae_loss_workload(cuda_dev, name):
    calls, problems = record(AE_LOSS_WORKLOADS[name], cuda_dev, ES.SIGS)
    ops_ = defaultdict(int)
    for p in problems:
        ops_[p["op"]] += 1
    print(f"\n{name}: {calls} calls, {len(problems)} distinct problems ({dict(ops_)})")
    assert any(p["op"] == "im2col3x3" and p["c"] == 3 for p in problems)
    if name != "lpips_min_side":
        assert any(p["op"] == "nchw_to_nhwc" and p["f16"] and not p["f32"] for p in problems)
    ES.run_sweep(problems, name)
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.timeout(TIMEOUT)
@pytest.mark.parametrize("name", NAMES)
def test_every_ae_loss_kernel_launch(cuda_dev, name):
    """lpips_scale, maxpool2x2, lpips_head and, for the full loss, im2col and every ae_loss_terms kind; at 256² the
    first LPIPS tap runs the 256-chunk grid (hw = 65536) and lpips_scale wraps its capped grid."""
    calls, problems = record(AE_LOSS_WORKLOADS[name], cuda_dev, SIGS)
    kinds = defaultdict(int)
    for p in problems:
        kinds[p["op"]] += 1
    print(f"\n{name}: {calls} calls, {len(problems)} distinct problems ({dict(kinds)})")
    assert {p["c"] for p in problems if p["op"] == "lpips_head"} == {64, 128, 256, 512}
    assert kinds["lpips_scale"] and kinds["maxpool2x2"]
    if name == "ae_loss_256":
        assert any(p["op"] == "lpips_head" and p["hw"] == 65536 for p in problems)
    if name == "ae_loss_72x104":
        assert any(p["op"] == "maxpool2x2" and (p["h"], p["w"]) == (9, 13) for p in problems)
    if name != "lpips_min_side":
        assert {p["kind"] for p in problems if p["op"] == "ae_loss_terms"} == {1, 2, 3}
        assert {(p["k"], p["stride"]) for p in problems if p["op"] == "im2col"} == {(4, 2), (4, 1)}
    run_sweep(problems, name)
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.timeout(TIMEOUT)
@pytest.mark.parametrize("name", NAMES)
def test_ae_loss_pre_wait_operands_are_packed_weights(cuda_dev, name):
    t0 = time.time()
    bad, n = audit_workload(name, AE_LOSS_WORKLOADS[name], cuda_dev)
    print(f"\n{name}: {n} gemm / groupnorm / layernorm calls audited, {len(bad)} violations, {time.time() - t0:.1f} s")
    assert n > 0
    assert not bad, "pre-wait operands outside packed weights (workload, op, slot, shape):\n" + \
        "\n".join(map(str, sorted(set(bad))))


# ------------------------------------------------------------------------------------------------ edges
def _p(op, **kw):
    base = {"lpips_scale": dict(a0=0, a1=0), "maxpool2x2": dict(ax=0), "lpips_head": dict(af=0, zeros=False),
            "im2col": dict(ax=0), "ae_loss_terms": dict(aa=0, ab=0, plant=False)}[op]
    return dict(dict(op=op, **base), **kw)


def edge_grid():
    ps = []
    # lpips_head: one pixel, one short of a 256-pixel chunk, one past it, one past 256 chunks; all-zero pixels; up to
    # 64 samples per batch (the per-sample fold runs 8 warps per block)
    for nb, hw, c in ((1, 1, 512), (2, 1, 64), (3, 255, 128), (2, 257, 256), (1, 65537, 64), (64, 257, 64),
                      (64, 3, 512), (9, 300, 128)):
        ps.append(_p("lpips_head", nb=nb, hw=hw, c=c))
        ps.append(_p("lpips_head", nb=nb, hw=hw, c=c, zeros=True))
    ps.append(_p("lpips_head", nb=2, hw=1000, c=256, af=8))
    # ae_loss_terms: n of 1, 255, 257 and 3 x 512²; KL at every latent width; logvar and logit edges planted
    for n in (1, 255, 257, 3 * 512 * 512):
        ps.append(_p("ae_loss_terms", kind=1, nb=2 if n > 1000 else 3, n=n, cc=1, aa=n % 4, ab=(n + 1) % 4))
        ps.append(_p("ae_loss_terms", kind=3, nb=1 if n > 1000 else 3, n=n, cc=32, plant=True))
        ps.append(_p("ae_loss_terms", kind=3, nb=2, n=n, cc=1, aa=1))
    for cc in (3, 4, 8, 16, 32, 64):
        for pix in (1, 85, 257):
            ps.append(_p("ae_loss_terms", kind=2, nb=3, n=pix * cc, cc=cc, plant=True))
    ps += [_p("ae_loss_terms", kind=2, nb=1, n=3 * 512 * 512, cc=3, plant=True),
           _p("ae_loss_terms", kind=2, nb=2, n=3 * 512 * 512, cc=64, aa=2)]
    # maxpool2x2: a NaN at each of the four window positions and each channel of two vectors, +-inf; odd sides
    ps += [_p("maxpool2x2", nb=1, h=4, w=2 * 64 + 1, c=16, special=True), _p("maxpool2x2", nb=2, h=5, w=7, c=8),
           _p("maxpool2x2", nb=3, h=2, w=2, c=520)]
    # im2col: the scalar path (c % 8 != 0) and k / stride / pad past the discriminator's 4 / 2 / 1, odd sides, kpad
    # past the next multiple of 64
    for c in (1, 3, 5):
        for k, s, pad in ((4, 2, 1), (3, 1, 0), (5, 3, 2), (1, 1, 0), (2, 2, 0), (7, 1, 3)):
            ps.append(_p("im2col", nb=2, h=11, w=9, c=c, k=k, stride=s, pad=pad, kpad=(k * k * c + 7) // 8 * 8 + 8,
                         ax=c % 3))
    for c in (8, 16, 72):
        for k, s, pad in ((3, 1, 0), (5, 3, 2), (4, 1, 1), (2, 2, 0), (4, 3, 3)):
            ps.append(_p("im2col", nb=2, h=10, w=13, c=c, k=k, stride=s, pad=pad, kpad=(k * k * c + 63) // 64 * 64 + 64))
    # lpips_scale: odd sides, a one-pixel image, inputs off 16-byte boundaries
    ps += [_p("lpips_scale", nb=3, h=7, w=5, a0=1, a1=3), _p("lpips_scale", nb=1, h=1, w=1)]
    return ps


@pytest.mark.gpu
@pytest.mark.timeout(TIMEOUT)
def test_ae_loss_kernel_edges(cuda_dev):
    run_sweep(edge_grid(), "edges")


@pytest.mark.gpu
def test_im2col_rejects_misaligned_vector_pointers(cuda_dev):
    """With c % 8 == 0 sdb_im2col moves 16-byte vectors: a pointer it cannot address so is an error returned before
    anything launches. The scalar path (c % 8 != 0) takes any fp16 pointer."""
    lib = L()
    before = lib.sdb_launch_count()
    x = ES._at((1, 6, 6, 8), 0, cuda_dev, torch.float16)
    o = torch.empty(9 * 128 + 8, dtype=torch.float16, device=cuda_dev)
    for k in (1, 2, 4):
        xm = ES._at((1, 6, 6, 8), k, cuda_dev, torch.float16)
        assert lib.sdb_im2col(P(xm), 1, 6, 6, 8, 4, 2, 1, 3, 3, 128, P(o), S()) != 0
        assert b"aligned" in lib.sdb_last_error()
        assert lib.sdb_im2col(P(x), 1, 6, 6, 8, 4, 2, 1, 3, 3, 128, P(o[k:]), S()) != 0
        assert b"aligned" in lib.sdb_last_error()
    assert lib.sdb_launch_count() == before
    xs = ES._at((1, 6, 6, 5), 1, cuda_dev, torch.float16)
    assert lib.sdb_im2col(P(xs), 1, 6, 6, 5, 4, 2, 1, 3, 3, 128, P(o[1:]), S()) == 0
    torch.cuda.synchronize()
    ref = im2col_ref(xs, 4, 2, 1, 128)
    assert ES._eq(o[1: 1 + ref.numel()].view_as(ref), ref)


# ------------------------------------------------------------------------------------------------ NaN propagation
@pytest.mark.gpu
@pytest.mark.parametrize("act", [ACT_RELU, ACT_LEAKY_RELU])
@pytest.mark.parametrize("geom", ["mm", "conv", "scalar"])
def test_nan_bias_column_propagates_through_relu_epilogues(cuda_dev, act, geom):
    """A NaN bias column is NaN in every output row, fp32 and fp16, as torch.relu / F.leaky_relu(0.2) keep it; every
    other element is finite. mm / conv take the TMA-store epilogue, scalar (n = 36) the scalar stores."""
    g = torch.Generator().manual_seed(31)
    if geom == "conv":
        a, n, taps = torch.randn(2, 8, 8, 64, generator=g).half(), 128, 9
        b = (torch.randn(n, 9 * 64, generator=g) * 24 ** -1).half()
    else:
        n = 36 if geom == "scalar" else 128
        a, taps = torch.randn(300, 640, generator=g).half(), 1
        b = (torch.randn(n, 640, generator=g) * 640 ** -0.5).half()
    bias = torch.randn(n, generator=g)
    bias[[3, n - 1]] = NAN
    o16, o32 = ops.gemm(a.to(cuda_dev), b.to(cuda_dev), taps=taps, bias=bias.to(cuda_dev), act=act, want_f16=True,
                        want_f32=True)
    if taps == 9:
        w = b.float().view(n, 3, 3, 64).permute(0, 3, 1, 2)
        v = F.conv2d(a.float().permute(0, 3, 1, 2), w, bias, padding=1).permute(0, 2, 3, 1).reshape(-1, n)
    else:
        v = a.float() @ b.float().t() + bias
    ref = torch.relu(v) if act == ACT_RELU else F.leaky_relu(v, 0.2)
    assert int(ref.isnan().sum()) == 2 * ref.shape[0]
    for o in (o32, o16):
        got = o.view(-1, n).cpu()
        assert torch.equal(got.isnan(), ref.isnan()), (int(got.isnan().sum()), int(ref.isnan().sum()))
        assert bool(torch.isfinite(got[:, :3]).all())


@pytest.mark.gpu
def test_nan_in_one_image_propagates_through_lpips(cuda_dev):
    """LPIPS of a batch whose second input image holds one NaN pixel is NaN for that sample alone, as the reference
    LPIPS (the oracle's restatement over torchvision's VGG16) reports it; the other samples keep their bits."""
    sys.path.insert(0, os.path.join(helpers.ROOT, "oracle"))
    import taming_loss_oracle as T
    sd = ae_loss.random_loss_state_dict(ae_loss.lpips_param_shapes(), 23)
    g = torch.Generator().manual_seed(7)
    x0, x1 = torch.rand(3, 3, 32, 32, generator=g) * 2 - 1, torch.rand(3, 3, 32, 32, generator=g) * 2 - 1
    x0n = x0.clone()
    x0n[1, 2, 5, 7] = NAN
    ref_m = T.LPIPS().eval()
    ref_m.load_state_dict(sd)
    with torch.no_grad():
        ref = ref_m(x0n, x1).view(-1)
    assert ref.isnan().tolist() == [False, True, False]
    lp = sdb200.LPIPS().load_weights(sd, cuda_dev)
    got = lp(x0n.to(cuda_dev), x1.to(cuda_dev)).view(-1).cpu()
    clean = lp(x0.to(cuda_dev), x1.to(cuda_dev)).view(-1).cpu()
    assert torch.equal(got.isnan(), ref.isnan()), got
    assert torch.equal(got[[0, 2]], clean[[0, 2]])


@pytest.mark.gpu
def test_nan_logvar_propagates_through_kl(cuda_dev):
    """A NaN logvar makes its sample's KL NaN, as torch.clamp keeps the NaN (distributions.py:28); the logvars past
    both clamps in the other samples stay finite."""
    g = torch.Generator().manual_seed(8)
    nb, h, w, cc = 3, 5, 6, 4
    m = torch.randn(nb, h, w, 2 * cc, generator=g)
    m[0, 1, 2, cc + 1] = 1e30
    m[2, 0, 0, cc] = -float("inf")
    m[1, 4, 5, cc + 3] = NAN
    mu, lv = m[..., :cc], torch.clamp(m[..., cc:], -30.0, 20.0)
    ref = 0.5 * (mu * mu + torch.exp(lv) - 1.0 - lv).double().sum((1, 2, 3))
    assert ref.isnan().tolist() == [False, True, False]
    got = ops.ae_loss_terms(m.to(cuda_dev), "kl", cc=cc)[0].cpu()
    assert torch.equal(got.isnan(), ref.isnan()), got


@pytest.mark.gpu
def test_nan_logit_propagates_through_every_logit_sum(cuda_dev):
    """A NaN logit makes all five sums of its sample NaN, as F.relu and F.softplus keep the NaN; a NaN outside column 0
    (not a logit) changes nothing."""
    g = torch.Generator().manual_seed(9)
    nb, n, cc = 3, 30, 32
    a = torch.randn(nb * n, cc, generator=g) * 8
    a[n + 7, 0] = NAN
    a[2 * n + 3, 1] = NAN
    lg = a[:, 0].view(nb, n)
    ref = torch.stack([lg.sum(1), F.relu(1.0 - lg).sum(1), F.relu(1.0 + lg).sum(1), F.softplus(-lg).sum(1),
                       F.softplus(lg).sum(1)])
    assert ref.isnan().tolist() == [[False, True, False]] * 5
    got = ops.ae_loss_terms(a.to(cuda_dev), "logits", n=n, cc=cc).cpu()
    assert torch.equal(got.isnan(), ref.isnan()), got


# ------------------------------------------------------------------------------------------------ CPU: the harness
def test_references_and_edges_cpu():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 7, 6, 3, generator=g).half()
    col = im2col_ref(x, 4, 2, 1, 56)
    assert col.shape == (2 * 3 * 3, 56) and bool((col[:, 48:] == 0).all())
    assert torch.equal(col[4, 5 * 3: 6 * 3], x[0, 2, 2])     # (oy, ox) = (1, 1), tap (ky, kx) = (1, 1): 2 o - 1 + k
    assert torch.equal(col[0, :3], torch.zeros(3, dtype=torch.float16))     # tap (0, 0) of (0, 0): padding
    mp = maxpool_operand(_p("maxpool2x2", nb=1, h=4, w=2 * 64 + 1, c=16, special=True), g)
    win = mp[0, :2, :128].float().view(2, 64, 2, 16).permute(1, 3, 0, 2).reshape(64, 16, 4)   # [window, ch, pos]
    nan = win.isnan()
    assert all(nan[j].nonzero().tolist() == [[j // 4, j % 4]] for j in range(64))
    assert 20.0 in LOGIT_EDGES and -20.0 in LOGIT_EDGES and _after(20.0, 1e9) > 20.0 and -1.0 in LOGIT_EDGES
    assert -30.0 in LOGVAR_EDGES and _after(-30.0, -1e9) < -30.0
    p = _ae_loss_terms_sig(torch.zeros(6 * 30, 32), "logits", n=30, cc=32)
    assert (p["kind"], p["nb"], p["n"], p["cc"]) == (3, 6, 30, 32)
    p = _ae_loss_terms_sig(torch.zeros(2, 4, 5, 8), "kl", cc=4)
    assert (p["kind"], p["nb"], p["n"], p["cc"]) == (2, 2, 80, 4)
    assert _lpips_head_sig(torch.zeros(4, 3, 5, 64, dtype=torch.float16), None, None, True)["hw"] == 15
    assert {q["op"] for q in edge_grid()} == set(RUN) == set(SIGS)
    # the KL / logit references reproduce the reference's element values
    q = _p("ae_loss_terms", kind=2, nb=1, n=12, cc=4, plant=True)
    a, _ = terms_operands(q, torch.Generator().manual_seed(1))
    v, extra = terms_reference(q, a, None)
    lv = a.view(1, 3, 8)[..., 4:].reshape(1, 12)
    assert torch.equal(lv[0], torch.tensor(LOGVAR_EDGES))
    assert bool(torch.isfinite(v).all()) and bool((extra > 0).all())
