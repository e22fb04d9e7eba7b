"""Launch ordering under programmatic dependent launch (PDL).

launch_pdl (csrc/host.h) and the GEMM launcher start every kernel with the programmatic-stream-serialization
attribute, and each of these kernels runs griddepcontrol.launch_dependents as its first statement: the next kernel's
prologue starts while this one runs, and since every kernel of a chain triggers early, kernel N may be resident while
N-1, N-2, ... still run. What a kernel reads before its griddepcontrol.wait (pdl_wait()) must therefore not be written by
any kernel that may still be in flight. The fp64 sweeps launch each kernel in isolation, after a synchronize, so none
of them can see a read that comes too early. This file checks the ordering four ways:

  1. (CPU) PRE_WAIT, the operands each PDL kernel reads ahead of its wait, checked against the kernel sources: every
     kernel launched through launch_pdl or the GEMM launcher is in the table, executes pdl_wait(), reads nothing before
     it that the table does not list, and does not return before it.
  2. (GPU, deterministic) at every gemm / groupnorm / layernorm call of the model workloads, the pre-wait operands (B
     unless b_dynamic, bias, gamma, beta) lie inside storage a stage packed as its weights; a negative control drops
     b_dynamic from one V^T call and must be flagged.
  3. (GPU) producer -> consumer pairs through the C entry points: a slow PDL GEMM writes a NaN-filled buffer, and a
     consumer launched right behind it reads a slice of that buffer in every operand that must be read after the wait;
     its output must equal, bit for bit, the same launch made after a synchronize. Chains of three put another PDL
     kernel between producer and consumer. Positive controls feed the producer's output into a pre-wait operand and
     must see a difference: otherwise the harness creates no overlap and the pairs prove nothing.
  4. (GPU) every model workload, the SD-v1 UNet through its CUDA graph and its C handle, and the C PLMS loop give the
     same bits in two fresh processes with SDB_PDL=1 and SDB_PDL=0 (tests/pdl_child.py).
"""
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import pytest
import torch

import helpers
from sdb200 import ops
from sdb200 import lib as _l
from sweeps import NAN, record
from workloads import ELEMENTWISE_WORKLOADS, GEMM_MODEL_WORKLOADS, _run_unet

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(helpers.ROOT, "stable-diffusion_b200", "csrc")

# ------------------------------------------------------------------------------------------------ 1. the contract
# kernel -> operands it reads before griddepcontrol.wait. "b if b_static": the GEMM's B producer warp skips the wait
# when the descriptor's b_dynamic is 0.
PRE_WAIT = {
    "gn_fold_kernel": set(),
    "gn_apply_kernel": {"gamma", "beta"},
    "gn_mod_apply_kernel": set(),
    "layernorm_v2_kernel": {"gamma", "beta"},
    "layernorm_kernel": set(),
    "splitk_epilogue_kernel": {"bias"},
    "attention_tc_kernel": set(),
    "gemm_tc_kernel": {"b if b_static"},
}
# PDL kernel roles that may finish without executing griddepcontrol.wait (they read only what PRE_WAIT lists)
NO_WAIT = {("gemm_tc_kernel", "B producer warp, b_static")}
# tensor maps -> the operand they load
TMAPS = {"tmQ": "q", "tmK": "k", "tmV": "vt", "tm.b": "b", "tm.a": "a", "amap": "a"}


def _strip_comments(s):
    s = re.sub(r"/\*.*?\*/", " ", s, flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def sources():
    return {f: _strip_comments(open(os.path.join(CSRC, f)).read())
            for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h"))}


def _close(s, i, o="(", c=")"):
    """Index of the bracket closing the one at s[i]."""
    depth = 0
    for j in range(i, len(s)):
        depth += (s[j] == o) - (s[j] == c)
        if depth == 0:
            return j
    raise ValueError("unbalanced")


def kernel(src, name):
    """(parameter text, body text) of the __global__ definition of `name`."""
    for s in src.values():
        for m in re.finditer(r"__global__[^;{}]*?\b%s\s*\(" % re.escape(name), s):
            j = _close(s, m.end() - 1)
            k = s.index("{", j)
            if s[j + 1:k].strip():
                continue
            return s[m.end():j], s[k + 1:_close(s, k, "{", "}")]
    raise AssertionError(f"no __global__ definition of {name}")


def _kernel_names(src):
    return {m.group(1) for s in src.values()
            for m in re.finditer(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(", s)}


def pdl_kernels(src):
    """Kernels launched through launch_pdl or cudaLaunchKernelEx (the GEMM launcher), template arguments dropped."""
    known = _kernel_names(src)
    found = set()
    for f, s in src.items():
        for m in re.finditer(r"\b(launch_pdl|cudaLaunchKernelEx)\s*\(\s*(?:&\w+\s*,\s*)?(\w+)", s):
            name = m.group(2)
            if name not in known:   # a variable: `auto kern = gemm_tc_kernel<BN, CG, KIND>;` earlier in the function
                a = list(re.finditer(r"\b%s\s*=\s*&?(\w+)" % re.escape(name), s[:m.start()]))
                if not a:
                    # only the generic launcher itself forwards a kernel it does not name
                    assert f == "host.h" and name in ("void", "kern"), (f, s[m.start():m.start() + 80])
                    continue
                name = a[-1].group(1)
            assert name in known, (f, name)
            found.add(name)
    return found


def pointer_params(params, src):
    """Names of the pointer parameters; a struct parameter `GemmArgs p` contributes p.<pointer field>."""
    out = set()
    for decl in params.split(","):
        words = re.findall(r"\w+", decl)
        if not words:
            continue
        if "*" in decl:
            out.add(words[-1])
        elif len(words) >= 2 and re.search(r"\bstruct\s+%s\s*\{" % words[-2], "".join(src.values())):
            body = re.search(r"\bstruct\s+%s\s*\{(.*?)\};" % words[-2], "".join(src.values()), re.S).group(1)
            for field in body.split(";"):
                if "*" in field:
                    out.update(f"{words[-1]}.{n}" for n in re.findall(r"\*\s*(?:const\s+)?(\w+)", field))
    return out


def reads(text, ptrs):
    """Operands `text` dereferences: a pointer indexed, offset, __ldg'd or reinterpret_cast; a tensor map in a TMA load.
    A null test (if (p.bias), p.ws ? ..) is not a read."""
    out = set()
    for p in ptrs:
        q = r"(?<![\w.])" + re.escape(p) + r"\b"
        if re.search(q + r"\s*[\[+]", text) or re.search(r"__ldg\(\s*&?\s*" + q, text) or \
                re.search(r"reinterpret_cast<[^>]*>\(\s*" + q + r"\s*\)", text):
            out.add(p.split(".")[-1])
    for m in re.finditer(r"\btma_load\w*\(([^;]*)\);", text):
        for arg in re.findall(r"&?\s*([\w.]+)", m.group(1)):
            if arg in TMAPS:
                out.add(TMAPS[arg])
    return out


def strip_lambdas(text):
    """(text with the bodies of `auto f = [&](...) {...};` removed, lambda names): a lambda runs where it is called."""
    names = []
    while True:
        m = re.search(r"\bauto\s+(\w+)\s*=\s*\[[^\]]*\]\s*\(", text)
        if not m:
            return text, names
        k = text.index("{", _close(text, m.end() - 1))
        e = _close(text, k, "{", "}")
        names.append(m.group(1))
        text = text[:m.start()] + text[e + 1:]


WAIT = re.compile(r"\bpdl_wait\s*\(\s*\)\s*;")


def roles(name, body):
    """[(role, text before its wait or None when it has none)]. The GEMM has three roles: the A producer, the B
    producer (which skips the wait when b_static) and the consumer warpgroups; the code before the role split (with
    its lambdas removed) runs ahead of every role's wait."""
    if name != "gemm_tc_kernel":
        m = WAIT.search(body)
        return [("kernel", body[:m.start()] if m else None)], set()
    split = re.search(r"if\s*\(\s*warp\s*==\s*A_WARP\s*\|\|\s*warp\s*==\s*B_WARP\s*\)\s*\{", body)
    assert split, "gemm_tc_kernel: the producer / consumer role split moved"
    prefix, lambdas = strip_lambdas(body[:split.start()])
    k = split.end() - 1
    prod = body[k + 1:_close(body, k, "{", "}")]
    rest = body[_close(body, k, "{", "}") + 1:]
    assert re.match(r"\s*else\s*\{", rest), "gemm_tc_kernel: the consumer branch moved"
    k2 = rest.index("{")
    cons = rest[k2 + 1:_close(rest, k2, "{", "}")]
    guard = re.search(r"if\s*\(\s*is_a\s*\|\|\s*!\s*p\.b_static\s*\)\s*\{\s*pdl_wait\s*\(\s*\)\s*;", prod)
    out = []
    mp = WAIT.search(prod)
    out.append(("A producer warp", prefix + prod[:mp.start()] if mp else None))
    if guard:
        # B skips the wait when b_static: every B load of the producer loop runs ahead of it
        out.append(("B producer warp, b_static", None))
        extra = {"b if b_static"} if "b" in reads(prod, set()) else set()
    else:
        out.append(("B producer warp", prefix + prod[:mp.start()] if mp else None))
        extra = set()
    mc = WAIT.search(cons)
    out.append(("consumer warpgroups", prefix + cons[:mc.start()] if mc else None))
    called = {n for n in lambdas for _, t in out if t is not None and re.search(r"\b%s\s*\(" % n, t)}
    assert not called, f"gemm_tc_kernel: epilogue lambdas called ahead of a wait: {sorted(called)}"
    return out, extra


def audit_sources(src):
    """[(kernel, role, problem)] for every PDL kernel; the pre-wait reads per kernel."""
    problems, seen = [], {}
    kernels = pdl_kernels(src)
    for k in sorted(kernels | set(PRE_WAIT)):
        if k not in kernels:
            problems.append((k, "-", "listed in PRE_WAIT but no longer launched with PDL"))
            continue
        if k not in PRE_WAIT:
            problems.append((k, "-", "launched with PDL but missing from PRE_WAIT"))
            continue
        params, body = kernel(src, k)
        if not WAIT.search(body):
            problems.append((k, "-", "no pdl_wait()"))
            continue
        ptrs = pointer_params(params, src)
        rs, extra = roles(k, body)
        got = set(extra)
        for role, text in rs:
            if text is None:
                if (k, role) not in NO_WAIT:
                    problems.append((k, role, "no pdl_wait() on this path"))
                continue
            got |= reads(text, ptrs)
            if re.search(r"\breturn\b", text):
                problems.append((k, role, "returns before pdl_wait()"))
        seen[k] = got
        if not got <= PRE_WAIT[k]:
            problems.append((k, "-", f"reads {sorted(got - PRE_WAIT[k])} before pdl_wait(); PRE_WAIT lists "
                                     f"{sorted(PRE_WAIT[k])}"))
    return problems, seen


def test_pre_wait_reads_match_the_table_cpu():
    problems, seen = audit_sources(sources())
    print("\npre-wait reads: " + "; ".join(f"{k} {sorted(v)}" for k, v in sorted(seen.items())))
    assert not problems, "\n".join(" | ".join(p) for p in problems)
    assert seen["gn_apply_kernel"] == {"gamma", "beta"} and seen["splitk_epilogue_kernel"] == {"bias"}
    assert seen["gemm_tc_kernel"] == {"b if b_static"}


MUTANTS = {   # name -> (file, [(text, replacement)], kernel, what audit_sources must report)
    "gn_apply: the wait below the first x read": ("norm.cu", [
        ("  pdl_wait();\n  if (cs0) {", "  if (cs0) {"),
        ("                      : *reinterpret_cast<const float4*>(x1 + r * c1 + (c - c0));\n",
         "                      : *reinterpret_cast<const float4*>(x1 + r * c1 + (c - c0));\n        pdl_wait();\n")],
        "gn_apply_kernel", "x0"),
    "attention: the wait after the Q TMA issue": ("attention_tc.cu", [
        ("  pdl_wait();   // q / k / v", "  //"),
        ("tma_load_4d(q_s + pn * (AQ * 128), &tmQ, &q_full, pn * 64, head, q0, b);",
         "tma_load_4d(q_s + pn * (AQ * 128), &tmQ, &q_full, pn * 64, head, q0, b);\n        pdl_wait();")],
        "attention_tc_kernel", "q"),
    "GEMM: the consumer-warp wait removed": ("gemm_kernel.cuh", [
        ("    pdl_wait();   // residual / FiLM", "    //")],
        "gemm_tc_kernel", "no pdl_wait() on this path"),
    "split-K epilogue: the wait after the partial-plane read": ("gemm_kernel.cuh", [
        ("  pdl_wait();\n  if (col < p.N) {", "  if (col < p.N) {"),
        ("#pragma unroll\n    for (int i = 0; i < 4; ++i) {\n      const int row = blockIdx.y * 32 + ty + 8 * i;\n",
         "  pdl_wait();\n#pragma unroll\n    for (int i = 0; i < 4; ++i) {\n      const int row = blockIdx.y * 32 + ty + 8 * i;\n")],
        "splitk_epilogue_kernel", "ws"),
    "a new PDL kernel": ("norm.cu", [
        ("softmax_rows_kernel<<<rows, 256, 0, st>>>(x, cols, scale, static_cast<__half*>(out_f16));",
         "SDB_CUDA(launch_pdl(softmax_rows_kernel, dim3(rows), dim3(256), 0, st, x, cols, scale, "
         "static_cast<__half*>(out_f16)));"),
        ("  const float* p = x + static_cast<size_t>(blockIdx.x) * cols;\n",
         "  pdl_wait();\n  const float* p = x + static_cast<size_t>(blockIdx.x) * cols;\n")],
        "softmax_rows_kernel", "missing from PRE_WAIT"),
}


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_source_audit_catches_mutant_cpu(name):
    """The audit on in-memory copies of the sources with one read moved ahead of its wait (nothing is compiled)."""
    f, edits, kern, what = MUTANTS[name]
    src = sources()
    raw = open(os.path.join(CSRC, f)).read()
    for old, new in edits:
        assert raw.count(old) == 1, (f, old)
        raw = raw.replace(old, new)
    src[f] = _strip_comments(raw)
    problems, _ = audit_sources(src)
    assert any(p[0] == kern and what in p[2] for p in problems), problems


# ------------------------------------------------------------------------------------------------ 2. weights only
class Weights:
    """Storage ranges of the tensors each stage packed as its weights (snapshotted when pack_weights returns); the
    tensors are kept alive, so freed weight memory is never reused by activations during the audit."""

    def __init__(self):
        self.spans, self.keep = [], []

    def add(self, obj, depth=0):
        if isinstance(obj, torch.Tensor):
            if obj.is_cuda:
                s = obj.untyped_storage()
                self.spans.append((s.data_ptr(), s.data_ptr() + s.nbytes()))
                self.keep.append(obj)
        elif depth < 16 and isinstance(obj, (list, tuple)):
            for v in obj:
                self.add(v, depth + 1)
        elif depth < 16 and isinstance(obj, dict):
            for v in obj.values():
                self.add(v, depth + 1)

    def has(self, t):
        lo = t.data_ptr()
        hi = lo + (sum((n - 1) * s for n, s in zip(t.shape, t.stride())) + 1) * t.element_size()
        return any(a <= lo and hi <= b for a, b in self.spans)


def _stage_classes():
    from sdb200.util import PackedStage
    out, todo = [], [PackedStage]
    while todo:
        c = todo.pop()
        out.append(c)
        todo.extend(c.__subclasses__())
    return [c for c in out if "pack_weights" in vars(c)]


def audit_workload(name, workload, dev):
    """(violations (workload, op, slot, shape), calls audited) of one eager run of workload(dev)."""
    W = Weights()
    bad = []

    def slot(op, what, t):
        if t is not None and not W.has(t):
            bad.append((name, op, what, tuple(t.shape)))

    def gemm(a0, b, **kw):
        if not kw.get("b_dynamic"):
            slot("gemm", "b", b)
        slot("gemm", "bias", kw.get("bias"))
        return {}

    def norm(op):
        def sig(x, gamma, beta, *a, **kw):
            slot(op, "gamma", gamma)
            slot(op, "beta", beta)
            return {}
        return sig

    def packer(orig):
        def pack_weights(self, device):
            r = orig(self, device)
            W.add(self.W)
            return r
        return pack_weights

    with pytest.MonkeyPatch.context() as mp:
        for c in _stage_classes():
            mp.setattr(c, "pack_weights", packer(vars(c)["pack_weights"]))
        n, _ = record(workload, dev, {"gemm": gemm, "groupnorm": norm("groupnorm"), "layernorm": norm("layernorm")})
    del W
    torch.cuda.empty_cache()
    return bad, n


AUDITED = {**ELEMENTWISE_WORKLOADS, **{"gemm_model_" + k: v for k, v in GEMM_MODEL_WORKLOADS.items()}}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(AUDITED))
def test_pre_wait_operands_are_packed_weights(cuda_dev, name):
    t0 = time.time()
    bad, n = audit_workload(name, AUDITED[name], cuda_dev)
    print(f"\n{name}: {n} gemm / groupnorm / layernorm calls audited, {len(bad)} violations, {time.time() - t0:.1f} s")
    assert not bad, "pre-wait operands outside packed weights (workload, op, slot, shape):\n" + \
        "\n".join(map(str, sorted(set(bad))))


@pytest.mark.gpu
def test_weight_audit_flags_a_dropped_b_dynamic(cuda_dev):
    """Negative control: the first V^T GEMM (B = the normalised activation, b_dynamic=True) of the attention-block
    UNet loses its flag; the audit must report exactly that call."""
    from sdb200 import arch
    dropped = []

    def workload(dev):
        with pytest.MonkeyPatch.context() as mp:
            inner = ops.gemm

            def gemm(a0, b, **kw):
                if kw.get("b_dynamic") and not dropped:
                    kw["b_dynamic"] = False
                    dropped.append(tuple(b.shape))
                return inner(a0, b, **kw)
            mp.setattr(ops, "gemm", gemm)
            return _run_unet(arch.TINY_ATTN_UNET, [(2, 4, 16, 16)], dev)

    bad, _ = audit_workload("tiny_attn_unet", workload, cuda_dev)
    assert dropped, "the workload made no b_dynamic GEMM call"
    assert bad == [("tiny_attn_unet", "gemm", "b", dropped[0])], bad


# ------------------------------------------------------------------------------------------------ 3. pairs
def L():
    return _l.load()


def S():
    return ops._stream()


def P(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def pdl_on():
    return not os.environ.get("SDB_PDL", "1").startswith("0")


PM, PN, PK = 2048, 1024, 32768   # the producer: 16 x 8 = 128 tiles of 128 x 128, one CTA each, K = 32768
PROD_SG = 1


def gemm_desc(a, b, n, *, a1=None, a2=None, taps=1, nb=1, h=1, w=None, bias=None, film=None, rps=0, residual=None,
              out16=None, out32=None, block_n=128, pair=1, splits=1, mode=0, ws=None, stats=None, sg=1, b_dynamic=0,
              stride=1, shift=0, in_hw=(0, 0), alpha=1.0):
    srcs = [t for t in (a, a1, a2) if t is not None]
    d = _l.GemmDesc()
    d.a0, d.a1, d.a2, d.a3 = [P(t) for t in srcs] + [None] * (4 - len(srcs))
    d.c0, d.c1, d.c2, d.c3 = [t.shape[-1] for t in srcs] + [0] * (4 - len(srcs))
    d.nb, d.h, d.w, d.taps = nb, h, (a.numel() // a.shape[-1] if w is None else w), taps
    d.b, d.n, d.alpha, d.bias = P(b), n, alpha, P(bias)
    d.film, d.ldf, d.rows_per_sample = P(film), (film.shape[-1] if film is not None else 0), rps
    d.residual, d.ldr = P(residual), (residual.shape[-1] if residual is not None else 0)
    d.out_f16, d.out_f32 = P(out16), P(out32)
    d.block_n, d.pair, d.splits, d.splitk_mode = block_n, pair, splits, mode
    if ws is not None:
        d.workspace, d.workspace_floats = P(ws), ws.numel()
    d.stats_out, d.stats_group = P(stats), sg
    d.b_dynamic, d.conv_stride, d.conv_shift = b_dynamic, stride, shift
    d.in_h, d.in_w = in_hw
    return d


def gemm_plan(d):
    plan = (C.c_int32 * 5)()
    _l.check(L().sdb_gemm_plan(C.byref(d), plan), "sdb_gemm_plan")
    return list(plan)


class Launch:
    """One C entry point call with its arguments bound (nothing but the ctypes call happens when it runs)."""

    def __init__(self, what, fn, *args, keep=()):
        self.what, self.fn, self.args, self.keep = what, fn, args, keep

    def __call__(self):
        return self.what, self.fn(*self.args, S())


def gemm_launch(what, d, keep):
    return Launch(what, L().sdb_gemm, C.byref(d), keep=(d, keep))


class Producer:
    """The slow PDL producer: an explicit-plan sdb_gemm (block_n 128, single CTAs, no split) over 128 tiles with
    K = 32768, writing fp16 and fp32 outputs and the per-tile GroupNorm statistics of its one 2048-row sample. It
    leaves sm_count - 128 SMs idle and triggers its dependents at CTA start."""

    def __init__(self, dev):
        g = torch.Generator(device=dev).manual_seed(77)
        self.a = (torch.rand(PM, PK, generator=g, device=dev) - 0.5).half()
        self.b = (torch.rand(PN, PK, generator=g, device=dev) - 0.5).half()
        self.out16 = torch.empty(PM * PN, dtype=torch.float16, device=dev)
        self.out32 = torch.empty(PM * PN, dtype=torch.float32, device=dev)
        d = gemm_desc(self.a, self.b, PN, out16=self.out16, out32=self.out32, rps=PM, alpha=1.0 / 16, sg=PROD_SG)
        d.stats_out = C.c_void_p(16)   # the plan only needs to know that statistics are wanted
        plan = gemm_plan(d)
        assert plan[:4] == [128, 1, 1, 0], plan
        self.T = plan[4]
        self.stats = torch.empty(1, self.T, PN // PROD_SG, 2, dtype=torch.float32, device=dev)
        d.stats_out = P(self.stats)
        self.d = d
        self.launch = gemm_launch("producer", d, ())

    def fill(self):
        for t in (self.out16, self.out32, self.stats):
            t.fill_(NAN)

    def f16(self, shape, off=0):
        n = torch.Size(shape).numel()
        return self.out16[off:off + n].view(shape)

    def f32(self, shape, off=0):
        n = torch.Size(shape).numel()
        return self.out32[off:off + n].view(shape)

    def measure(self):
        """Mean duration of one producer launch over 10, by CUDA events."""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        _l.check(self.launch()[1], "producer")
        e0.record()
        for _ in range(10):
            _l.check(self.launch()[1], "producer")
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 10 * 1e3


class Static:
    """The same views as Producer, over settled copies of its outputs (operands nothing in flight writes)."""

    def __init__(self, prod):
        self.out16, self.out32, self.stats, self.T = prod.out16.clone(), prod.out32.clone(), prod.stats.clone(), prod.T

    f16, f32 = Producer.f16, Producer.f32


class Bufs:
    """Seeded weights and NaN-filled outputs / workspaces of one pair."""

    def __init__(self, dev, seed):
        self.dev, self.g, self.outs, self.scratch = dev, torch.Generator(device=dev).manual_seed(seed), [], []

    def w16(self, *shape, scale=0.05):
        return (torch.randn(*shape, generator=self.g, device=self.dev) * scale).half()

    def w32(self, *shape, scale=1.0, mean=0.0):
        return torch.randn(*shape, generator=self.g, device=self.dev) * scale + mean

    def out(self, *shape, dtype=torch.float16):
        t = torch.empty(*shape, dtype=dtype, device=self.dev)
        self.outs.append(t)
        return t

    def ws(self, n):
        t = torch.empty(n, dtype=torch.float32, device=self.dev)
        self.scratch.append(t)
        return t


def _gn_ws(B, nb, groups):
    return B.ws(nb * (128 * groups * 2 + groups * 2 + 1))


# consumer builders: (src, B) -> [Launch]. src is the Producer (the operand is still being written) or Static.
def c_gemm_1x1(src, B):
    a, b = src.f16((512, 256)), B.w16(256, 256)
    return [gemm_launch("gemm A 1x1", gemm_desc(a, b, 256, out16=B.out(512, 256)), (a, b))]


def c_gemm_3x3(src, B):
    a, b = src.f16((2, 16, 16, 64)), B.w16(128, 9 * 64)
    return [gemm_launch("gemm A 3x3", gemm_desc(a, b, 128, taps=9, nb=2, h=16, w=16, out16=B.out(512, 128)), (a, b))]


def c_gemm_stride2(shift):
    def build(src, B):
        a, b = src.f16((1, 32, 32, 64)), B.w16(128, 9 * 64)
        ho = (32 + 1 - shift) // 2
        d = gemm_desc(a, b, 128, taps=9, nb=1, h=ho, w=ho, stride=2, shift=shift, in_hw=(32, 32),
                      out16=B.out(ho * ho, 128))
        return [gemm_launch(f"gemm A stride 2 shift {shift}", d, (a, b))]
    return build


def c_gemm_concat(src, B):
    a0, a1, b = B.w16(2, 16, 16, 64, scale=1.0), src.f16((2, 16, 16, 64)), B.w16(128, 9 * 128)
    d = gemm_desc(a0, b, 128, a1=a1, taps=9, nb=2, h=16, w=16, out32=B.out(512, 128, dtype=torch.float32))
    return [gemm_launch("gemm A second concat source", d, (a0, a1, b))]


def c_gemm_lo(src, B):
    hi, lo, b = B.w16(512, 256, scale=1.0), src.f16((512, 256)), B.w16(256, 3 * 256)
    d = gemm_desc(hi, b, 256, a1=lo, a2=hi, out32=B.out(512, 256, dtype=torch.float32))
    return [gemm_launch("gemm A lo plane (a1)", d, (hi, lo, b))]


def c_gemm_residual(src, B):
    a, b, r = B.w16(512, 256, scale=1.0), B.w16(256, 256), src.f32((512, 256))
    d = gemm_desc(a, b, 256, residual=r, out32=B.out(512, 256, dtype=torch.float32))
    return [gemm_launch("gemm residual", d, (a, b, r))]


def c_gemm_film(rps):
    def build(src, B):
        a, b, bias, f = B.w16(512, 256, scale=1.0), B.w16(256, 256), B.w32(256), src.f32(((512 + rps - 1) // rps, 256))
        d = gemm_desc(a, b, 256, bias=bias, film=f, rps=rps, out32=B.out(512, 256, dtype=torch.float32))
        return [gemm_launch(f"gemm FiLM rows_per_sample {rps}", d, (a, b, bias, f))]
    return build


def c_gemm_b_dynamic(b_dynamic):
    def build(src, B):
        a, b = B.w16(512, 256, scale=1.0), src.f16((256, 256))
        d = gemm_desc(a, b, 256, b_dynamic=b_dynamic, out16=B.out(512, 256))
        return [gemm_launch(f"gemm B b_dynamic={b_dynamic}", d, (a, b))]
    return build


def c_gemm_splitk(M, N, splits, mode):
    def build(src, B):
        a, b, bias = src.f16((M, 256)), B.w16(N, 256), B.w32(N)
        ws = B.ws(splits * M * N) if mode == 1 else None
        d = gemm_desc(a, b, N, bias=bias, out32=B.out(M, N, dtype=torch.float32), splits=splits, mode=mode, ws=ws,
                      block_n=160 if N % 160 == 0 else 128)
        assert gemm_plan(d)[2:4] == [splits, mode]
        return [gemm_launch(f"gemm split-K {splits} mode {mode} ({M} x {N})", d, (a, b, bias))]
    return build


def c_groupnorm_stats(groups):
    """GEMM statistics (the producer's) and x into sdb_groupnorm: gn_fold then gn_apply, or the fold inside gn_apply."""
    def build(src, B):
        x = src.f32((1, PM, PN))
        g, bt = B.w32(PN, scale=0.2, mean=1.0), B.w32(PN, scale=0.2)
        out = B.out(PM * PN)
        args = (P(x), None, PN, 0, 1, PM, groups, P(g), P(bt), C.c_float(1e-5), 1, P(out), None, None, None,
                P(_gn_ws(B, 1, groups)), P(src.stats), None, src.T, 0, PROD_SG)
        return [Launch(f"groupnorm fused statistics, {groups} groups", L().sdb_groupnorm, *args, keep=(x, g, bt))]
    return build


def c_groupnorm_own(src, B):
    """x0 static, x1 (the concat's second source) being written: the statistics pass, then gn_apply."""
    x0, x1 = B.w32(2, 256, 128), src.f32((2, 256, 256))
    g, bt = B.w32(384, scale=0.2, mean=1.0), B.w32(384, scale=0.2)
    raw = B.out(2 * 256 * 384)
    args = (P(x0), P(x1), 128, 256, 2, 256, 32, P(g), P(bt), C.c_float(1e-6), 0, P(B.out(2 * 256 * 384)), P(raw), None,
            None, P(_gn_ws(B, 2, 32)), None, None, 0, 0, 0)
    return [Launch("groupnorm own statistics, concat", L().sdb_groupnorm, *args, keep=(x0, x1, g, bt))]


def c_groupnorm_mod(resample, x_from_src=True):
    def build(src, B):
        # x and the statistics come from src, or from settled copies; the scale / shift rows are always src's
        x, stats = (src.out32, src.stats) if x_from_src else (B.settled.out32, B.settled.stats)
        sc, sh = src.f32((1, PN), 0), src.f32((1, PN), 5 * PN)
        g, bt = B.w32(PN, scale=0.2, mean=1.0), B.w32(PN, scale=0.2)
        opix = {0: PM, 1: PM // 4, 2: PM * 4}[resample]
        out = B.out(opix * PN)
        args = (P(x), PN, 1, 32, 64, 32, P(g), P(bt), C.c_float(1e-5), 1, P(sc), P(sh), PN, resample, P(out),
                P(_gn_ws(B, 1, 32)), P(stats), src.T, PROD_SG)
        what = f"groupnorm_mod {'x, ' if x_from_src else ''}scale / shift, resample {resample}"
        return [Launch(what, L().sdb_groupnorm_mod, *args, keep=(x, stats, sc, sh, g, bt))]
    return build


def c_layernorm(rows, c, gamma_from_src=False):
    def build(src, B):
        x = B.w32(rows, c) if gamma_from_src else src.f32((rows, c))
        g = src.f32((c,), 64) if gamma_from_src else B.w32(c, scale=0.2, mean=1.0)
        bt = B.w32(c, scale=0.2)
        args = (P(x), rows, c, P(g), P(bt), C.c_float(1e-5), P(B.out(rows * c)), P(B.out(rows * c, dtype=torch.float32)))
        what = f"layernorm {'gamma' if gamma_from_src else 'x'} {rows} x {c}"
        return [Launch(what, L().sdb_layernorm, *args, keep=(x, g, bt))]
    return build


def c_softmax(src, B):
    x = src.f32((256, 4096))
    return [Launch("softmax_rows x", L().sdb_softmax_rows, P(x), 256, 4096, C.c_float(0.125), P(B.out(256 * 4096)),
                   keep=(x,))]


def c_attention(heads, d, dpad, ntok, nb):
    """q | k as the two halves of one fused projection output, V^T as the permuted view of one [hd, nb * ntok] GEMM
    output, as the UNet's attention blocks lay them out."""
    def build(src, B):
        hd = heads * d
        nqk = nb * ntok * 2 * hd
        qk, vt = src.f16((nb, ntok, 2 * hd)), src.f16((hd, nb * ntok), (nqk + 63) // 64 * 64)
        out = B.out(nb * ntok * hd)
        a = _l.AttnDesc()
        a.q, a.k, a.vt, a.out = qk.data_ptr(), qk.data_ptr() + 2 * hd, vt.data_ptr(), out.data_ptr()
        a.batch, a.heads, a.nq, a.nkv, a.d, a.dpad = nb, heads, ntok, ntok, d, dpad
        a.ldq, a.ldk, a.ldvt, a.ldo = 2 * hd, 2 * hd, nb * ntok, hd
        a.q_batch_stride = a.k_batch_stride = ntok * 2 * hd
        a.vt_batch_stride, a.o_batch_stride = ntok, ntok * hd
        a.scale, a.causal, a.head_stride = d ** -0.5, 0, (d if heads > 1 else 0)
        return [Launch(f"attention dpad {dpad} (d {d}, {heads} heads, {ntok} tokens)", L().sdb_attention, C.byref(a),
                       keep=(a, qk, vt))]
    return build


PAIRS = {
    "gemm_a_1x1": c_gemm_1x1,
    "gemm_a_3x3": c_gemm_3x3,
    "gemm_a_stride2_shift0": c_gemm_stride2(0),
    "gemm_a_stride2_shift1": c_gemm_stride2(1),
    "gemm_a_concat_second": c_gemm_concat,
    "gemm_a_lo_plane": c_gemm_lo,
    "gemm_residual": c_gemm_residual,
    "gemm_film_row": c_gemm_film(128 * 3 // 4),     # 96 rows per sample: per-row FiLM reads
    "gemm_film_table": c_gemm_film(128),
    "gemm_b_dynamic": c_gemm_b_dynamic(1),
    "gemm_splitk_ws_32": c_gemm_splitk(512, 256, 4, 1),
    "gemm_splitk_ws_narrow": c_gemm_splitk(512, 320, 4, 1),
    "gemm_splitk_ws_wide": c_gemm_splitk(1152, 1280, 2, 1),
    "gemm_splitk_cluster": c_gemm_splitk(512, 256, 2, 2),
    "groupnorm_stats_in_apply": c_groupnorm_stats(32),
    "groupnorm_stats_fold": c_groupnorm_stats(16),
    "groupnorm_own_stats": c_groupnorm_own,
    "groupnorm_mod_x": c_groupnorm_mod(0),
    "groupnorm_mod_x_down": c_groupnorm_mod(1),
    "groupnorm_mod_scale_shift": c_groupnorm_mod(0, x_from_src=False),
    "layernorm_v2_320": c_layernorm(2048, 320),
    "layernorm_v2_1280": c_layernorm(1024, 1280),
    "layernorm_scalar_96": c_layernorm(4096, 96),
    "layernorm_scalar_1792": c_layernorm(1024, 1792),
    "softmax_rows": c_softmax,
    "attention_dpad64": c_attention(8, 40, 64, 512, 2),
    "attention_dpad128": c_attention(8, 80, 128, 256, 2),
    "attention_dpad192": c_attention(5, 160, 192, 256, 2),
    "attention_dpad384": c_attention(1, 384, 384, 256, 1),
    "attention_dpad512": c_attention(1, 512, 512, 256, 1),
    "attention_dpad576": c_attention(1, 576, 576, 256, 1),
    "attention_dpad960_stream_q": c_attention(1, 960, 960, 256, 1),
}
# the middle kernel of a chain of three, on settled operands: one per PDL family
MIDDLE = {
    "gemm_b_static": c_gemm_1x1,
    "gemm_narrow_tiles": lambda src, B: [gemm_launch("gemm 256 x 32, block_n 32", gemm_desc(
        src.f16((256, 64)), B.w16(32, 64), 32, block_n=32, out16=B.out(256, 32)), ())],
    "gemm_splitk_ws": c_gemm_splitk(512, 256, 4, 1),
    "gemm_splitk_cluster": c_gemm_splitk(512, 256, 2, 2),
    "groupnorm_fold_apply": c_groupnorm_stats(16),
    "groupnorm_mod": c_groupnorm_mod(0),
    "layernorm_v2": c_layernorm(2048, 320),
    "layernorm_scalar": c_layernorm(4096, 96),
    "attention": c_attention(8, 40, 64, 512, 2),
}
LAST = {"layernorm x": c_layernorm(1024, 1792), "gemm A": c_gemm_3x3}
CONTROLS = {"layernorm gamma": c_layernorm(1024, 768, gamma_from_src=True), "gemm B without b_dynamic": c_gemm_b_dynamic(0)}


def _bits(t):
    return t.contiguous().view(-1).view(torch.uint8)


def run(prod, launches, B, settle):
    """Fill every output and workspace with NaN, launch the producer, then `launches` back to back; settle=True
    synchronizes after the producer. Returns copies of the outputs."""
    prod.fill()
    for t in B.outs + B.scratch:
        t.fill_(NAN)
    torch.cuda.synchronize()
    rcs = [prod.launch()]
    if settle:
        torch.cuda.synchronize()
    for f in launches:
        rcs.append(f())
    torch.cuda.synchronize()
    for what, rc in rcs:
        _l.check(rc, what)
    return [o.clone() for o in B.outs]


@pytest.fixture(scope="module")
def harness(cuda_dev):
    if not pdl_on():
        pytest.skip("SDB_PDL=0: launches are plainly stream-ordered")
    prod = Producer(cuda_dev)
    prod.fill()
    _l.check(prod.launch()[1], "producer")
    torch.cuda.synchronize()
    us = prod.measure()
    print(f"\nproducer: {PM} x {PN} x {PK} over 128 CTAs on {torch.cuda.get_device_name()} "
          f"({torch.cuda.get_device_properties(0).multi_processor_count} SMs): {us:.0f} us per launch")
    return prod, Static(prod), {"producer_us": us}


def check_sequence(harness, build_list, seed, expect_equal=True):
    """Builds the launches (each builder gets src, the producer or its settled copy), runs them unsettled and settled,
    and returns (what, number of differing output elements)."""
    prod, static, _ = harness
    B = Bufs(prod.out16.device, seed)
    B.settled = static
    launches = []
    for src_is_prod, build in build_list:
        launches += build(prod if src_is_prod else static, B)
    torch.cuda.synchronize()
    run(prod, launches, B, settle=True)       # first launches: module loading, attributes
    ref = run(prod, launches, B, settle=True)
    got = run(prod, launches, B, settle=False)
    diff = sum(int((_bits(a) != _bits(b)).sum()) for a, b in zip(ref, got))
    finite = all(bool(torch.isfinite(r.float()).all()) for r in ref)
    return " -> ".join(f.what for f in launches), diff, finite


@pytest.mark.gpu
def test_producer_consumer_pairs(harness):
    t0 = time.time()
    rows = []
    for i, (name, build) in enumerate(sorted(PAIRS.items())):
        what, diff, finite = check_sequence(harness, [(True, build)], 100 + i)
        if diff or not finite:
            rows.append((name, what, f"{diff} bytes differ from the settled launch" if diff else "non-finite output"))
    print(f"\n{len(PAIRS)} producer -> consumer pairs, {len(rows)} failing, {time.time() - t0:.1f} s")
    assert not rows, "\n".join(" | ".join(map(str, r)) for r in rows)


@pytest.mark.gpu
def test_chains_of_three(harness):
    """Producer -> PDL kernel M on settled operands -> consumer of the producer's output: the consumer's wait covers
    the producer only through M's, so the ordering must carry through the whole chain."""
    t0 = time.time()
    rows, n = [], 0
    for i, (m, mid) in enumerate(sorted(MIDDLE.items())):
        for j, (c, last) in enumerate(sorted(LAST.items())):
            n += 1
            what, diff, finite = check_sequence(harness, [(False, mid), (True, last)], 200 + 10 * i + j)
            if diff or not finite:
                rows.append((m, c, what, f"{diff} bytes differ" if diff else "non-finite output"))
    print(f"\n{n} chains of three, {len(rows)} failing, {time.time() - t0:.1f} s")
    assert not rows, "\n".join(" | ".join(map(str, r)) for r in rows)


@pytest.mark.gpu
def test_positive_controls_see_the_overlap(harness):
    """The producer's output in a pre-wait operand must change the consumer's result: otherwise the producer ends
    before the consumer starts and the pairs above prove nothing (make the producer slower or leave more SMs idle)."""
    out = {}
    for i, (name, build) in enumerate(sorted(CONTROLS.items())):
        _, diff, finite = check_sequence(harness, [(True, build)], 300 + i)
        assert finite, name
        out[name] = diff
    print("\npositive controls, bytes differing from the settled launch: " +
          ", ".join(f"{k} {v}" for k, v in out.items()))
    # ptxas places layernorm_v2's gamma / beta loads (ld.global.nc) after the wait instruction in the sm_90a binary,
    # so that control reads settled values; the GEMM's B producer issues its TMA loads ahead of the wait
    assert out["gemm B without b_dynamic"], (
        "no overlap: the GEMM read the producer's output ahead of the wait and still saw only its final values, so "
        "the producer -> consumer pairs cannot see an early read")


# ------------------------------------------------------------------------------------------------ 4. PDL on / off
CHILD = os.path.join(HERE, "pdl_child.py")
CHILD_TIMEOUT = 1800


def child(pdl, out, args):
    env = dict(os.environ, SDB_PDL=pdl)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [CHILD, out] + list(args)
    r = subprocess.run(cmd, env=env, cwd=HERE, capture_output=True, text=True, timeout=CHILD_TIMEOUT)
    assert r.returncode == 0, f"SDB_PDL={pdl} child failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    with open(out) as fh:
        return json.load(fh)


@pytest.mark.gpu
def test_models_bit_equal_with_pdl_on_and_off(cuda_dev):
    import pdl_child
    names = sorted(pdl_child.ALL)
    t0 = time.time()
    with tempfile.TemporaryDirectory() as tmp:
        on = child("1", os.path.join(tmp, "on.json"), names)
        t1 = time.time()
        off = child("0", os.path.join(tmp, "off.json"), names)
        t2 = time.time()
        assert set(on) == set(off) == set(names)
        bad = [n for n in names if on[n] != off[n]]
        first = []
        for n in bad:
            a = child("1", os.path.join(tmp, "t1.json"), ["--trace", n])
            b = child("0", os.path.join(tmp, "t0.json"), ["--trace", n])
            k = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
            first.append((n, f"call {k}", a[k][0] if k < len(a) else "-", b[k][0] if k < len(b) else "-"))
    print(f"\n{len(names)} workloads digested with SDB_PDL=1 ({t1 - t0:.0f} s) and SDB_PDL=0 ({t2 - t1:.0f} s)")
    assert not bad, "outputs differ with PDL on and off (workload, first differing op call, op on, op off):\n" + \
        "\n".join(map(str, first))


def test_child_digest_cpu():
    """The child's digest sees every tensor of nested outputs and every bit of them, NaN payloads included."""
    import pdl_child
    x = torch.arange(12, dtype=torch.float32).view(3, 4)

    class Post:
        def __init__(self, m):
            self.mean, self.std = m, m * 2

    d0 = pdl_child.digest([x, (Post(x), {"b": x.half()})])
    y = x.clone()
    y.view(-1)[5] = torch.nextafter(y.view(-1)[5], torch.tensor(100.0))
    assert pdl_child.digest([y, (Post(x), {"b": x.half()})]) != d0
    assert pdl_child.digest([x, (Post(y), {"b": x.half()})]) != d0
    assert pdl_child.digest([x, (Post(x), {"b": x.half()})]) == d0
    n1 = torch.full((2,), float("nan"))
    n2 = n1.view(torch.int32).add(1).view(torch.float32)
    assert pdl_child.digest(n1) != pdl_child.digest(n2)
    assert set(pdl_child.EXTRA) <= set(pdl_child.ALL) and set(ELEMENTWISE_WORKLOADS) <= set(pdl_child.ALL)


def test_weight_spans_cpu():
    W = Weights()
    big = torch.zeros(100)
    W.spans.append((big.data_ptr(), big.data_ptr() + 400))
    assert W.has(big[10:20]) and W.has(big.view(10, 10)[:, 3]) and W.has(big)
    other = torch.zeros(4)
    assert not W.has(other)
    W.spans = [(big.data_ptr(), big.data_ptr() + 200)]
    assert W.has(big[:50]) and not W.has(big[:51]) and not W.has(big.view(10, 10)[:, 4])


def test_pair_table_covers_every_post_wait_operand_cpu():
    """Every operand read after the wait has a pair (GEMM A at every kind and layout, residual, both FiLM paths, dynamic
    B, both split-K paths, GroupNorm statistics and x, modulation, LayerNorm both kernels, softmax, attention at every
    DPAD class and streamed Q); every PDL family has a middle kernel."""
    need = {"gemm_a_1x1", "gemm_a_3x3", "gemm_a_stride2_shift0", "gemm_a_stride2_shift1", "gemm_a_concat_second",
            "gemm_a_lo_plane", "gemm_residual", "gemm_film_row", "gemm_film_table", "gemm_b_dynamic",
            "gemm_splitk_cluster", "groupnorm_stats_fold", "groupnorm_stats_in_apply", "groupnorm_own_stats",
            "groupnorm_mod_x", "groupnorm_mod_scale_shift", "softmax_rows", "attention_dpad960_stream_q"}
    assert need <= set(PAIRS)
    assert {k for k in PAIRS if k.startswith("gemm_splitk_ws")}
    assert {k for k in PAIRS if k.startswith("attention_dpad")} >= {f"attention_dpad{d}" for d in (64, 128, 192, 384, 512, 576)}
    assert {k for k in PAIRS if k.startswith("layernorm_v2")} and {k for k in PAIRS if k.startswith("layernorm_scalar")}
    fams = {"gemm", "splitk", "groupnorm", "groupnorm_mod", "layernorm_v2", "layernorm_scalar", "attention"}
    assert all(any(m.startswith(f) or f in m for m in MIDDLE) for f in fams)
    assert 96 % 64 and (PM // 128) * (PN // 128) == 128
