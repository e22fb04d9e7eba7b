"""Child process of test_pdl_order_gpu.py (not a test module): runs model workloads in a fresh process, with the
programmatic-launch attribute as the SDB_PDL environment variable of this process says, and writes a bit-level digest
of what each computes.

    python pdl_child.py OUT.json NAME [NAME ...]      {name: sha256 of every output tensor's bytes}
    python pdl_child.py OUT.json --trace NAME         [[op, sha256 of the op's outputs], ...] in call order

NAME is a key of workloads.ELEMENTWISE_WORKLOADS or of EXTRA below. The autotuner is off, so both settings of SDB_PDL
pick the same tile plans: their results must be equal bit for bit."""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

import helpers  # noqa: E402,F401  (puts the repository on sys.path)
from sdb200 import arch, ops  # noqa: E402
import workloads  # noqa: E402


def tensors(obj, depth=0):
    """The tensors inside obj (lists, tuples, dicts and plain objects, such as a posterior), in a fixed order."""
    if isinstance(obj, torch.Tensor):
        yield obj
    elif depth > 4 or obj is None:
        return
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            yield from tensors(v, depth + 1)
    elif isinstance(obj, dict):
        for k in sorted(obj, key=str):
            yield from tensors(obj[k], depth + 1)
    elif hasattr(obj, "__dict__") and not isinstance(obj, (torch.nn.Module, type)):
        for k in sorted(vars(obj)):
            yield from tensors(vars(obj)[k], depth + 1)


def digest(obj):
    h = hashlib.sha256()
    n = 0
    for t in tensors(obj):
        t = t.detach()
        h.update(f"{t.dtype}{tuple(t.shape)}".encode())
        h.update(t.contiguous().view(-1).view(torch.uint8).cpu().numpy().tobytes())
        n += 1
    return f"{n}:{h.hexdigest()}"


def _sdv1_unet(dev):
    net = workloads._unet(arch.SD_V1_UNET, dev)
    net.autotune = False
    g = torch.Generator(device=dev).manual_seed(21)
    x = torch.randn(2, 4, 64, 64, generator=g, device=dev)
    ctx = torch.randn(2, 77, 768, generator=g, device=dev)
    t = torch.tensor([981.0, 501.0], device=dev)
    return net, x, t, ctx


def _wl_sdv1_graph(dev):
    """SD-v1 UNet at (2, 4, 64, 64) through its captured CUDA graph: the capture, then two replays."""
    net, x, t, ctx = _sdv1_unet(dev)
    net.use_cuda_graph = True
    return [net(x, t, context=ctx), net(x * 0.5, t - 100, context=ctx)]


def _wl_sdv1_handle(dev):
    """The same UNet through its C handle (sdb_plan_* + sdb_unet_forward)."""
    net, x, t, ctx = _sdv1_unet(dev)
    h = net.c_handle(tuple(x.shape), ctx)
    try:
        return [h.forward(x, t).clone(), h.forward(x * 0.5, t - 100).clone()]
    finally:
        torch.cuda.synchronize()
        h.close()


def _wl_plms_tiny(dev):
    """Ten guided PLMS steps of the tiny text-to-image model in C (sdb_sample_plms)."""
    import sdb200
    from helpers import golden
    from test_pipeline_gpu import _tiny_ld
    ld = _tiny_ld(dev)
    ld.model.diffusion_model.autotune = False
    g = golden("pipeline_tiny.pt")
    c, uc, x_T = g["c"].to(dev), g["uc"].to(dev), g["x_T"].to(dev)
    h = ld.model.diffusion_model.c_handle((4, 4, 16, 16), torch.cat([uc, c]).contiguous())
    try:
        sampler = sdb200.PLMSSampler(ld)
        sampler.make_schedule(10, verbose=False)
        return h.sample_plms(x_T.contiguous().float(), sampler, scale=7.5, guided=True)
    finally:
        torch.cuda.synchronize()
        h.close()


EXTRA = {"sdv1_unet_graph": _wl_sdv1_graph, "sdv1_unet_handle": _wl_sdv1_handle, "plms_tiny": _wl_plms_tiny}
ALL = {**workloads.ELEMENTWISE_WORKLOADS, **EXTRA}


def traced(name, dev):
    """Runs one workload with every public ops function wrapped: the digest of each call's outputs, in call order."""
    calls = []
    originals = {}
    for k, fn in list(vars(ops).items()):
        if k.startswith("_") or not callable(fn) or isinstance(fn, type) or getattr(fn, "__module__", "") != ops.__name__:
            continue
        if k in ("launch_count", "add_graph_launches", "channel_stats", "tune_key", "tune_candidates",
                 "splitk_workspace"):
            continue

        def wrap(fn=fn, k=k):
            def call(*a, **kw):
                r = fn(*a, **kw)
                torch.cuda.synchronize()
                calls.append([k, digest(r)])
                return r
            return call
        originals[k] = fn
        setattr(ops, k, wrap())
    try:
        with torch.no_grad():
            calls.append(["result", digest(ALL[name](dev))])
    finally:
        for k, fn in originals.items():
            setattr(ops, k, fn)
    return calls


def main(argv):
    out_path, names = argv[0], argv[1:]
    dev = torch.device("cuda:0")
    ops.AUTOTUNE = False
    if names[0] == "--trace":
        result = traced(names[1], dev)
    else:
        result = {}
        for name in names:
            with torch.no_grad():
                result[name] = digest(ALL[name](dev))
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    with open(out_path, "w") as fh:
        json.dump(result, fh)


if __name__ == "__main__":
    main(sys.argv[1:])
