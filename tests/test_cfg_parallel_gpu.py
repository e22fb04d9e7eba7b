"""CFG-parallel latency mode (SURVEY 8f-2) on two GPUs: the guidance halves of every UNet evaluation run on two
GPUs and meet in the fused step kernel (NCCL all_gather, or peer loads over NVLink inside the kernel). Both ranks must
end with identical latents that match the reference PLMS / DPM-Solver outputs like the single-GPU path does.
Skipped on boxes with fewer than two GPUs (`gpurun --gpus 2 -- python -m pytest tests/test_cfg_parallel_gpu.py`)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


def _worker(rank, port, ret):
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, here)
    from helpers import golden, rel_l2
    from test_pipeline_gpu import _tiny_ld
    import sdb200
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=dev)
    try:
        ld = _tiny_ld(dev)
        g, gx = golden("pipeline_tiny.pt"), golden("samplers_ext.pt")
        c, uc, x_T = g["c"].to(dev), g["uc"].to(dev), g["x_T"].to(dev)
        errs = {}
        for mode in ("nccl", "p2p"):
            cp = sdb200.dist.CFGParallel(mode=mode, device=dev, max_numel=2 * 4 * 16 * 16)
            kw = dict(conditioning=c, batch_size=2, shape=[4, 16, 16], verbose=False, unconditional_guidance_scale=7.5,
                      unconditional_conditioning=uc, x_T=x_T)
            s, _ = sdb200.PLMSSampler(ld, cfg_parallel=cp).sample(S=10, eta=0.0, **kw)
            d, _ = sdb200.DPMSolverSampler(ld, cfg_parallel=cp).sample(S=20, **kw)
            for name, t, ref in (("plms10", s, g["plms10"]), ("dpm20", d, gx["dpm20_s7.5"])):
                both = [torch.empty_like(t) for _ in range(2)]
                dist.all_gather(both, t)
                assert torch.equal(both[0], both[1]), (mode, name)
                errs[f"{mode}_{name}"] = rel_l2(t, ref)
            assert cp.evals == 11 + 20
        ret.put((rank, errs))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def test_cfg_parallel_two_gpus(cuda_dev):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, port, ret)) for r in range(2)]
    [p.start() for p in procs]
    got = dict(ret.get(timeout=400) for _ in range(2))
    [p.join(120) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert got[0] == got[1]
    assert all(v < 3e-2 for v in got[0].values()), got[0]
