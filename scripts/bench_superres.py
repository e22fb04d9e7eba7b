#!/usr/bin/env python
"""LDM super-resolution (models/ldm/bsr_sr) speed on the H100 engine: the reference notebook's workload, a 256x256 input
to a 1024x1024 image (latent 256x256 in 3x3 tiles of 128x128 at stride 64, DDIM-100, eta 1, batch 1, LR conversion +
tiled sampling + tiled VQ-f4 decode), on seeded random weights and a seeded random input.
Also reports, with CUDA events: one tiled UNet evaluation (the 9 tiles of (3 + 3) x 128x128 as one graph-replayed batch)
and its TFLOP/s from the layer shapes; the same 9 tiles as 9 graph-replayed calls of one tile; the tiled decode; the
stitch kernels (sdb_patch_fold for eps at 256x256 and for the decode at 1024x1024, and the per-step sdb_patch_unfold).
Prints one JSON line with the card name and power limit read in the same run.

  python scripts/bench_superres.py --repeats 2 --out outputs/superres.json
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import arch, ops  # noqa: E402
from sdb200.samplers import DDIMSampler  # noqa: E402
from measure import card, emit, event_ms, unet_flops, wall_s  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=2)
    p.add_argument("--steps", type=int, default=100)
    p.add_argument("--size", type=int, default=256)
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    import superres as S
    dev = torch.device("cuda")
    m = S.load_model(random_init=True)
    u = m.model.diffusion_model
    u.use_cuda_graph = True
    sampler = DDIMSampler(m)
    g = np.random.default_rng(0)
    lrs = [torch.from_numpy(g.integers(0, 256, (1, a.size, a.size, 3), dtype=np.uint8)).to(dev)
           for _ in range(a.repeats + 1)]
    torch.manual_seed(0)
    with m.ema_scope():
        S.superresolve(m, sampler, lrs[0], steps=2)          # warm-up: autotune, graph capture, tables, decoder
        torch.cuda.synchronize()
        runs, events = iter(lrs[1:]), []

        def one_image():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            events.append(ev)
            ev[0].record()
            out = S.superresolve(m, sampler, next(runs), steps=a.steps, eta=1.0, return_latents=True)
            ev[1].record()
            return out
        times, (x, c, s, path) = wall_s(one_image, a.repeats)
        split = [e0.elapsed_time(e1) for e0, e1 in events]
    assert path == "split" and tuple(x.shape) == (1, 3, 4 * a.size, 4 * a.size) and bool(torch.isfinite(x).all())

    plan = m._split_plan((1, 3, a.size, a.size), 1, dev)
    dplan = m._split_plan((1, 3, a.size, a.size), 4, dev)
    n, ks = plan["n"], plan["ks"]
    gt = torch.Generator(device=dev).manual_seed(1)
    xt = torch.randn(n, 3, *ks, generator=gt, device=dev)
    ct = torch.randn(n, 3, *ks, generator=gt, device=dev)
    t = torch.full((n,), 501.0, device=dev)
    tiled = event_ms(lambda: u(xt, t, concat=ct), 20, warmup=2)
    one = [(xt[i:i + 1].contiguous(), t[i:i + 1].contiguous(), ct[i:i + 1].contiguous()) for i in range(n)]
    nine_calls = event_ms(lambda: [u(x1, t1, concat=c1) for x1, t1, c1 in one], 10, warmup=2)
    fl = unet_flops(arch.BSR_SR_UNET, n, *ks)
    decode = event_ms(lambda: m.decode_first_stage(s), 3, warmup=2)
    eps_tiles = u(xt, t, concat=ct)
    fold_eps = event_ms(lambda: ops.patch_fold(eps_tiles, plan["weight"], plan["norm"], plan["grid"], plan["stride"]), 50,
                        warmup=2)
    xl = torch.randn(1, 3, a.size, a.size, generator=gt, device=dev)
    unfold = event_ms(lambda: ops.patch_unfold(xl, ks, plan["stride"]), 50, warmup=2)
    kd = dplan["ks"][0] * 4
    dec_tiles = torch.randn(dplan["n"], kd, kd, 3, generator=gt, device=dev)
    sd = (dplan["stride"][0] * 4, dplan["stride"][1] * 4)
    fold_dec = event_ms(lambda: ops.patch_fold(dec_tiles, dplan["weight"], dplan["norm"], dplan["grid"], sd, nhwc=True),
                        20, warmup=2)
    res = dict(workload=f"bsr_sr LDM, {a.size}x{a.size} -> {4 * a.size}x{4 * a.size}, {plan['grid'][0]}x{plan['grid'][1]} "
                        f"tiles of {ks[0]}x{ks[1]} at stride {plan['stride'][0]}, DDIM-{a.steps} eta 1, batch 1, LR "
                        "conversion + tiled sampling + tiled VQ-f4 decode, random weights",
               images_per_s=1.0 / min(times), run_s=times, run_ms_events=split,
               unet_tiled_eval_ms_graph=tiled, unet_tiled_tflop=fl / 1e12, unet_tiled_tflops=fl / (tiled * 1e-3) / 1e12,
               unet_nine_single_tile_calls_ms_graph=nine_calls, tiled_decode_ms=decode,
               stitch_eps_fold_ms=fold_eps, stitch_decode_fold_ms=fold_dec, unfold_xt_ms=unfold,
               unet_chunk=plan["chunk"], decode_chunk=dplan["chunk"], **card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
