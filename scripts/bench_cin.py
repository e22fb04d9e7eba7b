#!/usr/bin/env python
"""Class-conditional ImageNet LDM sampling speed on the H100 engine: the notebook workload of scripts/sample_imagenet.py
(classes 25, 187, 448, 992, 6 samples per class, DDIM-20, eta 0; decode_first_stage included) on seeded random weights.
cin256-v2 (default) is guided at scale 3.0, so every UNet evaluation runs a batch of 12 at 64x64x3; --model cin256 (the
LDM-VQ-8, no unconditional label) samples unguided, a batch of 6 at 32x32x4.
Also reports one graph-replayed UNet evaluation at that batch (CUDA events) and every attention launch of one eager
evaluation from ops.PROFILE: time, algorithmic FLOPs (4 B heads nq nkv d) and tensor floor (FLOPs / 989 TFLOP/s, the
H100 SXM dense fp16 data-sheet rate), with the attention share of the evaluation. Prints one JSON line with the card
name and power limit read in the same run.

  python scripts/bench_cin.py --repeats 3 --out outputs/cin.json
  python scripts/bench_cin.py --model cin256 --repeats 3 --out outputs/cin256.json
"""
import argparse
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import ops  # noqa: E402
from measure import card, emit, event_ms, wall_s  # noqa: E402


def attention_launches(u, x, t, c, reps=5):
    """[(B, heads, nq, nkv, d, us, flops)] of one eager evaluation (median over reps) and the eager evaluation's ms."""
    runs, totals = [], []
    for _ in range(reps):
        ops.PROFILE = []
        totals.append(event_ms(lambda: u(x, t, context=c), 1))
        runs.append(ops.PROFILE)
    ops.PROFILE = None
    out = []
    for i, (kind, fl, _, _, shp) in enumerate(runs[0]):
        if kind == "attention":
            out.append((*shp, statistics.median(r[i][2].elapsed_time(r[i][3]) for r in runs) * 1e3, fl))
    return out, statistics.median(totals)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--out", type=str, default=None)
    p.add_argument("--model", choices=["cin256-v2", "cin256"], default="cin256-v2")
    a = p.parse_args()
    import sample_imagenet as S
    dev = torch.device("cuda")
    m = S.load_model(random_init=True, model=a.model)
    u = m.model.diffusion_model
    u.use_cuda_graph = True
    classes, n = [25, 187, 448, 992], 6
    scale = S.MODELS[a.model][2]
    torch.manual_seed(0)
    S.sample_classes(m, classes, n, ddim_steps=a.steps, scale=scale)   # warm-up: autotune, graph capture, first stage
    torch.cuda.synchronize()
    times, img = wall_s(lambda: S.sample_classes(m, classes, n, ddim_steps=a.steps, scale=scale), a.repeats)
    assert img.shape == (len(classes) * n, 3, 256, 256) and bool(torch.isfinite(img).all())
    labels = n * [1000] + n * [25] if scale != 1.0 else n * [25]
    nb = len(labels)
    x = torch.randn(nb, u.in_channels, u.image_size, u.image_size, device=dev)
    t = torch.full((nb,), 501.0, device=dev)
    c = m.get_learned_conditioning({"class_label": torch.tensor(labels, device=dev)})
    unet_ms = event_ms(lambda: u(x, t, context=c), 50, warmup=5)
    u.use_cuda_graph = False
    launches, eager_ms = attention_launches(u, x, t, c)
    attn_us = sum(r[5] for r in launches)
    rows = [dict(B=B, heads=H, nq=nq, nkv=nkv, d=d, us=round(us, 1), gflop=round(fl / 1e9, 3),
                 tensor_floor_us=round(fl / 989e12 * 1e6, 1)) for B, H, nq, nkv, d, us, fl in launches]
    for r in rows:
        print(f"attention B={r['B']} heads={r['heads']} nq={r['nq']} nkv={r['nkv']} d={r['d']}: {r['us']:7.1f} us, {r['gflop']:.2f} GFLOP, "
              f"tensor floor {r['tensor_floor_us']:.1f} us", file=sys.stderr)
    shp = f"{u.image_size}x{u.image_size}x{u.in_channels}"
    res = dict(workload=f"{a.model} LDM, classes {classes} x {n}, DDIM-{a.steps} eta 0, scale {scale} (UNet batch {nb} at "
                        f"{shp}), decode_first_stage, random weights",
               images_per_s=len(classes) * n / min(times), run_s=times, unet_eval_ms_graph=unet_ms,
               unet_eval_ms_eager_profiled=eager_ms, attention_us_eager=attn_us,
               attention_share_of_eager_eval=attn_us / 1e3 / eager_ms, attention_launches=rows, **card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
