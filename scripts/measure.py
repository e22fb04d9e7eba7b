"""What every bench script measures with: the card it ran on, CUDA-event and wall-clock timers, the algorithmic FLOPs of
one UNet evaluation, and the JSON line it prints. Bench scripts import these from here and never from each other."""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sdb200 import arch  # noqa: E402


def card():
    """The card's name, power limit and maximum SM clock, read in the same run as the numbers they go beside."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [v.strip() for v in q.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clk)
    except Exception as e:  # noqa: BLE001
        return dict(gpu=torch.cuda.get_device_name(), power_limit=f"unknown ({e})")


def event_ms(fn, reps, warmup=0):
    """Mean milliseconds per call of fn over reps calls after warmup untimed calls, between two CUDA events recorded in
    stream order (so no synchronize is needed after the warm-up)."""
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def wall_s(fn, repeats):
    """([seconds of each of `repeats` calls of fn, host clock around fn() and a device synchronize], the last call's
    result). The caller runs its warm-up first."""
    times, out = [], None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return times, out


def unet_flops(cfg, nb, h, w, n_ctx=0):
    """Algorithmic FLOPs (2 per multiply-add) of one UNet evaluation at batch nb on an h x w latent, walking
    arch.unet_plan: 3x3 convolutions, 1x1 skips, attention projections, Q K^T and P V over the tokens and the n_ctx
    context tokens, and the spatial transformers' GEGLU feed-forward, the last three once per transformer block. Norms,
    FiLM and pointwise work are not counted, nor are the cross-attention K / V projections of the context, which the
    engine computes once per context, not per evaluation. A layer kind without a count here raises."""
    plan = arch.unet_plan(cfg)
    px, total = h * w, 0

    def conv(cin, cout, k=9):
        return 2 * nb * px * k * cin * cout

    layers = [l for ls in plan["input"] for l in ls] + plan["middle"] + [l for ls in plan["output"] for l in ls]
    for kind, _, a in layers:
        if kind == "down" or kind == "res" and a["updown"] == "down":
            px //= 4
        elif kind == "up" or kind == "res" and a["updown"] == "up":
            px *= 4
        if kind == "conv_in":
            total += conv(a["cin"], a["cout"])
        elif kind == "res":
            total += conv(a["cin"], a["cout"]) + conv(a["cout"], a["cout"])
            total += conv(a["cin"], a["cout"], 1) if a["cin"] != a["cout"] else 0
        elif kind == "attn":            # qkv and proj_out
            total += conv(a["ch"], 4 * a["ch"], 1) + 4 * nb * px * px * a["ch"]
        elif kind == "st":              # proj in / out 2; per block attn1 q k v out 4, attn2 q out 2, ff c -> 8c, 4c -> c 12
            total += conv(a["ch"], (2 + 18 * a["depth"]) * a["ch"], 1) + a["depth"] * 4 * nb * px * (px + n_ctx) * a["ch"]
        elif kind in ("down", "up"):
            total += conv(a["ch"], a["ch"])
        else:
            raise ValueError(f"unet_flops: no FLOP count for layer kind {kind!r}")
    return total + conv(plan["out_ch"], cfg["out_channels"])


def emit(res, out=None):
    """Print res as one JSON line and, when out is a path, write the line to that file too."""
    line = json.dumps(res)
    print(line)
    if out:
        os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
        with open(out, "w") as f:
            f.write(line + "\n")
