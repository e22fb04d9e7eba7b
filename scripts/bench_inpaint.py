#!/usr/bin/env python
"""LDM inpainting (models/ldm/inpainting_big) speed on the H100 engine: the reference workload of scripts/inpaint.py at
512x512 (latent 128x128, DDIM-50, eta 0, batch 1, prepare + VQ encode + sampling + VQ decode + composite) on seeded
random weights and seeded synthetic image / mask pairs (a rectangle plus scattered pixels).
Also reports one graph-replayed UNet evaluation on the concat route at (1, 3 + 4, 128, 128) and (4, 3 + 4, 128, 128)
(CUDA events), the split of one image's time into prepare + encode / sampling / decode + composite, the FLOPs of one UNet
evaluation at batch 1 from the layer shapes (convolutions, 1x1 projections and attention matmuls) and the achieved
TFLOP/s. Prints one JSON line with the card name and power limit read in the same run.

  python scripts/bench_inpaint.py --repeats 3 --out outputs/inpaint.json
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import arch, ops  # noqa: E402
from sdb200.samplers import DDIMSampler  # noqa: E402
from bench_lsun import gpu_info  # noqa: E402


def unet_flops(cfg, h, w, nb=1):
    """Multiply-adds x 2 of one UNet evaluation: 3x3 / 1x1 convolutions and the attention blocks' projections, Q K^T and
    P V (norms, FiLM and elementwise work are not counted)."""
    plan = arch.unet_plan(cfg)
    conv = lambda cin, cout, px, k=9: 2 * k * cin * cout * px
    fl, px = 0, h * w

    def walk(layers):
        nonlocal fl, px
        for kind, _, a in layers:
            if kind == "conv_in":
                fl += conv(a["cin"], a["cout"], px)
            elif kind == "res":
                if a["updown"] == "down":
                    px //= 4
                elif a["updown"] == "up":
                    px *= 4
                fl += conv(a["cin"], a["cout"], px) + conv(a["cout"], a["cout"], px)
                if a["cin"] != a["cout"]:
                    fl += conv(a["cin"], a["cout"], px, 1)
            elif kind == "attn":
                ch = a["ch"]
                fl += conv(ch, 3 * ch, px, 1) + conv(ch, ch, px, 1) + 2 * 2 * px * px * ch
            elif kind == "down":
                px //= 4
                fl += conv(a["ch"], a["ch"], px)
            elif kind == "up":
                px *= 4
                fl += conv(a["ch"], a["ch"], px)

    for layers in plan["input"]:
        walk(layers)
    walk(plan["middle"])
    for layers in plan["output"]:
        walk(layers)
    fl += conv(plan["out_ch"], cfg["out_channels"], px)
    return nb * fl


def synthetic_pair(size, seed):
    g = np.random.default_rng(seed)
    image = g.integers(0, 256, (size, size, 3), dtype=np.uint8)
    mask = (g.random((size, size)) < 0.05).astype(np.uint8) * 255
    mask[size // 4: size // 2, size // 3: (2 * size) // 3] = 255
    return image, mask


def unet_ms(u, nb, hc, wc, dev, reps=30):
    x = torch.randn(nb, 3, hc, wc, device=dev)
    c = torch.randn(nb, 4, hc, wc, device=dev)
    t = torch.full((nb,), 501.0, device=dev)
    for _ in range(3):
        u(x, t, concat=c)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        u(x, t, concat=c)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--size", type=int, default=512)
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    import inpaint as S
    dev = torch.device("cuda")
    m = S.load_model(random_init=True)
    u = m.model.diffusion_model
    u.use_cuda_graph = True
    sampler = DDIMSampler(m)
    pairs = [synthetic_pair(a.size, i) for i in range(a.repeats + 1)]
    pairs = [(torch.from_numpy(i)[None].to(dev), torch.from_numpy(k)[None].to(dev)) for i, k in pairs]
    hc, wc = S.latent_size(m, a.size, a.size)
    torch.manual_seed(0)
    with m.ema_scope():
        S.inpaint(m, sampler, *pairs[0], steps=a.steps)        # warm-up: autotune, graph capture, first stage
        torch.cuda.synchronize()
        times, split = [], []
        for im, mk in pairs[1:]:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            t0 = time.perf_counter()
            ev[0].record()
            c = torch.empty((1, 4, hc, wc), device=dev)
            c[:, :3].copy_(m.cond_stage_model.encode(ops.inpaint_prepare(im, mk, c, 3)))
            ev[1].record()
            s, _ = sampler.sample(S=a.steps, conditioning=c, batch_size=1, shape=(3, hc, wc), verbose=False)
            ev[2].record()
            x = m.first_stage_model.decode(s, nhwc=True)
            out = ops.inpaint_composite(x, im, mk)
            ev[3].record()
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            split.append([ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
    assert out.shape == (1, a.size, a.size, 3)
    one = unet_ms(u, 1, hc, wc, dev)
    four = unet_ms(u, 4, hc, wc, dev)
    fl = unet_flops(arch.INPAINTING_BIG_UNET, hc, wc)
    best = int(np.argmin(times))
    res = dict(workload=f"inpainting_big LDM, {a.size}x{a.size} image, latent {hc}x{wc}, DDIM-{a.steps} eta 0, batch 1, "
                        "prepare + VQ encode + sampling + VQ decode + composite, random weights",
               images_per_s=1.0 / min(times), run_s=times,
               split_ms=dict(prepare_encode=split[best][0], sampling=split[best][1], decode_composite=split[best][2]),
               unet_eval_ms_graph_b1=one, unet_eval_ms_graph_b4=four, unet_gflop_b1=fl / 1e9,
               unet_tflops_b1=fl / (one * 1e-3) / 1e12, unet_tflops_b4=4 * fl / (four * 1e-3) / 1e12, **gpu_info())
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
