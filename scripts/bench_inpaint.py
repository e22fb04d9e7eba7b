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
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import arch, ops  # noqa: E402
from sdb200.samplers import DDIMSampler  # noqa: E402
from measure import card, emit, event_ms, unet_flops, wall_s  # noqa: E402


def synthetic_pair(size, seed):
    g = np.random.default_rng(seed)
    image = g.integers(0, 256, (size, size, 3), dtype=np.uint8)
    mask = (g.random((size, size)) < 0.05).astype(np.uint8) * 255
    mask[size // 4: size // 2, size // 3: (2 * size) // 3] = 255
    return image, mask


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
        runs, events = iter(pairs[1:]), []

        def one_image():
            im, mk = next(runs)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            events.append(ev)
            ev[0].record()
            c = torch.empty((1, 4, hc, wc), device=dev)
            c[:, :3].copy_(m.cond_stage_model.encode(ops.inpaint_prepare(im, mk, c, 3)))
            ev[1].record()
            s, _ = sampler.sample(S=a.steps, conditioning=c, batch_size=1, shape=(3, hc, wc), verbose=False)
            ev[2].record()
            x = m.first_stage_model.decode(s, nhwc=True)
            out = ops.inpaint_composite(x, im, mk)
            ev[3].record()
            return out
        times, out = wall_s(one_image, a.repeats)
        split = [[ev[i].elapsed_time(ev[i + 1]) for i in range(3)] for ev in events]
    assert out.shape == (1, a.size, a.size, 3)
    ms = {}
    for nb in (1, 4):       # one graph-replayed UNet evaluation on the concat route
        x = torch.randn(nb, 3, hc, wc, device=dev)
        c = torch.randn(nb, 4, hc, wc, device=dev)
        t = torch.full((nb,), 501.0, device=dev)
        ms[nb] = event_ms(lambda: u(x, t, concat=c), 30, warmup=3)
    one, four = ms[1], ms[4]
    fl = unet_flops(arch.INPAINTING_BIG_UNET, 1, hc, wc)
    best = int(np.argmin(times))
    res = dict(workload=f"inpainting_big LDM, {a.size}x{a.size} image, latent {hc}x{wc}, DDIM-{a.steps} eta 0, batch 1, "
                        "prepare + VQ encode + sampling + VQ decode + composite, random weights",
               images_per_s=1.0 / min(times), run_s=times,
               split_ms=dict(prepare_encode=split[best][0], sampling=split[best][1], decode_composite=split[best][2]),
               unet_eval_ms_graph_b1=one, unet_eval_ms_graph_b4=four, unet_gflop_b1=fl / 1e9,
               unet_tflops_b1=fl / (one * 1e-3) / 1e12, unet_tflops_b4=4 * fl / (four * 1e-3) / 1e12, **card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
