#!/usr/bin/env python
"""CelebA-HQ (VQ-f4 LDM) sampling speed on the H100 engine: scripts/sample_diffusion.py with the reference README's
CelebA-HQ settings (256^2 images, DDIM 50 steps, eta 0, batch 10) on seeded random weights, decode_first_stage included.
Also reports one UNet evaluation (graph replay, CUDA events) and the share of it spent in GEMMs whose K carries padded
64-wide steps (A sources 224, 672, ... channels wide), from per-GEMM CUDA events of one eager evaluation.
Prints one JSON line with the card name and power limit read in the same run. FFHQ and LSUN-Bedrooms run the same
network and first stage.

  python scripts/bench_celebahq.py --batches 3 --out outputs/celebahq.json
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import ops, pipeline  # noqa: E402
from sdb200.samplers import DDIMSampler  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402
from measure import card, emit, event_ms, wall_s  # noqa: E402


def padded_gemm_share(u, x, t):
    """(ms in GEMMs with a padded K step, ms in all GEMMs) of one eager evaluation, from per-launch CUDA events."""
    ops.PROFILE, ops.RECORD = [], []
    try:
        u(x, t)
        torch.cuda.synchronize()
        prof = [p for p in ops.PROFILE if p[0] == "gemm"]
        rec = ops.RECORD
    finally:
        ops.PROFILE, ops.RECORD = None, None
    assert len(prof) == len(rec)
    padded = total = 0.0
    for p, (d, _, _) in zip(prof, rec):
        ms = p[2].elapsed_time(p[3])
        total += ms
        if any(c % 64 for c in (d.c0, d.c1, d.c2, d.c3) if c):
            padded += ms
    return padded, total


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batches", type=int, default=3)
    p.add_argument("--batch_size", type=int, default=10)
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--eta", type=float, default=0.0)
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    import sample_diffusion as S
    dev = torch.device("cuda")
    m = instantiate_from_config(remap_config(S.celebahq_config()))
    m = pipeline.load_random_weights(m, dev, gen_device=dev).eval()
    u = m.model.diffusion_model
    u.use_cuda_graph = True
    shape = [a.batch_size, 3, 64, 64]
    sampler = DDIMSampler(m)

    def one_batch():
        with m.ema_scope():
            s, _ = sampler.sample(a.steps, batch_size=a.batch_size, shape=shape[1:], eta=a.eta, verbose=False)
        return m.decode_first_stage(s)
    torch.manual_seed(0)
    one_batch()                       # warm-up: autotune, graph capture, first stage
    torch.cuda.synchronize()
    times, img = wall_s(one_batch, a.batches)
    assert img.shape == (a.batch_size, 3, 256, 256) and bool(torch.isfinite(img).all())
    x = torch.randn(shape, device=dev)
    t = torch.full((a.batch_size,), 501.0, device=dev)
    unet_ms = event_ms(lambda: u(x, t), 50, warmup=5)
    # first stage alone: decode of one batch of latents
    z = torch.randn(shape, device=dev)
    dec_ms = event_ms(lambda: m.decode_first_stage(z), 3, warmup=1)
    u.use_cuda_graph = False
    padded_ms, gemm_ms = padded_gemm_share(u, x, t)
    res = dict(workload=f"CelebA-HQ VQ-f4 LDM 256x256 DDIM-{a.steps} eta={a.eta} batch {a.batch_size} (random weights), "
                        "sampling + decode_first_stage",
               images_per_s=a.batch_size / min(times), batch_s=times, unet_eval_ms=unet_ms, decode_ms=dec_ms,
               eager_gemm_ms=gemm_ms, eager_padded_k_gemm_ms=padded_ms, padded_k_share_of_unet_eval=padded_ms / unet_ms,
               **card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
