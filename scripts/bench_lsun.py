#!/usr/bin/env python
"""LSUN-Churches sampling speed on the H100 engine: scripts/sample_diffusion.py's default workload (256^2 images,
DDIM 50 steps, eta 1.0, batch 10) on seeded random weights, plus the time of one UNet evaluation from CUDA events.
Prints one JSON line with the card name and power limit read in the same run.

  python scripts/bench_lsun.py --batches 3 --out outputs/lsun.json
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sdb200 import pipeline  # noqa: E402
from sdb200.samplers import DDIMSampler  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402
from measure import card, emit, event_ms, wall_s  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batches", type=int, default=3)
    p.add_argument("--batch_size", type=int, default=10)
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--eta", type=float, default=1.0)
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import sample_diffusion as S
    dev = torch.device("cuda")
    m = instantiate_from_config(remap_config(S.lsun_churches_config()))
    m = pipeline.load_random_weights(m, dev, gen_device=dev).eval()
    u = m.model.diffusion_model
    m.scale_factor.fill_(0.22)
    u.use_cuda_graph = True
    shape = [a.batch_size, 4, 32, 32]
    sampler = DDIMSampler(m)

    def one_batch():
        with m.ema_scope():
            s, _ = sampler.sample(a.steps, batch_size=a.batch_size, shape=shape[1:], eta=a.eta, verbose=False)
        img = m.decode_first_stage(s)
        return img
    torch.manual_seed(0)
    one_batch()                       # warm-up: autotune, graph capture, VAE
    torch.cuda.synchronize()
    times, img = wall_s(one_batch, a.batches)
    assert img.shape == (a.batch_size, 3, 256, 256) and bool(torch.isfinite(img).all())
    # one UNet evaluation (graph replay) by CUDA events over many launches
    x = torch.randn(shape, device=dev)
    t = torch.full((a.batch_size,), 501.0, device=dev)
    unet_ms = event_ms(lambda: u(x, t), 50, warmup=5)
    res = dict(workload=f"LSUN-Churches 256x256 DDIM-{a.steps} eta={a.eta} batch {a.batch_size} (random weights), "
                        "sampling + decode_first_stage",
               images_per_s=a.batch_size / min(times), batch_s=times, unet_eval_ms=unet_ms, **card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
