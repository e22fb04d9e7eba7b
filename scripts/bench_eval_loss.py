#!/usr/bin/env python
"""Speed of the denoising-loss evaluation (LatentDiffusion.p_losses after the first-stage encode) on the H100 engine,
on seeded random weights: images/s of encode + posterior sample + per-sample-t noising + UNet + loss for SD-v1 at
512^2 (batch 8 and 32; the text context is encoded once outside the timed loop) and LSUN-Churches at 256^2 (batch 32),
and the per-launch time of the two loss kernels (sdb_q_sample_t, sdb_diffusion_loss) at SD-v1's batch-32 latent, from
CUDA events after warm-up. Prints one JSON line with the card name and power limit read in the same run.

  python scripts/bench_eval_loss.py --repeats 5 --out outputs/eval_loss.json
"""
import argparse
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sdb200 import ops, pipeline  # noqa: E402
from sdb200 import lib as _l  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402
from measure import card, emit, event_ms, wall_s  # noqa: E402


def sd_model(dev):
    m = pipeline.build_model()
    pipeline.load_random_weights(m, dev, gen_device=dev)
    return m.eval()


def lsun_model(dev):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import sample_diffusion as S
    m = instantiate_from_config(remap_config(S.lsun_churches_config()))
    m = pipeline.load_random_weights(m, dev, gen_device=dev).eval()
    m.scale_factor.fill_(0.22)
    return m


def images_per_s(m, nb, size, cond, repeats):
    dev = m.device
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand((nb, 3, size, size), generator=g, device=dev) * 2 - 1
    c = None if cond is None else cond.expand(nb, -1, -1).contiguous()
    m.model.diffusion_model.use_cuda_graph = True

    def step():
        z = m.get_first_stage_encoding(m.encode_first_stage(x))
        t = torch.randint(0, m.num_timesteps, (nb,), device=dev)
        return m.p_losses(z, c, t)[0]
    step()                                          # warm-up: autotune, graph capture
    torch.cuda.synchronize()
    times, loss = wall_s(step, repeats)
    assert torch.isfinite(loss)
    return nb / min(times), times


def kernel_us(dev, shape):
    """Per-launch microseconds of the two kernels through the C entry points (the ops wrappers add a host check of t)."""
    g = torch.Generator(device=dev).manual_seed(1)
    x, n = (torch.randn(shape, generator=g, device=dev) for _ in range(2))
    t = torch.randint(0, 1000, (shape[0],), generator=g, device=dev)
    tab = torch.rand(1000, generator=g, device=dev)
    out = torch.empty_like(x)
    loss = torch.empty((3, shape[0]), device=dev)
    L, s = _l.load(), lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda v: C.c_void_p(v.data_ptr())
    nb, per = shape[0], x[0].numel()
    q = event_ms(lambda: L.sdb_q_sample_t(P(x), P(n), P(t), P(tab), P(tab), nb, per, P(out), s()), 200, warmup=20)
    lo = event_ms(lambda: L.sdb_diffusion_loss(P(x), P(n), 2, P(t), P(tab), P(tab), nb, per, P(loss), s()), 200,
                  warmup=20)
    ops.diffusion_loss(x, n, "l2", t, tab, tab)          # the checked path runs too
    return q * 1e3, lo * 1e3


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=5)
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    dev = torch.device("cuda")
    res = {"workload": "p_losses after the first-stage encode (encode + posterior sample + q_sample_t + UNet + loss), "
                       "random weights, random t per sample"}
    sd = sd_model(dev)
    ids = torch.randint(0, 49406, (1, 77), generator=torch.Generator().manual_seed(2)).to(dev)
    ctx = sd.get_learned_conditioning(ids)
    for nb in (8, 32):
        ips, times = images_per_s(sd, nb, 512, ctx, a.repeats)
        res[f"sd_v1_512_b{nb}_images_per_s"], res[f"sd_v1_512_b{nb}_s"] = ips, times
    del sd
    torch.cuda.empty_cache()
    lsun = lsun_model(dev)
    ips, times = images_per_s(lsun, 32, 256, None, a.repeats)
    res["lsun_256_b32_images_per_s"], res["lsun_256_b32_s"] = ips, times
    res["q_sample_t_us"], res["diffusion_loss_us"] = kernel_us(dev, (32, 4, 64, 64))
    res.update(card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
