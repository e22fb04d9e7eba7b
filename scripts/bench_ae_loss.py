#!/usr/bin/env python
"""Speed of the first-stage validation loss on the H100 engine, on seeded random weights: images/s of
AutoencoderKL.validation_step (encode, posterior sample, decode, LPIPS, discriminator on both batches, loss terms) for
KL-f8 at 256^2 batch 16 and 512^2 batch 8, and LPIPS alone in images/s and TFLOP/s, its FLOPs counted here from the
VGG16 layer shapes (both inputs). Wall time to a device synchronize after warm-up. Prints one JSON line with the card
name and power limit read in the same run.

  python scripts/bench_ae_loss.py --repeats 5 --out outputs/ae_loss.json
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdb200  # noqa: E402
from sdb200 import ae_loss, arch  # noqa: E402
from measure import card, emit, wall_s  # noqa: E402


def lpips_flops(nb, h, w):
    """2 * MACs of the 13 VGG16 convs on both inputs of nb pairs (pools halve the sides, floor)."""
    total = 0
    for _, i, cin, cout in ae_loss.VGG16_CONVS:
        if i in (5, 10, 17, 24):
            h, w = h // 2, w // 2
        total += 2 * (2 * nb) * h * w * cout * cin * 9
    return total


def kl_f8(dev):
    m = sdb200.AutoencoderKL(**arch.FIRST_STAGES["kl-f8"])
    m.load_weights(arch.random_state_dict(m.shapes, 12, device=dev), dev)
    loss = sdb200.LPIPSWithDiscriminator(disc_start=50001, kl_weight=1.0e-6, disc_weight=0.5)
    loss.load_state_dict(ae_loss.random_loss_state_dict(ae_loss.loss_param_shapes(), 13))
    object.__setattr__(m, "loss", loss.to(dev).eval())
    return m


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=5)
    p.add_argument("--out")
    a = p.parse_args()
    dev = torch.device("cuda:0")
    res = card()
    m = kl_f8(dev)
    g = torch.Generator().manual_seed(0)
    for size, nb in ((256, 16), (512, 8)):
        batch = {"image": torch.rand(nb, size, size, 3, generator=g) * 2 - 1}
        step = lambda: m.validation_step(batch, 0)
        step()
        times, log = wall_s(step, a.repeats)
        res[f"validation_step_{size}_b{nb}_images_per_s"] = round(nb / min(times), 2)
        res[f"validation_step_{size}_b{nb}_rec_loss"] = float(log["val/rec_loss"])
        x0 = torch.rand(nb, 3, size, size, generator=g, device="cpu").to(dev) * 2 - 1
        x1 = torch.rand(nb, 3, size, size, generator=g, device="cpu").to(dev) * 2 - 1
        lp = m.loss.perceptual_loss
        lp(x0, x1)
        times, _ = wall_s(lambda: lp(x0, x1), a.repeats)
        t = min(times)
        res[f"lpips_{size}_b{nb}_images_per_s"] = round(nb / t, 2)
        res[f"lpips_{size}_b{nb}_tflops"] = round(lpips_flops(nb, size, size) / t / 1e12, 1)
        res[f"lpips_{size}_b{nb}_ms"] = round(1e3 * t, 3)
    emit(res, a.out)


if __name__ == "__main__":
    main()
