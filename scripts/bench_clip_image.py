#!/usr/bin/env python
"""Database-building speed of FrozenClipImageEmbedder on the H100 engine: CLIP ViT-L/14 image embeddings per second
(seeded random weights) at batch 64 and 256 from seeded 512² uint8 HWC images resident on the device, preprocessing
included (one sdb_clip_resize_patches launch for the batch, then the tower). Reports, by CUDA events:
  * images/s and the tower's TFLOP/s, with the FLOPs computed from the layer shapes (patch GEMM at K = 588, per layer
    the Q|K, V, out-projection, fc1 and fc2 GEMMs and 4 n^2 d per head of attention, the projection);
  * the preprocessing kernel alone: time per batch and per image, and the bytes it must move per image (the uint8
    source read once, the fp16 patch rows written) with the rate that implies.
Prints one JSON line with the card name and power limit read in the same run; --out also writes it to a file.

  python scripts/bench_clip_image.py --out outputs/clip_image.json
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sdb200  # noqa: E402
from sdb200 import arch  # noqa: E402
from sdb200.clip_image import _table  # noqa: E402
from measure import card, emit, event_ms  # noqa: E402


def tower_flops(cfg):
    """Algorithmic FLOPs of one image through the vision tower and the projection."""
    h, inter, L, P, S = (cfg[k] for k in ("hidden_size", "intermediate_size", "num_hidden_layers", "patch_size",
                                          "image_size"))
    g2 = (S // P) ** 2
    n = g2 + 1
    per_layer = 2 * n * h * (2 * h) + 2 * n * h * h + 4 * n * n * h + 2 * n * h * h + 2 * n * h * inter * 2
    return 2 * g2 * (3 * P * P) * h + L * per_layer + 2 * h * cfg["projection_dim"]


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    p.add_argument("--side", type=int, default=512)
    p.add_argument("--reps", type=int, default=10)
    p.add_argument("--out", type=str, default=None)
    opt = p.parse_args()
    dev = torch.device("cuda")
    cfg = arch.CLIP_VISION_PROJ
    emb = sdb200.FrozenClipImageEmbedder("ViT-L/14", config=cfg)
    emb.load_weights(arch.random_state_dict(emb.shapes, 16, device=dev), dev)
    flops = tower_flops(cfg)
    S, P, kpad = cfg["image_size"], cfg["patch_size"], emb.W["kpad"]
    res = dict(bench="clip_image", **card(), side=opt.side, gflop_per_image=round(flops / 1e9, 2), runs=[])
    g = torch.Generator(device=dev).manual_seed(0)
    for B in opt.batches:
        flat = torch.randint(0, 256, (B * opt.side * opt.side * 3,), dtype=torch.uint8, device=dev, generator=g)
        hw = [(opt.side, opt.side)] * B
        table = _table(hw, 3, flat.numel()).to(dev)
        ms = event_ms(lambda: emb.encode_packed(flat, hw), opt.reps, warmup=2)
        pre_ms = event_ms(lambda: emb.preprocess_patches(flat, table), 5 * opt.reps, warmup=1)
        bytes_img = opt.side * opt.side * 3 + (S // P) ** 2 * kpad * 2
        run = dict(batch=B, ms_per_batch=round(ms, 2), images_per_s=round(B / (ms * 1e-3), 1),
                   tflop_per_s=round(B * flops / (ms * 1e-3) / 1e12, 1),
                   preprocess_us_per_batch=round(pre_ms * 1e3, 1), preprocess_us_per_image=round(pre_ms * 1e3 / B, 3),
                   preprocess_bytes_per_image=bytes_img,
                   preprocess_gb_per_s=round(B * bytes_img / (pre_ms * 1e-3) / 1e9, 1),
                   preprocess_share=round(pre_ms / ms, 4))
        res["runs"].append(run)
        print(f"batch {B}: {run['images_per_s']} img/s, {run['tflop_per_s']} TFLOP/s; preprocess "
              f"{run['preprocess_us_per_batch']} us/batch ({run['preprocess_gb_per_s']} GB/s of {bytes_img} B/image)",
              file=sys.stderr)
        del flat
        torch.cuda.empty_cache()
    emit(res, opt.out)


if __name__ == "__main__":
    main()
