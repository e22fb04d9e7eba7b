"""Encode and decode throughput of the nine first-stage autoencoders of models/first_stage_models/* (seeded random
weights, 256x256 images, batch 16): images/s from CUDA events around `--iters` calls after `--warmup` calls, each
phase timed on its own. KL: encode = the posterior parameters, decode = decode(mean); VQ: encode = VQModel.encode
(quantized latent, indices, emb_loss), decode = VQModel.decode(quant). The card's name and power limit are printed in
the same run. One JSON line per config.

    python scripts/bench_first_stage.py [--batch 16] [--size 256] [--iters 10] [--warmup 3] [--only kl-f32 vq-f16]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdb200  # noqa: E402
from sdb200 import arch  # noqa: E402
from measure import card, event_ms  # noqa: E402


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=16)
    p.add_argument("--size", type=int, default=256)
    p.add_argument("--iters", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--only", nargs="*", default=None, help="config names (default: all nine)")
    opt = p.parse_args(argv)
    assert torch.cuda.is_available(), "bench_first_stage needs a CUDA device"
    dev = torch.device("cuda")
    c = card()
    print(f"# {c['gpu']}, {c['power_limit']}", flush=True)
    x = torch.randn(opt.batch, 3, opt.size, opt.size, generator=torch.Generator().manual_seed(0)).clamp(-1, 1).to(dev)
    for name in opt.only or sorted(arch.FIRST_STAGES):
        cfg = arch.FIRST_STAGES[name]
        if "n_embed" in cfg:
            model = sdb200.VQModel(**cfg)
            model.load_weights(arch.random_state_dict(model.shapes, 7, device=dev), dev)
            quant = model.encode(x)[0]
            enc, dec = (lambda: model.encode(x)), (lambda: model.decode(quant))
        else:
            model = sdb200.AutoencoderKL(**cfg)
            model.load_weights(arch.random_state_dict(model.shapes, 7, device=dev), dev)
            mean = model.encode(x).mean
            enc, dec = (lambda: model.encode(x).parameters), (lambda: model.decode(mean))
        te, td = (event_ms(fn, opt.iters, opt.warmup) / 1e3 for fn in (enc, dec))
        print(json.dumps({"config": name, "batch": opt.batch, "size": opt.size, "encode_img_s": round(opt.batch / te, 1),
                          "decode_img_s": round(opt.batch / td, 1), "encode_ms": round(te * 1e3, 2),
                          "decode_ms": round(td * 1e3, 2)}), flush=True)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
