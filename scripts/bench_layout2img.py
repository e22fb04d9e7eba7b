#!/usr/bin/env python
"""Layout-to-image LDM (models/ldm/layout2img-openimages256) sampling speed on the H100 engine, on seeded random weights.

User workload: scripts/layout2img.py at its defaults (LatentDiffusion.log_images' sampling: 256², DDIM-200, eta 1,
unguided, inside ema_scope()) for batches of 8 (log_images' N) and 24 (the config's batch size): images/s including the
BERT-512 encode of the 92 layout ids and the VQ-f4 decode with re-quantization. UNet evaluation: one graph-replayed
evaluation at each batch (CUDA events), with its FLOP/s from measure.unet_flops on the 92-token context. Prints one JSON
line with the card name and power limit read in the same run.

  python scripts/bench_layout2img.py --repeats 3 --out outputs/layout2img.json
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import arch, pipeline  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402
from layout2img import decode, layout2img_config, sample_latents, stand_in_ids  # noqa: E402
from measure import card, emit, event_ms, unet_flops, wall_s  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--batches", type=int, nargs="+", default=[8, 24])
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    dev = torch.device("cuda")
    model = instantiate_from_config(remap_config(layout2img_config()))
    pipeline.load_random_weights(model, dev, gen_device=dev)
    model.eval()
    u = model.model.diffusion_model
    u.use_cuda_graph = True
    res = dict(workload=f"layout2img-openimages256 LDM-VQ-4 (scripts/layout2img.py), 256², DDIM-{a.steps}, eta 1, "
                        f"unguided, BERT encode and VQ-f4 decode included, random weights", steps=a.steps)
    for B in a.batches:
        ids = stand_in_ids(model.cond_stage_model, B, 42)
        run = lambda: decode(model, sample_latents(model, ids, a.steps, 1.0))
        img = run()                                             # warm-up: autotune, graph capture, first stage
        torch.cuda.synchronize()
        times, img = wall_s(run, a.repeats)
        assert img.shape == (B, 3, 256, 256)
        c = model.get_learned_conditioning(ids.to(dev))
        g = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(B, 3, 64, 64, generator=g, device=dev)
        t = torch.full((B,), 501.0, device=dev)
        unet_ms = event_ms(lambda: u(x, t, context=c), 50, warmup=5)
        flops = unet_flops(arch.LAYOUT2IMG_UNET, B, 64, 64, 92)
        res[f"b{B}"] = dict(images_per_s=B / min(times), run_s=times, unet_batch=B, unet_eval_ms_graph=unet_ms,
                            unet_eval_gflop=flops / 1e9, unet_tflop_per_s=flops / (unet_ms * 1e-3) / 1e12)
        print(f"batch {B}: {B / min(times):.3f} images/s; UNet eval {unet_ms:.2f} ms, {flops / 1e9:.1f} GFLOP, "
              f"{flops / (unet_ms * 1e-3) / 1e12:.1f} TFLOP/s", file=sys.stderr)
    res.update(card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
