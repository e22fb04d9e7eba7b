#!/usr/bin/env python
"""Text-conditional LDM-VQ-4 (models/ldm/text2img256) sampling speed on the H100 engine, on seeded random weights.

User workload: scripts/txt2img.py --config models/ldm/text2img256/config.yaml --H 256 --W 256 --C 3 --f 4 --scale 5.0
(DDIM-50, eta 0) for 4 and 16 prompts: images/s including the BERT encode of [""]*B + prompts and the VQ-f4 decode with
re-quantization. UNet evaluation: one graph-replayed evaluation at the guidance batches 8 and 32 (CUDA events), with
its FLOP/s from the algorithmic FLOPs counted from the layer shapes below (convolutions, linear layers and attention
matmuls; normalisations and pointwise work are not counted; the cross-attention K / V projections of the context are
left out, because the engine computes them once per context, not per evaluation). Prints one JSON line with the card
name and power limit read in the same run.

  python scripts/bench_text2img256.py --repeats 3 --out outputs/text2img256.json
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import arch, pipeline  # noqa: E402
from sdb200.diffusion import LatentDiffusion  # noqa: E402
from bench_laion import event_ms  # noqa: E402
from bench_lsun import gpu_info  # noqa: E402
from txt2img import bert_uncond_ids, synthetic_bert_ids  # noqa: E402


def unet_flops(cfg, B, h, w, n_ctx):
    """Algorithmic FLOPs (2 per multiply-add) of one UNet evaluation at batch B on an h x w latent, walking arch.unet_plan:
    3x3 convolutions, 1x1 skips, the SpatialTransformers' projections, attention matmuls and feed-forward."""
    plan = arch.unet_plan(cfg)
    conv = lambda hw, cin, cout, k=9: 2 * B * hw * cin * cout * k
    total, ds = 0, 1

    def layer(kind, a, ds):
        hw = (h // ds) * (w // ds)
        if kind == "conv_in":
            return conv(hw, a["cin"], a["cout"])
        if kind == "res":
            f = conv(hw, a["cin"], a["cout"]) + conv(hw, a["cout"], a["cout"])
            return f + (conv(hw, a["cin"], a["cout"], 1) if a["cin"] != a["cout"] else 0)
        if kind == "st":
            c = a["ch"]
            lin = 2 * B * hw * c * c
            # proj_in, proj_out, attn1 q/k/v/out, attn2 q/out, ff (c -> 8c GEGLU, 4c -> c)
            return (2 + 4 + 2 + 12) * lin + 4 * B * hw * hw * c + 4 * B * hw * n_ctx * c
        if kind == "down":
            return conv(hw // 4, a["ch"], a["ch"])
        if kind == "up":
            return conv(hw * 4, a["ch"], a["ch"])
        raise ValueError(kind)

    for layers in plan["input"]:
        for kind, _, a in layers:
            total += layer(kind, a, ds)
            ds *= 2 if kind == "down" else 1
    for kind, _, a in plan["middle"]:
        total += layer(kind, a, ds)
    for layers in plan["output"]:
        for kind, _, a in layers:
            total += layer(kind, a, ds)
            ds //= 2 if kind == "up" else 1
    return total + conv(h * w, plan["out_ch"], cfg["out_channels"])


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--batches", type=int, nargs="+", default=[4, 16])
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    dev = torch.device("cuda")
    # the model node of models/ldm/text2img256/config.yaml
    model = LatentDiffusion(
        first_stage_config={"target": "sdb200.vq.VQModelInterface", "params": arch.VQ_F4},
        cond_stage_config={"target": "sdb200.bert.BERTEmbedder", "params": arch.TEXT2IMG256_BERT},
        unet_config={"target": "sdb200.unet.UNetModel", "params": arch.TEXT2IMG256_UNET},
        linear_start=0.0015, linear_end=0.0195, timesteps=1000, cond_stage_key="caption", conditioning_key="crossattn",
        image_size=64, channels=3)
    pipeline.load_random_weights(model, dev, gen_device=dev)
    model.eval()
    pipe = pipeline.Txt2Img(model, sampler="ddim", steps=a.steps, scale=5.0, height=256, width=256, eta=0.0, f=4,
                            channels=3)
    u = model.model.diffusion_model
    res = dict(workload=f"text2img256 LDM-VQ-4 (txt2img --config models/ldm/text2img256/config.yaml), 256², "
                        f"DDIM-{a.steps}, eta 0, scale 5.0, BERT encode and VQ-f4 decode included, random weights",
               steps=a.steps)
    for B in a.batches:
        ids, un = synthetic_bert_ids(B, 1234, dev), bert_uncond_ids(B, dev)
        g = torch.Generator(device=dev).manual_seed(0)
        x_T = torch.randn(B, 3, 64, 64, generator=g, device=dev)
        img = pipe(ids, un, x_T=x_T)                            # warm-up: autotune, graph capture, first stage
        torch.cuda.synchronize()
        times = []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            img = pipe(ids, un, x_T=x_T)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        assert img.shape == (B, 256, 256, 3)
        c = model.get_learned_conditioning(torch.cat([un, ids]))
        x = torch.randn(2 * B, 3, 64, 64, generator=g, device=dev)
        t = torch.full((2 * B,), 501.0, device=dev)
        for _ in range(5):
            u(x, t, context=c)
        unet_ms = event_ms(lambda: u(x, t, context=c), 50)
        flops = unet_flops(arch.TEXT2IMG256_UNET, 2 * B, 64, 64, 77)
        res[f"b{B}"] = dict(images_per_s=B / min(times), run_s=times, unet_batch=2 * B, unet_eval_ms_graph=unet_ms,
                            unet_eval_gflop=flops / 1e9, unet_tflop_per_s=flops / (unet_ms * 1e-3) / 1e12)
        print(f"{B} prompts: {B / min(times):.3f} images/s; UNet eval (batch {2 * B}) {unet_ms:.2f} ms, "
              f"{flops / 1e9:.1f} GFLOP, {flops / (unet_ms * 1e-3) / 1e12:.1f} TFLOP/s", file=sys.stderr)
    res.update(gpu_info())
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
