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
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import arch, pipeline  # noqa: E402
from sdb200.diffusion import LatentDiffusion  # noqa: E402
from measure import card, emit, event_ms, unet_flops, wall_s  # noqa: E402
from txt2img import bert_uncond_ids, synthetic_bert_ids  # noqa: E402


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
        times, img = wall_s(lambda: pipe(ids, un, x_T=x_T), a.repeats)
        assert img.shape == (B, 256, 256, 3)
        c = model.get_learned_conditioning(torch.cat([un, ids]))
        x = torch.randn(2 * B, 3, 64, 64, generator=g, device=dev)
        t = torch.full((2 * B,), 501.0, device=dev)
        unet_ms = event_ms(lambda: u(x, t, context=c), 50, warmup=5)
        flops = unet_flops(arch.TEXT2IMG256_UNET, 2 * B, 64, 64, 77)
        res[f"b{B}"] = dict(images_per_s=B / min(times), run_s=times, unet_batch=2 * B, unet_eval_ms_graph=unet_ms,
                            unet_eval_gflop=flops / 1e9, unet_tflop_per_s=flops / (unet_ms * 1e-3) / 1e12)
        print(f"{B} prompts: {B / min(times):.3f} images/s; UNet eval (batch {2 * B}) {unet_ms:.2f} ms, "
              f"{flops / 1e9:.1f} GFLOP, {flops / (unet_ms * 1e-3) / 1e12:.1f} TFLOP/s", file=sys.stderr)
    res.update(card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
