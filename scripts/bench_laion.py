#!/usr/bin/env python
"""LAION-400M text-to-image LDM sampling speed on the H100 engine: the workload of scripts/txt2img.py --laion400m
(512², PLMS-50, guidance scale 7.5, so every UNet evaluation runs a batch of 2B at 64x64x4 with a (77, 1280) BERT
context) at batch 1 and at the reference's default n_samples 3, on seeded random weights. images/s includes the BERT
encode of [""]*B + prompts and decode_first_stage. Also reports, by CUDA events, one graph-replayed UNet evaluation at
each batch and the BERT encode of cond + uncond. Prints one JSON line with the card name and power limit read in the
same run.

  python scripts/bench_laion.py --repeats 3 --out outputs/laion.json
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import pipeline  # noqa: E402
from measure import card, emit, event_ms, wall_s  # noqa: E402
from txt2img import bert_uncond_ids, synthetic_bert_ids  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--batches", type=int, nargs="+", default=[1, 3])
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    dev = torch.device("cuda")
    model = pipeline.build_laion_model()
    pipeline.load_random_weights(model, dev, gen_device=dev)
    model.eval()
    pipe = pipeline.Txt2Img(model, sampler="plms", steps=a.steps, scale=7.5, height=512, width=512)
    u, enc = model.model.diffusion_model, model.cond_stage_model
    res = dict(workload=f"LAION-400M LDM (txt2img --laion400m), 512², PLMS-{a.steps}, scale 7.5, BERT encode and "
                        "decode included, random weights", steps=a.steps)
    for B in a.batches:
        ids, un = synthetic_bert_ids(B, 1234, dev), bert_uncond_ids(B, dev)
        g = torch.Generator(device=dev).manual_seed(0)
        x_T = torch.randn(B, 4, 64, 64, generator=g, device=dev)
        img = pipe(ids, un, x_T=x_T)                            # warm-up: autotune, graph capture, first stage
        torch.cuda.synchronize()
        times, img = wall_s(lambda: pipe(ids, un, x_T=x_T), a.repeats)
        assert img.shape == (B, 512, 512, 3)
        both = torch.cat([un, ids])
        c = model.get_learned_conditioning(both)
        x = torch.randn(2 * B, 4, 64, 64, generator=g, device=dev)
        t = torch.full((2 * B,), 501.0, device=dev)
        unet_ms = event_ms(lambda: u(x, t, context=c), 50, warmup=5)
        bert_ms = event_ms(lambda: enc.encode(both), 20, warmup=3)
        res[f"b{B}"] = dict(images_per_s=B / min(times), run_s=times, unet_eval_ms_graph=unet_ms,
                            unet_batch=2 * B, bert_encode_ms=bert_ms, bert_tokens=tuple(both.shape))
        print(f"batch {B}: {B / min(times):.3f} images/s, UNet eval (batch {2 * B}) {unet_ms:.2f} ms, "
              f"BERT encode {tuple(both.shape)} {bert_ms:.2f} ms", file=sys.stderr)
    res.update(card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
