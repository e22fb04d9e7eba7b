#!/usr/bin/env python
"""img2img on the H100 engine with the reference script's flags (scripts/img2img.py:60-289):
encode_first_stage -> get_first_stage_encoding -> DDIM stochastic_encode(t_enc) -> decode -> decode_first_stage."""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdb200  # noqa: E402
from sdb200 import pipeline  # noqa: E402
from txt2img import load_model_from_config, synthetic_ids  # noqa: E402


def load_img(path):
    """scripts/img2img.py:48-57: resize to a multiple of 32, scale to [-1, 1], NCHW."""
    from PIL import Image
    image = Image.open(path).convert("RGB")
    w, h = image.size
    w, h = map(lambda x: x - x % 32, (w, h))
    image = image.resize((w, h), resample=Image.LANCZOS)
    image = np.array(image).astype(np.float32) / 255.0
    image = image[None].transpose(0, 3, 1, 2)
    return 2. * torch.from_numpy(image) - 1.


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--prompt", type=str, nargs="?", default="a painting of a virus monster playing guitar")
    p.add_argument("--init-img", type=str, nargs="?", help="path to the input image (random image if omitted)")
    p.add_argument("--outdir", type=str, nargs="?", default="outputs/img2img-samples")
    p.add_argument("--skip_save", action="store_true")
    p.add_argument("--ddim_steps", type=int, default=50)
    p.add_argument("--ddim_eta", type=float, default=0.0)
    p.add_argument("--n_iter", type=int, default=1)
    p.add_argument("--n_samples", type=int, default=2)
    p.add_argument("--scale", type=float, default=5.0)
    p.add_argument("--strength", type=float, default=0.75)
    p.add_argument("--config", type=str, default="configs/stable-diffusion/v1-inference.yaml")
    p.add_argument("--ckpt", type=str, default="models/ldm/stable-diffusion-v1/model.ckpt")
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of a checkpoint")
    p.add_argument("--unsafe-ckpt", action="store_true", help="allow full unpickling of a .ckpt (runs code from the file)")
    p.add_argument("--clip_vocab", type=str, default=None,
                   help="directory with the CLIP vocab.json + merges.txt (host-side BPE); default: transformers' local cache")
    p.add_argument("--size", type=int, default=512, help="side of the synthetic init image when --init-img is omitted")
    opt = p.parse_args()
    torch.manual_seed(opt.seed)
    device = torch.device("cuda")
    model = load_model_from_config(opt.config, opt.ckpt, device, random_init=opt.random_init, unsafe_ckpt=opt.unsafe_ckpt)
    pipe = pipeline.Img2Img(model, steps=opt.ddim_steps, scale=opt.scale, strength=opt.strength, eta=opt.ddim_eta)
    B = opt.n_samples
    if opt.init_img:
        init = load_img(opt.init_img).to(device).repeat(B, 1, 1, 1)
    else:
        init = (torch.rand(B, 3, opt.size, opt.size, device=device) * 2 - 1)
    enc = model.cond_stage_model
    if opt.clip_vocab:
        enc.version, enc.tokenizer = opt.clip_vocab, None
    try:
        ids = enc._tokenize(B * [opt.prompt]).to(device)
        un = enc._tokenize(B * [""]).to(device)
    except RuntimeError as e:
        print(f"tokenizer unavailable ({e}); using seeded token ids")
        ids = synthetic_ids(B, 1234, device)
        un = torch.full((B, 77), 49407, dtype=torch.long, device=device)
        un[:, 0] = 49406
    os.makedirs(opt.outdir, exist_ok=True)
    tic = time.time()
    for n in range(opt.n_iter):
        img = pipe(init, ids, un)
        if not opt.skip_save:
            from PIL import Image
            for i, x in enumerate(img.cpu().numpy()):
                Image.fromarray(x.astype(np.uint8)).save(os.path.join(opt.outdir, f"{n:03}_{i:03}.png"))
    torch.cuda.synchronize()
    print(f"{opt.n_iter * B} images in {time.time() - tic:.2f} s")


if __name__ == "__main__":
    main()
