"""Encode and reconstruct images with a first-stage autoencoder of models/first_stage_models/*/config.yaml (KL-f4 / f8
/ f16 / f32, VQ-f4 / f4-noattn / f8 / f8-n256 / f16), from the reference's YAML unchanged.

Images are preprocessed as the reference's data modules do (x / 127.5 - 1, NCHW). Reconstructions are written as PNG:
for a KL first stage the decode of the posterior mode, for a VQ first stage VQModel.forward's dec (encode, quantize,
decode). With --save_latents a latents.pt is written too: the KL posterior mean, or the VQ pre-quant latent and the
code indices (flat over b*h*w of each image, as VQModel.encode returns them), keyed by output name.

    python scripts/autoencode.py --config models/first_stage_models/vq-f16/config.yaml --ckpt model.ckpt \
        --indir images/ --outdir outputs/autoencode --save_latents
    python scripts/autoencode.py --config models/first_stage_models/kl-f32/config.yaml --random_init --n_samples 2
"""
from __future__ import annotations

import argparse
import glob
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdb200  # noqa: E402
from sdb200 import arch, checkpoint  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402

IMAGE_EXTS = (".png", ".jpg", ".jpeg")


def downsampling_factor(node):
    """2^(levels - 1): every Encoder level but the last halves the image (model.py:368-432)."""
    return 2 ** (len(node["params"]["ddconfig"]["ch_mult"]) - 1)


def check_size(h, w, f, what="image"):
    if h % f or w % f or h <= 0 or w <= 0:
        raise ValueError(f"{what}: {h}x{w} is not a multiple of the first stage's downsampling factor {f} in both sides")


def preprocess(u8):
    """uint8 [n, H, W, 3] -> fp32 NCHW in [-1, 1] (x / 127.5 - 1)."""
    return (u8.float() / 127.5 - 1.0).permute(0, 3, 1, 2).contiguous()


def to_uint8(x):
    """fp32 NCHW -> uint8 [n, H, W, 3]: clamp to [-1, 1], (x + 1) / 2, 255 * x truncated (custom_to_pil)."""
    x = (torch.clamp(x.detach().float().cpu(), -1.0, 1.0) + 1.0) / 2.0
    return (255 * x.permute(0, 2, 3, 1)).numpy().astype(np.uint8)


def load_model(config, ckpt=None, random_init=False, seed=0, device="cuda"):
    node = checkpoint.load_config(config)
    if random_init:
        model = instantiate_from_config(remap_config(node))
        model.load_weights(arch.random_state_dict(model.shapes, seed), device)
    else:
        model = checkpoint.load_model_from_config(config, ckpt, device=device)
    if not isinstance(model, (sdb200.AutoencoderKL, sdb200.VQModel)) or isinstance(model, sdb200.VQModelInterface):
        raise ValueError(f"{node['target']} is not a first-stage autoencoder (AutoencoderKL or VQModel)")
    return model, node


@torch.no_grad()
def reconstruct(model, x, save_latents=False):
    """(reconstruction NCHW fp32, latents dict or None) of the fp32 NCHW batch x on the model's device."""
    if isinstance(model, sdb200.AutoencoderKL):
        post = model.encode(x)
        mode = post.mode()
        return model.decode(mode), ({"mean": mode.cpu()} if save_latents else None)
    dec, _, ind = model(x, return_pred_indices=True)
    lat = {"h": model.encode_to_prequant(x).cpu(), "indices": ind.cpu()} if save_latents else None
    return dec, lat


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--config", type=str, required=True, help="first-stage YAML (models/first_stage_models/*/config.yaml)")
    p.add_argument("--ckpt", type=str, default=None, help="its checkpoint (.ckpt / .safetensors)")
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of a checkpoint")
    p.add_argument("--indir", type=str, default=None, help="dir of images (.png / .jpg); default: a synthetic batch")
    p.add_argument("--n_samples", type=int, default=4, help="synthetic batch size")
    p.add_argument("--H", type=int, default=256, help="synthetic image height")
    p.add_argument("--W", type=int, default=256, help="synthetic image width")
    p.add_argument("--seed", type=int, default=42, help="seed of the random weights and of the synthetic batch")
    p.add_argument("--outdir", type=str, default="outputs/autoencode", help="dir to write results to")
    p.add_argument("--save_latents", action="store_true", help="also write latents.pt")
    return p


def check_args(opt):
    """The argument and size checks, all before anything is built. Returns (node, inputs): inputs is a list of
    (name, uint8 [1, H, W, 3]) per image of --indir, or one ("synthetic", uint8 [n, H, W, 3]) batch."""
    if opt.random_init == (opt.ckpt is not None):
        raise ValueError("pass --ckpt, or --random_init")
    node = checkpoint.load_config(opt.config)
    f = downsampling_factor(node)
    if opt.indir is None:
        if opt.n_samples < 1:
            raise ValueError("--n_samples must be at least 1")
        check_size(opt.H, opt.W, f, "--H x --W")
        g = torch.Generator().manual_seed(opt.seed + 1)
        return node, [("synthetic", torch.randint(0, 256, (opt.n_samples, opt.H, opt.W, 3), generator=g,
                                                  dtype=torch.uint8))]
    from PIL import Image
    paths = sorted(p for p in glob.glob(os.path.join(opt.indir, "*")) if p.lower().endswith(IMAGE_EXTS))
    if not paths:
        raise ValueError(f"no .png / .jpg images in {opt.indir}")
    inputs = []
    for path in paths:
        u8 = torch.from_numpy(np.array(Image.open(path).convert("RGB")))[None]
        check_size(u8.shape[1], u8.shape[2], f, path)
        inputs.append((os.path.splitext(os.path.basename(path))[0], u8))
    return node, inputs


def main(argv=None):
    from PIL import Image
    opt = get_parser().parse_args(argv)
    _, inputs = check_args(opt)
    model, node = load_model(opt.config, opt.ckpt, opt.random_init, opt.seed)
    dev = model.W["device"]
    os.makedirs(opt.outdir, exist_ok=True)
    written, latents = [], {}
    t0 = time.time()
    for name, u8 in inputs:
        x = preprocess(u8).to(dev)
        dec, lat = reconstruct(model, x, opt.save_latents)
        for i, img in enumerate(to_uint8(dec)):
            out_name = name if u8.shape[0] == 1 else f"{name}_{i:04d}"
            outpath = os.path.join(opt.outdir, out_name + ".png")
            Image.fromarray(img).save(outpath)
            written.append(outpath)
        if lat is not None:
            latents[name] = lat
        print(f"{name}: {tuple(x.shape)} -> {tuple(dec.shape)}")
    if opt.save_latents:
        torch.save(latents, os.path.join(opt.outdir, "latents.pt"))
    print(f"{node['target']}: {len(written)} reconstructions in {time.time() - t0:.2f} s, written to {opt.outdir}")
    return written


if __name__ == "__main__":
    main()
