"""Validation loss of a KL first stage (AutoencoderKL.validation_step, autoencoder.py:372-383) on the H100 engine:
reconstruct through the sampled posterior, then LPIPSWithDiscriminator's two calls (LPIPS over VGG16, the PatchGAN
discriminator, KL), printing the val/* dict averaged over the batches, as Lightning averages it over a validation epoch.

The loss is built from the YAML's lossconfig and loaded from the checkpoint's loss.* tensors; global_step (which sets
disc_factor against disc_start) is the checkpoint's, or --global_step. Images come from --indir (center-cropped and
resized to --size, x / 127.5 - 1) or, without it, a seeded synthetic batch. Posterior sampling is for 4 latent channels
(KL-f8, autoencoder_kl_32x32x4).

    python scripts/eval_autoencoder.py --config models/first_stage_models/kl-f8/config.yaml --ckpt model.ckpt \
        --indir images/ --batch_size 8
    python scripts/eval_autoencoder.py --config models/first_stage_models/kl-f8/config.yaml --random_init --size 64
"""
from __future__ import annotations

import argparse
import glob
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdb200  # noqa: E402
from sdb200 import ae_loss, arch, checkpoint  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402

IMAGE_EXTS = (".png", ".jpg", ".jpeg")


def load(config, ckpt=None, random_init=False, seed=0, device="cuda"):
    """(AutoencoderKL with its loss attached). random_init: seeded weights for the stage and the loss."""
    node = checkpoint.load_config(config)
    if random_init:
        model = instantiate_from_config(remap_config(node))
        model.load_weights(arch.random_state_dict(model.shapes, seed), device)
        loss = instantiate_from_config(remap_config(node["params"]["lossconfig"]))
        loss.load_state_dict(ae_loss.random_loss_state_dict(ae_loss.loss_param_shapes(
            loss.discriminator.n_layers, loss.discriminator.layers[0][1]), seed + 1))
        loss = loss.to(device).eval()
        object.__setattr__(model, "loss", loss)
    else:
        model = checkpoint.load_model_from_config(config, ckpt, device=device)
        checkpoint.load_first_stage_loss(model, config, ckpt, device=device)
    if not isinstance(model, sdb200.AutoencoderKL):
        raise SystemExit(f"{node['target']}: eval_autoencoder.py takes a KL first stage (AutoencoderKL)")
    return model


def image_batches(indir, size, batch_size):
    from PIL import Image
    paths = sorted(p for p in glob.glob(os.path.join(indir, "*")) if p.lower().endswith(IMAGE_EXTS))
    if not paths:
        raise SystemExit(f"no {'/'.join(IMAGE_EXTS)} images in {indir}")
    imgs = []
    for p in paths:
        im = Image.open(p).convert("RGB")
        s = min(im.size)
        left, top = (im.size[0] - s) // 2, (im.size[1] - s) // 2
        im = im.crop((left, top, left + s, top + s)).resize((size, size), Image.BICUBIC)
        imgs.append(torch.from_numpy(np.array(im)))
    for i in range(0, len(imgs), batch_size):
        yield torch.stack(imgs[i:i + batch_size])


def synthetic_batches(n_batches, batch_size, size, seed):
    g = torch.Generator().manual_seed(seed)
    for _ in range(n_batches):
        yield torch.randint(0, 256, (batch_size, size, size, 3), generator=g, dtype=torch.uint8)


def get_parser():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--config", required=True, help="KL first-stage YAML (with its lossconfig)")
    p.add_argument("--ckpt", help="checkpoint with the stage's and the loss's (loss.*) tensors")
    p.add_argument("--random_init", action="store_true", help="seeded stand-in weights instead of a checkpoint")
    p.add_argument("--indir", help="folder of images; default: a seeded synthetic batch")
    p.add_argument("--size", type=int, default=256)
    p.add_argument("--batch_size", type=int, default=4)
    p.add_argument("--n_batches", type=int, default=1, help="synthetic batches")
    p.add_argument("--global_step", type=int, help="override the checkpoint's global_step")
    p.add_argument("--seed", type=int, default=42, help="weights (random_init), synthetic images and posterior noise")
    return p


def main(argv=None):
    opt = get_parser().parse_args(argv)
    if not opt.random_init and not opt.ckpt:
        raise SystemExit("give --ckpt or --random_init")
    model = load(opt.config, opt.ckpt, opt.random_init, opt.seed)
    if opt.global_step is not None:
        model.global_step = opt.global_step
    batches = (image_batches(opt.indir, opt.size, opt.batch_size) if opt.indir
               else synthetic_batches(opt.n_batches, opt.batch_size, opt.size, opt.seed))
    torch.manual_seed(opt.seed)   # the posterior draws its noise on the CPU generator
    sums, n = {}, 0
    for i, u8 in enumerate(batches):
        log = model.validation_step({model.image_key: u8.float() / 127.5 - 1.0}, i)
        for k, v in log.items():
            sums[k] = sums.get(k, 0.0) + float(v)
        n += 1
    res = {k: v / n for k, v in sums.items()}
    print(json.dumps({"batches": n, "global_step": model.global_step, **res}))
    return res


if __name__ == "__main__":
    main()
