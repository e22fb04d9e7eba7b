#!/usr/bin/env python
"""The denoising loss of an LDM on a set of images (the val/loss_simple, val/loss_vlb and val/loss numbers main.py logs
for the reference, with their _ema twins), e.g.

  python scripts/eval_loss.py --config configs/latent-diffusion/lsun_churches-ldm-kl-8.yaml \
      --ckpt models/ldm/lsun_churches256/model.ckpt --indir data/churches --n_samples 512

Default mode: the reference's objective, validation_step on each batch: one uniformly drawn t and one noise draw per
image, on the raw weights and again inside ema_scope() on the EMA weights (each with its own draws, as the reference).
With --timesteps 0,250,500,750,999 every image is evaluated at every listed t with one shared noise draw per image,
raw and EMA, giving a loss-against-timestep table.

Images: --indir (PNG / JPEG, resized to the model's image size and scaled to [-1, 1]) or a seeded synthetic batch.
Conditioning by the config's cond_stage_key: none (unconditional models), `class_label` (--class_label, or a labels
file of one integer per image, or seeded labels), or `caption` (--from-file, one caption per line, tokenized by the
cond stage; --clip_vocab / --bert_vocab as in txt2img.py). With --random_init every stage gets seeded random weights.
Writes a JSON file (--out) and prints a summary.
"""
import argparse
import glob
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdb200  # noqa: E402
from sdb200 import pipeline  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402

KEYS = ("loss_simple", "loss_vlb", "loss")


def load_model(opt, device):
    if opt.random_init:
        print("--random_init: seeded random-init weights")
        model = instantiate_from_config(remap_config(sdb200.checkpoint.load_config(opt.config)))
        return pipeline.load_random_weights(model, device, gen_device=device).eval()
    if not opt.ckpt or not os.path.exists(opt.ckpt):
        raise FileNotFoundError(f"checkpoint {opt.ckpt!r} does not exist (pass --ckpt, or --random_init)")
    return sdb200.checkpoint.load_model_from_config(opt.config, opt.ckpt, device=device)


def image_size(model):
    dd = model.first_stage_model.cfg["ddconfig"]
    return model.image_size * 2 ** (len(dd["ch_mult"]) - 1)


def load_images(opt, n, size):
    """[n, size, size, 3] fp32 in [-1, 1]: the images of --indir (sorted, cycled), or seeded uniform noise."""
    if not opt.indir:
        g = torch.Generator().manual_seed(opt.seed)
        return torch.rand((n, size, size, 3), generator=g) * 2 - 1
    from PIL import Image
    paths = sorted(p for p in glob.glob(os.path.join(opt.indir, "*")) if p.lower().endswith((".png", ".jpg", ".jpeg")))
    if not paths:
        raise FileNotFoundError(f"no PNG / JPEG images in {opt.indir}")
    out = []
    for i in range(n):
        img = Image.open(paths[i % len(paths)]).convert("RGB").resize((size, size), resample=Image.BICUBIC)
        out.append(torch.from_numpy(np.asarray(img, dtype=np.float32) / 127.5 - 1.0))
    return torch.stack(out)


def conditioning(opt, model, n):
    """The batch entries the cond stage reads, for n images."""
    key = model.cond_stage_key
    if model.model.conditioning_key is None:
        return {}
    if key == "class_label":
        if opt.labels:
            labels = torch.tensor([int(v) for v in open(opt.labels).read().split()], dtype=torch.long)
        elif opt.class_label is not None:
            labels = torch.full((n,), opt.class_label, dtype=torch.long)
        else:
            labels = torch.randint(0, model.cond_stage_model.n_classes, (n,),
                                   generator=torch.Generator().manual_seed(opt.seed + 1))
        if labels.numel() < n:
            labels = labels.repeat(-(-n // labels.numel()))
        return {key: labels[:n]}
    if key == "caption":
        if not opt.from_file:
            raise ValueError("caption-conditional models need --from-file (one caption per line)")
        enc = model.cond_stage_model
        if opt.clip_vocab and hasattr(enc, "version"):
            enc.version, enc.tokenizer = opt.clip_vocab, None
        if opt.bert_vocab and hasattr(enc, "vocab_dir"):
            enc.vocab_dir, enc.tokenizer = opt.bert_vocab, None
        lines = [ln.strip() for ln in open(opt.from_file) if ln.strip()]
        return {key: [lines[i % len(lines)] for i in range(n)]}
    raise NotImplementedError(f"eval_loss.py: cond_stage_key {key!r}: supported are unconditional, class_label and "
                              "caption models (call LatentDiffusion.p_losses with the conditioning for others)")


def batches(images, cond, bs):
    for i in range(0, images.shape[0], bs):
        b = {"image": images[i:i + bs]}
        for k, v in cond.items():
            b[k] = v[i:i + bs]
        yield b


@torch.no_grad()
def random_t(model, images, cond, bs):
    """Mean of validation_step's dict over the batches, weighted by batch size."""
    total, n = {}, 0
    for i, b in enumerate(batches(images, cond, bs)):
        d = model.validation_step(b, i)
        nb = b["image"].shape[0]
        for k, v in d.items():
            total[k] = total.get(k, 0.0) + float(v) * nb
        n += nb
    return {k: v / n for k, v in total.items()}


@torch.no_grad()
def per_timestep(model, images, cond, bs, timesteps):
    """Every image at every t with one noise draw per image: mean loss_simple / loss_vlb / loss, raw and EMA."""
    acc = {t: {} for t in timesteps}
    n = 0
    for b in batches(images, cond, bs):
        z, c = model.get_input(b, model.first_stage_key)
        if c is not None and model.cond_stage_trainable:
            c = model.get_learned_conditioning(c)
        noise = torch.randn_like(z)
        nb = z.shape[0]
        for t in timesteps:
            tt = torch.full((nb,), t, dtype=torch.long, device=z.device)
            _, raw = model.p_losses(z, c, tt, noise=noise)
            with model.ema_scope():
                _, ema = model.p_losses(z, c, tt, noise=noise)
            for suffix, d in (("", raw), ("_ema", ema)):
                for k in KEYS:
                    acc[t][k + suffix] = acc[t].get(k + suffix, 0.0) + float(d[f"val/{k}"]) * nb
        n += nb
    return [{"t": t, **{k: v / n for k, v in acc[t].items()}} for t in timesteps]


def get_parser():
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--config", type=str, required=True, help="model config YAML (the reference's)")
    p.add_argument("--ckpt", type=str, default=None, help="checkpoint (.ckpt or .safetensors)")
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of a checkpoint")
    p.add_argument("--indir", type=str, default=None, help="directory of images (default: a seeded synthetic batch)")
    p.add_argument("--batch_size", type=int, default=8)
    p.add_argument("--n_samples", type=int, default=32, help="images evaluated")
    p.add_argument("--seed", type=int, default=42, help="seed of the images, labels, t and noise draws")
    p.add_argument("--timesteps", type=str, default=None, help="comma-separated t: loss-against-t table mode")
    p.add_argument("--class_label", type=int, default=None, help="class of every image (class-conditional models)")
    p.add_argument("--labels", type=str, default=None, help="file of integer class labels, one per image")
    p.add_argument("--from-file", dest="from_file", type=str, default=None, help="captions, one per line")
    p.add_argument("--clip_vocab", type=str, default=None, help="directory with the CLIP vocab.json + merges.txt")
    p.add_argument("--bert_vocab", type=str, default=None, help="directory with the bert-base-uncased vocab.txt")
    p.add_argument("--out", type=str, default="outputs/eval_loss/eval_loss.json", help="JSON result file")
    return p


def main(argv=None):
    opt = get_parser().parse_args(argv)
    if not os.path.exists(opt.config):
        raise FileNotFoundError(f"--config {opt.config} does not exist")
    torch.manual_seed(opt.seed)
    device = torch.device("cuda")
    model = load_model(opt, device)
    size = image_size(model)
    images = load_images(opt, opt.n_samples, size)
    cond = conditioning(opt, model, opt.n_samples)
    res = {"config": opt.config, "ckpt": None if opt.random_init else opt.ckpt, "n_samples": opt.n_samples,
           "image_size": size, "loss_type": model.loss_type, "seed": opt.seed}
    if opt.timesteps:
        ts = [int(v) for v in opt.timesteps.split(",")]
        bad = [t for t in ts if not 0 <= t < model.num_timesteps]
        if bad:
            raise IndexError(f"--timesteps {bad} outside [0, {model.num_timesteps})")
        res["per_t"] = per_timestep(model, images, cond, opt.batch_size, ts)
        print(f"{'t':>5} " + " ".join(f"{k:>16}" for k in ("loss_simple", "loss_simple_ema", "loss_vlb", "loss_vlb_ema")))
        for r in res["per_t"]:
            print(f"{r['t']:>5} " + " ".join(f"{r[k]:>16.6g}" for k in ("loss_simple", "loss_simple_ema", "loss_vlb",
                                                                         "loss_vlb_ema")))
    else:
        res["loss"] = random_t(model, images, cond, opt.batch_size)
        for k, v in res["loss"].items():
            print(f"{k:>22} {v:.6g}")
    os.makedirs(os.path.dirname(os.path.abspath(opt.out)), exist_ok=True)
    with open(opt.out, "w") as f:
        json.dump(res, f, indent=1)
    print(f"wrote {opt.out}")
    return res


if __name__ == "__main__":
    main()
