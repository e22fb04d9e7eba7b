"""Semantic image synthesis (segmentation map -> image) on the H100 engine with the LDM semantic-synthesis models
(models/ldm/semantic_synthesis256/config.yaml, and semantic_synthesis512, the landscape model):

  python scripts/semantic_synthesis.py map.png --outdir outputs/semantic --ckpt models/ldm/semantic_synthesis256/model.ckpt

A label map is a PNG of mode L or P whose pixel values are class ids < 182 (the convention of taming's sflckr /
landscapes data: the id is the one-hot channel). RGB maps and out-of-range ids are rejected. Per map: one kernel
(sdb_seg_labels_rescale) turns the uint8 ids into the cond stage's output, SpatialRescaler's two bilinear x0.5 stages
and 182 -> 3 channel map of the one-hot, at the latent size, without building the one-hot; DDIM with log_images'
defaults (--steps 200, --eta 1, no guidance, inside ema_scope()) samples --n_samples latents from x_T ~ N(0, 1), the
conditioning concatenated to x_t; the VQ-f4 first stage decodes them, written as PNGs converted as
sample_diffusion.py's custom_to_pil does.

Size rule: both sides must be multiples of 16 (the f4 first stage times the UNet's two downsamplings); square or not.
Maps larger than the training size are sampled convolutionally at full size, the paper's landscape use (e.g. 512x1024
with the 512 model). The reference's split_input_params tiling is not used.

The config is built in code (semantic_config, the 256 model's `model:` node); --config reads a reference YAML instead.
With --random_init no checkpoint is read and every stage gets seeded random weights; --tiny swaps in the small test
members (arch.TINY_SEMANTIC_UNET, TINY_VQ_F4, TINY_SEMANTIC_COND).
"""
import argparse
import glob
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdb200  # noqa: E402
from sdb200 import arch, pipeline  # noqa: E402
from sdb200.samplers import DDIMSampler  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402


def semantic_config(unet_cfg=None, vq_cfg=None, cond_cfg=None, image_size=None):
    """models/ldm/semantic_synthesis256/config.yaml, `model:` node (reference targets); image_size 128 with the
    first stage's monitor is semantic_synthesis512's."""
    u = dict(unet_cfg or arch.SEMANTIC_SYNTHESIS_UNET)
    if image_size is not None:
        u["image_size"] = image_size
    v = dict(vq_cfg or arch.VQ_F4)
    fs = {**v, "lossconfig": {"target": "torch.nn.Identity"}}
    if image_size == 128:
        fs["monitor"] = "val/rec_loss"
    return {"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        "linear_start": 0.0015, "linear_end": 0.0205, "log_every_t": 100, "timesteps": 1000, "loss_type": "l1",
        "first_stage_key": "image", "cond_stage_key": "segmentation", "image_size": u["image_size"], "channels": 3,
        "concat_mode": True, "cond_stage_trainable": True,
        "unet_config": {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": u},
        "first_stage_config": {"target": "ldm.models.autoencoder.VQModelInterface", "params": fs},
        "cond_stage_config": {"target": "ldm.modules.encoders.modules.SpatialRescaler",
                              "params": dict(cond_cfg or arch.SEMANTIC_SYNTHESIS_COND)}}}


def size_multiple(model):
    """Side multiple a label map needs: the first stage's downsampling times the UNet's."""
    f = 1 << (len(model.first_stage_model.cfg["ddconfig"]["ch_mult"]) - 1)
    return f << (len(model.model.diffusion_model.cfg["channel_mult"]) - 1)


def check_size(h, w, multiple=16):
    if h <= 0 or w <= 0 or h % multiple or w % multiple:
        raise ValueError(f"a {h}x{w} label map: both sides must be multiples of {multiple}")


def read_label_map(path, n_classes=182):
    """A label PNG (mode L or P, pixel value = class id) -> uint8 [H, W]. ValueError for other modes or ids
    >= n_classes."""
    from PIL import Image
    img = Image.open(path)
    if img.mode not in ("L", "P"):
        raise ValueError(f"{path}: label maps are single-channel PNGs of mode L or P holding class ids; got mode "
                         f"{img.mode}")
    lab = np.array(img)
    if lab.ndim != 2 or lab.dtype != np.uint8:
        raise ValueError(f"{path}: expected 8-bit class ids, got {lab.dtype} {lab.shape}")
    if lab.size and int(lab.max()) >= n_classes:
        raise ValueError(f"{path}: class id {int(lab.max())} out of range (the model has {n_classes} classes)")
    return lab


def load_model(ckpt=None, random_init=False, tiny=False, config=None, device="cuda", image_size=None):
    dev = torch.device(device)
    if config is not None:
        if random_init or tiny:
            raise ValueError("--config is read with --ckpt")
        return sdb200.checkpoint.load_model_from_config(config, ckpt, device=dev)
    node = (semantic_config(arch.TINY_SEMANTIC_UNET, arch.TINY_VQ_F4, arch.TINY_SEMANTIC_COND) if tiny else
            semantic_config(image_size=image_size))
    if not random_init:
        return sdb200.checkpoint.load_model_from_config({"model": node}, ckpt, device=dev)
    return pipeline.load_random_weights(instantiate_from_config(remap_config(node)), dev, gen_device=dev).eval()


@torch.no_grad()
def synthesize(model, sampler, labels, n_samples=1, steps=200, eta=1.0, x_T=None, return_latents=False):
    """labels integer [nb, H, W] (class ids) -> the decoded images fp32 NCHW [nb * n_samples, 3, H, W] in [-1, 1]
    (quantized decode), sample i * n_samples + j from map i, as log_images samples them. return_latents also returns
    (conditioning, DDIM sample)."""
    nb, h, w = labels.shape
    check_size(h, w, size_multiple(model))
    c = model.get_learned_conditioning(labels)
    if n_samples > 1:
        c = c.repeat_interleave(n_samples, 0)
    samples, _ = sampler.sample(S=steps, conditioning=c, batch_size=c.shape[0], shape=tuple(c.shape[1:]), eta=eta,
                                verbose=False, x_T=x_T)
    x = model.decode_first_stage(samples)
    return (x, c, samples) if return_latents else x


def to_pil(x):
    """sample_diffusion.py's custom_to_pil: clamp to [-1, 1], (x + 1) / 2, 255 * x truncated to uint8."""
    from PIL import Image
    x = torch.clamp(x.detach().cpu(), -1., 1.)
    x = (x + 1.) / 2.
    return Image.fromarray((255 * x.permute(1, 2, 0).numpy()).astype(np.uint8)).convert("RGB")


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("label_map", type=str, nargs="?", help="a label PNG (mode L or P, pixel values = class ids)")
    p.add_argument("--indir", type=str, default=None, help="dir of label PNGs")
    p.add_argument("--outdir", type=str, default="outputs/semantic_synthesis", help="dir to write results to")
    p.add_argument("--n_samples", type=int, default=1, help="samples per label map")
    p.add_argument("--steps", type=int, default=200, help="number of ddim sampling steps")
    p.add_argument("--eta", type=float, default=1.0, help="ddim eta")
    p.add_argument("--ckpt", type=str, default=None, help="checkpoint (models/ldm/semantic_synthesis256/model.ckpt)")
    p.add_argument("--config", type=str, default=None,
                   help="reference YAML (default: models/ldm/semantic_synthesis256/config.yaml)")
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of a checkpoint")
    p.add_argument("--tiny", action="store_true", help="the small test configuration (with --random_init)")
    p.add_argument("--no_cuda_graph", action="store_true", help="eager kernel launches instead of CUDA-graph replay")
    return p


def main(argv=None):
    opt = get_parser().parse_args(argv)
    if not opt.random_init and not opt.ckpt:
        raise ValueError("pass --ckpt, or --random_init")
    if opt.tiny and not opt.random_init:
        raise ValueError("--tiny needs --random_init")
    if (opt.label_map is None) == (opt.indir is None):
        raise ValueError("pass one label map, or --indir")
    maps = [opt.label_map] if opt.label_map else sorted(
        p for p in glob.glob(os.path.join(opt.indir, "*")) if p.lower().endswith(".png"))
    print(f"Found {len(maps)} inputs.")
    model = load_model(opt.ckpt, opt.random_init, opt.tiny, opt.config)
    model.model.diffusion_model.use_cuda_graph = not opt.no_cuda_graph
    n_classes = model.cond_stage_model.in_channels
    multiple = size_multiple(model)
    labels = []
    for path in maps:           # every map is checked before any sampling
        lab = read_label_map(path, n_classes)
        check_size(*lab.shape, multiple)
        labels.append(lab)
    sampler = DDIMSampler(model)
    os.makedirs(opt.outdir, exist_ok=True)
    written = []
    t0 = time.time()
    with model.ema_scope():
        for path, lab in zip(maps, labels):
            x = synthesize(model, sampler, torch.from_numpy(lab)[None], n_samples=opt.n_samples, steps=opt.steps,
                           eta=opt.eta)
            stem = os.path.splitext(os.path.basename(path))[0]
            for j in range(x.shape[0]):
                outpath = os.path.join(opt.outdir, f"{stem}_{j:02d}.png")
                to_pil(x[j]).save(outpath)
                written.append(outpath)
            print(f"{path}: {lab.shape[1]}x{lab.shape[0]}, {x.shape[0]} samples")
    print(f"{len(written)} images in {time.time() - t0:.2f} s, written to {opt.outdir}")
    return written


if __name__ == "__main__":
    main()
