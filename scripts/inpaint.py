"""Inpainting on the H100 engine: the reference's scripts/inpaint.py (models/ldm/inpainting_big/config.yaml,
models/ldm/inpainting_big/last.ckpt):

  python scripts/inpaint.py --indir data/inpainting_examples --outdir outputs/inpainting_results --ckpt last.ckpt

Every `<name>_mask.png` in --indir pairs with `<name>.png`; each pair is inpainted on its own (DDIM, --steps, eta 0, no
guidance, inside ema_scope()) and written to --outdir/<name>.png. Per image: PIL decodes the PNGs (convert("RGB") /
convert("L")) on the host; one kernel pair builds the masked image and the resized ±1 mask channel of the conditioning
(sdb_inpaint_prepare); the VQ encoder fills the other three channels; the UNet reads x_t and the conditioning as two
sources; after the VQ decode one kernel forms the uint8 composite (sdb_inpaint_composite).
The config is built in code (inpaint_config). With --random_init no checkpoint is read and every stage gets seeded random
weights; --tiny swaps in the small test members (arch.TINY_INPAINT_UNET, TINY_VQ_NOATTN).
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
from sdb200 import arch, ops, pipeline  # noqa: E402
from sdb200.samplers import DDIMSampler  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402


def inpaint_config(unet_cfg=None, vq_cfg=None):
    """models/ldm/inpainting_big/config.yaml, `model:` node (reference targets, the DummyLoss included)."""
    u = dict(unet_cfg or arch.INPAINTING_BIG_UNET)
    v = dict(vq_cfg or arch.VQ_F4_NOATTN)
    return {"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        "linear_start": 0.0015, "linear_end": 0.0205, "log_every_t": 100, "timesteps": 1000, "loss_type": "l1",
        "first_stage_key": "image", "cond_stage_key": "masked_image", "image_size": u["image_size"], "channels": 3,
        "concat_mode": True, "monitor": "val/loss",
        "unet_config": {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": u},
        "first_stage_config": {"target": "ldm.models.autoencoder.VQModelInterface", "params": {
            **v, "monitor": "val/rec_loss", "lossconfig": {"target": "ldm.modules.losses.contperceptual.DummyLoss"}}},
        "cond_stage_config": "__is_first_stage__"}}


def load_model(ckpt=None, random_init=False, tiny=False, device="cuda"):
    dev = torch.device(device)
    node = inpaint_config(arch.TINY_INPAINT_UNET, arch.TINY_VQ_NOATTN) if tiny else inpaint_config()
    if not random_init:
        return sdb200.checkpoint.load_model_from_config({"model": node}, ckpt, device=dev)
    return pipeline.load_random_weights(instantiate_from_config(remap_config(node)), dev, gen_device=dev).eval()


def latent_size(model, h, w):
    """The VQ encoder's output size: every Downsample (pad right / bottom by 1, 3x3 stride 2) halves, rounding down."""
    n = len(model.first_stage_model.cfg["ddconfig"]["ch_mult"]) - 1
    return h >> n, w >> n


@torch.no_grad()
def inpaint(model, sampler, image, mask, steps=50, x_T=None, return_latents=False):
    """image uint8 [nb, h, w, 3] (RGB), mask uint8 [nb, h, w] (L), cuda tensors -> uint8 [nb, h, w, 3]: the reference
    loop body on a batch. return_latents also returns (conditioning, DDIM sample, decoded image NHWC)."""
    fs = model.cond_stage_model            # is model.first_stage_model (__is_first_stage__)
    nb, h, w, _ = image.shape
    hc, wc = latent_size(model, h, w)
    c = torch.empty((nb, 4, hc, wc), dtype=torch.float32, device=image.device)
    masked = ops.inpaint_prepare(image.contiguous(), mask.contiguous(), c, 3)       # channel 3: the resized ±1 mask
    enc = fs.encode(masked)
    assert tuple(enc.shape) == (nb, 3, hc, wc), tuple(enc.shape)
    c[:, :3].copy_(enc)
    samples, _ = sampler.sample(S=steps, conditioning=c, batch_size=nb, shape=(3, hc, wc), verbose=False, x_T=x_T)
    x = model.first_stage_model.decode(samples, scale=1. / float(model.scale_factor), nhwc=True)
    out = ops.inpaint_composite(x, image.contiguous(), mask.contiguous())
    return (out, c, samples, x) if return_latents else out


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--indir", type=str, nargs="?", help="dir containing image-mask pairs (`example.png` and `example_mask.png`)")
    p.add_argument("--outdir", type=str, nargs="?", help="dir to write results to")
    p.add_argument("--steps", type=int, default=50, help="number of ddim sampling steps")
    p.add_argument("--ckpt", type=str, default=None, help="inpainting_big checkpoint (models/ldm/inpainting_big/last.ckpt)")
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of a checkpoint")
    p.add_argument("--tiny", action="store_true", help="the small test configuration (with --random_init)")
    p.add_argument("--no_cuda_graph", action="store_true", help="eager kernel launches instead of CUDA-graph replay")
    return p


def main(argv=None):
    from PIL import Image
    opt = get_parser().parse_args(argv)
    if not opt.random_init and not opt.ckpt:
        raise ValueError("pass --ckpt, or --random_init")
    if opt.tiny and not opt.random_init:
        raise ValueError("--tiny needs --random_init")
    masks = sorted(glob.glob(os.path.join(opt.indir, "*_mask.png")))
    images = [x.replace("_mask.png", ".png") for x in masks]
    print(f"Found {len(masks)} inputs.")
    model = load_model(opt.ckpt, opt.random_init, opt.tiny)
    model.model.diffusion_model.use_cuda_graph = not opt.no_cuda_graph
    sampler = DDIMSampler(model)
    dev = model.device
    os.makedirs(opt.outdir, exist_ok=True)
    written = []
    t0 = time.time()
    with model.ema_scope():
        for image, mask in zip(images, masks):
            outpath = os.path.join(opt.outdir, os.path.split(image)[1])
            im = torch.from_numpy(np.array(Image.open(image).convert("RGB")))[None].to(dev)
            mk = torch.from_numpy(np.array(Image.open(mask).convert("L")))[None].to(dev)
            out = inpaint(model, sampler, im, mk, steps=opt.steps)
            Image.fromarray(out[0].cpu().numpy()).save(outpath)
            written.append(outpath)
    print(f"{len(written)} images in {time.time() - t0:.2f} s, written to {opt.outdir}")
    return written


if __name__ == "__main__":
    main()
