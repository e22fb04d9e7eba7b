"""4x super-resolution on the H100 engine with the LDM-BSR model (models/ldm/bsr_sr/config.yaml), as the reference's
notebook_helpers.py runs it (get_cond, run, make_convolutional_sample):

  python scripts/superres.py data/example_conditioning/superresolution/sample_0.jpg --outdir outputs/superres --ckpt last.ckpt

Per image: PIL decodes it to RGB on the host; one kernel converts it to the conditioning 2 * (u / 255) - 1 at the latent
size (sdb_lr_prepare; the cond stage is the identity); DDIM (--steps, --eta, no guidance, inside ema_scope()) samples a
latent of the input's size from x_T ~ N(0, 1); the VQ-f4 first stage decodes it (quantized) to 4x the size, written as
a PNG converted as sample_diffusion.py does.

Which path runs (printed per image):
  * split, when both sides are >= 128: the UNet and the decoder run on 128x128 latent tiles at stride 64, blended with
    the reference's split_input_params weighting (ks 128, stride 64, vqf 4, clip weights 0.01 / 0.5). The tiles must
    cover the image, i.e. (side - 128) % 64 == 0, or the run raises ValueError, where the reference writes NaN.
  * plain otherwise, which needs sides that are multiples of 8 (the UNet's three downsamplings).
The reference splits as soon as the 4x output is >= 128 on both sides, i.e. from 32 input pixels on, and then fails for
every side below 128 (its tiles may not be larger than the latent). Running those sizes - 64x64, the model's training
size, among them - on the plain path is this script's one deliberate extension; everywhere the reference produces an
image, the path and the result are the reference's.

The config is built in code (superres_config); --config reads a reference YAML instead. With --random_init no
checkpoint is read and every stage gets seeded random weights; --tiny swaps in the small test members
(arch.TINY_BSR_UNET, TINY_VQ_F4).
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
from sdb200.diffusion import split_geometry  # noqa: E402
from sdb200.samplers import DDIMSampler  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402

SPLIT_MIN = 128


def superres_config(unet_cfg=None, vq_cfg=None):
    """models/ldm/bsr_sr/config.yaml, `model:` node (reference targets)."""
    u = dict(unet_cfg or arch.BSR_SR_UNET)
    v = dict(vq_cfg or arch.VQ_F4)
    return {"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        "linear_start": 0.0015, "linear_end": 0.0155, "log_every_t": 100, "timesteps": 1000, "loss_type": "l2",
        "first_stage_key": "image", "cond_stage_key": "LR_image", "image_size": u["image_size"], "channels": 3,
        "concat_mode": True, "cond_stage_trainable": False,
        "unet_config": {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": u},
        "first_stage_config": {"target": "ldm.models.autoencoder.VQModelInterface", "params": {
            **v, "monitor": "val/rec_loss", "lossconfig": {"target": "torch.nn.Identity"}}},
        "cond_stage_config": {"target": "torch.nn.Identity"}}}


def split_params(ks=128, stride=64, vqf=4):
    """run()'s split_input_params (notebook_helpers.py)."""
    return {"ks": (ks, ks), "stride": (stride, stride), "vqf": vqf, "patch_distributed_vq": True, "tie_braker": False,
            "clip_max_weight": 0.5, "clip_min_weight": 0.01, "clip_max_tie_weight": 0.5, "clip_min_tie_weight": 0.01}


def choose_path(h, w, ks=SPLIT_MIN, stride=64, levels=4):
    """"split" or "plain" for an h x w low-resolution image (the latent size); ValueError for a size neither runs."""
    if h >= ks and w >= ks:
        split_geometry(h, w, split_params(ks, stride), 1)      # raises for uncovered sizes
        return "split"
    m = 1 << (levels - 1)
    if h % m or w % m:
        raise ValueError(f"plain path: the {h}x{w} input must have sides that are multiples of {m}")
    return "plain"


def load_model(ckpt=None, random_init=False, tiny=False, config=None, device="cuda"):
    dev = torch.device(device)
    if config is not None:
        if random_init or tiny:
            raise ValueError("--config is read with --ckpt")
        return sdb200.checkpoint.load_model_from_config(config, ckpt, device=dev)
    node = superres_config(arch.TINY_BSR_UNET, arch.TINY_VQ_F4) if tiny else superres_config()
    if not random_init:
        return sdb200.checkpoint.load_model_from_config({"model": node}, ckpt, device=dev)
    return pipeline.load_random_weights(instantiate_from_config(remap_config(node)), dev, gen_device=dev).eval()


@torch.no_grad()
def superresolve(model, sampler, lr_u8, steps=100, eta=1.0, x_T=None, return_latents=False, split=None):
    """lr_u8 uint8 [nb, h, w, 3] (RGB, cuda) -> the decoded image fp32 NCHW [nb, 3, 4h, 4w] in [-1, 1] (quantized
    decode), as run() / make_convolutional_sample compute it. split: None picks the path by choose_path, a dict of
    split_input_params forces a tiled geometry (the tests' small ones). return_latents also returns (conditioning,
    DDIM sample, path)."""
    nb, h, w, _ = lr_u8.shape
    unet = model.model.diffusion_model
    if split is None:
        path = choose_path(h, w, levels=len(unet.cfg["channel_mult"]))
        split = split_params() if path == "split" else None
    path = "plain" if split is None else "split"
    if split is None:
        if hasattr(model, "split_input_params"):
            del model.split_input_params
    else:
        model.split_input_params = split
    c = model.get_learned_conditioning(ops.lr_prepare(lr_u8.contiguous()))     # Identity cond stage
    samples, _ = sampler.sample(S=steps, conditioning=c, batch_size=nb, shape=(3, h, w), eta=eta, verbose=False,
                                x_T=x_T)
    x = model.decode_first_stage(samples)
    return (x, c, samples, path) if return_latents else x


def to_pil(x):
    """sample_diffusion.py's custom_to_pil: clamp to [-1, 1], (x + 1) / 2, 255 * x truncated to uint8."""
    from PIL import Image
    x = torch.clamp(x.detach().cpu(), -1., 1.)
    x = (x + 1.) / 2.
    return Image.fromarray((255 * x.permute(1, 2, 0).numpy()).astype(np.uint8)).convert("RGB")


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("image", type=str, nargs="?", help="a low-resolution image")
    p.add_argument("--indir", type=str, default=None, help="dir of low-resolution images (.png / .jpg)")
    p.add_argument("--outdir", type=str, default="outputs/superres", help="dir to write results to")
    p.add_argument("--steps", type=int, default=100, help="number of ddim sampling steps")
    p.add_argument("--eta", type=float, default=1.0, help="ddim eta")
    p.add_argument("--ckpt", type=str, default=None, help="bsr_sr checkpoint (models/ldm/bsr_sr/model.ckpt)")
    p.add_argument("--config", type=str, default=None, help="reference YAML (default: models/ldm/bsr_sr/config.yaml)")
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
    if (opt.image is None) == (opt.indir is None):
        raise ValueError("pass one image, or --indir")
    images = [opt.image] if opt.image else sorted(
        p for p in glob.glob(os.path.join(opt.indir, "*")) if p.lower().endswith((".png", ".jpg", ".jpeg")))
    print(f"Found {len(images)} inputs.")
    model = load_model(opt.ckpt, opt.random_init, opt.tiny, opt.config)
    model.model.diffusion_model.use_cuda_graph = not opt.no_cuda_graph
    sampler = DDIMSampler(model)
    dev = model.device
    os.makedirs(opt.outdir, exist_ok=True)
    written = []
    t0 = time.time()
    with model.ema_scope():
        for image in images:
            lr = torch.from_numpy(np.array(Image.open(image).convert("RGB")))[None].to(dev)
            x, _, _, path = superresolve(model, sampler, lr, steps=opt.steps, eta=opt.eta, return_latents=True)
            outpath = os.path.join(opt.outdir, os.path.splitext(os.path.basename(image))[0] + ".png")
            to_pil(x[0]).save(outpath)
            print(f"{image}: {lr.shape[2]}x{lr.shape[1]} -> {x.shape[3]}x{x.shape[2]}, {path} path")
            written.append(outpath)
    print(f"{len(written)} images in {time.time() - t0:.2f} s, written to {opt.outdir}")
    return written


if __name__ == "__main__":
    main()
