#!/usr/bin/env python
"""Unconditional LDM sampling on the H100 engine with the reference script's flags (scripts/sample_diffusion.py of
CompVis/stable-diffusion), e.g. the LSUN-Churches KL-f8 model:

  python scripts/sample_diffusion.py -r models/ldm/lsun_churches256/model.ckpt -n 50 -c 50 -e 1.0 -l outputs/lsun

or the VQ-f4 models (CelebA-HQ, FFHQ, LSUN-Bedrooms: configs/latent-diffusion/*-ldm-vq-4.yaml), e.g.

  python scripts/sample_diffusion.py -r models/ldm/celeba256/model.ckpt -n 50 -c 50 -e 0 -l outputs/celeba

-r is a checkpoint (its directory holds config.yaml) or a logdir holding model.ckpt and config.yaml. DDIM with eta
(default 1.0) or, with -v, the ancestral sampler over all training steps (progressive_denoising). Sampling runs inside
ema_scope(), so checkpoints with EMA copies sample with them. With --random_init no checkpoint is read: every stage with
weights gets seeded random weights (the config comes from -r, --config, or the built-in LSUN-Churches values).
Samples are written as sample_XXXXXX.png and one .npz of uint8 NHWC images, converted exactly as the reference does.
"""
import argparse
import datetime
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


def lsun_churches_config(unet_cfg=None, vae_cfg=None):
    """models/ldm/lsun_churches256/config.yaml, `model:` node (reference targets)."""
    u = dict(unet_cfg or arch.LSUN_CHURCHES_UNET)
    v = dict(vae_cfg or arch.SD_V1_VAE)
    return {"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        "linear_start": 0.0015, "linear_end": 0.0155, "num_timesteps_cond": 1, "log_every_t": 200, "timesteps": 1000,
        "loss_type": "l1", "first_stage_key": "image", "cond_stage_key": "image", "image_size": u["image_size"],
        "channels": 4, "cond_stage_trainable": False, "concat_mode": False, "scale_by_std": True,
        "monitor": "val/loss_simple_ema",
        "unet_config": {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": u},
        "first_stage_config": {"target": "ldm.models.autoencoder.AutoencoderKL",
                               "params": {**v, "monitor": "val/rec_loss", "lossconfig": {"target": "torch.nn.Identity"}}},
        "cond_stage_config": "__is_unconditional__"}}


def celebahq_config(unet_cfg=None, vq_cfg=None):
    """configs/latent-diffusion/celebahq-ldm-vq-4.yaml, `model:` node (reference targets); the FFHQ and LSUN-Bedrooms
    configs differ only in their data and first-stage ckpt_path."""
    u = dict(unet_cfg or arch.CELEBAHQ_UNET)
    v = dict(vq_cfg or arch.VQ_F4)
    return {"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        "linear_start": 0.0015, "linear_end": 0.0195, "num_timesteps_cond": 1, "log_every_t": 200, "timesteps": 1000,
        "first_stage_key": "image", "image_size": u["image_size"], "channels": u["in_channels"],
        "monitor": "val/loss_simple_ema",
        "unet_config": {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": u},
        "first_stage_config": {"target": "ldm.models.autoencoder.VQModelInterface",
                               "params": {**v, "ckpt_path": "models/first_stage_models/vq-f4/model.ckpt",
                                          "lossconfig": {"target": "torch.nn.Identity"}}},
        "cond_stage_config": "__is_unconditional__"}}


def custom_to_pil(x):
    """sample_diffusion.py custom_to_pil: clamp, (x + 1) / 2, 255 * x truncated to uint8."""
    from PIL import Image
    x = x.detach().cpu()
    x = torch.clamp(x, -1., 1.)
    x = (x + 1.) / 2.
    x = x.permute(1, 2, 0).numpy()
    x = (255 * x).astype(np.uint8)
    return Image.fromarray(x).convert("RGB")


def custom_to_np(x):
    """sample_diffusion.py custom_to_np: ((x + 1) * 127.5).clamp(0, 255) cast to uint8, NHWC."""
    sample = x.detach().cpu()
    sample = ((sample + 1) * 127.5).clamp(0, 255).to(torch.uint8)
    return sample.permute(0, 2, 3, 1).contiguous()


@torch.no_grad()
def make_convolutional_sample(model, batch_size, vanilla=False, custom_steps=None, eta=1.0):
    unet = model.model.diffusion_model
    shape = [batch_size, unet.in_channels, unet.image_size, unet.image_size]
    log = {}
    with model.ema_scope("Plotting"):
        t0 = time.time()
        if vanilla:
            sample, _ = model.progressive_denoising(None, shape, verbose=False)
        else:
            sample, _ = DDIMSampler(model).sample(custom_steps, batch_size=shape[0], shape=shape[1:], eta=eta,
                                                  verbose=False)
        torch.cuda.synchronize()
        t1 = time.time()
    log["sample"] = model.decode_first_stage(sample)
    log["time"] = t1 - t0
    log["throughput"] = sample.shape[0] / (t1 - t0)
    print(f'Throughput for this batch: {log["throughput"]}')
    return log


def save_logs(logs, path, n_saved=0, key="sample"):
    for x in logs[key]:
        custom_to_pil(x).save(os.path.join(path, f"{key}_{n_saved:06}.png"))
        n_saved += 1
    return n_saved


def run(model, logdir, batch_size=50, vanilla=False, custom_steps=None, eta=None, n_samples=50000, nplog=None):
    if vanilla:
        print(f"Using Vanilla DDPM sampling with {model.num_timesteps} sampling steps.")
    else:
        print(f"Using DDIM sampling with {custom_steps} sampling steps and eta={eta}")
    tstart = time.time()
    n_saved = len(glob.glob(os.path.join(logdir, "*.png"))) - 1
    if model.cond_stage_model is not None:
        raise NotImplementedError("Currently only sampling for unconditional models supported.")
    all_images = []
    print(f"Running unconditional sampling for {n_samples} samples")
    for _ in range(n_samples // batch_size):
        logs = make_convolutional_sample(model, batch_size=batch_size, vanilla=vanilla, custom_steps=custom_steps,
                                         eta=eta)
        n_saved = save_logs(logs, logdir, n_saved=n_saved, key="sample")
        all_images.extend([custom_to_np(logs["sample"])])
        if n_saved >= n_samples:
            print(f"Finish after generating {n_saved} samples")
            break
    all_img = np.concatenate(all_images, axis=0)[:n_samples]
    shape_str = "x".join([str(x) for x in all_img.shape])
    np.savez(os.path.join(nplog, f"{shape_str}-samples.npz"), all_img)
    print(f"sampling of {n_saved} images finished in {(time.time() - tstart) / 60.:.2f} minutes.")


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("-r", "--resume", type=str, nargs="?", help="load from logdir or checkpoint in logdir")
    p.add_argument("-n", "--n_samples", type=int, nargs="?", help="number of samples to draw", default=50000)
    p.add_argument("-e", "--eta", type=float, nargs="?", default=1.0,
                   help="eta for ddim sampling (0.0 yields deterministic sampling)")
    p.add_argument("-v", "--vanilla_sample", default=False, action="store_true",
                   help="vanilla sampling (default option is DDIM sampling)?")
    p.add_argument("-l", "--logdir", type=str, nargs="?", help="extra logdir", default="none")
    p.add_argument("-c", "--custom_steps", type=int, nargs="?", help="number of steps for ddim and fastdpm sampling",
                   default=50)
    p.add_argument("--batch_size", type=int, nargs="?", help="the bs", default=10)
    p.add_argument("--config", type=str, default=None, help="model config YAML (default: <logdir>/config.yaml)")
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of a checkpoint")
    p.add_argument("--seed", type=int, default=None, help="torch seed of the sampling noise")
    p.add_argument("--no_cuda_graph", action="store_true", help="eager kernel launches instead of CUDA-graph replay")
    return p


def main(argv=None):
    opt = get_parser().parse_args(argv)
    now = datetime.datetime.now().strftime("%Y-%m-%d-%H-%M-%S")
    ckpt, logdir = None, None
    if opt.resume:
        if not os.path.exists(opt.resume):
            raise ValueError(f"Cannot find {opt.resume}")
        if os.path.isfile(opt.resume):
            logdir = os.path.dirname(opt.resume) or "."
            ckpt = opt.resume
        else:
            logdir = opt.resume.rstrip("/")
            ckpt = os.path.join(logdir, "model.ckpt")
        print(f"Logdir is {logdir}")
    elif not opt.random_init:
        raise ValueError("pass -r (checkpoint or logdir), or --random_init")
    config = opt.config or (os.path.join(logdir, "config.yaml") if logdir else None)
    if config is not None and not os.path.exists(config):
        raise FileNotFoundError(f"config {config} does not exist")
    if opt.seed is not None:
        torch.manual_seed(opt.seed)
    dev = torch.device("cuda")
    if opt.random_init:
        node = sdb200.checkpoint.load_config(config) if config else lsun_churches_config()
        print("--random_init: seeded random-init weights (images will be noise-like)")
        model = pipeline.load_random_weights(instantiate_from_config(remap_config(node)), dev, gen_device=dev).eval()
        global_step = None
    else:
        model = sdb200.checkpoint.load_model_from_config(config, ckpt, device=dev)
        global_step = model.load_info.get("global_step")
    model.model.diffusion_model.use_cuda_graph = not opt.no_cuda_graph
    print(f"global step: {global_step}")
    base = opt.logdir if opt.logdir != "none" else (logdir or "outputs/sample_diffusion")
    logdir = os.path.join(base, "samples", f"{global_step if global_step is not None else 0:08}", now)
    imglogdir = os.path.join(logdir, "img")
    numpylogdir = os.path.join(logdir, "numpy")
    os.makedirs(imglogdir, exist_ok=True)
    os.makedirs(numpylogdir, exist_ok=True)
    print(75 * "=")
    print(f"logging to: {logdir}")
    run(model, imglogdir, eta=opt.eta, vanilla=opt.vanilla_sample, n_samples=opt.n_samples,
        custom_steps=opt.custom_steps, batch_size=opt.batch_size, nplog=numpylogdir)
    print("done.")
    return logdir


if __name__ == "__main__":
    main()
