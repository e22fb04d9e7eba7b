"""Class-conditional ImageNet sampling on the H100 engine: the sampling cell of the reference's
scripts/latent_imagenet_diffusion.ipynb (configs/latent-diffusion/cin256-v2.yaml, models/ldm/cin256-v2/model.ckpt):

  python scripts/sample_imagenet.py --ckpt models/ldm/cin256-v2/model.ckpt --outdir outputs/imagenet
  python scripts/sample_imagenet.py --model cin256 --ckpt models/ldm/cin256/model.ckpt --outdir outputs/imagenet

Classes 25, 187, 448, 992, six samples per class, DDIM-20, eta 0, classifier-free guidance scale 3.0 with the
unconditional conditioning taken from label 1000, inside ema_scope(); decode_first_stage, clamp((x + 1) / 2, 0, 1), and
one PNG grid (one row per class, 2-pixel padding, as torchvision's make_grid) written with numpy / PIL.
--model cin256 is the LDM-VQ-8 (models/ldm/cin256/config.yaml): 1000 classes and no unconditional label, so it samples
unguided (scale 1.0, no unconditional conditioning); any other --scale is an error. Its config leaves use_ema on, so the
checkpoint's EMA weights are the ones sampled.
The configs are built in code (cin_config, cin256_f8_config). With --random_init no checkpoint is read and every stage
gets seeded random weights; --tiny swaps in the small test members (arch.TINY_CIN_UNET, TINY_VQ, TINY_CIN_COND, or
arch.TINY_CIN_F8_UNET, TINY_VQ_F8, TINY_CIN_F8_COND with --model cin256).
"""
import argparse
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


def cin_config(unet_cfg=None, vq_cfg=None, cond_cfg=None):
    """configs/latent-diffusion/cin256-v2.yaml, `model:` node (reference targets)."""
    u = dict(unet_cfg or arch.CIN256_V2_UNET)
    v = dict(vq_cfg or arch.VQ_F4)
    c = dict(cond_cfg or arch.CIN256_V2_COND)
    return {"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        "linear_start": 0.0015, "linear_end": 0.0195, "num_timesteps_cond": 1, "log_every_t": 200, "timesteps": 1000,
        "first_stage_key": "image", "cond_stage_key": "class_label", "image_size": u["image_size"],
        "channels": u["in_channels"], "cond_stage_trainable": True, "conditioning_key": "crossattn",
        "monitor": "val/loss", "use_ema": False,
        "unet_config": {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": u},
        "first_stage_config": {"target": "ldm.models.autoencoder.VQModelInterface",
                               "params": {**v, "lossconfig": {"target": "torch.nn.Identity"}}},
        "cond_stage_config": {"target": "ldm.modules.encoders.modules.ClassEmbedder", "params": c}}}


def cin256_f8_config(unet_cfg=None, vq_cfg=None, cond_cfg=None):
    """models/ldm/cin256/config.yaml (= configs/latent-diffusion/cin-ldm-vq-f8.yaml), `model:` node (reference targets).
    use_ema is left at its default (True): the checkpoint carries model_ema.*."""
    u = dict(unet_cfg or arch.CIN256_F8_UNET)
    v = dict(vq_cfg or arch.VQ_F8)
    c = dict(cond_cfg or arch.CIN256_F8_COND)
    node = cin_config(u, v, c)
    node["params"]["monitor"] = "val/loss_simple_ema"
    del node["params"]["use_ema"]
    return node


MODELS = {"cin256-v2": (cin_config, (arch.TINY_CIN_UNET, arch.TINY_VQ, arch.TINY_CIN_COND), 3.0),
          "cin256": (cin256_f8_config, (arch.TINY_CIN_F8_UNET, arch.TINY_VQ_F8, arch.TINY_CIN_F8_COND), 1.0)}


def load_model(ckpt=None, random_init=False, tiny=False, device="cuda", model="cin256-v2"):
    dev = torch.device(device)
    make, tiny_cfgs, _ = MODELS[model]
    node = make(*tiny_cfgs) if tiny else make()
    if not random_init:
        return sdb200.checkpoint.load_model_from_config({"model": node}, ckpt, device=dev)
    return pipeline.load_random_weights(instantiate_from_config(remap_config(node)), dev, gen_device=dev).eval()


def make_grid(images, nrow, padding=2):
    """[N, 3, H, W] in [0, 1] -> uint8 HWC grid of ceil(N / nrow) rows x nrow columns (torchvision's layout, pad 0)."""
    n, c, h, w = images.shape
    rows = (n + nrow - 1) // nrow
    grid = np.zeros((rows * (h + padding) + padding, nrow * (w + padding) + padding, c), dtype=np.uint8)
    arr = (255. * images.permute(0, 2, 3, 1).cpu().numpy()).astype(np.uint8)   # the notebook's 255. * grid, truncated
    for i in range(n):
        y, x = padding + (i // nrow) * (h + padding), padding + (i % nrow) * (w + padding)
        grid[y: y + h, x: x + w] = arr[i]
    return grid


@torch.no_grad()
def sample_classes(model, classes, n_samples_per_class, ddim_steps=20, ddim_eta=0.0, scale=3.0):
    """The notebook's loop: one DDIM batch per class, guided by label 1000's conditioning unless scale is 1.0;
    returns [len(classes) * n, 3, H, W] in [0, 1]."""
    unet = model.model.diffusion_model
    shape = [unet.in_channels, unet.image_size, unet.image_size]
    sampler = DDIMSampler(model)
    key = model.cond_stage_key
    out = []
    with model.ema_scope():
        uc = None
        if scale != 1.0:
            uc = model.get_learned_conditioning({key: torch.tensor(n_samples_per_class * [1000]).to(model.device)})
        for class_label in classes:
            xc = torch.tensor(n_samples_per_class * [class_label])
            c = model.get_learned_conditioning({key: xc.to(model.device)})
            samples_ddim, _ = sampler.sample(S=ddim_steps, conditioning=c, batch_size=n_samples_per_class, shape=shape,
                                             verbose=False, unconditional_guidance_scale=scale,
                                             unconditional_conditioning=uc, eta=ddim_eta)
            x = model.decode_first_stage(samples_ddim)
            out.append(torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0))
    return torch.cat(out)


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--model", choices=sorted(MODELS), default="cin256-v2",
                   help="cin256-v2 (VQ-f4, guided) or cin256 (the LDM-VQ-8, unguided)")
    p.add_argument("--ckpt", type=str, default=None,
                   help="checkpoint (models/ldm/cin256-v2/model.ckpt or models/ldm/cin256/model.ckpt)")
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of a checkpoint")
    p.add_argument("--tiny", action="store_true", help="the small test configuration (with --random_init)")
    p.add_argument("--outdir", type=str, default="outputs/imagenet")
    p.add_argument("--classes", type=int, nargs="+", default=[25, 187, 448, 992])
    p.add_argument("--n_samples_per_class", type=int, default=6)
    p.add_argument("--ddim_steps", type=int, default=20)
    p.add_argument("--ddim_eta", type=float, default=0.0)
    p.add_argument("--scale", type=float, default=None,
                   help="classifier-free guidance scale (default 3.0; cin256 has no unconditional label: 1.0 only)")
    p.add_argument("--seed", type=int, default=None, help="torch seed of the sampling noise")
    p.add_argument("--no_cuda_graph", action="store_true", help="eager kernel launches instead of CUDA-graph replay")
    return p


def main(argv=None):
    from PIL import Image
    opt = get_parser().parse_args(argv)
    if not opt.random_init and not opt.ckpt:
        raise ValueError("pass --ckpt, or --random_init")
    if opt.tiny and not opt.random_init:
        raise ValueError("--tiny needs --random_init")
    scale = MODELS[opt.model][2] if opt.scale is None else opt.scale
    if opt.model == "cin256" and scale != 1.0:
        raise ValueError("cin256 has no unconditional label (n_classes 1000): it samples unguided, --scale 1.0")
    if opt.seed is not None:
        torch.manual_seed(opt.seed)
    model = load_model(opt.ckpt, opt.random_init, opt.tiny, model=opt.model)
    model.model.diffusion_model.use_cuda_graph = not opt.no_cuda_graph
    t0 = time.time()
    images = sample_classes(model, opt.classes, opt.n_samples_per_class, opt.ddim_steps, opt.ddim_eta, scale)
    torch.cuda.synchronize()
    dt = time.time() - t0
    print(f"{images.shape[0]} images in {dt:.2f} s ({images.shape[0] / dt:.2f} img/s)")
    os.makedirs(opt.outdir, exist_ok=True)
    path = os.path.join(opt.outdir, "grid.png")
    Image.fromarray(make_grid(images, nrow=opt.n_samples_per_class)).save(path)
    print(f"wrote {path}")
    return path


if __name__ == "__main__":
    main()
