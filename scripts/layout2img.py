#!/usr/bin/env python
"""Layout-to-image sampling on the H100 engine with the layout-to-image LDM (models/ldm/layout2img-openimages256):

  python scripts/layout2img.py --ckpt models/ldm/layout2img-openimages256/model.ckpt --tokens layout.pt
  python scripts/layout2img.py --random_init --n_samples 4

The model is conditioned on 92 bounding-box token ids per image (cond_stage_key coordinates_bbox): a BERTEmbedder with
use_tokenizer False embeds them as they are. The ids come from the OpenImages conditional builder, which is not part of
this project: --tokens reads them from a .pt or .npy file of integer ids of shape [92] (one layout, repeated
--n_samples times) or [B, 92] (one sample per row). Ids outside [0, vocab_size) or rows of another length are rejected
with BERTEmbedder.check_ids' error. --random_init samples seeded random weights, on seeded stand-in ids unless --tokens
is given.

Sampling follows the reference's only sampling path for this model, LatentDiffusion.log_images (ddpm.py:1251-1305):
DDIM, 200 steps, eta 1, unguided (the model has no unconditional layout, so there is no guidance scale), inside
ema_scope() (the checkpoint's model_ema.* weights when it has them), then decode_first_stage with re-quantization and
clamp((x + 1) / 2, 0, 1), written as PNGs under --outdir/samples. When --config is the reference's default path and that
file is absent, the built-in copy of its model node (layout2img_config) is used.
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

DEFAULT_CONFIG = "models/ldm/layout2img-openimages256/config.yaml"
DEFAULT_CKPT = "models/ldm/layout2img-openimages256/model.ckpt"


def layout2img_config(unet_cfg=None, vq_cfg=None, bert_cfg=None):
    """models/ldm/layout2img-openimages256/config.yaml, `model:` node (reference targets)."""
    u = dict(unet_cfg or arch.LAYOUT2IMG_UNET)
    v = dict(vq_cfg or arch.VQ_F4)
    b = dict(bert_cfg or arch.LAYOUT2IMG_BERT)
    return {"base_learning_rate": 2.0e-06, "target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        "linear_start": 0.0015, "linear_end": 0.0205, "log_every_t": 100, "timesteps": 1000, "loss_type": "l1",
        "first_stage_key": "image", "cond_stage_key": "coordinates_bbox", "image_size": u["image_size"],
        "channels": u["in_channels"], "conditioning_key": "crossattn", "cond_stage_trainable": True,
        "unet_config": {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": u},
        "first_stage_config": {"target": "ldm.models.autoencoder.VQModelInterface",
                               "params": {**v, "monitor": "val/rec_loss",
                                          "lossconfig": {"target": "torch.nn.Identity"}}},
        "cond_stage_config": {"target": "ldm.modules.encoders.modules.BERTEmbedder",
                              "params": {**b, "use_tokenizer": False}},
        "monitor": "val/loss_simple_ema"}}


def load_model(config, ckpt, device, random_init=False, unsafe_ckpt=False):
    """The model --config names (a reference YAML, or layout2img_config when the default path is absent), with the
    checkpoint's weights (.ckpt or .safetensors; model_ema.* become the UNet's "ema" set) or seeded random weights."""
    if config and not os.path.exists(config):
        if config != DEFAULT_CONFIG:
            raise FileNotFoundError(f"--config {config} does not exist")
        config = None                         # the reference's default path is absent here: built-in values
    cfg = config if config else {"model": layout2img_config()}
    if random_init:
        print("--random_init: seeded random-init weights (images will be noise-like)")
        model = instantiate_from_config(remap_config(sdb200.checkpoint.load_config(cfg)))
        pipeline.load_random_weights(model, device, gen_device=device)
        return model.eval()
    if not ckpt or not os.path.exists(ckpt):
        raise FileNotFoundError(f"checkpoint {ckpt!r} does not exist (pass --ckpt, or --random_init for seeded random "
                                "weights)")
    return sdb200.checkpoint.load_model_from_config(cfg, ckpt, device=device, allow_pickle=unsafe_ckpt)


def check_layout_ids(bert, ids):
    """Integer ids [B, max_seq_len] on the host, validated by BERTEmbedder.check_ids (dtype, rank, range, at most
    max_seq_len ids); the layout model also needs exactly max_seq_len ids per row."""
    ids = bert.check_ids(ids)
    n = bert.cfg["max_seq_len"]
    if ids.shape[1] != n:
        raise ValueError(f"BERTEmbedder: need B >= 1 and 1 <= n <= {n} tokens (got {tuple(ids.shape)}); this model "
                         f"takes exactly {n} bounding-box token ids per sample")
    return ids


def read_token_file(path, n_samples):
    """Ids of a .pt (a tensor) or .npy file: shape [n] is one layout repeated n_samples times, [B, n] one per row.
    Other ranks are passed on unchanged, for check_layout_ids to reject."""
    if path.endswith(".npy"):
        ids = torch.from_numpy(np.load(path, allow_pickle=False))
    elif path.endswith(".pt"):
        ids = torch.load(path, map_location="cpu", weights_only=True)
        if not torch.is_tensor(ids):
            raise TypeError(f"{path}: expected a tensor of token ids, got {type(ids).__name__}")
    else:
        raise ValueError(f"{path}: --tokens takes a .pt or .npy file")
    return ids.unsqueeze(0).repeat(n_samples, 1) if ids.dim() == 1 else ids


def stand_in_ids(bert, n_samples, seed):
    """Seeded stand-in layout ids: n_samples rows of max_seq_len ids in [0, vocab_size)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, bert.cfg["vocab_size"], (n_samples, bert.cfg["max_seq_len"]), generator=g)


@torch.no_grad()
def sample_latents(model, ids, ddim_steps=200, ddim_eta=1.0, x_T=None):
    """log_images' sampling: c = the cond stage of the ids, unguided DDIM inside ema_scope()."""
    unet = model.model.diffusion_model
    shape = [unet.in_channels, unet.image_size, unet.image_size]
    c = model.get_learned_conditioning(ids.to(model.device))
    with model.ema_scope():
        samples, _ = DDIMSampler(model).sample(S=ddim_steps, conditioning=c, batch_size=ids.shape[0], shape=shape,
                                               verbose=False, eta=ddim_eta, x_T=x_T)
    return samples


@torch.no_grad()
def decode(model, samples):
    """decode_first_stage (the VQ first stage re-quantizes) and clamp((x + 1) / 2, 0, 1): [B, 3, H, W] in [0, 1]."""
    return torch.clamp((model.decode_first_stage(samples) + 1.0) / 2.0, min=0.0, max=1.0)


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--config", type=str, default=DEFAULT_CONFIG)
    p.add_argument("--ckpt", type=str, default=DEFAULT_CKPT)
    p.add_argument("--tokens", type=str, default=None,
                   help=".pt or .npy file of integer bounding-box token ids, shape [92] or [B, 92]")
    p.add_argument("--random_init", action="store_true",
                   help="seeded random weights instead of a checkpoint (and seeded stand-in ids without --tokens)")
    p.add_argument("--n_samples", type=int, default=8, help="samples of a [92] layout or of the stand-in ids")
    p.add_argument("--ddim_steps", type=int, default=200)
    p.add_argument("--ddim_eta", type=float, default=1.0)
    p.add_argument("--seed", type=int, default=42, help="seed of the sampling noise and of the stand-in ids")
    p.add_argument("--outdir", type=str, default="outputs/layout2img-samples")
    p.add_argument("--skip_save", action="store_true", help="do not write the PNGs")
    p.add_argument("--no_cuda_graph", action="store_true", help="eager kernel launches instead of CUDA-graph replay")
    p.add_argument("--unsafe_ckpt", action="store_true",
                   help="allow arbitrary pickled objects in a .ckpt (only for checkpoints you trust)")
    return p


def main(argv=None):
    from PIL import Image
    opt = get_parser().parse_args(argv)
    if opt.tokens is None and not opt.random_init:
        raise SystemExit("error: pass --tokens FILE with the layout's token ids (or --random_init for stand-in ids)")
    torch.manual_seed(opt.seed)
    dev = torch.device("cuda")
    model = load_model(opt.config, opt.ckpt, dev, random_init=opt.random_init, unsafe_ckpt=opt.unsafe_ckpt)
    bert = model.cond_stage_model
    if opt.tokens is not None:
        ids = check_layout_ids(bert, read_token_file(opt.tokens, opt.n_samples))
    else:
        ids = stand_in_ids(bert, opt.n_samples, opt.seed)
        print(f"seeded token ids (seed {opt.seed}) in place of a layout")
    model.model.diffusion_model.use_cuda_graph = not opt.no_cuda_graph
    t0 = time.time()
    images = decode(model, sample_latents(model, ids, opt.ddim_steps, opt.ddim_eta))
    torch.cuda.synchronize()
    dt = time.time() - t0
    print(f"{images.shape[0]} images in {dt:.2f} s ({images.shape[0] / dt:.2f} img/s)")
    if opt.skip_save:
        return []
    out = os.path.join(opt.outdir, "samples")
    os.makedirs(out, exist_ok=True)
    base = len(os.listdir(out))
    paths = []
    for i, img in enumerate((255. * images.permute(0, 2, 3, 1)).to(torch.uint8).cpu().numpy()):
        paths.append(os.path.join(out, f"{base + i:05}.png"))
        Image.fromarray(img).save(paths[-1])
    print(f"wrote {len(paths)} images to {out}")
    return paths


if __name__ == "__main__":
    main()
