"""Retrieval-augmented text-to-image sampling on the H100 engine: the reference's scripts/knn2img.py
(configs/retrieval-augmented-diffusion/768x768.yaml, models/rdm/rdm768x768/model.ckpt):

  python scripts/knn2img.py --prompt "a happy bear reading a newspaper, oil on canvas" --clip_vocab <dir> \
      --clip_ckpt <clip-vit-large-patch14 model.safetensors> [--use_neighbors --knn 10 --database artbench-surrealism]

The prompt is encoded by FrozenCLIPTextEmbedder (CLIP ViT-L/14's projected, normalised text embedding, (B, 1, 768)).
With --use_neighbors the Searcher (sdb200.retrieval) loads data/rdm/retrieval_databases/<database>/*.npz, takes the
--knn rows of the largest dot product with the normalised query, exactly, on the GPU, and appends their normalised
embeddings: (B, 1 + knn, 768). --database_dir DIR reads the shards from DIR instead (a database built by
scripts/build_rdm_database.py, which the fixed --database names cannot point at). The unconditional conditioning is
zeros_like(c) when --scale is not 1; DDIM (or PLMS) samples the [16, H/16, W/16] latent inside ema_scope() on the CUDA-graph path, and decode_first_stage (KL-f16) gives the
images, written as samples/NNNNN.png and one grid per --n_iter, as the reference does.

CLIP's weights are read in the transformers CLIPModel layout (`text_model.*`, `text_projection.weight`; the vision
tower's keys are ignored) from --clip_ckpt; --clip_vocab is a directory with CLIP's vocab.json + merges.txt. With
--random_init no checkpoint is read and every stage gets seeded random weights (--tiny: the small test members).
--n_repeat is parsed and unused, as in the reference.
"""
import argparse
import os
import sys
import time
from itertools import islice

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import sdb200  # noqa: E402
from sample_imagenet import make_grid  # noqa: E402
from sdb200 import arch, pipeline  # noqa: E402
from sdb200.retrieval import DATABASES, Searcher  # noqa: E402
from sdb200.samplers import DDIMSampler, PLMSSampler  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402


def rdm_config(unet_cfg=None, vae_cfg=None):
    """configs/retrieval-augmented-diffusion/768x768.yaml, `model:` node (reference targets)."""
    u = dict(unet_cfg or arch.RDM_UNET)
    v = dict(vae_cfg or arch.KL_F16)
    return {"base_learning_rate": 0.0001, "target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        "linear_start": 0.0015, "linear_end": 0.015, "num_timesteps_cond": 1, "log_every_t": 200, "timesteps": 1000,
        "first_stage_key": "jpg", "cond_stage_key": "nix", "image_size": u["image_size"], "channels": u["in_channels"],
        "cond_stage_trainable": False, "conditioning_key": "crossattn", "monitor": "val/loss_simple_ema",
        "scale_by_std": False, "scale_factor": 0.22765929,
        "unet_config": {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": u},
        "first_stage_config": {"target": "ldm.models.autoencoder.AutoencoderKL",
                               "params": {"monitor": "val/rec_loss", **v, "lossconfig": {"target": "torch.nn.Identity"}}},
        "cond_stage_config": {"target": "torch.nn.Identity"}}}


def load_model(ckpt=None, random_init=False, tiny=False, device="cuda", unsafe_ckpt=False):
    dev = torch.device(device)
    node = rdm_config(arch.TINY_RDM_UNET, arch.TINY_KL_F16) if tiny else rdm_config()
    if not random_init:
        return sdb200.checkpoint.load_model_from_config({"model": node}, ckpt, device=dev, allow_pickle=unsafe_ckpt)
    return pipeline.load_random_weights(instantiate_from_config(remap_config(node)), dev, gen_device=dev).eval()


def load_clip(clip_ckpt=None, clip_vocab=None, random_init=False, tiny=False, device="cuda", unsafe_ckpt=False):
    """FrozenCLIPTextEmbedder('ViT-L/14') with its weights from a transformers CLIPModel checkpoint, or seeded."""
    cfg = arch.TINY_CLIP_TEXT_PROJ if tiny else arch.CLIP_TEXT_PROJ
    enc = sdb200.FrozenCLIPTextEmbedder(version=clip_vocab or "ViT-L/14", config=cfg)
    if clip_ckpt:
        sd, _ = sdb200.checkpoint.read_state_dict(clip_ckpt, allow_pickle=unsafe_ckpt)
        return enc.load_weights(sd, device)
    if not random_init:
        raise ValueError("pass --clip_ckpt (CLIP ViT-L/14 in the transformers CLIPModel layout), or --random_init")
    return enc.load_weights(arch.random_state_dict(enc.shapes, 13, device=torch.device(device)), device)


def chunk(it, size):
    it = iter(it)
    return iter(lambda: tuple(islice(it, size)), ())


@torch.no_grad()
def sample(model, clip_encoder, prompts, searcher=None, knn=10, ddim_steps=50, plms=False, eta=0.0, scale=5.0, H=768,
           W=768):
    """One batch of the reference's loop; returns the decoded images [B, 3, H, W] in [0, 1] and the conditioning."""
    dev = model.device
    c = clip_encoder.encode(list(prompts))
    if searcher is not None:
        nn_dict = searcher(c, knn)
        c = torch.cat([c, torch.from_numpy(nn_dict["nn_embeddings"]).to(dev).float()], dim=1)
    uc = torch.zeros_like(c) if scale != 1.0 else None
    shape = [16, H // 16, W // 16]
    sampler = PLMSSampler(model) if plms else DDIMSampler(model)
    samples, _ = sampler.sample(S=ddim_steps, conditioning=c, batch_size=c.shape[0], shape=shape, verbose=False,
                                unconditional_guidance_scale=scale, unconditional_conditioning=uc, eta=eta)
    x = model.decode_first_stage(samples)
    return torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0), c


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("--prompt", type=str, nargs="?", default="a painting of a virus monster playing guitar")
    p.add_argument("--outdir", type=str, nargs="?", default="outputs/txt2img-samples")
    p.add_argument("--skip_grid", action="store_true")
    p.add_argument("--ddim_steps", type=int, default=50)
    p.add_argument("--n_repeat", type=int, default=1, help="parsed and unused, as in the reference")
    p.add_argument("--plms", action="store_true")
    p.add_argument("--ddim_eta", type=float, default=0.0)
    p.add_argument("--n_iter", type=int, default=1)
    p.add_argument("--H", type=int, default=768)
    p.add_argument("--W", type=int, default=768)
    p.add_argument("--n_samples", type=int, default=3)
    p.add_argument("--n_rows", type=int, default=0)
    p.add_argument("--scale", type=float, default=5.0)
    p.add_argument("--from-file", type=str)
    p.add_argument("--config", type=str, default=None,
                   help="a reference config YAML (default: the built-in values of configs/retrieval-augmented-diffusion/"
                        "768x768.yaml)")
    p.add_argument("--ckpt", type=str, default="models/rdm/rdm768x768/model.ckpt")
    p.add_argument("--clip_type", type=str, default="ViT-L/14")
    p.add_argument("--database", type=str, default="artbench-surrealism", choices=DATABASES)
    p.add_argument("--database_dir", type=str, default=None,
                   help="a database directory of .npz shards (e.g. from scripts/build_rdm_database.py); overrides the "
                        "--database path")
    p.add_argument("--use_neighbors", default=False, action="store_true")
    p.add_argument("--knn", default=10, type=int)
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of checkpoints")
    p.add_argument("--tiny", action="store_true", help="the small test configuration (with --random_init)")
    p.add_argument("--seed", type=int, default=None, help="torch seed of the sampling noise")
    p.add_argument("--clip_vocab", type=str, default=None, help="directory with the CLIP vocab.json + merges.txt")
    p.add_argument("--clip_ckpt", type=str, default=None,
                   help="CLIP ViT-L/14 weights in the transformers CLIPModel layout (.safetensors or .ckpt)")
    p.add_argument("--unsafe-ckpt", action="store_true", help="allow full unpickling of a .ckpt (runs code from the file)")
    p.add_argument("--no_cuda_graph", action="store_true", help="eager kernel launches instead of CUDA-graph replay")
    return p


def main(argv=None):
    from PIL import Image
    opt = get_parser().parse_args(argv)
    if opt.clip_type != "ViT-L/14":
        raise NotImplementedError(f"--clip_type {opt.clip_type}: the model was trained on ViT-L/14 embeddings")
    if opt.tiny and not opt.random_init:
        raise ValueError("--tiny needs --random_init")
    if opt.H % 16 or opt.W % 16:
        raise ValueError(f"--H / --W must be multiples of 16 (the KL-f16 first stage), got {opt.H} x {opt.W}")
    if opt.use_neighbors and opt.knn < 1:
        raise ValueError("--knn must be at least 1")
    if opt.plms and opt.ddim_eta != 0:
        raise ValueError("ddim_eta must be 0 for PLMS")
    if opt.seed is not None:
        torch.manual_seed(opt.seed)
    device = torch.device("cuda")
    if opt.config and not opt.random_init:
        model = sdb200.checkpoint.load_model_from_config(opt.config, opt.ckpt, device=device,
                                                         allow_pickle=opt.unsafe_ckpt)
    else:
        model = load_model(opt.ckpt, opt.random_init, opt.tiny, device, opt.unsafe_ckpt)
    model.model.diffusion_model.use_cuda_graph = not opt.no_cuda_graph
    clip_encoder = load_clip(opt.clip_ckpt, opt.clip_vocab, opt.random_init, opt.tiny, device, opt.unsafe_ckpt)

    batch_size = opt.n_samples
    n_rows = opt.n_rows if opt.n_rows > 0 else batch_size
    if not opt.from_file:
        data = [batch_size * [opt.prompt]]
    else:
        with open(opt.from_file, "r") as f:
            data = list(chunk(f.read().splitlines(), batch_size))
    sample_path = os.path.join(opt.outdir, "samples")
    os.makedirs(sample_path, exist_ok=True)
    base_count = len(os.listdir(sample_path))
    grid_count = len(os.listdir(opt.outdir)) - 1
    searcher = Searcher(opt.database, device=device, path=opt.database_dir) if opt.use_neighbors else None

    written = []
    t0 = time.time()
    n_images = 0
    with model.ema_scope():
        for _ in range(opt.n_iter):
            all_samples = []
            for prompts in data:
                x, _ = sample(model, clip_encoder, prompts, searcher, opt.knn, opt.ddim_steps, opt.plms, opt.ddim_eta,
                              opt.scale, opt.H, opt.W)
                n_images += x.shape[0]
                arr = (255. * x.permute(0, 2, 3, 1).cpu().numpy()).astype(np.uint8)
                for a in arr:
                    path = os.path.join(sample_path, f"{base_count:05}.png")
                    Image.fromarray(a).save(path)
                    written.append(path)
                    base_count += 1
                all_samples.append(x)
            if not opt.skip_grid:
                path = os.path.join(opt.outdir, f"grid-{grid_count:04}.png")
                Image.fromarray(make_grid(torch.cat(all_samples), nrow=n_rows)).save(path)
                written.append(path)
                grid_count += 1
    torch.cuda.synchronize()
    dt = time.time() - t0
    print(f"{n_images} images in {dt:.2f} s ({n_images / dt:.2f} img/s)")
    print(f"Your samples are ready and waiting for you here: \n{opt.outdir} \nEnjoy.")
    return written


if __name__ == "__main__":
    main()
