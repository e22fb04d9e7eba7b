#!/usr/bin/env python
"""txt2img on the H100 engine with the reference script's flags (scripts/txt2img.py:98-235 of CompVis/stable-diffusion).

  python scripts/txt2img.py --prompt "a photograph of an astronaut riding a horse" --plms --ckpt sd-v1-4.ckpt

With --random_init the three stages get seeded random weights (no checkpoint ships offline); without the CLIP vocabulary
files the prompt is replaced by seeded token ids (--token_seed). Post-processing as in the reference script
(txt2img.py:317-327), on the GPU: the invisible watermark ("StableDiffusionV1", dwtDct) is always embedded unless
--no_watermark; the safety checker runs when its weights are supplied (--safety_ckpt: a diffusers
StableDiffusionSafetyChecker state dict, .safetensors or tensors-only pickle) - no weights ship offline.

--laion400m switches to the LAION-400M model as the reference does (configs/latent-diffusion/txt2img-1p4B-eval.yaml,
models/ldm/text2img-large/model.ckpt, outputs/txt2img-samples-laion400m): BERT-conditioned UNet, same KL-f8 first stage.

Any text-conditional LDM config runs through --config, e.g. the LDM-VQ-4 text-to-image model (BERT-640 text encoder,
VQ-f4 first stage, 64x64x3 latent):

  python scripts/txt2img.py --config models/ldm/text2img256/config.yaml --ckpt models/ldm/text2img256/model.ckpt \
      --H 256 --W 256 --C 3 --f 4 --scale 5.0 --plms --prompt "a virus monster is playing guitar, oil on canvas"

The tokenizer follows the cond stage's class. A FrozenCLIPEmbedder uses the CLIP BPE (--clip_vocab); without it,
seeded CLIP stand-in ids are used. A BERTEmbedder uses the uncased WordPiece vocabulary of --bert_vocab (or the locally
cached bert-base-uncased files); without one, seeded stand-in ids [CLS] r... [SEP] [PAD]... are used and the empty
prompt is [CLS] [SEP] [PAD].... --random_init builds the model --config names with seeded weights; the built-in SD-v1
and LAION values are used only when the reference's default path of either config is absent. --C and --f must match
the model (the UNet's in_channels and the first stage's downsampling factor). The script samples the raw weights, also
for a config with use_ema: a checkpoint's model_ema.* set is loaded, and model.ema_scope() switches to it, but the
sampling loop here does not enter that scope (the reference script does, so its samples of such a checkpoint come from
the EMA weights).
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sdb200  # noqa: E402
from sdb200 import pipeline  # noqa: E402
from sdb200.util import instantiate_from_config, remap_config  # noqa: E402
from sdb200.safety import StableDiffusionSafetyChecker, WatermarkEncoder, put_watermark  # noqa: E402

DEFAULT_CONFIG = "configs/stable-diffusion/v1-inference.yaml"
LAION_CONFIG = "configs/latent-diffusion/txt2img-1p4B-eval.yaml"
LAION_CKPT = "models/ldm/text2img-large/model.ckpt"
LAION_OUTDIR = "outputs/txt2img-samples-laion400m"
BERT_CLS, BERT_SEP, BERT_PAD = 101, 102, 0          # bert-base-uncased [CLS] / [SEP] / [PAD]


def apply_laion400m(opt):
    """txt2img.py:237-241: --laion400m replaces config, checkpoint and output directory."""
    if opt.laion400m:
        print("Falling back to LAION 400M model...")
        opt.config = LAION_CONFIG
        opt.ckpt = LAION_CKPT
        opt.outdir = LAION_OUTDIR
    return opt


def load_model_from_config(config, ckpt, device, verbose=False, random_init=False, unsafe_ckpt=False):
    """scripts/txt2img.py:49-66 via sdb200.checkpoint (pickled .ckpt or .safetensors, reference YAML or built-in values
    of v1-inference.yaml / txt2img-1p4B-eval.yaml when the reference's default path of either is absent). Seeded random
    weights are used only on request (--random_init), for the model the config names: a missing checkpoint or config
    path is an error."""
    laion = config == LAION_CONFIG
    if config and not os.path.exists(config):
        if config not in (DEFAULT_CONFIG, LAION_CONFIG):
            raise FileNotFoundError(f"--config {config} does not exist")
        config = None                         # the reference's default path is absent here: built-in values
    if random_init:
        print("--random_init: seeded random-init weights (images will be noise-like)")
        if config:
            model = instantiate_from_config(remap_config(sdb200.checkpoint.load_config(config)))
        else:
            model = pipeline.build_laion_model() if laion else pipeline.build_model()
        pipeline.load_random_weights(model, device, gen_device=device)
        return model.eval()
    if not ckpt or not os.path.exists(ckpt):
        raise FileNotFoundError(f"checkpoint {ckpt!r} does not exist (pass --ckpt, or --random_init for seeded random "
                                "weights)")
    cfg = config if config else {"model": pipeline.laion_model_config() if laion else pipeline.v1_model_config()}
    return sdb200.checkpoint.load_model_from_config(cfg, ckpt, device=device, verbose=verbose, allow_pickle=unsafe_ckpt)


def synthetic_ids(n, seed, device):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 49406, (n, 77), generator=g)
    ids[:, 0] = 49406
    ids[:, 20:] = 49407
    return ids.to(device)


def synthetic_bert_ids(n, seed, device, vocab_size=30522):
    """Stand-in bert-base-uncased ids: [CLS], 19 seeded word-piece ids (999 .. vocab_size - 1; 103 .. for a vocabulary
    of at most 2000 rows), [SEP], [PAD]..."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.full((n, 77), BERT_PAD, dtype=torch.long)
    ids[:, 0] = BERT_CLS
    ids[:, 1:20] = torch.randint(999 if vocab_size > 2000 else 103, vocab_size, (n, 19), generator=g)
    ids[:, 20] = BERT_SEP
    return ids.to(device)


def bert_uncond_ids(n, device):
    """The empty prompt as bert-base-uncased tokenises it: [CLS] [SEP] [PAD]..."""
    ids = torch.full((n, 77), BERT_PAD, dtype=torch.long)
    ids[:, 0], ids[:, 1] = BERT_CLS, BERT_SEP
    return ids.to(device)


def text_encoder_kind(model):
    """"bert" or "clip" from the class of the model's cond stage; a model that is not text-conditional is an error."""
    enc = model.cond_stage_model
    if isinstance(enc, sdb200.BERTEmbedder):
        return "bert"
    if isinstance(enc, sdb200.FrozenCLIPEmbedder):
        return "clip"
    raise SystemExit(f"error: the cond stage {type(enc).__name__} is not a text encoder (BERTEmbedder or "
                     "FrozenCLIPEmbedder); txt2img samples text-conditional models only")


def stand_in_ids(kind, enc, n, seed, device):
    """Seeded (prompt ids, empty-prompt ids) for the cond stage when no tokenizer vocabulary is available."""
    if kind == "bert":
        return synthetic_bert_ids(n, seed, device, enc.cfg["vocab_size"]), bert_uncond_ids(n, device)
    un = torch.full((n, 77), 49407, dtype=torch.long, device=device)
    un[:, 0] = 49406
    return synthetic_ids(n, seed, device), un


def check_latent_shape(model, C, f):
    """--C must be the UNet's in_channels and --f the first stage's downsampling factor 2 ** (len(ch_mult) - 1)."""
    want_c = model.model.diffusion_model.in_channels
    want_f = 2 ** (len(model.first_stage_model.cfg["ddconfig"]["ch_mult"]) - 1)
    if (C, f) != (want_c, want_f):
        raise SystemExit(f"error: --C {C} --f {f} do not match the model: pass --C {want_c} --f {want_f} (the UNet's "
                         f"in_channels and the first stage's downsampling factor)")


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--prompt", type=str, nargs="?", default="a painting of a virus monster playing guitar")
    p.add_argument("--outdir", type=str, nargs="?", default="outputs/txt2img-samples")
    p.add_argument("--skip_grid", action="store_true")
    p.add_argument("--skip_save", action="store_true", help="do not save individual samples. For speed measurements.")
    p.add_argument("--ddim_steps", type=int, default=50)
    p.add_argument("--plms", action="store_true")
    p.add_argument("--dpm_solver", action="store_true")
    p.add_argument("--laion400m", action="store_true")
    p.add_argument("--fixed_code", action="store_true")
    p.add_argument("--ddim_eta", type=float, default=0.0)
    p.add_argument("--n_iter", type=int, default=2)
    p.add_argument("--H", type=int, default=512)
    p.add_argument("--W", type=int, default=512)
    p.add_argument("--C", type=int, default=4)
    p.add_argument("--f", type=int, default=8)
    p.add_argument("--n_samples", type=int, default=3)
    p.add_argument("--n_rows", type=int, default=0)
    p.add_argument("--scale", type=float, default=7.5)
    p.add_argument("--from-file", type=str)
    p.add_argument("--config", type=str, default=DEFAULT_CONFIG)
    p.add_argument("--ckpt", type=str, default="models/ldm/stable-diffusion-v1/model.ckpt")
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of a checkpoint")
    p.add_argument("--unsafe-ckpt", action="store_true", help="allow full unpickling of a .ckpt (runs code from the file)")
    p.add_argument("--precision", type=str, choices=["full", "autocast"], default="autocast")
    p.add_argument("--clip_vocab", type=str, default=None,
                   help="directory with the CLIP vocab.json + merges.txt (host-side BPE); default: transformers' local cache")
    p.add_argument("--bert_vocab", type=str, default=None,
                   help="directory with the bert-base-uncased vocab.txt (any BERTEmbedder cond stage); default: the "
                        "local Hugging Face cache")
    p.add_argument("--token_seed", type=int, default=1234, help="seed of the stand-in token ids (no tokenizer offline)")
    p.add_argument("--safety_ckpt", type=str, default=None,
                   help="state dict of diffusers' StableDiffusionSafetyChecker: flagged images are blanked (txt2img.py:88-95)")
    p.add_argument("--no_watermark", action="store_true", help="do not embed the invisible watermark (txt2img.py:261-264)")
    opt = apply_laion400m(p.parse_args(argv))
    torch.manual_seed(opt.seed)           # seed_everything (txt2img.py:243)
    device = torch.device("cuda")
    model = load_model_from_config(opt.config, opt.ckpt, device, random_init=opt.random_init, unsafe_ckpt=opt.unsafe_ckpt)
    kind = text_encoder_kind(model)
    check_latent_shape(model, opt.C, opt.f)
    sampler = "dpm_solver" if opt.dpm_solver else ("plms" if opt.plms else "ddim")
    pipe = pipeline.Txt2Img(model, sampler=sampler, steps=opt.ddim_steps, scale=opt.scale,
                            height=opt.H, width=opt.W, eta=opt.ddim_eta, f=opt.f, channels=opt.C)
    safety_checker = None
    if opt.safety_ckpt:
        if not os.path.exists(opt.safety_ckpt):
            raise FileNotFoundError(f"--safety_ckpt {opt.safety_ckpt} does not exist")
        ssd, _ = sdb200.checkpoint.read_state_dict(opt.safety_ckpt, allow_pickle=opt.unsafe_ckpt)
        safety_checker = StableDiffusionSafetyChecker().load_weights(ssd, device)
    wm_encoder = None
    if not opt.no_watermark:
        print("Creating invisible watermark encoder (see https://github.com/ShieldMnt/invisible-watermark)...")
        wm_encoder = WatermarkEncoder()
        wm_encoder.set_watermark("bytes", "StableDiffusionV1".encode("utf-8"))
    os.makedirs(opt.outdir, exist_ok=True)
    sample_path = os.path.join(opt.outdir, "samples")
    os.makedirs(sample_path, exist_ok=True)
    B = opt.n_samples
    if opt.from_file:
        with open(opt.from_file) as f:
            prompts = f.read().splitlines()
    else:
        prompts = [opt.prompt]
    enc = model.cond_stage_model
    if opt.clip_vocab and kind == "clip":
        enc.version, enc.tokenizer = opt.clip_vocab, None
    if opt.bert_vocab and kind == "bert":
        enc.vocab_dir, enc.tokenizer = opt.bert_vocab, None
    start_code = torch.randn([B, opt.C, opt.H // opt.f, opt.W // opt.f], device=device) if opt.fixed_code else None
    base_count = len(os.listdir(sample_path))
    tic = time.time()
    n_img = 0
    for n in range(opt.n_iter):
        for pi, prompt in enumerate(prompts):
            try:
                ids = enc._tokenize(B * [prompt]).to(device)
                un = enc._tokenize(B * [""]).to(device)
            except RuntimeError as e:
                if n == 0 and pi == 0:
                    print(f"tokenizer unavailable ({e}); using seeded token ids")
                ids, un = stand_in_ids(kind, enc, B, opt.token_seed + pi, device)
            x_T = start_code if start_code is not None else torch.randn(
                [B, opt.C, opt.H // opt.f, opt.W // opt.f], device=device)      # plms.py:124
            if safety_checker is not None:       # check_safety on the fp32 image, then 255 * x -> uint8 (txt2img.py:317-322)
                x01 = pipe(ids, un if opt.scale != 1.0 else None, x_T=x_T, return_image01=True)
                x01, has_nsfw = safety_checker.check_safety(x01)
                if any(has_nsfw):
                    print(f"safety checker: {sum(has_nsfw)} of {B} images blanked")
                img = (255.0 * x01).to(torch.uint8)
            else:
                img = pipe(ids, un if opt.scale != 1.0 else None, x_T=x_T)       # uint8 [B, H, W, 3]
            img = put_watermark(img, wm_encoder)                                 # txt2img.py:324
            n_img += B
            if not opt.skip_save:
                from PIL import Image
                for x in img.cpu().numpy():
                    Image.fromarray(x.astype(np.uint8)).save(os.path.join(sample_path, f"{base_count:05}.png"))
                    base_count += 1
    torch.cuda.synchronize()
    toc = time.time()
    print(f"Your samples are ready and waiting for you here: \n{opt.outdir} \n"
          f"{n_img} images in {toc - tic:.2f} s ({n_img / (toc - tic):.2f} images/s). Enjoy.")
    return opt.outdir


if __name__ == "__main__":
    main()
