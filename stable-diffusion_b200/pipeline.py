"""Script-level call sequences of the reference (scripts/txt2img.py:289-327, scripts/img2img.py:225-270) as callable
pipelines over the H100 engine: conditioning -> sampler -> first-stage decode -> uint8 image.

Inputs are token ids (the tokenizer vocabulary is a host-side, third-party asset; see clip.py) and, optionally, the
start noise x_T so results do not depend on batch size or world size (SURVEY.md Appendix D).
"""
from __future__ import annotations

import torch

from . import arch, ops
from .diffusion import LatentDiffusion
from .samplers import DDIMSampler, DPMSolverSampler, PLMSSampler

V1_PARAMS = dict(linear_start=0.00085, linear_end=0.0120, num_timesteps_cond=1, log_every_t=200, timesteps=1000,
                 first_stage_key="jpg", cond_stage_key="txt", image_size=64, channels=4, cond_stage_trainable=False,
                 conditioning_key="crossattn", monitor="val/loss_simple_ema", scale_factor=0.18215, use_ema=False)


def v1_model_config(unet_cfg=None, vae_cfg=None, clip_cfg=None):
    """The `model:` node of configs/stable-diffusion/v1-inference.yaml as a dict, with the reference's target names
    (sdb200.checkpoint / LatentDiffusion map them onto the sdb200 classes)."""
    return {"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": dict(
        V1_PARAMS,
        unet_config={"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": dict(unet_cfg or arch.SD_V1_UNET)},
        first_stage_config={"target": "ldm.models.autoencoder.AutoencoderKL", "params": dict(vae_cfg or arch.SD_V1_VAE)},
        cond_stage_config={"target": "ldm.modules.encoders.modules.FrozenCLIPEmbedder",
                           "params": {"config": dict(clip_cfg or arch.SD_V1_CLIP)}})}


def build_model(unet_cfg=None, vae_cfg=None, clip_cfg=None):
    """LatentDiffusion with the v1-inference.yaml parameters (configs/stable-diffusion/v1-inference.yaml)."""
    return LatentDiffusion(
        first_stage_config={"target": "sdb200.vae.AutoencoderKL", "params": dict(vae_cfg or arch.SD_V1_VAE)},
        cond_stage_config={"target": "sdb200.clip.FrozenCLIPEmbedder", "params": {"config": dict(clip_cfg or arch.SD_V1_CLIP)}},
        unet_config={"target": "sdb200.unet.UNetModel", "params": dict(unet_cfg or arch.SD_V1_UNET)}, **V1_PARAMS)


# configs/latent-diffusion/txt2img-1p4B-eval.yaml: the LAION-400M model (scripts/txt2img.py --laion400m)
LAION_PARAMS = dict(V1_PARAMS, first_stage_key="image", cond_stage_key="caption", image_size=32,
                    cond_stage_trainable=True)


def laion_model_config(unet_cfg=None, vae_cfg=None, bert_cfg=None):
    """The `model:` node of configs/latent-diffusion/txt2img-1p4B-eval.yaml as a dict, with the reference's target
    names (used when that YAML is not at hand)."""
    bert = dict(bert_cfg or arch.LAION_BERT)
    return {"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": dict(
        LAION_PARAMS,
        unet_config={"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel",
                     "params": dict(unet_cfg or arch.LAION_UNET)},
        first_stage_config={"target": "ldm.models.autoencoder.AutoencoderKL", "params": dict(vae_cfg or arch.SD_V1_VAE)},
        cond_stage_config={"target": "ldm.modules.encoders.modules.BERTEmbedder", "params": bert})}


def build_laion_model(unet_cfg=None, vae_cfg=None, bert_cfg=None):
    """LatentDiffusion with the txt2img-1p4B-eval.yaml parameters: UNet (context 1280), KL-f8, BERTEmbedder."""
    return LatentDiffusion(
        first_stage_config={"target": "sdb200.vae.AutoencoderKL", "params": dict(vae_cfg or arch.SD_V1_VAE)},
        cond_stage_config={"target": "sdb200.bert.BERTEmbedder", "params": dict(bert_cfg or arch.LAION_BERT)},
        unet_config={"target": "sdb200.unet.UNetModel", "params": dict(unet_cfg or arch.LAION_UNET)}, **LAION_PARAMS)


def load_random_weights(model, device, seeds=(11, 12, 13), gen_device=None):
    """Seeded synthetic weights for a LatentDiffusion (no checkpoint offline): the UNet, first stage and cond stage get
    seeds[0], seeds[1] and seeds[2]. A cond stage that is the first stage (__is_first_stage__) is loaded once, with the
    first stage's seed, and stages without `shapes` (Identity, no cond stage) hold no weights. gen_device='cuda' draws
    on the GPU, which gives other numbers than the CPU default."""
    gd = gen_device or "cpu"
    stages = [model.model.diffusion_model, model.first_stage_model]
    if model.cond_stage_model is not model.first_stage_model:
        stages.append(model.cond_stage_model)
    for stage, seed in zip(stages, seeds):
        if getattr(stage, "shapes", None):
            stage.load_weights(arch.random_state_dict(stage.shapes, seed, device=gd), device)
    return model.to(device)


class Txt2Img:
    """scripts/txt2img.py main loop for one batch: uc/c = cond stage (CLIP or BERT) of ids -> sampler.sample -> decode_first_stage ->
    clamp((x+1)/2, 0, 1) -> 255*x uint8 (HWC)."""

    def __init__(self, model, sampler="plms", steps=50, scale=7.5, height=512, width=512, eta=0.0, f=8, channels=4,
                 cuda_graph=True):
        self.model = model
        self.sampler = {"plms": PLMSSampler, "ddim": DDIMSampler, "dpm_solver": DPMSolverSampler}[sampler](model)
        self.steps, self.scale, self.eta = steps, scale, eta
        self.shape = [channels, height // f, width // f]
        model.model.diffusion_model.use_cuda_graph = bool(cuda_graph)

    @torch.no_grad()
    def __call__(self, ids, uncond_ids=None, x_T=None, return_latent=False, return_image01=False):
        """ids / uncond_ids: int64 [B, 77] (device). Returns uint8 [B, H, W, 3] on the device; return_image01=True
        returns the fp32 image clamp((x + 1) / 2, 0, 1) instead (what txt2img.py:317-319 hands to check_safety)."""
        m = self.model
        B = ids.shape[0]
        if self.scale != 1.0:
            assert uncond_ids is not None
            both = m.get_learned_conditioning(torch.cat([uncond_ids, ids]))   # one CLIP pass for [""]*B and prompts
            uc, c = both[:B].contiguous(), both[B:].contiguous()
        else:
            uc, c = None, m.get_learned_conditioning(ids)
        samples, _ = self.sampler.sample(S=self.steps, conditioning=c, batch_size=B, shape=self.shape, verbose=False,
                                         unconditional_guidance_scale=self.scale, unconditional_conditioning=uc,
                                         eta=self.eta, x_T=x_T)
        if return_latent:
            return samples
        x = m.first_stage_model.decode(samples, scale=1. / m.scale_factor, nhwc=True)
        if return_image01:
            return torch.clamp((x + 1.0) / 2.0, min=0.0, max=1.0)
        return ops.to_uint8(x)


class Img2Img:
    """scripts/img2img.py: encode -> stochastic_encode(t_enc) -> DDIM decode -> first-stage decode."""

    def __init__(self, model, steps=50, scale=5.0, strength=0.75, eta=0.0, cuda_graph=True):
        assert 0. <= strength <= 1., "can only work with strength in [0.0, 1.0]"
        self.model = model
        self.sampler = DDIMSampler(model)
        self.steps, self.scale, self.eta = steps, scale, eta
        self.t_enc = int(strength * steps)
        model.model.diffusion_model.use_cuda_graph = bool(cuda_graph)

    @torch.no_grad()
    def __call__(self, init_image, ids, uncond_ids=None, enc_noise=None, noise=None):
        """init_image: fp32 [B, 3, H, W] in [-1, 1] (device); returns uint8 [B, H, W, 3]."""
        m = self.model
        B = ids.shape[0]
        init_latent = m.get_first_stage_encoding(m.encode_first_stage(init_image), noise=enc_noise)
        self.sampler.make_schedule(ddim_num_steps=self.steps, ddim_eta=self.eta, verbose=False)
        if self.scale != 1.0:
            both = m.get_learned_conditioning(torch.cat([uncond_ids, ids]))
            uc, c = both[:B].contiguous(), both[B:].contiguous()
        else:
            uc, c = None, m.get_learned_conditioning(ids)
        z_enc = self.sampler.stochastic_encode(init_latent, torch.tensor([self.t_enc] * B), noise=noise)
        z = self.sampler.decode(z_enc, c, self.t_enc, unconditional_guidance_scale=self.scale,
                                unconditional_conditioning=uc)
        x = m.first_stage_model.decode(z, scale=1. / m.scale_factor, nhwc=True)
        return ops.to_uint8(x)
