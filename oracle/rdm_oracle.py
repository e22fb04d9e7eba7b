"""ORACLE — test infrastructure only. The retrieval-augmented diffusion model (configs/retrieval-augmented-diffusion/
768x768.yaml, scripts/knn2img.py) as plain functional PyTorch on state dicts:

- `unet_forward`: cin_f8_oracle's spatial-transformer UNet with heads of num_head_channels (here 32), cross-attending
  to the [text | neighbours] context.
- `kl_encode_moments`, `kl_decode`, `decode_first_stage`: AutoencoderKL (autoencoder.py:285-333) on cin_f8_oracle's
  Encoder / Decoder with AttnBlocks inside the levels (KL-f16: at 16x16).
- `ddim_sample` (any eta, replayed noise draws) and `plms_sample` with classifier-free guidance on a model's own
  alphas_cumprod (linear_end 0.015).
- `clip_text_embed`: FrozenCLIPTextEmbedder.forward (modules.py:182-187): ldm_oracle's CLIP text tower, the EOT row,
  text_projection, L2 normalisation.
Pinned against the unmodified reference by oracle/make_golden_rdm.py (tests/golden/rdm.pt)."""
from __future__ import annotations

import numpy as np
import torch

import cin_f8_oracle as F8
from ldm_oracle import _conv, _guided_eps, clip_text
from uncond_oracle import ddim_sample_uncond

unet_forward = F8.unet_forward


def kl_encode_moments(sd, x):
    """AutoencoderKL.encode before the posterior: quant_conv(encoder(x)) = [mean | logvar]."""
    return _conv(F8.vae_encoder(sd, x), sd, "quant_conv", padding=0)


def kl_decode(sd, z):
    """AutoencoderKL.decode: decoder(post_quant_conv(z))."""
    return F8.vae_decoder(sd, _conv(z, sd, "post_quant_conv", padding=0))


def decode_first_stage(sd, z, scale_factor=0.22765929):
    return kl_decode(sd, 1. / scale_factor * z)


def ddim_sample(model_fn, x_T, c, uc, scale, alphas_cumprod, S, eta, noises):
    """Guided DDIMSampler.sample (ddim.py:78-204): eta > 0 adds sigma_t * noises[j] at step j."""
    return ddim_sample_uncond(lambda x, t: _guided_eps(model_fn, x, t, c, uc, scale), x_T, alphas_cumprod, S, eta,
                              noises)


def plms_sample(model_fn, x_T, c, uc, scale, alphas_cumprod, S):
    """Guided PLMSSampler.sample (plms.py:114-236, eta 0) on the given alphas_cumprod."""
    ts = np.asarray(list(range(0, 1000, 1000 // S))) + 1
    ac = alphas_cumprod.numpy().astype(np.float64)
    a, ap = ac[ts], np.asarray([ac[0]] + ac[ts[:-1]].tolist())
    f = lambda v: float(np.float32(v))
    sc = dict(alphas=[f(v) for v in a], alphas_prev=[f(v) for v in ap], sigmas=[0.0] * S,
              sqrt_one_minus_alphas=[f(v) for v in np.sqrt(1. - a)])
    from ldm_oracle import _x_prev
    time_range = np.flip(ts)
    img, old_eps, b = x_T, [], x_T.shape[0]
    for i, step in enumerate(time_range):
        index = S - i - 1
        t = torch.full((b,), int(step), dtype=torch.long)
        t_next = torch.full((b,), int(time_range[min(i + 1, S - 1)]), dtype=torch.long)
        e_t = _guided_eps(model_fn, img, t, c, uc, scale)
        if not old_eps:
            x_prev, _ = _x_prev(img, e_t, sc, index)
            e_prime = (e_t + _guided_eps(model_fn, x_prev, t_next, c, uc, scale)) / 2
        elif len(old_eps) == 1:
            e_prime = (3 * e_t - old_eps[-1]) / 2
        elif len(old_eps) == 2:
            e_prime = (23 * e_t - 16 * old_eps[-1] + 5 * old_eps[-2]) / 12
        else:
            e_prime = (55 * e_t - 59 * old_eps[-1] + 37 * old_eps[-2] - 9 * old_eps[-3]) / 24
        img, _ = _x_prev(img, e_prime, sc, index)
        old_eps.append(e_t)
        if len(old_eps) >= 4:
            old_eps.pop(0)
    return img


def clip_text_embed(sd, ids, num_heads):
    """encode_text + normalisation: the final-LayerNorm output at argmax(ids), @ text_projection^T, / its L2 norm."""
    h = clip_text(sd, ids, num_heads)
    pooled = h[torch.arange(h.shape[0]), ids.argmax(dim=-1)]
    z = pooled @ sd["text_projection.weight"].t()
    return z / torch.linalg.norm(z, dim=1, keepdim=True)
