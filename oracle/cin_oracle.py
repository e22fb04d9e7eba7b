"""ORACLE — test infrastructure only. The class-conditional ImageNet LDM (configs/latent-diffusion/cin256-v2.yaml) as
plain functional PyTorch on state dicts: the ClassEmbedder (ldm/modules/encoders/modules.py:19-32) and DDIM with
classifier-free guidance on an arbitrary schedule (ddim.py:78-204 with unconditional_conditioning). The UNet is
ldm_oracle.unet_forward with num_heads 1 (legacy dim_head = ch), the first stage vq_oracle.decode_first_stage.
Pinned against the unmodified reference by oracle/make_golden_cin.py (tests/golden/cin.pt)."""
from __future__ import annotations

import numpy as np
import torch


def class_embed(sd, labels):
    """ClassEmbedder.forward: embedding(batch[key][:, None]) -> [B, 1, embed_dim]."""
    return sd["embedding.weight"][labels.long()][:, None]


def ddim_sample_guided(model_fn, x_T, c, uc, scale, alphas_cumprod, S):
    """DDIMSampler.sample, eta 0, with guidance: e = e_u + scale (e_c - e_u) from one [uc; c] batch (ddim.py:171-178).
    model_fn(x, t, context) -> eps."""
    step = 1000 // S
    ts = np.asarray(list(range(0, 1000, step))) + 1
    ac = alphas_cumprod.numpy()
    a = ac[ts]
    ap = np.asarray([ac[0]] + ac[ts[:-1]].tolist())
    f = lambda v: torch.tensor(float(np.float32(v)))
    x = x_T
    b = x.shape[0]
    for j, t in enumerate(np.flip(ts)):
        index = S - j - 1
        tt = torch.full((2 * b,), int(t), dtype=torch.long)
        e_u, e_c = model_fn(torch.cat([x] * 2), tt, torch.cat([uc, c])).chunk(2)
        e = e_u + scale * (e_c - e_u)
        a_t, a_prev = f(a[index]), f(ap[index])
        p0 = (x - torch.sqrt(1. - a_t) * e) / a_t.sqrt()
        x = a_prev.sqrt() * p0 + (1. - a_prev).sqrt() * e
    return x
