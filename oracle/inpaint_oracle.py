"""ORACLE — test infrastructure only. Never imported by the product path (stable-diffusion_b200/).

CPU fp32 restatement of the per-image steps of the reference's scripts/inpaint.py (models/ldm/inpainting_big):
`make_batch` on decoded uint8 arrays (PIL's decoding and convert("RGB") / convert("L") stay with the caller),
the conditioning's mask channel (F.interpolate, nearest, to the latent size) and the final composite.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def make_batch(image_u8, mask_u8):
    """image uint8 [h, w, 3], mask uint8 [h, w] -> {"image", "mask", "masked_image"}, each NCHW fp32 mapped x*2-1."""
    image = image_u8.astype(np.float32) / 255.0
    image = torch.from_numpy(image[None].transpose(0, 3, 1, 2))
    mask = mask_u8.astype(np.float32) / 255.0
    mask = mask[None, None]
    mask[mask < 0.5] = 0
    mask[mask >= 0.5] = 1
    mask = torch.from_numpy(mask)
    masked_image = (1 - mask) * image
    batch = {"image": image, "mask": mask, "masked_image": masked_image}
    return {k: v * 2.0 - 1.0 for k, v in batch.items()}


def mask_channel(batch_mask, size):
    """cc = F.interpolate(batch["mask"], size=c.shape[-2:]) (default mode: nearest)."""
    return F.interpolate(batch_mask, size=tuple(size))


def composite(batch, x_dec):
    """The script's output image: uint8 [h, w, 3] of (1 - mask) * image + mask * predicted, times 255, truncated."""
    image = torch.clamp((batch["image"] + 1.0) / 2.0, min=0.0, max=1.0)
    mask = torch.clamp((batch["mask"] + 1.0) / 2.0, min=0.0, max=1.0)
    predicted_image = torch.clamp((x_dec + 1.0) / 2.0, min=0.0, max=1.0)
    inpainted = (1 - mask) * image + mask * predicted_image
    inpainted = inpainted.cpu().numpy().transpose(0, 2, 3, 1)[0] * 255
    return inpainted.astype(np.uint8)
