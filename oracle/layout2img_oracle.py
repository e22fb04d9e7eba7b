"""ORACLE — test infrastructure only. The UNet of the layout-to-image LDM (models/ldm/layout2img-openimages256/config.yaml)
as plain functional PyTorch on state dicts: the spatial-transformer UNet with heads of `num_head_channels` whose
SpatialTransformers hold `transformer_depth` BasicTransformerBlocks (attention.py:239-241), run in order between proj_in
and proj_out (attention.py:250-261). The blocks, ResBlocks and layout walk are ldm_oracle's; only the number of blocks
differs from cin_f8_oracle's UNet, and with one block the result is the same to the bit.
Pinned against the unmodified reference by oracle/make_golden_layout2img.py (tests/golden/layout2img.pt)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ldm_oracle import _conv, _gn, _unet_layout, basic_transformer_block, resblock, timestep_embedding


def spatial_transformer(sd, pre, x, context, heads):
    """SpatialTransformer.forward (GroupNorm eps 1e-6): every transformer_blocks.{i} of the state dict, in order."""
    b, c, h, w = x.shape
    x_in = x
    x = _gn(x, sd, pre + ".norm", 1e-6)
    x = _conv(x, sd, pre + ".proj_in", padding=0)
    x = x.permute(0, 2, 3, 1).reshape(b, h * w, c)
    i = 0
    while f"{pre}.transformer_blocks.{i}.norm1.weight" in sd:
        x = basic_transformer_block(sd, f"{pre}.transformer_blocks.{i}", x, context, heads)
        i += 1
    x = x.reshape(b, h, w, c).permute(0, 3, 1, 2)
    x = _conv(x, sd, pre + ".proj_out", padding=0)
    return x + x_in


def _run_block(sd, pre, h, emb, context, nhc):
    subs = sorted({int(k[len(pre) + 1:].split(".")[0]) for k in sd if k.startswith(pre + ".")})
    for s in subs:
        p = f"{pre}.{s}"
        if p + ".in_layers.0.weight" in sd:
            h = resblock(sd, p, h, emb)
        elif p + ".transformer_blocks.0.norm1.weight" in sd:
            h = spatial_transformer(sd, p, h, context, h.shape[1] // nhc)
        elif p + ".op.weight" in sd:
            h = _conv(h, sd, p + ".op", stride=2, padding=1)
        elif p + ".conv.weight" in sd:
            h = _conv(F.interpolate(h, scale_factor=2, mode="nearest"), sd, p + ".conv")
        elif p + ".weight" in sd:
            h = _conv(h, sd, p)
        else:
            raise KeyError(p)
    return h


def unet_forward(sd, x, timesteps, context, num_head_channels=32):
    """UNetModel.forward (openaimodel.py:710-742), every SpatialTransformer with ch / num_head_channels heads and all of
    its blocks."""
    mc = sd["time_embed.0.weight"].shape[1]
    emb = F.linear(timestep_embedding(timesteps, mc), sd["time_embed.0.weight"], sd["time_embed.0.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.2.weight"], sd["time_embed.2.bias"])
    in_idx, out_idx = _unet_layout(sd)
    hs = []
    h = x.float()
    for i in in_idx:
        h = _run_block(sd, f"input_blocks.{i}", h, emb, context, num_head_channels)
        hs.append(h)
    h = _run_block(sd, "middle_block", h, emb, context, num_head_channels)
    for i in out_idx:
        h = _run_block(sd, f"output_blocks.{i}", torch.cat([h, hs.pop()], dim=1), emb, context, num_head_channels)
    return _conv(F.silu(_gn(h, sd, "out.0", 1e-5)), sd, "out.2")
