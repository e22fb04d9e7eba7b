"""ORACLE — test infrastructure only. The class-conditional ImageNet LDM-VQ-8 (models/ldm/cin256/config.yaml) as plain
functional PyTorch on state dicts:

- `unet_forward`: the spatial-transformer UNet with heads of `num_head_channels` (openaimodel.py:537-545: ch //
  num_head_channels heads of d = num_head_channels, legacy or not), cross-attention on the ClassEmbedder's context.
- `vae_encoder` / `vae_decoder`: Encoder / Decoder (model.py:368-568) with the AttnBlocks inside the levels at
  attn_resolutions, each after its ResnetBlock (model.py:446-449, 557-560); `vq_encode`, `vq_decode`,
  `decode_first_stage` as in vq_oracle on top of them.
Pinned against the unmodified reference by oracle/make_golden_cin_f8.py (tests/golden/cin_f8.pt)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ldm_oracle import (_conv, _gn, _levels, _unet_layout, _vae_attn, _vae_resnet, resblock, spatial_transformer,
                        timestep_embedding)
from vq_oracle import quantize


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
    """UNetModel.forward (openaimodel.py:710-742), every SpatialTransformer with ch / num_head_channels heads."""
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


def _level(sd, pre, h):
    """The ResnetBlocks of one level, each followed by its AttnBlock where the level has them."""
    for b in _levels(sd, pre + ".block"):
        h = _vae_resnet(sd, f"{pre}.block.{b}", h)
        if f"{pre}.attn.{b}.q.weight" in sd:
            h = _vae_attn(sd, f"{pre}.attn.{b}", h)
    return h


def vae_encoder(sd, x, pre="encoder"):
    """Encoder.forward, model.py:434-459."""
    h = _conv(x, sd, pre + ".conv_in")
    for lvl in _levels(sd, pre + ".down"):
        h = _level(sd, f"{pre}.down.{lvl}", h)
        if f"{pre}.down.{lvl}.downsample.conv.weight" in sd:
            h = _conv(F.pad(h, (0, 1, 0, 1), mode="constant", value=0), sd, f"{pre}.down.{lvl}.downsample.conv",
                      stride=2, padding=0)
    h = _vae_resnet(sd, pre + ".mid.block_1", h)
    h = _vae_attn(sd, pre + ".mid.attn_1", h)
    h = _vae_resnet(sd, pre + ".mid.block_2", h)
    return _conv(F.silu(_gn(h, sd, pre + ".norm_out", 1e-6)), sd, pre + ".conv_out")


def vae_decoder(sd, z, pre="decoder"):
    """Decoder.forward, model.py:535-568."""
    h = _conv(z, sd, pre + ".conv_in")
    h = _vae_resnet(sd, pre + ".mid.block_1", h)
    h = _vae_attn(sd, pre + ".mid.attn_1", h)
    h = _vae_resnet(sd, pre + ".mid.block_2", h)
    for lvl in reversed(_levels(sd, pre + ".up")):
        h = _level(sd, f"{pre}.up.{lvl}", h)
        if f"{pre}.up.{lvl}.upsample.conv.weight" in sd:
            h = _conv(F.interpolate(h, scale_factor=2.0, mode="nearest"), sd, f"{pre}.up.{lvl}.upsample.conv")
    return _conv(F.silu(_gn(h, sd, pre + ".norm_out", 1e-6)), sd, pre + ".conv_out")


def vq_encode(sd, x):
    """VQModelInterface.encode (autoencoder.py:269-272): encoder -> quant_conv."""
    return _conv(vae_encoder(sd, x), sd, "quant_conv", padding=0)


def vq_decode(sd, h, force_not_quantize=False):
    """VQModelInterface.decode (autoencoder.py:274-282)."""
    quant = h if force_not_quantize else quantize(h, sd["quantize.embedding.weight"])[0]
    return vae_decoder(sd, _conv(quant, sd, "post_quant_conv", padding=0))


def decode_first_stage(sd, z, scale_factor=1.0):
    """LatentDiffusion.decode_first_stage with a VQ first stage (ddpm.py:713, 760-761)."""
    return vq_decode(sd, 1. / scale_factor * z)
