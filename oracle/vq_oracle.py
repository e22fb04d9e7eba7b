"""ORACLE — test infrastructure only. Never imported by the product path (stable-diffusion_b200/).

CPU fp32 restatement of the VQ-f4 latent diffusion models of CompVis/stable-diffusion (configs/latent-diffusion/
celebahq-ldm-vq-4.yaml and its FFHQ / LSUN-bedrooms siblings):

- `VectorQuantizer2`: taming-transformers' quantizer (taming/modules/vqvae/quantize.py, legacy=True, no remap,
  sane_index_shape False), restated from its published form. taming is neither vendored by the reference nor installed
  here, so its parity with that package is not pinned; oracle/make_golden_vq.py installs this class as
  `ldm.models.autoencoder.VectorQuantizer`, and the reference's own VQModelInterface, Encoder / Decoder and
  LatentDiffusion run unmodified around it.
- `unet_forward`: the unconditional AttentionBlock UNet with heads of `num_head_channels` channels
  (openaimodel.py:542-556), plain ResBlocks.
- `vq_encode` / `vq_decode` / `decode_first_stage`: VQModelInterface (autoencoder.py:264-282) and
  LatentDiffusion.decode_first_stage (ddpm.py:705-763) on a state dict.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

import uncond_oracle as U
from ldm_oracle import _conv, _gn, timestep_embedding, vae_decoder, vae_encoder


class VectorQuantizer2(nn.Module):
    """taming VectorQuantizer2 at inference (legacy loss order, no remap): nearest codebook entry by
    ||z||^2 + ||e||^2 - 2 z.e, lowest index on ties (torch.argmin), straight-through output z + (z_q - z)."""

    def __init__(self, n_e, e_dim, beta, remap=None, unknown_index="random", sane_index_shape=False, legacy=True):
        super().__init__()
        assert remap is None and not sane_index_shape and legacy
        self.n_e, self.e_dim, self.beta, self.legacy = n_e, e_dim, beta, legacy
        self.remap, self.sane_index_shape = remap, sane_index_shape
        self.embedding = nn.Embedding(self.n_e, self.e_dim)
        self.embedding.weight.data.uniform_(-1.0 / self.n_e, 1.0 / self.n_e)

    def forward(self, z, temp=None, rescale_logits=False, return_logits=False):
        z = z.permute(0, 2, 3, 1).contiguous()
        z_flattened = z.view(-1, self.e_dim)
        d = torch.sum(z_flattened ** 2, dim=1, keepdim=True) + torch.sum(self.embedding.weight ** 2, dim=1) - \
            2 * torch.einsum("bd,dn->bn", z_flattened, self.embedding.weight.t())
        min_encoding_indices = torch.argmin(d, dim=1)
        z_q = self.embedding(min_encoding_indices).view(z.shape)
        loss = torch.mean((z_q.detach() - z) ** 2) + self.beta * torch.mean((z_q - z.detach()) ** 2)
        z_q = z + (z_q - z).detach()
        z_q = z_q.permute(0, 3, 1, 2).contiguous()
        return z_q, loss, (None, None, min_encoding_indices)

    def get_codebook_entry(self, indices, shape):
        z_q = self.embedding(indices)
        if shape is not None:
            z_q = z_q.view(shape).permute(0, 3, 1, 2).contiguous()
        return z_q


def quantize(z, embedding):
    """VectorQuantizer2.forward on a codebook tensor: (z_q NCHW, flat indices)."""
    q = VectorQuantizer2(embedding.shape[0], embedding.shape[1], 0.25)
    q.embedding.weight.data.copy_(embedding)
    with torch.no_grad():
        z_q, _, (_, _, idx) = q(z)
    return z_q, idx


def vq_encode(sd, x):
    """VQModelInterface.encode (autoencoder.py:269-272): encoder -> quant_conv."""
    return _conv(vae_encoder(sd, x), sd, "quant_conv", padding=0)


def vq_decode(sd, h, force_not_quantize=False):
    """VQModelInterface.decode (autoencoder.py:274-282)."""
    quant = h if force_not_quantize else quantize(h, sd["quantize.embedding.weight"])[0]
    return vae_decoder(sd, _conv(quant, sd, "post_quant_conv", padding=0))


def decode_first_stage(sd, z, scale_factor=1.0, force_not_quantize=False):
    """LatentDiffusion.decode_first_stage with a VQ first stage (ddpm.py:713, 760-761)."""
    return vq_decode(sd, 1. / scale_factor * z, force_not_quantize)


def unet_forward(sd, cfg, x, timesteps):
    """UNetModel.forward (openaimodel.py:710-742) of the unconditional AttentionBlock UNet with plain ResBlocks and
    AttentionBlocks of ch / num_head_channels heads (openaimodel.py:542-556: legacy passes num_head_channels on)."""
    mc, mult, nrb = cfg["model_channels"], cfg["channel_mult"], cfg["num_res_blocks"]
    nhc, attn_res = cfg["num_head_channels"], set(cfg["attention_resolutions"])
    attn = lambda pre, h: U.attention_block(sd, pre, h, h.shape[1] // nhc)
    emb = F.linear(timestep_embedding(timesteps, mc), sd["time_embed.0.weight"], sd["time_embed.0.bias"])
    emb = F.linear(F.silu(emb), sd["time_embed.2.weight"], sd["time_embed.2.bias"])
    h = _conv(x.float(), sd, "input_blocks.0.0")
    hs = [h]
    idx, ds = 1, 1
    for level in range(len(mult)):
        for _ in range(nrb):
            h = U.resblock(sd, f"input_blocks.{idx}.0", h, emb)
            if ds in attn_res:
                h = attn(f"input_blocks.{idx}.1", h)
            hs.append(h)
            idx += 1
        if level != len(mult) - 1:
            h = _conv(h, sd, f"input_blocks.{idx}.0.op", stride=2, padding=1)
            hs.append(h)
            idx += 1
            ds *= 2
    h = U.resblock(sd, "middle_block.0", h, emb)
    h = attn("middle_block.1", h)
    h = U.resblock(sd, "middle_block.2", h, emb)
    idx = 0
    for level in reversed(range(len(mult))):
        for i in range(nrb + 1):
            h = U.resblock(sd, f"output_blocks.{idx}.0", torch.cat([h, hs.pop()], dim=1), emb)
            sub = 1
            if ds in attn_res:
                h = attn(f"output_blocks.{idx}.1", h)
                sub = 2
            if level and i == nrb:
                h = _conv(F.interpolate(h, scale_factor=2, mode="nearest"), sd, f"output_blocks.{idx}.{sub}.conv")
                ds //= 2
            idx += 1
    return _conv(F.silu(_gn(h, sd, "out.0", 1e-5)), sd, "out.2")
