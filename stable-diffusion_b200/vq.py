"""H100-native VQModelInterface (the first stage of the VQ-f4 / VQ-f8 LDMs): drop-in for
`ldm.models.autoencoder.VQModelInterface` (autoencoder.py:14-44, 264-282) with taming's VectorQuantizer2 (legacy,
no remap). State-dict keys unchanged (`encoder.*`, `decoder.*`, `quantize.embedding.weight`, `quant_conv.*`,
`post_quant_conv.*`); the loss is training-only and its keys are ignored.

The Encoder / Decoder are the AutoencoderKL ones (vae.ConvAutoencoder), including AttnBlocks inside the levels at
ddconfig.attn_resolutions (VQ-f8: one per ResnetBlock of the 32x32 level). The quantizer is one kernel (sdb_vq_quantize):
nearest codebook entry by sum(z^2) + sum(e^2) - 2 z.e with the lowest index winning ties, and the straight-through
value z + (e - z) in fp32, as the reference computes it. sum(e^2) is computed once per weight load.
"""
from __future__ import annotations

import torch

from . import ops
from .arch import vq_param_shapes
from .vae import ConvAutoencoder


class VQModelInterface(ConvAutoencoder):
    def __init__(self, embed_dim, ddconfig, lossconfig=None, n_embed=None, ckpt_path=None, ignore_keys=(),
                 image_key="image", colorize_nlabels=None, monitor=None, batch_resize_range=None, scheduler_config=None,
                 lr_g_factor=1.0, remap=None, sane_index_shape=False, use_ema=False):
        # ckpt_path is accepted and ignored, as by AutoencoderKL: the LDM checkpoint carries the first stage's weights
        # under first_stage_model.* (the FFHQ / LSUN-bedrooms configs even point it at a .yaml)
        if remap is not None or sane_index_shape or use_ema:
            raise NotImplementedError("sdb200.VQModelInterface: remap, sane_index_shape and use_ema are not supported")
        assert n_embed is not None, "n_embed is required"
        assert not ddconfig["double_z"], "VQ first stages have double_z False"
        cfg = dict(embed_dim=embed_dim, n_embed=n_embed, ddconfig=dict(ddconfig))
        super().__init__(vq_param_shapes(cfg))
        self.cfg = cfg
        self.embed_dim, self.n_embed = embed_dim, n_embed
        self.image_key = image_key

    @torch.no_grad()
    def pack_weights(self, device):
        super().pack_weights(device)
        e = self._host_sd["quantize.embedding.weight"].detach().to(device=device, dtype=torch.float32).contiguous()
        self.W["codebook"] = e
        self.W["code_sq"] = (e.double() ** 2).sum(1).float().contiguous()

    def _quantize_nhwc(self, zh, scale=1.0, want_indices=False):
        return ops.vq_quantize(zh, self.W["codebook"], self.W["code_sq"], scale=float(scale), want_indices=want_indices)

    # ------------------------------------------------------------------ public API
    @torch.no_grad()
    def encode(self, x):
        """VQModelInterface.encode: encoder -> quant_conv, the unquantized latent h (NCHW fp32)."""
        assert self.W is not None and x.is_cuda, "sdb200.VQModelInterface runs on CUDA only (no CPU fallback)"
        W = self.W
        return ops.nhwc_to_nchw(ops.pointwise_small(self._encoder(x), W["quant_w"], W["quant_b"]))

    @torch.no_grad()
    def quantize(self, h):
        """VectorQuantizer2.forward at inference: (z_q, loss, (perplexity, min_encodings, indices)) with the
        training-only loss and the unused perplexity / encodings None; indices are flat over b*h*w."""
        assert self.W is not None and h.is_cuda, "sdb200.VQModelInterface runs on CUDA only (no CPU fallback)"
        zh, _ = ops.nchw_to_nhwc(h.contiguous().float())
        zq, idx = self._quantize_nhwc(zh, want_indices=True)
        return ops.nhwc_to_nchw(zq), None, (None, None, idx)

    @torch.no_grad()
    def decode(self, h, force_not_quantize=False, scale=1.0, nhwc=False):
        """VQModelInterface.decode on h*scale (scale: decode_first_stage's 1 / scale_factor): quantize unless
        force_not_quantize, post_quant_conv, decoder. NCHW fp32 in / out (nhwc=True keeps the NHWC output)."""
        out = self._decoder(self.post_quant(h, force_not_quantize, scale))
        return out if nhwc else ops.nhwc_to_nchw(out)

    @torch.no_grad()
    def post_quant(self, h, force_not_quantize=False, scale=1.0):
        """The per-pixel head of decode: quantize h*scale (unless force_not_quantize), then post_quant_conv; NCHW fp32
        in, the decoder's NHWC fp32 input out."""
        assert self.W is not None and h.is_cuda, "sdb200.VQModelInterface runs on CUDA only (no CPU fallback)"
        W = self.W
        zh, _ = ops.nchw_to_nhwc(h.contiguous().float())
        if force_not_quantize:
            return ops.pointwise_small(zh, W["pq_w"], W["pq_b"], alpha=float(scale))
        return ops.pointwise_small(self._quantize_nhwc(zh, scale), W["pq_w"], W["pq_b"])
