"""H100-native VQ first stages: drop-ins for `ldm.models.autoencoder.VQModel` (autoencoder.py:14-122: the standalone
first stages of models/first_stage_models/vq-*) and its subclass `VQModelInterface` (autoencoder.py:264-282: the first
stage of the VQ-f4 / VQ-f8 LDMs), with taming's VectorQuantizer2 (legacy, no remap). State-dict keys unchanged
(`encoder.*`, `decoder.*`, `quantize.embedding.weight`, `quant_conv.*`, `post_quant_conv.*`); the loss is training-only
and its keys are ignored.

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

BETA = 0.25   # VQModel builds VectorQuantizer(n_embed, embed_dim, beta=0.25) (autoencoder.py:40)


class VQModel(ConvAutoencoder):
    def __init__(self, embed_dim, ddconfig, lossconfig=None, n_embed=None, ckpt_path=None, ignore_keys=(),
                 image_key="image", colorize_nlabels=None, monitor=None, batch_resize_range=None, scheduler_config=None,
                 lr_g_factor=1.0, remap=None, sane_index_shape=False, use_ema=False):
        # ckpt_path is accepted and ignored, as by AutoencoderKL: weights come through load_state_dict (an LDM checkpoint
        # carries them under first_stage_model.*; the FFHQ / LSUN-bedrooms configs even point ckpt_path at a .yaml)
        if remap is not None or sane_index_shape or use_ema:
            raise NotImplementedError(f"sdb200.{type(self).__name__}: remap, sane_index_shape and use_ema are not "
                                      "supported")
        assert n_embed is not None, "n_embed is required"
        assert not ddconfig["double_z"], "VQ first stages have double_z False"
        cfg = dict(embed_dim=embed_dim, n_embed=n_embed, ddconfig=dict(ddconfig))
        super().__init__(vq_param_shapes(cfg))
        self.cfg = cfg
        self.embed_dim, self.n_embed = embed_dim, n_embed
        self.image_key = image_key

    def _need_cuda(self, t):
        assert self.W is not None and t.is_cuda, f"sdb200.{type(self).__name__} runs on CUDA only (no CPU fallback)"

    @torch.no_grad()
    def pack_weights(self, device):
        super().pack_weights(device)
        e = self._host_sd["quantize.embedding.weight"].detach().to(device=device, dtype=torch.float32).contiguous()
        self.W["codebook"] = e
        self.W["code_sq"] = (e.double() ** 2).sum(1).float().contiguous()

    def _quantize_nhwc(self, zh, scale=1.0, want_indices=False):
        return ops.vq_quantize(zh, self.W["codebook"], self.W["code_sq"], scale=float(scale), want_indices=want_indices)

    def _prequant_nhwc(self, x):
        """encoder -> quant_conv: the unquantized latent, fp32 NHWC."""
        self._need_cuda(x)
        W = self.W
        return ops.pointwise_small(self._encoder(x), W["quant_w"], W["quant_b"])

    # ------------------------------------------------------------------ public API (VQModel, autoencoder.py:96-122)
    @torch.no_grad()
    def encode_to_prequant(self, x):
        """encoder -> quant_conv, the unquantized latent h (NCHW fp32)."""
        return ops.nhwc_to_nchw(self._prequant_nhwc(x))

    @torch.no_grad()
    def encode(self, x):
        """VQModel.encode: (quant, emb_loss, (None, None, indices)) — quantize(encode_to_prequant(x))."""
        zh = self._prequant_nhwc(x)
        zq, idx = self._quantize_nhwc(zh, want_indices=True)
        # VectorQuantizer2's legacy loss at inference: mean((e - z)^2) + beta * mean((e - z)^2), e the selected entries
        loss = (1.0 + BETA) * torch.mean((self.W["codebook"][idx].view_as(zh) - zh) ** 2)
        return ops.nhwc_to_nchw(zq), loss, (None, None, idx)

    @torch.no_grad()
    def quantize(self, h):
        """VectorQuantizer2.forward at inference: (z_q, loss, (perplexity, min_encodings, indices)) with the
        training-only loss and the unused perplexity / encodings None; indices are flat over b*h*w."""
        self._need_cuda(h)
        zh, _ = ops.nchw_to_nhwc(h.contiguous().float())
        zq, idx = self._quantize_nhwc(zh, want_indices=True)
        return ops.nhwc_to_nchw(zq), None, (None, None, idx)

    @torch.no_grad()
    def get_codebook_entry(self, indices, shape):
        """VectorQuantizer2.get_codebook_entry: the codebook rows of int64 `indices` [b*h*w], as NCHW fp32 for
        shape (b, h, w, e_dim). Indices outside [0, n_embed) raise IndexError."""
        b, h, w, e = shape
        if indices.dtype != torch.int64 or indices.numel() != b * h * w or e != self.embed_dim:
            raise ValueError(f"indices: int64 with b*h*w = {b * h * w} entries and e_dim {self.embed_dim} expected, got "
                             f"{indices.dtype} with {indices.numel()} entries and e_dim {e}")
        flat = indices.reshape(-1)
        if flat.numel() and not bool(((flat >= 0) & (flat < self.n_embed)).all()):
            raise IndexError(f"code indices must lie in [0, {self.n_embed})")
        self._need_cuda(indices)
        # an exact row copy of b*h*w x e_dim floats (the embedding lookup), before the decoder's kernels
        return ops.nhwc_to_nchw(self.W["codebook"][flat].view(b, h, w, e))

    @torch.no_grad()
    def decode(self, quant):
        """VQModel.decode: post_quant_conv then the decoder, no re-quantization (unlike VQModelInterface.decode).
        NCHW fp32 in / out."""
        self._need_cuda(quant)
        W = self.W
        zh, _ = ops.nchw_to_nhwc(quant.contiguous().float())
        return ops.nhwc_to_nchw(self._decoder(ops.pointwise_small(zh, W["pq_w"], W["pq_b"])))

    @torch.no_grad()
    def decode_code(self, code_b):
        """Decode int64 code indices of shape (b, h, w). The reference calls `self.quantize.embed_code`, which taming's
        VectorQuantizer2 does not have (it raises AttributeError); this does what the method means instead:
        get_codebook_entry(code_b, (b, h, w, e_dim)), then decode. Indices outside [0, n_embed) raise IndexError
        before anything is launched."""
        if not isinstance(code_b, torch.Tensor) or code_b.dim() != 3 or code_b.dtype != torch.int64:
            raise ValueError("decode_code: code_b must be an int64 tensor of shape (b, h, w)")
        b, h, w = code_b.shape
        return self.decode(self.get_codebook_entry(code_b.reshape(-1), (b, h, w, self.embed_dim)))

    def forward(self, input, return_pred_indices=False):
        quant, diff, (_, _, ind) = self.encode(input)
        dec = self.decode(quant)
        if return_pred_indices:
            return dec, diff, ind
        return dec, diff


class VQModelInterface(VQModel):
    """VQModelInterface (autoencoder.py:264-282): encode returns the unquantized latent, decode quantizes first."""

    @torch.no_grad()
    def encode(self, x):
        """VQModelInterface.encode: encoder -> quant_conv, the unquantized latent h (NCHW fp32)."""
        return self.encode_to_prequant(x)

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
        self._need_cuda(h)
        W = self.W
        zh, _ = ops.nchw_to_nhwc(h.contiguous().float())
        if force_not_quantize:
            return ops.pointwise_small(zh, W["pq_w"], W["pq_b"], alpha=float(scale))
        return ops.pointwise_small(self._quantize_nhwc(zh, scale), W["pq_w"], W["pq_b"])
