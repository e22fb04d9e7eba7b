"""H100-native CLIP image embedder: drop-in for `ldm.modules.encoders.modules.FrozenClipImageEmbedder`
(modules.py:197-229), the retriever of the retrieval-augmented model whose embeddings make up its databases
(scripts/knn2img.py Searcher.load_retriever). `forward(x)` = CLIP ViT-L/14's `encode_image(preprocess(x))`:
fp32 [B, 3, H, W] in [-1, 1] -> fp32 [B, 768], unnormalised.

preprocess is kornia.geometry.resize(x, (224, 224), 'bicubic', align_corners=True, antialias=False) (the whole image,
aspect ratio not kept), (x + 1) / 2, then CLIP's mean / std. With antialias=False kornia's resize is
F.interpolate(mode='bicubic', align_corners=True); sdb_clip_resize_patches restates torch's CUDA bicubic and writes
the normalised values straight into the fp16 patch rows of the patch-embedding GEMM, for a ragged batch (every image
at its own size) in one launch. The tower then runs batched: patch GEMM -> sdb_vit_embed (class token + positions for
all B images) -> pre-LN -> the encoder layers of clip.encoder_layers (quick-GELU) -> class-token gather -> post-LN ->
visual projection. `encode_uint8(images)` takes uint8 HWC images (x / 127.5 - 1 is applied in the kernel), the input
of scripts/build_rdm_database.py.

Weights are read in the transformers `CLIPModel` layout of the checkpoint knn2img.py reads (`vision_model.*`,
`visual_projection.weight`); the text tower's keys are ignored. There is no CPU fallback.
"""
from __future__ import annotations

import torch

from . import ops
from .arch import CLIP_IMAGE_MEAN, CLIP_IMAGE_STD, CLIP_VISION_PROJ, clip_vision_proj_param_shapes
from .clip import encoder_layers, pack_clip_layers
from .ops import ACT_QUICK_GELU
from .util import PackedStage


class FrozenClipImageEmbedder(PackedStage):
    drop_prefixes = ("vision_model.embeddings.position_ids", "text_model.", "text_projection.", "logit_scale")

    def __init__(self, model, jit=False, device="cuda", antialias=False, config=None):
        """model: the CLIP name (only "ViT-L/14", the retriever knn2img.py builds). jit is accepted for the reference's
        signature and has no effect (OpenAI's TorchScript file is not read). antialias=True is not implemented."""
        super().__init__()
        if model != "ViT-L/14":
            raise NotImplementedError(f"FrozenClipImageEmbedder: model {model!r} (only 'ViT-L/14' is implemented)")
        if antialias:
            raise NotImplementedError("FrozenClipImageEmbedder: antialias=True is not implemented (the reference "
                                      "default, antialias=False, is)")
        self.model_name, self.jit, self.device, self.antialias = model, jit, device, antialias
        self.cfg = dict(config or CLIP_VISION_PROJ)
        self.shapes = clip_vision_proj_param_shapes(self.cfg)
        self.mean, self.std = tuple(CLIP_IMAGE_MEAN), tuple(CLIP_IMAGE_STD)

    @torch.no_grad()
    def pack_weights(self, device):
        sd = {k: v.detach().to(device=device, dtype=torch.float32) for k, v in self._host_sd.items()}
        f32 = lambda k: sd[k].contiguous()
        cfg = self.cfg
        h, P = cfg["hidden_size"], cfg["patch_size"]
        kpad = (3 * P * P + 63) // 64 * 64
        wp = torch.zeros((h, kpad), dtype=torch.float16, device=device)
        wp[:, : 3 * P * P] = sd["vision_model.embeddings.patch_embedding.weight"].reshape(h, -1).half()
        pos = f32("vision_model.embeddings.position_embedding.weight")
        self.W = {"device": device, "w_patch": wp, "kpad": kpad, "pos_patches": pos[1:].contiguous(),
                  "cls_pos": (sd["vision_model.embeddings.class_embedding"] + pos[0]).contiguous(),
                  "ln_pre": (f32("vision_model.pre_layrnorm.weight"), f32("vision_model.pre_layrnorm.bias")),
                  "ln_post": (f32("vision_model.post_layernorm.weight"), f32("vision_model.post_layernorm.bias")),
                  "layers": pack_clip_layers(sd, "vision_model.encoder.layers", cfg["num_hidden_layers"]),
                  "w_proj": sd["visual_projection.weight"].half().contiguous()}

    def preprocess_patches(self, src, table, want_resized=False):
        """The packed images src (fp32 NCHW or uint8 HWC each) with table int64 cuda [B, 3] = (H, W, element offset)
        -> (fp16 patch rows, fp32 [B, 3, S, S] resized values before (x + 1) / 2 or None)."""
        return ops.clip_resize_patches(src, table, self.cfg["image_size"], self.cfg["patch_size"], self.W["kpad"],
                                       self.mean, self.std, want_resized=want_resized)

    @torch.no_grad()
    def embed_patches(self, patches, B):
        """fp16 patch rows [B * (S/P)^2, kpad] -> fp32 [B, projection_dim]."""
        W, cfg = self.W, self.cfg
        h, heads, eps = cfg["hidden_size"], cfg["num_attention_heads"], cfg["layer_norm_eps"]
        d = h // heads
        assert d == 64, "CLIP vision heads are 64 wide"
        n = (cfg["image_size"] // cfg["patch_size"]) ** 2 + 1
        _, pe = ops.gemm(patches, W["w_patch"], want_f32=True)                      # [B * (n - 1), h]
        x = ops.vit_embed(pe, W["cls_pos"], W["pos_patches"], B)                    # [B * n, h]
        _, x = ops.layernorm(x, *W["ln_pre"], eps=eps, want_f32=True)
        x = encoder_layers(x, W["layers"], B, heads=heads, d=d, eps=eps, act=ACT_QUICK_GELU)
        _, pooled = ops.layernorm(ops.rows_gather(x, B, n), *W["ln_post"], eps=eps, want_f32=True)
        return ops.linear_small(pooled, W["w_proj"])

    @torch.no_grad()
    def encode_packed(self, flat_u8, hw):
        """flat_u8: uint8 cuda, the HWC images back to back; hw: their (H, W) -> fp32 [len(hw), projection_dim]."""
        # pinned, so the upload does not wait for the work already queued on the stream
        table = _table(hw, 3, flat_u8.numel()).pin_memory().to(flat_u8.device, non_blocking=True)
        patches, _ = self.preprocess_patches(flat_u8, table)
        return self.embed_patches(patches, len(hw))

    @torch.no_grad()
    def encode_uint8(self, images):
        """images: list of uint8 [H_i, W_i, 3] tensors (host or device, any sizes) -> fp32 [B, projection_dim]."""
        assert self.W is not None, "load weights first"
        assert images and all(t.dtype == torch.uint8 and t.dim() == 3 and t.shape[2] == 3 for t in images), \
            "encode_uint8 takes a non-empty list of uint8 [H, W, 3] tensors"
        dev = self.W["device"]
        hw = [(int(t.shape[0]), int(t.shape[1])) for t in images]
        if all(t.is_cuda for t in images):
            flat = torch.cat([t.reshape(-1) for t in images])
        else:
            host = torch.empty(sum(h * w * 3 for h, w in hw), dtype=torch.uint8, pin_memory=True)
            off = 0
            for t in images:
                host[off:off + t.numel()].copy_(t.reshape(-1))
                off += t.numel()
            flat = host.to(dev, non_blocking=True)
        return self.encode_packed(flat, hw)

    @torch.no_grad()
    def forward(self, x):
        """x: fp32 cuda [B, 3, H, W] in [-1, 1] -> fp32 [B, projection_dim] (CLIP's encode_image, unnormalised)."""
        assert self.W is not None and x.is_cuda, "sdb200.FrozenClipImageEmbedder runs on CUDA only (no CPU fallback)"
        assert x.dim() == 4 and x.shape[1] == 3, f"need [B, 3, H, W], got {tuple(x.shape)}"
        x = x.float().contiguous()
        B, _, H, W = x.shape
        table = _table([(H, W)] * B, 3, x.numel()).pin_memory().to(x.device, non_blocking=True)
        patches, _ = self.preprocess_patches(x, table)
        return self.embed_patches(patches, B)

    def encode(self, x):
        return self(x)


def _table(hw, channels, total):
    """int64 [B, 3] = (H, W, element offset) of images of (H, W) x channels elements packed back to back."""
    rows, off = [], 0
    for h, w in hw:
        assert h > 0 and w > 0, f"empty image {h} x {w}"
        rows.append((h, w, off))
        off += h * w * channels
    assert off == total, f"packed buffer holds {total} elements, the images {off}"
    return torch.tensor(rows, dtype=torch.int64)
