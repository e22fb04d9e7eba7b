"""ORACLE tooling: generate tests/golden/clip_image.pt for FrozenClipImageEmbedder (the retriever of the
retrieval-augmented model, ldm/modules/encoders/modules.py:197-229).

Run in the build container:  python oracle/make_golden_clip_image.py

The reference's encode_image is CLIP ViT-L/14's vision tower + visual projection, third-party code: it is pinned
against the installed transformers CLIPVisionModelWithProjection (`image_embeds`) on seeded random weights
(stable-diffusion_b200/arch.random_state_dict), tiny and full size. Its preprocess is kornia.geometry.resize(bicubic,
align_corners=True, antialias=False), restated as F.interpolate(mode='bicubic', align_corners=True) (kornia is not
installed; DESIGN.md states that link), then (x + 1) / 2 and CLIP's mean / std.

Inputs are seeded uint8 images stored in the file, read as x = u8 / 127.5 - 1 (IEEE fp32 division on the host) at a
size other than the tower's, so the resize runs. Contents per config: the key and shape list of the vision tower and
projection (CLIPVisionModelWithProjection.state_dict(), position_ids buffers excluded), the uint8 inputs, and the
image_embeds (the full-size ones stored as fp16 to keep the file small: that rounding is below 3e-4 rel-L2).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SEED = 15
CASES = (("tiny", arch.TINY_CLIP_VISION_PROJ, (3, 70, 90)), ("vitl14", arch.CLIP_VISION_PROJ, (2, 200, 256)))


def to_pixels(u8):
    """uint8 [B, 3, H, W] -> x in [-1, 1] (fp32 host division, as the kernel's uint8 path)."""
    return torch.from_numpy(u8.astype(np.float32) / np.float32(127.5) - np.float32(1.0))


def preprocess(x, size):
    """FrozenClipImageEmbedder.preprocess with kornia's antialias=False resize written as F.interpolate."""
    x = F.interpolate(x, size=(size, size), mode="bicubic", align_corners=True)
    x = (x + 1.0) / 2.0
    mean = torch.tensor(arch.CLIP_IMAGE_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(arch.CLIP_IMAGE_STD).view(1, 3, 1, 1)
    return (x - mean) / std


def main():
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    out = {}
    for tag, cfg, (B, H, W) in CASES:
        hf_cfg = CLIPVisionConfig(hidden_size=cfg["hidden_size"], intermediate_size=cfg["intermediate_size"],
                                  num_hidden_layers=cfg["num_hidden_layers"], num_attention_heads=cfg["num_attention_heads"],
                                  image_size=cfg["image_size"], patch_size=cfg["patch_size"],
                                  projection_dim=cfg["projection_dim"], hidden_act="quick_gelu",
                                  layer_norm_eps=cfg["layer_norm_eps"])
        model = CLIPVisionModelWithProjection(hf_cfg).eval()
        keys = [(k, tuple(v.shape)) for k, v in model.state_dict().items() if "position_ids" not in k]
        sd = arch.random_state_dict(arch.clip_vision_proj_param_shapes(cfg), SEED)
        missing, unexpected = model.load_state_dict(sd, strict=False)
        assert not unexpected and all("position_ids" in m for m in missing), (missing, unexpected)
        rng = np.random.default_rng(700 + len(tag))
        # smooth structure plus noise, so the bicubic taps see both gradients and edges
        yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
        base = 127.5 + 100 * np.sin(6 * xx + 4 * yy)[None, None] * rng.uniform(0.3, 1.0, (B, 3, 1, 1))
        u8 = np.clip(base + rng.normal(0, 25, (B, 3, H, W)), 0, 255).astype(np.uint8)
        with torch.no_grad():
            emb = model(pixel_values=preprocess(to_pixels(u8), cfg["image_size"])).image_embeds
        full = tag != "tiny"
        print(f"{tag}: {len(keys)} keys, embeds {tuple(emb.shape)} std {float(emb.std()):.3f}"
              + (f", fp16 storage rel-L2 {float((emb.half().float() - emb).norm() / emb.norm()):.1e}" if full else ""))
        out[tag] = dict(keys=keys, images_u8=torch.from_numpy(u8), image_embeds=emb.half() if full else emb, seed=SEED)
    path = os.path.join(OUT, "clip_image.pt")
    torch.save(out, path)
    print(f"wrote {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
