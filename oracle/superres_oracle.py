"""ORACLE: CPU fp32 restatement of the reference's super-resolution path (notebook_helpers.py get_cond, and the
split_input_params tiling of LatentDiffusion: meshgrid / delta_border / get_weighting / get_fold_unfold, ddpm.py:564-651;
the split apply_model, ddpm.py:891-992; the split decode_first_stage, ddpm.py:705-763). Written from the reference's
definitions with torch's Unfold / Fold; the model and the decoder are callables supplied by the caller."""
from __future__ import annotations

import numpy as np
import torch


def lr_image(image_u8):
    """get_cond("superresolution"): ToTensor (uint8 HWC -> fp32 CHW / 255), 2c - 1, batch of one, NCHW."""
    c = torch.from_numpy(np.ascontiguousarray(image_u8)).permute(2, 0, 1).float().div(255)
    return (2. * c - 1.)[None]


def meshgrid(h, w):
    y = torch.arange(0, h).view(h, 1, 1).expand(h, w, 1)
    x = torch.arange(0, w).view(1, w, 1).expand(h, w, 1)
    return torch.cat([y, x], dim=-1)


def delta_border(h, w):
    arr = meshgrid(h, w) / torch.tensor([h - 1, w - 1]).view(1, 1, 2)
    lo = arr.min(dim=-1, keepdim=True)[0]
    hi = (1 - arr).min(dim=-1, keepdim=True)[0]
    return torch.cat([lo, hi], dim=-1).min(dim=-1)[0]


def get_weighting(h, w, ly, lx, p):
    """[1, h*w, ly*lx]: the clipped border distance of every tile pixel, times the clipped tile-grid distance with
    tie_braker."""
    wt = torch.clip(delta_border(h, w), p["clip_min_weight"], p["clip_max_weight"]).view(1, h * w, 1).repeat(1, 1, ly * lx)
    if p["tie_braker"]:
        lw = torch.clip(delta_border(ly, lx), p["clip_min_tie_weight"], p["clip_max_tie_weight"])
        wt = wt * lw.view(1, 1, ly * lx)
    return wt


def get_fold_unfold(shape, ks, stride, p, uf=1):
    """(fold, unfold, normalization [1, 1, H, W], weighting [1, 1, kh, kw, L]); fold works at ks*uf / stride*uf. As in
    the reference, the uf > 1 fold kernel is ks[0]*uf on both sides."""
    _, _, h, w = shape
    ly = (h - ks[0]) // stride[0] + 1
    lx = (w - ks[1]) // stride[1] + 1
    unfold = torch.nn.Unfold(kernel_size=ks, dilation=1, padding=0, stride=stride)
    if uf == 1:
        fold = torch.nn.Fold(output_size=(h, w), kernel_size=ks, dilation=1, padding=0, stride=stride)
    else:
        fold = torch.nn.Fold(output_size=(h * uf, w * uf), kernel_size=(ks[0] * uf, ks[0] * uf), dilation=1, padding=0,
                             stride=(stride[0] * uf, stride[1] * uf))
    kh, kw = ks[0] * uf, ks[1] * uf
    weighting = get_weighting(kh, kw, ly, lx, p)
    normalization = fold(weighting).view(1, 1, h * uf, w * uf)
    return fold, unfold, normalization, weighting.view(1, 1, kh, kw, ly * lx)


def split_apply(model_fn, x, t, c, p):
    """The split apply_model with concat conditioning: model_fn(x_tile, t, c_tile) per tile, weighted, folded, divided
    by the normalization."""
    ks, stride = tuple(p["ks"]), tuple(p["stride"])
    fold, unfold, norm, weighting = get_fold_unfold(x.shape, ks, stride, p)
    z = unfold(x)
    z = z.view(z.shape[0], -1, ks[0], ks[1], z.shape[-1])
    cz = unfold(c)
    cz = cz.view(cz.shape[0], -1, ks[0], ks[1], cz.shape[-1])
    o = torch.stack([model_fn(z[..., i], t, cz[..., i]) for i in range(z.shape[-1])], dim=-1)
    o = o * weighting
    return fold(o.view(o.shape[0], -1, o.shape[-1])) / norm


def split_decode(decode_fn, z, p):
    """The split decode_first_stage (patch_distributed_vq): decode_fn per latent tile at uf = vqf, kernel and stride
    reduced to the latent first."""
    ks, stride, uf = tuple(p["ks"]), tuple(p["stride"]), p["vqf"]
    _, _, h, w = z.shape
    if ks[0] > h or ks[1] > w:
        ks = (min(ks[0], h), min(ks[1], w))
    if stride[0] > h or stride[1] > w:
        stride = (min(stride[0], h), min(stride[1], w))
    fold, unfold, norm, weighting = get_fold_unfold(z.shape, ks, stride, p, uf=uf)
    t = unfold(z)
    t = t.view(t.shape[0], -1, ks[0], ks[1], t.shape[-1])
    o = torch.stack([decode_fn(t[..., i]) for i in range(t.shape[-1])], dim=-1)
    o = o * weighting
    return fold(o.view(o.shape[0], -1, o.shape[-1])) / norm


def notebook_params(ks=128, stride=64, vqf=4, tie_braker=False):
    """run()'s split_input_params (notebook_helpers.py), with a free geometry."""
    return {"ks": (ks, ks), "stride": (stride, stride), "vqf": vqf, "patch_distributed_vq": True,
            "tie_braker": tie_braker, "clip_max_weight": 0.5, "clip_min_weight": 0.01, "clip_max_tie_weight": 0.5,
            "clip_min_tie_weight": 0.01}
