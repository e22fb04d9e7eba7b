"""ORACLE: CPU fp32 functional restatement of the semantic-synthesis cond stage (SpatialRescaler,
ldm/modules/encoders/modules.py:106-134) as the reference's data pipeline feeds it: label ids -> one-hot
(np.eye(n)[labels], ddpm.py:329-335 get_input's NCHW float) -> n_stages x F.interpolate(scale_factor=0.5, bilinear)
-> channel_mapper 1x1 conv. Also the seeded inputs the goldens and tests share."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def one_hot(labels, n_classes):
    """int [B, H, W] -> fp32 NCHW [B, n_classes, H, W] (get_input: rearrange b h w c -> b c h w, contiguous, float)."""
    return F.one_hot(torch.as_tensor(labels).long(), n_classes).permute(0, 3, 1, 2).contiguous().float()


def spatial_rescale(x, n_stages, weight=None, bias=None):
    """SpatialRescaler.forward on fp32 NCHW x; weight [cout, cin, 1, 1] (or None: no channel mapper)."""
    for _ in range(n_stages):
        x = F.interpolate(x, scale_factor=0.5, mode="bilinear")
    if weight is not None:
        x = F.conv2d(x, weight, bias)
    return x


def cond_from_labels(labels, sd, cfg):
    """The cond stage on label ids: one-hot, then spatial_rescale with the state dict's channel mapper."""
    return spatial_rescale(one_hot(labels, cfg["in_channels"]), cfg["n_stages"], sd.get("channel_mapper.weight"),
                           sd.get("channel_mapper.bias"))


def voronoi_labels(h, w, n_classes, seed, n_points=24):
    """uint8 [h, w]: a Voronoi partition of n_points seeded sites, each labelled with a random class id - regions
    with straight borders, like a segmentation map."""
    g = np.random.default_rng(seed)
    ys, xs = g.uniform(0, h, n_points), g.uniform(0, w, n_points)
    ids = g.integers(0, n_classes, n_points)
    yy, xx = np.mgrid[0:h, 0:w]
    d = (yy[..., None] - ys) ** 2 + (xx[..., None] - xs) ** 2
    return ids[d.argmin(-1)].astype(np.uint8)


def all_ids_labels(h, w, n_classes, seed):
    """uint8 [h, w] holding every id in [0, n_classes) (h * w >= n_classes), in seeded random places."""
    assert h * w >= n_classes
    g = np.random.default_rng(seed)
    return (g.permutation(h * w) % n_classes).reshape(h, w).astype(np.uint8)


def soft_map(shape, seed):
    """fp32 NCHW: softmax over the channels of seeded N(0, 2^2) logits."""
    return torch.softmax(2.0 * torch.randn(shape, generator=torch.Generator().manual_seed(seed)), dim=1)
