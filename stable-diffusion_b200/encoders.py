"""H100-native cond stages that are not text encoders.

ClassEmbedder, the cond stage of the class-conditional ImageNet LDM: drop-in for
`ldm.modules.encoders.modules.ClassEmbedder` (constructor `(embed_dim, n_classes=1000, key='class')`,
`forward(batch, key=None)` = `nn.Embedding(n_classes, embed_dim)(batch[key][:, None])`, state-dict key
`embedding.weight`).

The context it produces has ONE token per sample; UNetModel.context_kv turns such a context into one residual vector
per SpatialTransformer. The gather is sdb_embed_tokens with one token position and a zero position row. That kernel
clamps ids, so labels are validated on the host first: out-of-range labels raise IndexError, as nn.Embedding does.

SpatialRescaler, the cond stage of the semantic-synthesis LDMs: drop-in for
`ldm.modules.encoders.modules.SpatialRescaler` (see the class).
"""
from __future__ import annotations

import torch

from . import ops
from .util import PackedStage


class ClassEmbedder(PackedStage):
    def __init__(self, embed_dim, n_classes=1000, key="class"):
        super().__init__()
        self.key = key
        self.embed_dim, self.n_classes = int(embed_dim), int(n_classes)
        self.shapes = {"embedding.weight": (self.n_classes, self.embed_dim)}

    @torch.no_grad()
    def pack_weights(self, device):
        table = self._host_sd["embedding.weight"].detach().to(device=device, dtype=torch.float32).contiguous()
        self.W = {"device": device, "table": table,
                  "pos": torch.zeros((1, self.embed_dim), dtype=torch.float32, device=device)}

    @torch.no_grad()
    def forward(self, batch, key=None):
        """fp32 [B, 1, embed_dim]: the table rows of the labels batch[key] (shape [B])."""
        assert self.W is not None, "weights not loaded (load_state_dict / load_weights, then .cuda())"
        labels = batch[self.key if key is None else key]
        labels = torch.as_tensor(labels)
        if labels.dtype.is_floating_point or labels.dtype == torch.bool or labels.dim() != 1:
            raise TypeError(f"ClassEmbedder: class labels must be a 1-D integer tensor (got {labels.dtype}, "
                            f"shape {tuple(labels.shape)})")
        host = labels.detach().to("cpu", torch.int64)
        if host.numel() and (int(host.min()) < 0 or int(host.max()) >= self.n_classes):
            raise IndexError(f"ClassEmbedder: class labels must lie in [0, {self.n_classes}) "
                             f"(got {host.min().item()} .. {host.max().item()})")
        ids = host.to(self.W["device"]).view(-1, 1).contiguous()
        out = ops.embed_tokens(ids, self.W["table"], self.W["pos"])
        return out.view(-1, 1, self.embed_dim)


class SpatialRescaler(PackedStage):
    """Drop-in for `ldm.modules.encoders.modules.SpatialRescaler` (modules.py:106-134): n_stages bilinear x0.5
    interpolations, then the optional `channel_mapper` 1x1 conv in_channels -> out_channels (state-dict keys
    `channel_mapper.weight` [out, in, 1, 1] and, with bias, `channel_mapper.bias`). Only the configuration every
    reference config uses is served: method 'bilinear', multiplier 0.5, n_stages <= 3; others raise
    NotImplementedError.

    forward / encode take either
      * a float NCHW map [B, in_channels, H, W] (the reference's input: one-hot or soft maps) -> sdb_spatial_rescale, or
      * integer label ids [B, H, W] -> sdb_seg_labels_rescale: the same result as on their one-hot
        (np.eye(in_channels)[ids], ddpm.py:329-335), which is never materialised. Needs the channel mapper and
        in_channels <= 256. Ids are checked on the host: negative or >= in_channels raises IndexError, as the one-hot
        would.
    Output fp32 NCHW [B, out_channels (or C), H >> n_stages, W >> n_stages]."""

    MAX_STAGES = 3

    def __init__(self, n_stages=1, method="bilinear", multiplier=0.5, in_channels=3, out_channels=None, bias=False):
        super().__init__()
        assert n_stages >= 0
        if method != "bilinear" or float(multiplier) != 0.5:
            raise NotImplementedError(f"SpatialRescaler: method {method!r} with multiplier {multiplier}: only "
                                      "'bilinear' with multiplier 0.5 is supported")
        if n_stages > self.MAX_STAGES:
            raise NotImplementedError(f"SpatialRescaler: n_stages {n_stages} > {self.MAX_STAGES}")
        self.n_stages, self.method, self.multiplier = int(n_stages), method, float(multiplier)
        self.in_channels = int(in_channels)
        self.remap_output = out_channels is not None
        self.out_channels = int(out_channels) if self.remap_output else None
        self.shapes = {}
        if self.remap_output:
            self.shapes["channel_mapper.weight"] = (self.out_channels, self.in_channels, 1, 1)
            if bias:
                self.shapes["channel_mapper.bias"] = (self.out_channels,)
        if not self.shapes:   # nothing to load: .cuda() packs right away
            self._host_sd = {}

    @torch.no_grad()
    def pack_weights(self, device):
        W = {"device": device, "weight": None, "bias": None}
        if self.remap_output:
            W["weight"] = self._host_sd["channel_mapper.weight"].detach().to(device=device, dtype=torch.float32).view(
                self.out_channels, self.in_channels).contiguous()
            if "channel_mapper.bias" in self._host_sd:
                W["bias"] = self._host_sd["channel_mapper.bias"].detach().to(device=device,
                                                                             dtype=torch.float32).contiguous()
        self.W = W

    def check_labels(self, labels):
        """Integer label ids [B, H, W] (any device) -> uint8 ids on the host; IndexError for ids outside
        [0, in_channels), before any kernel sees them."""
        labels = torch.as_tensor(labels)
        if labels.dtype.is_floating_point or labels.dtype == torch.bool or labels.dim() != 3:
            raise TypeError(f"SpatialRescaler: label maps are integer [B, H, W] (got {labels.dtype}, "
                            f"shape {tuple(labels.shape)})")
        host = labels.detach().to("cpu")
        if host.numel():
            lo, hi = int(host.min()), int(host.max())
            if lo < 0 or hi >= self.in_channels:
                raise IndexError(f"SpatialRescaler: label ids must lie in [0, {self.in_channels}) "
                                 f"(got {lo} .. {hi})")
        return host.to(torch.uint8)

    @torch.no_grad()
    def forward(self, x):
        assert self.W is not None, "weights not loaded (load_state_dict / load_weights, then .cuda())"
        dev = self.W["device"]
        x = torch.as_tensor(x)
        if not x.dtype.is_floating_point:
            if not self.remap_output:
                raise NotImplementedError("SpatialRescaler: label-map input needs the channel mapper (out_channels)")
            if self.in_channels > 256:
                raise NotImplementedError(f"SpatialRescaler: label-map input with {self.in_channels} > 256 classes")
            ids = self.check_labels(x).to(dev).contiguous()
            return ops.seg_labels_rescale(ids, self.in_channels, self.n_stages, self.W["weight"], self.W["bias"])
        if x.dim() != 4 or (self.remap_output and x.shape[1] != self.in_channels):
            raise ValueError(f"SpatialRescaler: expected a float map [B, {self.in_channels}, H, W], "
                             f"got {tuple(x.shape)}")
        x = x.to(device=dev, dtype=torch.float32).contiguous()
        return ops.spatial_rescale(x, self.n_stages, self.W["weight"], self.W["bias"])

    def encode(self, x):
        return self(x)
