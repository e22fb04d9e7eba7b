"""H100-native ClassEmbedder, the cond stage of the class-conditional ImageNet LDM: drop-in for
`ldm.modules.encoders.modules.ClassEmbedder` (constructor `(embed_dim, n_classes=1000, key='class')`,
`forward(batch, key=None)` = `nn.Embedding(n_classes, embed_dim)(batch[key][:, None])`, state-dict key
`embedding.weight`).

The context it produces has ONE token per sample; UNetModel.context_kv turns such a context into one residual vector
per SpatialTransformer. The gather is sdb_embed_tokens with one token position and a zero position row. That kernel
clamps ids, so labels are validated on the host first: out-of-range labels raise IndexError, as nn.Embedding does.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops
from .util import adopt_state_dict


class ClassEmbedder(nn.Module):
    def __init__(self, embed_dim, n_classes=1000, key="class"):
        super().__init__()
        self.key = key
        self.embed_dim, self.n_classes = int(embed_dim), int(n_classes)
        self.shapes = {"embedding.weight": (self.n_classes, self.embed_dim)}
        self.W = None
        self._host_sd = None

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        sd = adopt_state_dict(self, state_dict, prefix, missing_keys, unexpected_keys, error_msgs)
        if sd is None:
            return
        self._host_sd = sd
        if self.W is not None:
            self.pack_weights(self.W["device"])

    def load_weights(self, sd, device):
        for k, shape in self.shapes.items():
            assert k in sd and tuple(sd[k].shape) == tuple(shape), k
        self._host_sd = {k: sd[k] for k in self.shapes}
        self.pack_weights(torch.device(device))
        return self

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        probe = fn(torch.empty(0))
        if probe.is_cuda and self._host_sd is not None and (self.W is None or self.W["device"] != probe.device):
            self.pack_weights(probe.device)
        return r

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
