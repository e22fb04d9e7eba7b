"""ORACLE — test infrastructure only. The BERTEmbedder of the LAION-400M LDM (ldm/modules/encoders/modules.py:80-103,
ldm/modules/x_transformer.py TransformerWrapper + Encoder, return_embeddings=True) as plain functional PyTorch on a state
dict with the reference's keys (`transformer.*`): token + absolute position embedding, pre-LayerNorm residual pairs of
8-head (d = 64) unmasked self-attention and Linear -> exact GELU -> Linear, final LayerNorm. Pinned against the
unmodified reference by oracle/make_golden_laion.py (tests/golden/laion.pt)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

HEADS, DIM_HEAD, EPS = 8, 64, 1e-5


def bert_embed(sd, ids):
    """ids int64 [B, n] -> fp32 [B, n, dim]."""
    B, n = ids.shape
    x = sd["transformer.token_emb.weight"][ids] + sd["transformer.pos_emb.emb.weight"][:n][None]
    dim = x.shape[-1]
    j = 0
    while f"transformer.attn_layers.layers.{j}.0.weight" in sd:
        p = f"transformer.attn_layers.layers.{j}"
        y = F.layer_norm(x, (dim,), sd[p + ".0.weight"], sd[p + ".0.bias"], EPS)
        if j % 2 == 0:
            split = lambda t: t.view(B, n, HEADS, DIM_HEAD).transpose(1, 2)
            q, k, v = (split(y @ sd[f"{p}.1.{w}.weight"].t()) for w in ("to_q", "to_k", "to_v"))
            att = torch.softmax(q @ k.transpose(-1, -2) * DIM_HEAD ** -0.5, dim=-1)
            o = (att @ v).transpose(1, 2).reshape(B, n, HEADS * DIM_HEAD)
            x = x + o @ sd[p + ".1.to_out.weight"].t() + sd[p + ".1.to_out.bias"]
        else:
            h = F.gelu(y @ sd[p + ".1.net.0.0.weight"].t() + sd[p + ".1.net.0.0.bias"])
            x = x + h @ sd[p + ".1.net.2.weight"].t() + sd[p + ".1.net.2.bias"]
        j += 1
    return F.layer_norm(x, (dim,), sd["transformer.norm.weight"], sd["transformer.norm.bias"], EPS)
