"""H100-native BERTEmbedder, the cond stage of the LAION-400M text-to-image LDM: drop-in for
`ldm.modules.encoders.modules.BERTEmbedder` (modules.py:80-103; configs/latent-diffusion/txt2img-1p4B-eval.yaml:
n_embed 1280, n_layer 32).

The reference wraps `x_transformer.TransformerWrapper(num_tokens, max_seq_len, Encoder(dim, depth))` with
`return_embeddings=True`: token + absolute position embedding, `depth` pairs of pre-LayerNorm residual layers
('a': 8 heads of 64, no bias on q/k/v, no mask; 'f': Linear -> exact GELU -> Linear), a final LayerNorm. It runs here
on the kernels of clip.py: fp32 LayerNorm -> fp16 operand, wgmma GEMMs with fused bias / exact-GELU / fp32-residual
epilogues, the fused attention kernel (d = 64, not causal: [PAD] positions are attended to, as in the reference).
State-dict keys are the reference's (`transformer.*`); `transformer.to_logits.*` is never used by the embedding and
is accepted and dropped.

Tokenisation (use_tokenizer=True) is the uncased WordPiece of tokenizer.BertWordPieceTokenizer, from a directory with
the bert-base-uncased vocab.txt (`vocab_dir`) or from the locally cached Hugging Face files; without a vocabulary,
string input raises and token ids have to be passed.
"""
from __future__ import annotations

import os

import torch

from . import ops
from .arch import bert_param_shapes
from .clip import encoder_layers
from .ops import ACT_GELU
from .util import PackedStage

HEADS, DIM_HEAD = 8, 64          # x_transformer.py DEFAULT_DIM_HEAD and AttentionLayers' heads: fixed by the config
LN_EPS = 1e-5


class BERTEmbedder(PackedStage):
    # to_logits is part of the reference's state dict but not of the embedding: not required, dropped when present
    drop_prefixes = ("transformer.to_logits.",)

    def __init__(self, n_embed, n_layer, vocab_size=30522, max_seq_len=77, device="cuda", use_tokenizer=True,
                 embedding_dropout=0.0, vocab_dir=None):
        super().__init__()
        self.cfg = dict(n_embed=int(n_embed), n_layer=int(n_layer), vocab_size=int(vocab_size),
                        max_seq_len=int(max_seq_len))
        self.device = device
        self.use_tknz_fn = bool(use_tokenizer)
        self.embedding_dropout = float(embedding_dropout)   # dropout is inactive at inference (eval mode)
        self.vocab_dir = vocab_dir
        self.tokenizer = None
        self.shapes = {k: v for k, v in bert_param_shapes(self.cfg).items() if not k.startswith(self.drop_prefixes)}

    def freeze(self):
        return self

    @torch.no_grad()
    def pack_weights(self, device):
        sd = self._host_sd
        f32 = lambda k: sd[k].detach().to(device=device, dtype=torch.float32).contiguous()
        f16 = lambda k: sd[k].detach().to(device=device, dtype=torch.float16).contiguous()
        p = "transformer.attn_layers.layers"
        W = {"device": device, "tok": f32("transformer.token_emb.weight"), "pos": f32("transformer.pos_emb.emb.weight"),
             "layers": []}
        for i in range(self.cfg["n_layer"]):
            a, f = f"{p}.{2 * i}", f"{p}.{2 * i + 1}"
            W["layers"].append({
                "ln1": (f32(f"{a}.0.weight"), f32(f"{a}.0.bias")),
                "w_qk": torch.cat([f16(f"{a}.1.to_q.weight"), f16(f"{a}.1.to_k.weight")], 0).contiguous(),
                "w_v": f16(f"{a}.1.to_v.weight"),
                "w_o": f16(f"{a}.1.to_out.weight"), "b_o": f32(f"{a}.1.to_out.bias"),
                "ln2": (f32(f"{f}.0.weight"), f32(f"{f}.0.bias")),
                "w_fc1": f16(f"{f}.1.net.0.0.weight"), "b_fc1": f32(f"{f}.1.net.0.0.bias"),
                "w_fc2": f16(f"{f}.1.net.2.weight"), "b_fc2": f32(f"{f}.1.net.2.bias")})
        W["ln_f"] = (f32("transformer.norm.weight"), f32("transformer.norm.bias"))
        self.W = W

    def check_ids(self, ids):
        """Host-side validation: sdb_embed_tokens clamps ids, so anything out of range raises here."""
        ids = torch.as_tensor(ids)
        if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool or ids.dim() != 2:
            raise TypeError(f"BERTEmbedder: token ids must be a 2-D integer tensor [B, n] (got {ids.dtype}, "
                            f"shape {tuple(ids.shape)})")
        B, n = ids.shape
        if B == 0 or not 1 <= n <= self.cfg["max_seq_len"]:
            raise ValueError(f"BERTEmbedder: need B >= 1 and 1 <= n <= {self.cfg['max_seq_len']} tokens "
                             f"(got {tuple(ids.shape)})")
        host = ids.detach().to("cpu", torch.int64)
        lo, hi = int(host.min()), int(host.max())
        if lo < 0 or hi >= self.cfg["vocab_size"]:
            raise IndexError(f"BERTEmbedder: token ids must lie in [0, {self.cfg['vocab_size']}) (got {lo} .. {hi})")
        return host

    @torch.no_grad()
    def encode_ids(self, ids):
        """ids: integer [B, n <= max_seq_len] -> fp32 [B, n, n_embed] on the weights' device."""
        assert self.W is not None, "weights not loaded (load_state_dict / load_weights, then .cuda())"
        assert self.W["device"].type == "cuda", "sdb200.BERTEmbedder runs on CUDA only (no CPU fallback)"
        W = self.W
        ids = self.check_ids(ids).to(W["device"]).contiguous()
        B, n = ids.shape
        x = ops.embed_tokens(ids, W["tok"], W["pos"])                                  # [B*n, n_embed] fp32
        x = encoder_layers(x, W["layers"], B, heads=HEADS, d=DIM_HEAD, eps=LN_EPS, act=ACT_GELU)
        _, z = ops.layernorm(x, *W["ln_f"], eps=LN_EPS, want_f32=True)
        return z.view(B, n, self.cfg["n_embed"])

    def _tokenize(self, text):
        """list[str] -> int64 [B, max_seq_len] as BERTTokenizer (modules.py:63-67): truncation, max_length padding."""
        if self.tokenizer is None:
            from .tokenizer import BertWordPieceTokenizer
            path = os.path.join(str(self.vocab_dir), "vocab.txt") if self.vocab_dir else _cached_vocab()
            if not path or not os.path.exists(path):
                raise RuntimeError("the bert-base-uncased vocabulary is not available offline; pass a directory with "
                                   "its vocab.txt as vocab_dir (txt2img.py --bert_vocab), or token ids")
            tok = BertWordPieceTokenizer(path, self.cfg["max_seq_len"])
            if len(tok) > self.cfg["vocab_size"]:
                raise ValueError(f"{path} has {len(tok)} entries, more than vocab_size {self.cfg['vocab_size']}")
            self.tokenizer = tok
        if isinstance(text, str):
            text = [text]
        if not all(isinstance(t, str) for t in text):
            raise TypeError("BERTEmbedder: text must be a string or a list of strings")
        return torch.tensor(self.tokenizer(list(text), self.cfg["max_seq_len"]), dtype=torch.long)

    def forward(self, text):
        ids = text if (torch.is_tensor(text) or not self.use_tknz_fn) else self._tokenize(text)
        return self.encode_ids(ids)

    def encode(self, text):
        return self(text)


def _cached_vocab():
    """vocab.txt of bert-base-uncased in the local Hugging Face cache, if any (a lookup only: nothing is downloaded)."""
    try:
        from huggingface_hub import try_to_load_from_cache
        p = try_to_load_from_cache("bert-base-uncased", "vocab.txt")
    except Exception:   # noqa: BLE001 - no hub client or no cache: no vocabulary
        return None
    return p if isinstance(p, str) else None
