"""H100-native CLIP ViT-L/14 text encoder: drop-in for `ldm.modules.encoders.modules.FrozenCLIPEmbedder`
(modules.py:137-162: `encode(text) -> (B, 77, 768)` = CLIPTextModel(...).last_hidden_state).

The arithmetic the reference delegates to third-party `transformers` (CLIPTextModel: token+position embedding,
12 pre-LN causal self-attention layers with quick-GELU MLP, final LayerNorm) runs on the same kernel family as the
UNet: fp32 LayerNorm -> fp16 operand, wgmma GEMMs with fused bias / quick-GELU / residual epilogues, the fused
wgmma attention kernel with a causal mask. The value bias is folded through out_proj at pack time
(softmax rows sum to 1). State-dict keys are transformers' (`text_model.*`), found under
`cond_stage_model.transformer.` in an SD checkpoint.

Tokenisation stays on the host with HF's CLIPTokenizer when its vocabulary files are available; there is no
vocabulary in this offline image, so `encode_ids` takes token ids directly (tests and the benchmark use seeded ids).
"""
from __future__ import annotations

import os

import torch
import torch.nn as nn

from . import ops
from .arch import CLIP_TEXT_PROJ, SD_V1_CLIP, clip_param_shapes, clip_text_proj_param_shapes
from .ops import ACT_QUICK_GELU
from .util import PackedStage


def pack_clip_layers(sd, prefix, n_layers):
    """The layer dicts of encoder_layers from HF CLIP encoder layers `{prefix}.{i}.*` (transformers' CLIPEncoderLayer
    keys; sd: fp32 tensors on the target device)."""
    f32 = lambda k: sd[k].contiguous()
    f16 = lambda k: sd[k].half().contiguous()
    layers = []
    for i in range(n_layers):
        p = f"{prefix}.{i}"
        wo = sd[p + ".self_attn.out_proj.weight"]
        layers.append({
            "ln1": (f32(p + ".layer_norm1.weight"), f32(p + ".layer_norm1.bias")),
            "ln2": (f32(p + ".layer_norm2.weight"), f32(p + ".layer_norm2.bias")),
            "w_qk": torch.cat([sd[p + ".self_attn.q_proj.weight"], sd[p + ".self_attn.k_proj.weight"]], 0).half().contiguous(),
            "b_qk": torch.cat([sd[p + ".self_attn.q_proj.bias"], sd[p + ".self_attn.k_proj.bias"]]).contiguous(),
            "w_v": f16(p + ".self_attn.v_proj.weight"),
            "w_o": wo.half().contiguous(),
            # softmax rows sum to 1: the value bias passes through the attention unchanged -> fold it through out_proj
            "b_o": (sd[p + ".self_attn.out_proj.bias"] + wo @ sd[p + ".self_attn.v_proj.bias"]).contiguous(),
            "w_fc1": f16(p + ".mlp.fc1.weight"), "b_fc1": f32(p + ".mlp.fc1.bias"),
            "w_fc2": f16(p + ".mlp.fc2.weight"), "b_fc2": f32(p + ".mlp.fc2.bias")})
    return layers


def encoder_layers(x, layers, B, *, heads, d, eps, act, causal=False):
    """Pre-LN transformer encoder layers (CLIP text and vision towers, BERTEmbedder) over the fp32 residual stream
    x [B*n, hidden]; returns the stream. Per layer: LayerNorm -> Q|K GEMM (bias "b_qk" when the layer has one) and V
    GEMM (its bias folded into "b_o") -> attention of `heads` heads of width d -> out-projection + residual ->
    LayerNorm -> fc1 with the `act` epilogue -> fc2 + residual. The attention width heads * d need not be hidden."""
    n, w = x.shape[0] // B, heads * d
    for L in layers:
        y = ops.layernorm(x, *L["ln1"], eps=eps)
        qk, _ = ops.gemm(y, L["w_qk"], bias=L.get("b_qk"), want_f16=True)            # [B*n, 2w]
        v, _ = ops.gemm(y, L["w_v"], want_f16=True)
        qk3 = qk.view(B, n, 2 * w)
        vt = ops.transpose_f16(v.view(B, n, w))                                       # [B, w, pad8(n)]
        o = ops.attention(qk3[:, :, :w], qk3[:, :, w:], vt, heads=heads, d=d, dpad=d, nq=n, nkv=n, scale=d ** -0.5,
                          causal=causal)
        _, x = ops.gemm(o.view(-1, w), L["w_o"], bias=L["b_o"], residual=x, want_f32=True)
        y = ops.layernorm(x, *L["ln2"], eps=eps)
        g, _ = ops.gemm(y, L["w_fc1"], bias=L["b_fc1"], act=act, want_f16=True)
        _, x = ops.gemm(g, L["w_fc2"], bias=L["b_fc2"], residual=x, want_f32=True)
    return x


class _Transformer(nn.Module):
    """Holds the `text_model.*` keys so the checkpoint prefix `cond_stage_model.transformer.` resolves."""

    def __init__(self, owner):
        super().__init__()
        object.__setattr__(self, "_owner", owner)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        self._owner._adopt(state_dict, prefix, missing_keys, unexpected_keys, error_msgs)


class FrozenCLIPEmbedder(PackedStage):
    # text_model.embeddings.position_ids is a buffer of older transformers versions (present in sd-v1 checkpoints)
    drop_prefixes = ("text_model.embeddings.position_ids",)

    def __init__(self, version="openai/clip-vit-large-patch14", device="cuda", max_length=77, config=None):
        super().__init__()
        self.cfg = dict(config or SD_V1_CLIP)
        self.version = version
        self.device = device
        self.max_length = max_length
        self.shapes = clip_param_shapes(self.cfg)
        self.transformer = _Transformer(self)
        self.tokenizer = None

    def _load_from_state_dict(self, *args):
        nn.Module._load_from_state_dict(self, *args)   # the keys sit one module below, in the shim, which adopts them

    def freeze(self):
        return self

    @torch.no_grad()
    def pack_weights(self, device):
        sd = {k: v.detach().to(device=device, dtype=torch.float32) for k, v in self._host_sd.items()}
        f32 = lambda k: sd[k].contiguous()
        self.W = {"device": device, "tok": f32("text_model.embeddings.token_embedding.weight"),
                  "pos": f32("text_model.embeddings.position_embedding.weight"),
                  "layers": pack_clip_layers(sd, "text_model.encoder.layers", self.cfg["num_hidden_layers"]),
                  "ln_f": (f32("text_model.final_layer_norm.weight"), f32("text_model.final_layer_norm.bias"))}

    def check_ids(self, ids):
        """Host-side validation before any launch. sdb_embed_tokens reads position row i for token i, so a sequence
        longer than the position table raises here, as do non-integer and non-2-D ids. It clamps ids to the vocabulary,
        so ids outside [0, vocab_size) raise here too when they are on the host (tokenizer output, or ids handed to
        forward / encode_ids from the CPU); ids already on the GPU are not read back, since that would stall the
        stream once per prompt."""
        if not torch.is_tensor(ids) or ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool \
                or ids.dim() != 2:
            raise TypeError(f"{type(self).__name__}: token ids must be a 2-D integer tensor [B, n] (got "
                            f"{getattr(ids, 'dtype', type(ids))}, shape {tuple(getattr(ids, 'shape', ()))})")
        B, n = ids.shape
        n_pos = self.cfg["max_position_embeddings"]
        if B == 0 or not 1 <= n <= n_pos:
            raise ValueError(f"{type(self).__name__}: need B >= 1 and 1 <= n <= {n_pos} tokens (got {tuple(ids.shape)})")
        if not ids.is_cuda:
            lo, hi = int(ids.min()), int(ids.max())
            if lo < 0 or hi >= self.cfg["vocab_size"]:
                raise IndexError(f"{type(self).__name__}: token ids must lie in [0, {self.cfg['vocab_size']}) "
                                 f"(got {lo} .. {hi})")

    @torch.no_grad()
    def encode_ids(self, ids):
        """ids: integer [B, n <= max_position_embeddings] (host ids are checked, then moved) -> fp32 [B, n, hidden] on
        the GPU."""
        assert self.W is not None, "weights not loaded (load_state_dict / load_weights, then .cuda())"
        self.check_ids(ids)
        W = self.W
        ids = ids.to(W["device"], torch.int64)
        B, n = ids.shape
        h = self.cfg["hidden_size"]
        heads = self.cfg["num_attention_heads"]
        d = h // heads
        assert d == 64, "CLIP text heads are 64 wide"
        eps = self.cfg["layer_norm_eps"]
        x = ops.embed_tokens(ids.contiguous(), W["tok"], W["pos"])                     # [B*n, h] fp32
        x = encoder_layers(x, W["layers"], B, heads=heads, d=d, eps=eps, act=ACT_QUICK_GELU, causal=True)
        _, z = ops.layernorm(x, *W["ln_f"], eps=eps, want_f32=True)
        return z.view(B, n, h)

    def _tokenize(self, text):
        """list[str] -> int64 [B, max_length] ids as `modules.py:153-156` (truncation, max_length padding).
        `version` may be a directory holding vocab.json + merges.txt (host-side BPE in tokenizer.py, no third-party
        code); otherwise the locally cached transformers tokenizer of that name is used, as the reference does."""
        if self.tokenizer is None:
            if os.path.isdir(str(self.version)) and os.path.exists(os.path.join(str(self.version), "vocab.json")):
                from .tokenizer import CLIPBPETokenizer
                self.tokenizer = CLIPBPETokenizer.from_dir(str(self.version), self.max_length)
            else:
                try:
                    from transformers import CLIPTokenizer
                    tok = CLIPTokenizer.from_pretrained(self.version, local_files_only=True)
                    if len(tok) < 49408:  # transformers >= 5 silently builds an empty tokenizer when files are missing
                        raise FileNotFoundError(f"vocabulary has {len(tok)} entries")
                    self.tokenizer = tok
                except Exception as e:  # no vocabulary offline
                    raise RuntimeError(f"CLIP tokenizer files for {self.version} are not available offline ({e}); pass "
                                       "a directory with vocab.json + merges.txt as `version`, or token ids to "
                                       "encode_ids()") from e
        if isinstance(text, str):
            text = [text]
        from .tokenizer import CLIPBPETokenizer
        if isinstance(self.tokenizer, CLIPBPETokenizer):
            return torch.tensor(self.tokenizer(list(text), self.max_length), dtype=torch.long)
        batch = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=True,
                               return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
        return batch["input_ids"]

    def forward(self, text):
        if torch.is_tensor(text):
            ids = text
        else:
            ids = self._tokenize(text)
        return self.encode_ids(ids)

    def encode(self, text):
        return self(text)


class FrozenCLIPTextEmbedder(FrozenCLIPEmbedder):
    """Drop-in for `ldm.modules.encoders.modules.FrozenCLIPTextEmbedder` (modules.py:165-194), the text encoder of the
    retrieval-augmented model (scripts/knn2img.py): `encode(text) -> (B, 1, projection_dim)`, CLIP's `encode_text`
    (the text tower above, the final LayerNorm, the row at the EOT token, `@ text_projection`) divided by its L2 norm.

    Weights are read in the transformers `CLIPModel` layout of the same ViT-L/14 checkpoint: `text_model.*` and
    `text_projection.weight`; the vision tower's keys are ignored. Prompts are tokenized as `clip.tokenize`: BOS +
    tokens + EOT, zero padding, and an error for prompts longer than max_length tokens. `version` is a directory with
    the CLIP vocab.json + merges.txt (or `tokenizer` a CLIPBPETokenizer). n_repeat copies the embedding along the token
    axis, as the reference's encode (knn2img.py keeps 1)."""

    drop_prefixes = FrozenCLIPEmbedder.drop_prefixes + ("vision_model.", "visual_projection.", "logit_scale")
    _load_from_state_dict = PackedStage._load_from_state_dict   # the keys sit at this level: no `transformer.` shim

    def __init__(self, version="ViT-L/14", device="cuda", max_length=77, n_repeat=1, normalize=True, config=None,
                 tokenizer=None):
        super().__init__(version=version, device=device, max_length=max_length, config=config or CLIP_TEXT_PROJ)
        del self.transformer
        self.shapes = clip_text_proj_param_shapes(self.cfg)
        self.n_repeat, self.normalize = n_repeat, normalize
        self.tokenizer = tokenizer

    @torch.no_grad()
    def pack_weights(self, device):
        super().pack_weights(device)
        self.W["proj"] = self._host_sd["text_projection.weight"].to(device=device, dtype=torch.float16).contiguous()

    def tokenize(self, text):
        """list[str] -> int64 [B, max_length] as `clip.tokenize(text)` (truncate=False)."""
        if self.tokenizer is None:
            from .tokenizer import CLIPBPETokenizer
            if not os.path.exists(os.path.join(str(self.version), "vocab.json")):
                raise RuntimeError(f"CLIP vocabulary not found: pass a directory with vocab.json + merges.txt as "
                                   f"`version` (got {self.version!r}), or token ids to encode_ids()")
            self.tokenizer = CLIPBPETokenizer.from_dir(str(self.version), self.max_length)
        tok = self.tokenizer
        if isinstance(text, str):
            text = [text]
        ids = torch.zeros((len(text), self.max_length), dtype=torch.long)
        for i, t in enumerate(text):
            row = [tok.bos_id] + tok.tokenize_ids(t) + [tok.eos_id]
            if len(row) > self.max_length:
                raise RuntimeError(f"Input {t} is too long for context length {self.max_length}")
            ids[i, :len(row)] = torch.tensor(row)
        return ids

    @torch.no_grad()
    def encode_ids(self, ids):
        """ids: integer [B, n] (host ids are checked, then moved), EOT = the largest id of each row -> fp32
        [B, projection_dim] on the GPU, normalised when `normalize` (the reference's forward)."""
        self.check_ids(ids)
        ids = ids.to(self.W["device"], torch.int64).contiguous()
        h = super().encode_ids(ids)                                                     # [B, n, hidden], final LN
        pooled = ops.rows_pool(h.view(-1, h.shape[-1]), ids)                           # the EOT rows
        z = ops.linear_small(pooled, self.W["proj"])
        return ops.rows_pool(z, normalize=True) if self.normalize else z

    def forward(self, text):
        ids = text if torch.is_tensor(text) else self.tokenize(text)
        return self.encode_ids(ids)

    def encode(self, text):
        z = self(text)
        if z.ndim == 2:
            z = z[:, None, :]
        return z.expand(-1, self.n_repeat, -1).contiguous() if self.n_repeat != 1 else z
