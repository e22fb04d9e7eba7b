"""H100-native UNet for the SD-v1 denoising loop and the unconditional attention-block LDMs: drop-in for the
reference's `ldm.modules.diffusionmodules.openaimodel.UNetModel` (constructor kwargs openaimodel.py:443-469,
`forward(x, timesteps, context)` openaimodel.py:710-742, state-dict keys unchanged).

Two members of the reference's UNet family run: the SD-v1 spatial-transformer UNet (cross-attention on a context, with
num_heads heads, or heads of num_head_channels as in the cin256 LDM-VQ-8; one BasicTransformerBlock per
SpatialTransformer, or three as in layout2img-openimages256), and
the unconditional AttentionBlock UNet (use_spatial_transformer=False, e.g. LSUN-Churches) with any combination of
use_scale_shift_norm and resblock_updown, or with plain ResBlocks and heads of num_head_channels (the VQ-f4 models).

Nothing here computes with torch: forward() only sequences the hand-written sm_90a kernels of libsdb200.so
(ops.py). torch provides device memory and the current stream. nn.Module is used solely so that the reference's
`load_state_dict` / `instantiate_from_config` plumbing (ldm/util.py:78-93, scripts/txt2img.py:49-66) sees this
object; there are no nn layers and no parameters.

Data layout: activations NHWC; the residual stream is fp32, tensor-core operands are fp16 (fp32 accumulate);
GroupNorm/LayerNorm statistics, softmax, FiLM and residual adds are fp32 (SURVEY.md §7.3-1).
"""
from __future__ import annotations

import math

import torch

from . import ops
from .arch import unet_param_shapes, unet_plan
from .ops import ACT_GEGLU, ACT_SILU
from .util import PackedStage


def _dpad(d):
    return (d + 63) // 64 * 64


def _pad64(w):
    """Zero columns up to the GEMM's 64-wide K step for a source width that is a multiple of 32 but not of 64 (the GEMM
    reads the tail of such a source as zeros); other widths are returned unchanged."""
    c = w.shape[-1]
    return torch.nn.functional.pad(w, (0, 32)) if c % 64 == 32 else w


def _pack_conv3(w):  # [Cout, Cin, 3, 3] -> [Cout, 9*Cin'], k = (ky*3+kx)*Cin' + c, Cin' = Cin padded by _pad64
    return _pad64(w.permute(0, 2, 3, 1)).reshape(w.shape[0], -1).contiguous().half()


def _pack_conv3_padk(w, kpad):  # small-Cin convs through im2col: k = (ky*3+kx)*Cin + c, K zero-padded to kpad
    p = torch.zeros((w.shape[0], kpad), dtype=torch.float16, device=w.device)
    p[:, : 9 * w.shape[1]] = w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).half()
    return p


def _pack_heads(w, heads, d, dpad):  # [heads*d, K] -> [heads*dpad, K], zero rows between heads
    """The head-padded layout (head_stride = dpad) that sdb_attention still accepts; the engine packs heads at stride
    d."""
    K = w.shape[1]
    p = torch.zeros((heads, dpad, K), dtype=torch.float16, device=w.device)
    p[:, :d] = w.reshape(heads, d, K).half()
    return p.reshape(heads * dpad, K).contiguous()


def _hilo(w):
    hi = w.half()
    return hi, (w - hi.float()).half()


def _pack_hilo_1x1(w):  # [N, K] fp32 -> [N, 3K] = [W_hi | W_hi | W_lo], multiplied by A = [A_hi | A_lo | A_hi]
    hi, lo = _hilo(w)
    return torch.cat([_pad64(hi), _pad64(hi), _pad64(lo)], dim=1).contiguous()


def _pack_hilo_conv3(w):  # [N, C, 3, 3] fp32 -> [N, 9 * 3C], per tap [W_hi | W_hi | W_lo]
    wk = w.permute(0, 2, 3, 1).reshape(w.shape[0], 9, w.shape[1])
    hi, lo = _hilo(wk)
    return torch.cat([_pad64(hi), _pad64(hi), _pad64(lo)], dim=2).reshape(w.shape[0], -1).contiguous()


def _geglu_tile(inner):
    """Accumulator tile width of the GEGLU GEMM: 256 ([128 value | 128 gate], CTA-pair tiles) when the inner width
    allows, else 128."""
    return 256 if inner % 128 == 0 else 128


def _pack_geglu(w, b):  # [8C, C]: rows [0,4C) value, [4C,8C) gate -> per accumulator tile [half value | half gate]
    inner = w.shape[0] // 2
    half = _geglu_tile(inner) // 2
    assert inner % half == 0
    idx = torch.arange(inner, device=w.device).reshape(-1, half)
    perm = torch.cat([idx, idx + inner], dim=1).reshape(-1)
    return w[perm].contiguous().half(), b[perm].contiguous().float()


class UNetModel(PackedStage):
    # "fp16x3": the 1x1 convs that act on the raw residual stream (ResBlock skip_connection, SpatialTransformer
    # proj_in / proj_out) and the final 320->4 conv run with hi/lo-split fp16 operands (three tensor-core passes,
    # ~fp32 operand precision); everything else single-pass fp16. These few layers (5% of the FLOPs) carry ~60% of the
    # fp16 operand-rounding error of eps (DESIGN.md, numerics). "fp16": single pass everywhere (eps rel-L2 ~1.2e-3).
    PRECISION = "fp16x3"

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, num_classes=None,
                 use_checkpoint=False, use_fp16=False, num_heads=-1, num_head_channels=-1, num_heads_upsample=-1,
                 use_scale_shift_norm=False, resblock_updown=False, use_new_attention_order=False,
                 use_spatial_transformer=False, transformer_depth=1, context_dim=None, n_embed=None, legacy=True):
        super().__init__()
        # same argument checks as the reference (openaimodel.py:471-489)
        if use_spatial_transformer:
            assert context_dim is not None, "Fool!! You forgot to include the dimension of your cross-attention conditioning..."
        if context_dim is not None:
            assert use_spatial_transformer, "Fool!! You forgot to use the spatial transformer for your cross-attention conditioning..."
            context_dim = list(context_dim) if isinstance(context_dim, (list, tuple)) else context_dim
        if num_heads == -1:
            assert num_head_channels != -1, "Either num_heads or num_head_channels has to be set"
        # the sdb200 path covers the configuration SD v1 ships (v1-inference.yaml:29-44) and the unconditional
        # AttentionBlock family (models/ldm/lsun_churches256/config.yaml: scale-shift norm, up/down ResBlocks;
        # configs/latent-diffusion/*-ldm-vq-4.yaml: plain ResBlocks with num_head_channels). Spatial transformers take
        # num_head_channels when it alone sets the heads (models/ldm/cin256: num_heads left at -1); the reference
        # silently ignores num_heads when both are given, so that combination is rejected.
        plain = not (use_spatial_transformer or use_scale_shift_norm or resblock_updown)
        st_nhc = use_spatial_transformer and num_heads == -1
        unsupported = dict(dims=dims != 2, num_classes=num_classes is not None, n_embed=n_embed is not None,
                           num_head_channels=num_head_channels != -1 and not (plain or st_nhc), dropout=dropout != 0,
                           conv_resample=not conv_resample, use_new_attention_order=bool(use_new_attention_order),
                           num_heads_upsample=num_heads_upsample not in (-1, num_heads))
        if use_spatial_transformer:
            # depth 1 (every other spatial-transformer LDM) and 3 (layout2img-openimages256) are the published ones
            unsupported.update(resblock_updown=resblock_updown, use_scale_shift_norm=use_scale_shift_norm,
                               transformer_depth=transformer_depth not in (1, 3))
        bad = [k for k, v in unsupported.items() if v]
        if bad:
            raise NotImplementedError("sdb200.UNetModel supports the SD-v1 UNet and the unconditional AttentionBlock UNet "
                                      f"configurations only; unsupported: {bad}")
        self.cfg = dict(image_size=image_size, in_channels=in_channels, model_channels=model_channels,
                        out_channels=out_channels, num_res_blocks=num_res_blocks,
                        attention_resolutions=list(attention_resolutions), channel_mult=list(channel_mult),
                        num_heads=num_heads, num_head_channels=num_head_channels,
                        use_spatial_transformer=bool(use_spatial_transformer),
                        transformer_depth=int(transformer_depth) if use_spatial_transformer else 1,
                        context_dim=context_dim, legacy=legacy, use_scale_shift_norm=bool(use_scale_shift_norm),
                        resblock_updown=bool(resblock_updown))
        self.conditional = bool(use_spatial_transformer)   # cross-attention on a context; otherwise forward(x, t)
        self.image_size = image_size
        self.in_channels, self.model_channels, self.out_channels = in_channels, model_channels, out_channels
        self.num_heads = num_heads
        self.context_dim = context_dim
        self.dtype = torch.float32
        self.plan = unet_plan(self.cfg)
        self.shapes = unet_param_shapes(self.cfg)
        self.precision = self.PRECISION
        # channels per fused GroupNorm-statistics entry: every channel count of the UNet (and of its skip concats) is a
        # multiple of model_channels, so the 32 groups always tile into entries of model_channels / 32 channels
        self._sg = model_channels // 32 if model_channels % 32 == 0 else 1
        if not self.conditional or all(bn % self._sg for bn in (64, 128, 160, 256)):
            # entries must also divide the GEMM tile widths (the GEMM drops the fused statistics otherwise): 192
            # channels -> 6 per group -> entries of 2; SD-v1's 10 divides the 160-wide tiles
            self._sg = math.gcd(self._sg, 16)
        self._ctx_ref = None    # the context tensor whose cross-attention K/V are cached (strong reference)
        self._ctx_ver = -1
        self._ctx_kv = None
        self._kv_static = {}
        self._graphs = {}
        self._arena = None
        self._side = None       # side stream of the FiLM chain (forked / joined inside every forward, graph-capturable)
        self._alt_sd = {}       # other weight sets of the same architecture by name (the EMA copy), host tensors
        self._packed = {}       # name -> (packed weights, captured graphs) of the sets not in use
        self._active = "raw"
        self.use_cuda_graph = False   # replay one captured graph per UNet evaluation (set by the pipeline / bench)
        self.autotune = True          # graph mode: pick (block_n, split-K) per GEMM problem by measurement before capture

    # ------------------------------------------------------------------ weights
    def set_weight_set(self, name, sd):
        """Register another state dict of this architecture (UNetModel keys) under `name`, e.g. the EMA weights."""
        self._alt_sd[name] = self._checked(sd, f"weight set {name}")
        self._packed.pop(name, None)

    def has_weight_set(self, name):
        return name in self._alt_sd

    @torch.no_grad()
    def use_weight_set(self, name="raw"):
        """Run on the weights registered under `name` ("raw": the loaded state dict). Each set is packed once and keeps
        its own captured CUDA graphs, so switching back and forth costs no repacking."""
        if name == self._active:
            return
        assert name == "raw" or name in self._alt_sd, f"no weight set {name}"
        if self.W is not None:
            self._packed[self._active] = (self.W, self._graphs)
            dev = self.W["device"]
            if name in self._packed:
                self.W, self._graphs = self._packed.pop(name)
                self._ctx_ref = None      # cross-attention K / V are recomputed with this set's weights
            else:
                self._active = name
                self.pack_weights(dev, keep_sets=True)
        self._active = name

    @torch.no_grad()
    def pack_weights(self, device, keep_sets=False):
        if not keep_sets:       # fresh weights: every packed set is stale
            self._packed = {}
            self._active = "raw"
        src = self._host_sd if self._active == "raw" else self._alt_sd[self._active]
        sd = {k: v.detach().to(device=device, dtype=torch.float32) for k, v in src.items()}
        W = {"device": device}
        f32 = lambda k: sd[k].contiguous()
        f16 = lambda k: sd[k].half().contiguous()
        x3 = self.precision == "fp16x3"
        W["x3"] = x3
        one = (lambda w: _pack_hilo_1x1(w)) if x3 else (lambda w: w.half().contiguous())
        mc = self.model_channels
        W["te0_w"], W["te0_b"] = f16("time_embed.0.weight"), f32("time_embed.0.bias")
        W["te2_w"], W["te2_b"] = f16("time_embed.2.weight"), f32("time_embed.2.bias")
        emb_w, emb_b, emb_off = [], [], {}
        off = 0

        def pack_res(pre, a):
            nonlocal off
            r = {"cin": a["cin"], "cout": a["cout"], "ss": a.get("ss", False), "updown": a.get("updown")}
            assert r["updown"] is None or a["cin"] == a["cout"]
            r["gn1"] = (f32(pre + ".in_layers.0.weight"), f32(pre + ".in_layers.0.bias"))
            r["w1"], r["b1"] = _pack_conv3(sd[pre + ".in_layers.2.weight"]), f32(pre + ".in_layers.2.bias")
            r["gn2"] = (f32(pre + ".out_layers.0.weight"), f32(pre + ".out_layers.0.bias"))
            r["w2"], r["b2"] = _pack_conv3(sd[pre + ".out_layers.3.weight"]), f32(pre + ".out_layers.3.bias")
            if a["cin"] != a["cout"]:
                r["ws"] = one(sd[pre + ".skip_connection.weight"].reshape(a["cout"], a["cin"]))
                r["bs"] = f32(pre + ".skip_connection.bias")
            emb_w.append(sd[pre + ".emb_layers.1.weight"].half())
            emb_b.append(sd[pre + ".emb_layers.1.bias"])
            r["film_off"] = off
            off += 2 * a["cout"] if r["ss"] else a["cout"]     # [scale | shift] with use_scale_shift_norm
            return r

        def pack_attn(pre, a):
            """AttentionBlock (openaimodel.py:278-324) with QKVAttentionLegacy: qkv rows are [head][q | k | v][ch]. They
            are repacked into head-major Q|K and V weights for the flash kernel. The V bias is folded into proj_out:
            softmax rows sum to one, so P (V + 1 b_v^T) = P V + 1 b_v^T, and proj_out(o + b_v) = W_p o + (W_p b_v + b_p)."""
            ch, d = a["ch"], a["dhead"]
            hh = a["heads"]
            dp = _dpad(d)
            w = sd[pre + ".qkv.weight"].reshape(hh, 3, d, ch)
            b = sd[pre + ".qkv.bias"].reshape(hh, 3, d)
            s = {"ch": ch, "d": d, "dpad": dp, "heads": hh}
            s["gn"] = (f32(pre + ".norm.weight"), f32(pre + ".norm.bias"))
            s["w_qk"] = w[:, :2].transpose(0, 1).reshape(2 * hh * d, ch).half().contiguous()
            s["b_qk"] = b[:, :2].transpose(0, 1).reshape(-1).float().contiguous()
            s["w_v"] = w[:, 2].reshape(hh * d, ch).half().contiguous()
            wp = sd[pre + ".proj_out.weight"].reshape(ch, ch)
            s["w_proj"] = wp.half().contiguous()
            s["b_proj"] = (sd[pre + ".proj_out.bias"].double() + wp.double() @ b[:, 2].reshape(-1).double()).float().contiguous()
            return s

        def pack_block(tb):
            """One BasicTransformerBlock (attention.py:196-215)."""
            b = {"tb": tb}
            for i in (1, 2, 3):
                b[f"ln{i}"] = (f32(f"{tb}.norm{i}.weight"), f32(f"{tb}.norm{i}.bias"))
            b["w_qk1"] = torch.cat([sd[tb + ".attn1.to_q.weight"], sd[tb + ".attn1.to_k.weight"]], 0).half().contiguous()
            b["w_v1"] = f16(tb + ".attn1.to_v.weight")
            b["w_o1"], b["b_o1"] = f16(tb + ".attn1.to_out.0.weight"), f32(tb + ".attn1.to_out.0.bias")
            b["w_q2"] = f16(tb + ".attn2.to_q.weight")
            b["w_k2"] = f16(tb + ".attn2.to_k.weight")
            b["w_v2"] = f16(tb + ".attn2.to_v.weight")
            b["w_o2"], b["b_o2"] = f16(tb + ".attn2.to_out.0.weight"), f32(tb + ".attn2.to_out.0.bias")
            b["w_ff1"], b["b_ff1"] = _pack_geglu(sd[tb + ".ff.net.0.proj.weight"], sd[tb + ".ff.net.0.proj.bias"])
            b["w_ff2"], b["b_ff2"] = f16(tb + ".ff.net.2.weight"), f32(tb + ".ff.net.2.bias")
            return b

        def pack_st(pre, a):
            """SpatialTransformer with the plan's heads of dhead channels (num_heads, or ch / num_head_channels) and its
            `depth` BasicTransformerBlocks in order."""
            ch, d = a["ch"], a["dhead"]
            dp = _dpad(d)
            s = {"ch": ch, "d": d, "dpad": dp, "heads": a["heads"]}
            s["gn"] = (f32(pre + ".norm.weight"), f32(pre + ".norm.bias"))
            s["w_in"], s["b_in"] = one(sd[pre + ".proj_in.weight"].reshape(ch, ch)), f32(pre + ".proj_in.bias")
            s["w_out"], s["b_out"] = one(sd[pre + ".proj_out.weight"].reshape(ch, ch)), f32(pre + ".proj_out.bias")
            s["blocks"] = [pack_block(f"{pre}.transformer_blocks.{i}") for i in range(a["depth"])]
            return s

        def pack_layers(layers):
            out = []
            for kind, pre, a in layers:
                if kind == "conv_in":
                    # K = 9 * in_channels zero-padded to the GEMM's 64-wide K step (64 up to 7 channels, 192 for 16)
                    kpad = (9 * a["cin"] + 63) // 64 * 64
                    out.append((kind, {"w": _pack_conv3_padk(sd[pre + ".weight"], kpad), "b": f32(pre + ".bias"),
                                       "cout": a["cout"]}))
                elif kind == "res":
                    out.append((kind, pack_res(pre, a)))
                elif kind == "st":
                    out.append((kind, pack_st(pre, a)))
                elif kind == "attn":
                    out.append((kind, pack_attn(pre, a)))
                elif kind == "down":
                    out.append((kind, {"w": _pack_conv3(sd[pre + ".op.weight"]), "b": f32(pre + ".op.bias"), "ch": a["ch"]}))
                elif kind == "up":
                    out.append((kind, {"w": _pack_conv3(sd[pre + ".conv.weight"]), "b": f32(pre + ".conv.bias"), "ch": a["ch"]}))
            return out

        W["input"] = [pack_layers(l) for l in self.plan["input"]]
        W["middle"] = pack_layers(self.plan["middle"])
        W["output"] = [pack_layers(l) for l in self.plan["output"]]
        W["gn_out"] = (f32("out.0.weight"), f32("out.0.bias"))
        W["w_out"] = _pack_hilo_conv3(sd["out.2.weight"]) if x3 else _pack_conv3(sd["out.2.weight"])
        W["b_out"] = f32("out.2.bias")
        W["emb_w"] = torch.cat(emb_w, 0).contiguous()
        W["emb_b"] = torch.cat(emb_b, 0).float().contiguous()
        W["st_list"] = [p for grp in W["input"] + [W["middle"]] + W["output"] for k, p in grp if k == "st"]
        self.W = W
        self._ctx_ref = None
        self._kv_static = {}
        self._graphs = {}

    # ------------------------------------------------------------------ blocks
    def _film(self, t):
        """time_embed MLP + all 22 emb_layers in three weight-streaming launches (fp32 activations)."""
        W = self.W
        te = ops.timestep_embedding_f32(t, self.model_channels)
        h = ops.linear_small(te, W["te0_w"], W["te0_b"], act=ACT_SILU)
        # ResBlocks only ever consume SiLU(emb) (openaimodel.py:217-218), so apply it in this epilogue
        h = ops.linear_small(h, W["te2_w"], W["te2_b"], act=ACT_SILU)
        return ops.linear_small(h, W["emb_w"], W["emb_b"])          # [N, sum(Cout)] fp32

    def _res(self, r, h, skip, film, emit_f16=False):
        """ResBlock._forward (openaimodel.py:255-275); `skip` is the UNet skip tensor concatenated along C.
        emit_f16: the last GEMM also writes an fp16 copy of the block output (operand of a following stride-2 conv).
        Up / down blocks resample inside the first GroupNorm kernel (h_upd) and through sdb_resample_f32 (x_upd); with
        scale-shift norm the FiLM vector modulates the second GroupNorm instead of being added by the first conv."""
        x3 = self.W["x3"] and "ws" in r
        raw = raw_lo = None
        if r["updown"] is not None:
            assert skip is None
            mode = 1 if r["updown"] == "down" else 2
            hn = ops.groupnorm_mod(h, *r["gn1"], resample=mode, eps=1e-5, silu=True)
            h = ops.resample_f32(h, mode)
        elif x3:
            hn, raw, _, raw_lo = ops.groupnorm(h, *r["gn1"], x1=skip, eps=1e-5, silu=True, want_raw_lo=True)
        else:
            hn, raw = ops.groupnorm(h, *r["gn1"], x1=skip, eps=1e-5, silu=True, want_raw="ws" in r)
        nb, H, Wd, _ = h.shape
        fo, co = r["film_off"], r["cout"]
        _, h1 = ops.gemm(hn, r["w1"], taps=9, bias=r["b1"], film=None if r["ss"] else film[:, fo: fo + co], want_f32=True,
                         splits=-1, want_stats=True, stats_group=self._sg)
        h1 = h1.view(nb, H, Wd, co)
        if r["ss"]:
            hn2 = ops.groupnorm_mod(h1, *r["gn2"], scale=film[:, fo: fo + co], shift=film[:, fo + co: fo + 2 * co],
                                    eps=1e-5, silu=True)
        else:
            hn2, _ = ops.groupnorm(h1, *r["gn2"], eps=1e-5, silu=True)
        if x3:    # skip 1x1 conv on the raw stream: [x_hi | x_lo | x_hi] . [W_hi | W_hi | W_lo]
            _, res = ops.gemm(raw, r["ws"], a1=raw_lo, a2=raw, bias=r["bs"], want_f32=True, splits=-1)
        elif "ws" in r:
            _, res = ops.gemm(raw, r["ws"], bias=r["bs"], want_f32=True, splits=-1)
        else:
            assert skip is None
            res = h.view(-1, r["cout"])
        o16, out = ops.gemm(hn2, r["w2"], taps=9, bias=r["b2"], residual=res, want_f32=True, want_f16=emit_f16, splits=-1,
                            want_stats=True, stats_group=self._sg)
        out = out.view(nb, H, Wd, r["cout"])
        if emit_f16:
            out._sdb_f16 = o16.view(nb, H, Wd, r["cout"])
        return out

    def _st(self, s, x, kvs, emit_f16=False):
        """SpatialTransformer.forward (attention.py:250-261): GroupNorm and proj_in, the BasicTransformerBlocks in order
        (one cross-attention K / V^T of `kvs` each) on the fp32 token stream, then proj_out and the residual. A block
        before the last writes its feed-forward output in fp32 for the next block's LayerNorm; the last one's goes to
        proj_out as fp16 (hi / lo in fp16x3)."""
        nb, H, Wd, ch = x.shape
        ntok = H * Wd
        x3 = self.W["x3"]
        if x3:
            xn, _, xn_lo, _ = ops.groupnorm(x, *s["gn"], eps=1e-6, silu=False, want_lo=True)
            _, t = ops.gemm(xn, s["w_in"], a1=xn_lo, a2=xn, bias=s["b_in"], want_f32=True, splits=-1)
        else:
            xn, _ = ops.groupnorm(x, *s["gn"], eps=1e-6, silu=False)
            _, t = ops.gemm(xn, s["w_in"], bias=s["b_in"], want_f32=True, splits=-1)       # tokens [M, ch] fp32
        blocks = s["blocks"]
        assert len(kvs) == len(blocks)
        for b, kv in zip(blocks[:-1], kvs[:-1]):
            t2, g = self._block(s, b, t, kv, nb, ntok)
            _, t = ops.gemm(g, b["w_ff2"], bias=b["b_ff2"], residual=t2, want_f32=True, splits=-1)
        b = blocks[-1]
        t2, g = self._block(s, b, t, kvs[-1], nb, ntok)
        if x3:
            t3, _, t3_lo = ops.gemm(g, b["w_ff2"], bias=b["b_ff2"], residual=t2, want_lo=True, splits=-1)
            o16, out = ops.gemm(t3, s["w_out"], a1=t3_lo, a2=t3, bias=s["b_out"], residual=x.view(-1, ch), want_f32=True,
                                want_f16=emit_f16, splits=-1, rows_per_sample=ntok, want_stats=True, stats_group=self._sg)
        else:
            t3, _ = ops.gemm(g, b["w_ff2"], bias=b["b_ff2"], residual=t2, want_f16=True, splits=-1)
            o16, out = ops.gemm(t3, s["w_out"], bias=s["b_out"], residual=x.view(-1, ch), want_f32=True,
                                want_f16=emit_f16, splits=-1, rows_per_sample=ntok, want_stats=True, stats_group=self._sg)
        out = out.view(nb, H, Wd, ch)
        if emit_f16:
            out._sdb_f16 = o16.view(nb, H, Wd, ch)
        return out

    def _block(self, s, b, t0, kv, nb, ntok):
        """BasicTransformerBlock._forward (attention.py:211-215) on the fp32 tokens t0 up to the feed-forward's GEGLU:
        returns the residual stream after both attentions (fp32) and the GEGLU output (fp16), whose second linear layer
        the caller runs with the output form it needs."""
        ch = s["ch"]
        heads, d, dp = s["heads"], s["d"], s["dpad"]
        hd = heads * d                                                                     # heads packed at stride d
        scale = d ** -0.5
        # --- self attention
        y = ops.layernorm(t0, *b["ln1"])
        qk, _ = ops.gemm(y, b["w_qk1"], want_f16=True)                                     # [M, 2*hd]
        qk3 = qk.view(nb, ntok, 2 * hd)
        if ntok % 8 == 0:
            # V^T straight out of the tensor cores by swapping the operand roles: [hd, M] = Wv . y^T
            vt, _ = ops.gemm(b["w_v1"], y, want_f16=True, b_dynamic=True)
            vt3 = vt.view(hd, nb, ntok).permute(1, 0, 2)                                   # [nb, hd, ntok] (strided view)
        else:  # TMA needs 16-byte aligned strides: tiny token counts go through an explicit transpose
            v, _ = ops.gemm(y, b["w_v1"], want_f16=True)
            vt3 = ops.transpose_f16(v.view(nb, ntok, hd))
        o = ops.attention(qk3[:, :, :hd], qk3[:, :, hd:], vt3, heads=heads, d=d, dpad=dp, nq=ntok, nkv=ntok, scale=scale,
                          head_stride=d)
        k2, vt2, nkv = kv
        if k2 is None:
            # one-token context (context_kv): attn2(LN2(t1), c) = u per sample, added as the FiLM operand of the attn1
            # out-projection, which then yields t2 = t0 + attn1 + u directly
            _, t2 = ops.gemm(o.view(-1, ch), b["w_o1"], bias=b["b_o1"], film=vt2, rows_per_sample=ntok, residual=t0,
                             want_f32=True, splits=-1)
        else:
            _, t1 = ops.gemm(o.view(-1, ch), b["w_o1"], bias=b["b_o1"], residual=t0, want_f32=True, splits=-1)
            # --- cross attention (K / V^T of the context are precomputed per prompt)
            y = ops.layernorm(t1, *b["ln2"])
            q, _ = ops.gemm(y, b["w_q2"], want_f16=True)
            o = ops.attention(q.view(nb, ntok, hd), k2, vt2, heads=heads, d=d, dpad=dp, nq=ntok, nkv=nkv, scale=scale,
                              head_stride=d)
            _, t2 = ops.gemm(o.view(-1, ch), b["w_o2"], bias=b["b_o2"], residual=t1, want_f32=True, splits=-1)
        # --- GEGLU feed-forward
        y = ops.layernorm(t2, *b["ln3"])
        g, _ = ops.gemm(y, b["w_ff1"], bias=b["b_ff1"], act=ACT_GEGLU, want_f16=True,
                        block_n=_geglu_tile(b["w_ff1"].shape[0] // 2))
        return t2, g

    def _attn(self, s, x, emit_f16=False):
        """AttentionBlock._forward (openaimodel.py:318-324) with QKVAttentionLegacy (:347-372) on the flash kernel.
        The reference scales q and k by ch^-0.25 each; the kernel applies ch^-0.5 to the product."""
        nb, H, Wd, ch = x.shape
        ntok = H * Wd
        heads, d, dp = s["heads"], s["d"], s["dpad"]
        hd = heads * d                                                                     # heads packed at stride d
        xn, _ = ops.groupnorm(x, *s["gn"], eps=1e-5, silu=False)
        xm = xn.view(-1, ch)
        qk, _ = ops.gemm(xm, s["w_qk"], bias=s["b_qk"], want_f16=True)                     # [M, 2*hd]
        qk3 = qk.view(nb, ntok, 2 * hd)
        if ntok % 8 == 0:
            vt, _ = ops.gemm(s["w_v"], xm, want_f16=True, b_dynamic=True)                    # V^T [hd, M]
            vt3 = vt.view(hd, nb, ntok).permute(1, 0, 2)
        else:  # TMA needs 16-byte aligned strides: the 4x4 / 2x2 levels go through an explicit transpose
            v, _ = ops.gemm(xm, s["w_v"], want_f16=True)
            vt3 = ops.transpose_f16(v.view(nb, ntok, hd))
        o = ops.attention(qk3[:, :, :hd], qk3[:, :, hd:], vt3, heads=heads, d=d, dpad=dp, nq=ntok, nkv=ntok,
                          scale=d ** -0.5, head_stride=d)
        o16, out = ops.gemm(o.view(-1, ch), s["w_proj"], bias=s["b_proj"], residual=x.view(-1, ch), want_f32=True,
                            want_f16=emit_f16, splits=-1, rows_per_sample=ntok, want_stats=True, stats_group=self._sg)
        out = out.view(nb, H, Wd, ch)
        if emit_f16:
            out._sdb_f16 = o16.view(nb, H, Wd, ch)
        return out

    def _one_token_weights(self):
        """[sum ch, context_dim] fp16 / [sum ch] fp32: W_o2 W_v2 of every SpatialTransformer (folded in fp64) and b_o2,
        stacked so that u = W c + b for all of them is one weight-streaming launch."""
        W = self.W
        if "u_w" not in W:      # from the fp32 weights of the set in use: one fp16 rounding of the product
            src = self._host_sd if self._active == "raw" else self._alt_sd[self._active]
            f64 = lambda k: src[k].to(device=W["device"], dtype=torch.float64)
            tbs = [s["blocks"][0] for s in W["st_list"]]
            W["u_w"] = torch.cat([(f64(b["tb"] + ".attn2.to_out.0.weight") @ f64(b["tb"] + ".attn2.to_v.weight")).half()
                                  for b in tbs], 0).contiguous()
            W["u_b"] = torch.cat([b["b_o2"] for b in tbs], 0).contiguous()
        return W["u_w"], W["u_b"]

    def context_kv(self, context, static=False):
        """Cross-attention K and V^T for every BasicTransformerBlock of every SpatialTransformer, in execution order
        (x/t independent: once per prompt). static=True writes into persistent per-shape buffers, one per block, so
        captured CUDA graphs stay valid across prompts.
        A one-token context (the ClassEmbedder's) makes the softmax over one key exactly 1, so attn2(x, c) =
        to_out(to_v(c)) does not depend on x: each SpatialTransformer gets (None, u [nb, ch], 1) with
        u = W_o2 W_v2 c + b_o2 instead of K / V^T. That fold is made for single-block transformers only: no published
        model pairs a one-token context with deeper ones."""
        nb, nkv, cd = context.shape
        bufs = self._kv_static.setdefault((nb, nkv), {}) if static else {}
        if nkv == 1:
            if self.cfg["transformer_depth"] != 1:
                raise NotImplementedError("a one-token context (ClassEmbedder) with transformer_depth "
                                          f"{self.cfg['transformer_depth']}: only depth 1 is supported")
            w, b = self._one_token_weights()
            u = ops.linear_small(context.contiguous().float().view(nb, cd), w, b, out=bufs.get("u"))
            bufs["u"] = u
            out, off = [], 0
            for s in self.W["st_list"]:
                out.append((None, u[:, off: off + s["ch"]], 1))
                off += s["ch"]
            return out
        ctx16 = ops.cast_f16(context.contiguous().float().view(nb * nkv, cd))
        ld = (nkv + 7) // 8 * 8
        out = []
        for i, (s, b) in enumerate((s, b) for s in self.W["st_list"] for b in s["blocks"]):
            hd = s["heads"] * s["d"]
            if i not in bufs:
                bufs[i] = (torch.empty((nb * nkv, hd), dtype=torch.float16, device=context.device),
                           torch.empty((nb * nkv, hd), dtype=torch.float16, device=context.device),
                           torch.empty((nb, hd, ld), dtype=torch.float16, device=context.device))
            kb, vb, vtb = bufs[i]
            ops.gemm(ctx16, b["w_k2"], out_f16=kb)
            ops.gemm(ctx16, b["w_v2"], out_f16=vb)
            ops.transpose_f16(vb.view(nb, nkv, hd), out=vtb)
            out.append((kb.view(nb, nkv, hd), vtb, nkv))
        return out

    def set_context(self, context):
        """Cache the cross-attention K/V for `context` ([uncond; cond] batch). forward() reuses them for the same
        tensor object (unmodified since) or for a tensor with equal contents; the cached tensor is kept alive, so a new
        prompt can never alias it through a recycled allocation."""
        self._ctx_kv = self.context_kv(context, static=True)
        self._ctx_ref, self._ctx_ver = context, context._version
        return self._ctx_kv

    def _context_cached(self, context):
        ref = self._ctx_ref
        if ref is None or self._ctx_kv is None:
            return False
        if context is ref:
            return context._version == self._ctx_ver
        # a different tensor object (the reference samplers build torch.cat([uc, c]) every step, plms.py:182-185):
        # compare contents - a 2x77x768 compare is far cheaper than 32 projection GEMMs
        return (ref._version == self._ctx_ver and context.shape == ref.shape and context.dtype == ref.dtype
                and context.device == ref.device and bool(torch.equal(context, ref)))

    def _run_layers(self, layers, h, skip, film, kvs, st_idx, emit_f16=False):
        """emit_f16: the block's output feeds a Downsample next, whose stride-2 conv reads an fp16 copy through TMA."""
        for li, (kind, p) in enumerate(layers):
            last = emit_f16 and li == len(layers) - 1
            if kind == "res":
                h = self._res(p, h, skip, film, emit_f16=last)
                skip = None
            elif kind == "st":
                n = len(p["blocks"])
                h = self._st(p, h, kvs[st_idx[0]: st_idx[0] + n], emit_f16=last)
                st_idx[0] += n
            elif kind == "attn":
                h = self._attn(p, h, emit_f16=last)
            elif kind == "down":
                # Downsample (openaimodel.py:149-153): 3x3, stride 2, pad 1, straight from the NHWC activation through
                # strided TMA boxes (element strides {1,2,2,1}); no im2col buffer
                nb, H, Wd, c = h.shape
                h16 = getattr(h, "_sdb_f16", None)
                if h16 is None:
                    h16 = ops.cast_f16(h)
                _, o = ops.gemm(h16, p["w"], taps=9, conv_stride=2, bias=p["b"], want_f32=True, splits=-1, want_stats=True, stats_group=self._sg)
                h = o.view(nb, (H + 1) // 2, (Wd + 1) // 2, c)
            elif kind == "up":
                nb, H, Wd, c = h.shape
                up = ops.upsample2x(h)
                _, o = ops.gemm(up, p["w"], taps=9, bias=p["b"], want_f32=True, splits=-1, want_stats=True, stats_group=self._sg)
                h = o.view(nb, 2 * H, 2 * Wd, c)
            elif kind == "conv_in":
                if isinstance(h, tuple):    # concat route: (x, conditioning), both NCHW, one im2col for the pair
                    nb, _, H, Wd = h[0].shape
                    col = ops.im2col3x3_concat(h[0], h[1], p["w"].shape[1])
                else:
                    nb, H, Wd, c = h.shape
                    col = ops.im2col3x3(h, 1, 1, H, Wd, p["w"].shape[1])
                _, o = ops.gemm(col, p["w"], bias=p["b"], want_f32=True, rows_per_sample=H * Wd, want_stats=True, stats_group=self._sg)
                h = o.view(nb, H, Wd, p["cout"])
        return h

    # ------------------------------------------------------------------ forward
    def _forward_impl(self, x, t, kvs, concat=None):
        """x NCHW fp32, t fp32 [nb], kvs from context_kv, concat: NCHW fp32 channels that follow x's (or None) -> eps
        NCHW fp32. Pure kernel sequence (graph-capturable)."""
        nb, _, H, Wd = x.shape
        if self._arena is None:
            self._arena = ops.StatsArena(x.device)
        self._arena.reset()          # one memset for all fused GroupNorm statistics of this evaluation
        ops.ARENA = self._arena
        try:
            return self._forward_body(x, t, kvs, concat)
        finally:
            ops.ARENA = None

    def _forward_body(self, x, t, kvs, concat=None):
        nb, _, H, Wd = x.shape
        # The FiLM chain (timestep embedding -> time_embed MLP -> all emb_layers, three weight-streaming launches, ~37 us)
        # depends on t only: it runs on a side stream next to nchw->nhwc / conv_in and joins before the first ResBlock.
        cur = torch.cuda.current_stream()
        if self._side is None:
            self._side = torch.cuda.Stream()
        side = self._side
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            film = self._film(t)
        film.record_stream(cur)
        h = (x, concat) if concat is not None else ops.nchw_to_nhwc(x)[0]
        W = self.W
        hs = []
        st_idx = [0]
        joined = False
        for bi, layers in enumerate(W["input"]):
            if not joined and any(kind != "conv_in" for kind, _ in layers):
                cur.wait_stream(side)
                joined = True
            nxt = W["input"][bi + 1] if bi + 1 < len(W["input"]) else None
            h = self._run_layers(layers, h, None, film, kvs, st_idx, emit_f16=bool(nxt) and nxt[0][0] == "down")
            hs.append(h)
        if not joined:
            cur.wait_stream(side)
        h = self._run_layers(W["middle"], h, None, film, kvs, st_idx)
        for layers in W["output"]:
            h = self._run_layers(layers, h, hs.pop(), film, kvs, st_idx)
        if W["x3"]:
            hn, _, hn_lo, _ = ops.groupnorm(h, *W["gn_out"], eps=1e-5, silu=True, want_lo=True)
            _, o = ops.gemm(hn, W["w_out"], a1=hn_lo, a2=hn, taps=9, bias=W["b_out"], want_f32=True)
        else:
            hn, _ = ops.groupnorm(h, *W["gn_out"], eps=1e-5, silu=True)
            _, o = ops.gemm(hn, W["w_out"], taps=9, bias=W["b_out"], want_f32=True)
        return ops.nhwc_to_nchw(o.view(nb, H, Wd, self.out_channels))

    def _graph_for(self, shape, kvs, concat_shape=None, ctx_tokens=None):
        """Capture one UNet evaluation (~400 kernels) as a CUDA graph with static x / t / eps / K,V buffers, and a static
        conditioning buffer on the concat route. The static K,V buffers are per context token count, so a conditional
        UNet keeps one graph per (shape, ctx_tokens): text-only and text + neighbours contexts share a latent shape."""
        key = shape if concat_shape is None else (shape, concat_shape)
        if ctx_tokens is not None:
            key = (key, ctx_tokens)
        g = self._graphs.get(key)
        if g is None:
            dev = self.W["device"]
            sx = torch.zeros(shape, dtype=torch.float32, device=dev)
            st = torch.zeros((shape[0],), dtype=torch.float32, device=dev)
            sc = None if concat_shape is None else torch.zeros(concat_shape, dtype=torch.float32, device=dev)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):      # warm-up outside capture: cudaFuncSetAttribute, allocator pools,
                ops.AUTOTUNE = self.autotune   # and one-time (block_n, split-K) selection per GEMM problem
                try:
                    self._forward_impl(sx, st, kvs, sc)
                finally:
                    ops.AUTOTUNE = False
                self._forward_impl(sx, st, kvs, sc)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            n0 = ops.launch_count()
            with torch.cuda.graph(graph):
                out = self._forward_impl(sx, st, kvs, sc)
            g = {"graph": graph, "x": sx, "t": st, "c": sc, "out": out, "launches": ops.launch_count() - n0, "kvs": kvs}
            self._graphs[key] = g
        return g

    # ------------------------------------------------------------------ handle-level C entry (include/sdb200.h)
    @torch.no_grad()
    def c_handle(self, shape, context=None):
        """Build the C-side handle of one guided evaluation for latents of `shape` = (n, c, h, w) and the given context
        (None for the unconditional model):
        walks the model once between sdb_plan_begin / sdb_plan_end (every launch is recorded with its arguments; the
        pass doubles as warm-up), then wraps the plan and its static x / t / eps buffers in an sdb_unet. Afterwards
        `sdb_unet_forward(handle, x, t, eps, stream)` and `sdb_sample_plms` run without any Python on the hot path.
        All intermediates of the recorded pass live in a private memory pool owned by the returned object."""
        import ctypes as C
        from . import lib as _l
        lib = _l.load()
        dev = self.W["device"]
        self._check_context(context, shape[0])
        kvs = self.set_context(context) if self.conditional else None
        x = torch.zeros(shape, dtype=torch.float32, device=dev)
        t = torch.zeros((shape[0],), dtype=torch.float32, device=dev)
        ops.AUTOTUNE = self.autotune
        try:
            self._forward_impl(x, t, kvs)       # (block_n, split-K) selection happens outside the recording
        finally:
            ops.AUTOTUNE = False
        torch.cuda.synchronize()
        pool = torch.cuda.MemPool()
        plan = C.c_void_p()
        with torch.cuda.use_mem_pool(pool):
            _l.check(lib.sdb_plan_begin(C.byref(plan)), "sdb_plan_begin")
            try:
                eps = self._forward_impl(x, t, kvs)
            finally:
                _l.check(lib.sdb_plan_end(plan), "sdb_plan_end")
        torch.cuda.synchronize()
        h = C.c_void_p()
        _l.check(lib.sdb_unet_create(plan, C.c_void_p(x.data_ptr()), C.c_void_p(t.data_ptr()), C.c_void_p(eps.data_ptr()),
                                     shape[0], shape[1], eps.shape[1], shape[2], shape[3], C.byref(h)), "sdb_unet_create")
        return CUNet(h, plan, pool, (x, t, eps, kvs, context), int(lib.sdb_plan_size(plan)))

    def _check_context(self, context, nb):
        if not self.conditional:
            if context is not None:
                raise ValueError("this UNet is unconditional (no spatial transformer): call forward(x, t) without a context")
            return
        assert context is not None and context.shape[0] == nb and context.shape[2] == self.context_dim

    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, concat=None, **kwargs):
        """eps = UNet(x, t[, context]). concat: NCHW channels that follow x's in the UNet input (DiffusionWrapper's
        "concat" conditioning): forward(x, t, concat=c) equals forward(cat([x, c], 1), t) without building the concat."""
        assert y is None, "must specify y if and only if the model is class-conditional"
        assert self.W is not None, "weights not loaded (load_state_dict / load_weights, then .cuda())"
        if not x.is_cuda:
            raise RuntimeError("sdb200.UNetModel runs on CUDA (sm_90a) only; there is no CPU fallback")
        cin = x.shape[1] + (0 if concat is None else concat.shape[1])
        assert x.dim() == 4 and cin == self.in_channels, (tuple(x.shape), self.in_channels)
        if concat is not None:
            assert not self.conditional, "concat conditioning with a spatial-transformer UNet is not supported"
            assert concat.dim() == 4 and concat.shape[0] == x.shape[0] and concat.shape[2:] == x.shape[2:], \
                (tuple(concat.shape), tuple(x.shape))
        self._check_context(context, x.shape[0])
        nb, _, H, Wd = x.shape
        lv = len(self.cfg["channel_mult"]) - 1
        assert H % (1 << lv) == 0 and Wd % (1 << lv) == 0, "latent size must be divisible by 2^(levels-1)"
        if not self.conditional:
            return self._forward_uncond(x, timesteps, concat)
        cached = self._context_cached(context)
        if self.use_cuda_graph:
            if not cached:
                self.set_context(context)
            g = self._graph_for(tuple(x.shape), self._ctx_kv, ctx_tokens=context.shape[1])
            assert g["kvs"] is self._ctx_kv or all(a[1].data_ptr() == b[1].data_ptr() for a, b in zip(g["kvs"], self._ctx_kv))
            if x.data_ptr() != g["x"].data_ptr():
                g["x"].copy_(x)
            g["t"].copy_(timesteps)
            g["graph"].replay()
            ops.add_graph_launches(g["launches"])
            # a fresh tensor, as the reference returns: callers may keep eps across evaluations (the reference's PLMS
            # history does when guidance is off, plms.py:159-162), the graph's static output buffer is overwritten
            return g["out"].clone() if x.dtype == torch.float32 else g["out"].to(x.dtype)
        kvs = self._ctx_kv if cached else self.context_kv(context)
        t = timesteps.to(torch.float32).contiguous()
        eps = self._forward_impl(x.contiguous().float(), t, kvs)
        return eps.to(x.dtype)

    def graph_inputs(self, shape, concat_shape=None):
        """Graph mode, no spatial transformer: the static x and conditioning buffers (the latter None without concat) of
        the graph captured for these shapes, capturing it first. A caller that writes its next input straight into them
        skips forward()'s copy. None in eager mode."""
        if not self.use_cuda_graph or self.conditional:
            return None
        g = self._graph_for(tuple(shape), None, None if concat_shape is None else tuple(concat_shape))
        return g["x"], g["c"]

    def _forward_uncond(self, x, timesteps, concat=None):
        if self.use_cuda_graph:
            g = self._graph_for(tuple(x.shape), None, None if concat is None else tuple(concat.shape))
            if x.data_ptr() != g["x"].data_ptr():
                g["x"].copy_(x)
            if concat is not None and concat.data_ptr() != g["c"].data_ptr():
                g["c"].copy_(concat)
            g["t"].copy_(timesteps)
            g["graph"].replay()
            ops.add_graph_launches(g["launches"])
            return g["out"].clone() if x.dtype == torch.float32 else g["out"].to(x.dtype)
        t = timesteps.to(torch.float32).contiguous()
        c = None if concat is None else concat.contiguous().float()
        return self._forward_impl(x.contiguous().float(), t, None, c).to(x.dtype)


class CUNet:
    """Owner of an sdb_unet handle (include/sdb200.h): the C plan, its CUDA graph and the memory pool holding every
    intermediate buffer of the recorded evaluation."""

    def __init__(self, handle, plan, pool, keep, n_launches):
        self.handle, self.plan, self.pool, self.keep, self.n_launches = handle, plan, pool, keep, n_launches
        self.x, self.t, self.eps = keep[0], keep[1], keep[2]

    def forward(self, x, t, out=None):
        """eps = UNet(x, t) through sdb_unet_forward on the current stream (x, t: fp32 cuda tensors)."""
        import ctypes as C
        from . import lib as _l
        lib = _l.load()
        if out is None:
            out = torch.empty_like(self.eps)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _l.check(lib.sdb_unet_forward(self.handle, C.c_void_p(x.data_ptr()), C.c_void_p(t.data_ptr()),
                                      C.c_void_p(out.data_ptr()), st), "sdb_unet_forward")
        return out

    def sample_plms(self, x_T, sampler, scale, guided=True):
        """Whole PLMS trajectory in C (sdb_sample_plms) with the schedule of an sdb200 PLMSSampler on which
        make_schedule() has been called. Returns (x_0 latent, pred_x0)."""
        import ctypes as C
        import numpy as np
        from . import lib as _l
        lib = _l.load()
        b = x_T.shape[0]
        rep = 2 if guided else 1
        per = x_T.numel()
        work = torch.empty((5 + 2 * rep) * per, dtype=torch.float32, device=x_T.device)
        x_out, p0 = torch.empty_like(x_T), torch.empty_like(x_T)
        arr = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.float32))
        ts, al, ap = arr(sampler.ddim_timesteps), arr(sampler.ddim_alphas), arr(sampler.ddim_alphas_prev)
        sq, sg = arr(sampler.ddim_sqrt_one_minus_alphas), arr(sampler.ddim_sigmas)
        fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
        d = _l.PlmsDesc()
        d.unet, d.x, d.x_out, d.pred_x0_out, d.work = self.handle, x_T.data_ptr(), x_out.data_ptr(), p0.data_ptr(), work.data_ptr()
        d.batch, d.n_steps, d.guided, d.scale = b, len(ts), 1 if guided else 0, float(scale)
        d.timesteps, d.alphas, d.alphas_prev, d.sqrt_one_minus_alphas, d.sigmas = fp(ts), fp(al), fp(ap), fp(sq), fp(sg)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _l.check(lib.sdb_sample_plms(C.byref(d), st), "sdb_sample_plms")
        torch.cuda.current_stream().synchronize()   # the host schedule arrays and `work` must outlive the enqueued work
        return x_out, p0

    def close(self):
        from . import lib as _l
        if self.handle is not None:
            lib = _l.load()
            lib.sdb_unet_destroy(self.handle)
            lib.sdb_plan_destroy(self.plan)
            self.handle = self.plan = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
