"""H100-native first-stage loss: drop-ins for taming's `LPIPS` (VGG16 trunk) and `NLayerDiscriminator`, and for
`ldm.modules.losses.LPIPSWithDiscriminator` (contperceptual.py), forward only, in eval mode, as Lightning's validation
runs them. State-dict keys follow taming's layout: `scaling_layer.{shift,scale}`, `net.slice{1..5}.<torchvision
features index>.{weight,bias}`, `lin{0..4}.model.1.weight` for LPIPS; `main.<index>.*` for the discriminator; `logvar`,
`perceptual_loss.*` and `discriminator.main.*` for the combined loss.

The convs run on the wgmma kernels (sdb_gemm) with ReLU / LeakyReLU(0.2) in the epilogue and fp16 activations between
layers: VGG's 3x3 convs as implicit GEMMs (conv1_1's 3 channels through im2col), the discriminator's 4x4 convs through
sdb_im2col. The LPIPS heads, max-pools, input scaling and every per-sample sum are the kernels of
include/sdb200_ae_loss.h; the per-sample -> batch combination is done on the host in fp64.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from . import ops
from .arch import random_state_dict as _random_sd
from .lib import ACT_LEAKY_RELU, ACT_RELU
from .util import PackedStage

# torchvision vgg16().features: (slice, index, c_in, c_out) of the 13 convs; a 2x2 max-pool precedes the first conv of
# slices 2-5, and the ReLU output of each slice's last conv is one LPIPS tap (relu1_2 .. relu5_3)
VGG16_CONVS = (("slice1", 0, 3, 64), ("slice1", 2, 64, 64),
               ("slice2", 5, 64, 128), ("slice2", 7, 128, 128),
               ("slice3", 10, 128, 256), ("slice3", 12, 256, 256), ("slice3", 14, 256, 256),
               ("slice4", 17, 256, 512), ("slice4", 19, 512, 512), ("slice4", 21, 512, 512),
               ("slice5", 24, 512, 512), ("slice5", 26, 512, 512), ("slice5", 28, 512, 512))
LPIPS_CHANNELS = (64, 128, 256, 512, 512)
LPIPS_SHIFT = (-0.030, -0.088, -0.188)   # taming lpips.py ScalingLayer
LPIPS_SCALE = (0.458, 0.450, 0.450)
LPIPS_MIN_SIDE = 16                      # four 2x2 pools leave one pixel
BN_EPS = 1e-5


def lpips_param_shapes():
    s = {"scaling_layer.shift": (1, 3, 1, 1), "scaling_layer.scale": (1, 3, 1, 1)}
    for sl, i, cin, cout in VGG16_CONVS:
        s[f"net.{sl}.{i}.weight"] = (cout, cin, 3, 3)
        s[f"net.{sl}.{i}.bias"] = (cout,)
    for k, c in enumerate(LPIPS_CHANNELS):
        s[f"lin{k}.model.1.weight"] = (1, c, 1, 1)
    return s


def discriminator_layers(input_nc=3, ndf=64, n_layers=3):
    """NLayerDiscriminator's convs (taming discriminator/model.py): (index in `main`, c_in, c_out, stride, has_bias,
    BatchNorm index or None, LeakyReLU after)."""
    out = [(0, input_nc, ndf, 2, True, None, True)]
    idx, mult = 2, 1
    for n in range(1, n_layers):
        prev, mult = mult, min(2 ** n, 8)
        out.append((idx, ndf * prev, ndf * mult, 2, False, idx + 1, True))
        idx += 3
    prev, mult = mult, min(2 ** n_layers, 8)
    out.append((idx, ndf * prev, ndf * mult, 1, False, idx + 1, True))
    out.append((idx + 3, ndf * mult, 1, 1, True, None, False))
    return out


def discriminator_param_shapes(input_nc=3, ndf=64, n_layers=3):
    s = {}
    for i, cin, cout, _, bias, bn, _ in discriminator_layers(input_nc, ndf, n_layers):
        s[f"main.{i}.weight"] = (cout, cin, 4, 4)
        if bias:
            s[f"main.{i}.bias"] = (cout,)
        if bn is not None:
            for k in ("weight", "bias", "running_mean", "running_var"):
                s[f"main.{bn}.{k}"] = (cout,)
            s[f"main.{bn}.num_batches_tracked"] = ()
    return s


def loss_param_shapes(disc_num_layers=3, disc_in_channels=3):
    """The state dict of LPIPSWithDiscriminator (the `loss.*` tensors of a KL first-stage checkpoint)."""
    s = {"logvar": ()}
    s.update({"perceptual_loss." + k: v for k, v in lpips_param_shapes().items()})
    s.update({"discriminator." + k: v
              for k, v in discriminator_param_shapes(disc_in_channels, 64, disc_num_layers).items()})
    return s


def random_loss_state_dict(shapes, seed, logvar=0.0):
    """Seeded stand-in loss weights (arch.random_state_dict) with the values that must not be random: LPIPS's scaling
    constants, logvar, BatchNorm running statistics (variance 0.5 .. 1.5) and num_batches_tracked 0; the lin heads are
    non-negative, as LPIPS's trained heads are."""
    sd = _random_sd({k: v for k, v in shapes.items() if not k.endswith("num_batches_tracked")}, seed)
    g = torch.Generator().manual_seed(seed)
    for k, shp in shapes.items():
        if k.endswith("scaling_layer.shift"):
            sd[k] = torch.tensor(LPIPS_SHIFT).view(shp)
        elif k.endswith("scaling_layer.scale"):
            sd[k] = torch.tensor(LPIPS_SCALE).view(shp)
        elif k == "logvar":
            sd[k] = torch.tensor(float(logvar))
        elif k.endswith("running_mean"):
            sd[k] = 0.1 * torch.randn(shp, generator=g)
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(shp, generator=g)
        elif k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(0, dtype=torch.int64)
        elif ".model.1.weight" in k:
            sd[k] = sd[k].abs()
        elif ".weight" in k and len(shp) == 1:     # BatchNorm gain
            sd[k] = 1.0 + 0.02 * torch.randn(shp, generator=g)
    return {k: sd[k] for k in shapes}


def _pack_conv_padk(w, kpad):
    """[c_out, c_in, k, k] -> fp16 [c_out, kpad], column (ky * k + kx) * c_in + c (the im2col order), zero tail."""
    p = torch.zeros((w.shape[0], kpad), dtype=torch.float16, device=w.device)
    p[:, : w[0].numel()] = w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).half()
    return p


def _pack_conv3(w):
    """[c_out, c_in, 3, 3] -> fp16 [c_out, 9 * c_in], k = (ky * 3 + kx) * c_in + c (the implicit GEMM's taps = 9)."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous().half()


def _kpad(k):
    return (k + 63) // 64 * 64


def _check_images(in0, in1, what):
    for t, n in ((in0, "in0"), (in1, "in1")):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dim() == 4 and t.shape[1] == 3):
            raise ValueError(f"{what}: {n} must be a CUDA NCHW tensor with 3 channels, got "
                             f"{tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__}")
    if in0.shape != in1.shape:
        raise ValueError(f"{what}: the two image batches differ in shape: {tuple(in0.shape)} vs {tuple(in1.shape)}")
    if in0.shape[0] < 1:
        raise ValueError(f"{what}: empty batch")


class LPIPS(PackedStage):
    """taming.modules.losses.lpips.LPIPS: forward(in0, in1) -> [B, 1, 1, 1], images in [-1, 1]. Sides of at least 16
    pixels (four 2x2 pools leave one); non-square sizes work. Dropout in front of the lin heads is identity (eval)."""

    def __init__(self, use_dropout=True):
        super().__init__()
        self.shapes = lpips_param_shapes()

    @torch.no_grad()
    def pack_weights(self, device):
        sd = {k: v.detach().to(device=device, dtype=torch.float32) for k, v in self._host_sd.items()}
        W = {"device": device, "shift": sd["scaling_layer.shift"].reshape(3).contiguous(),
             "scale": sd["scaling_layer.scale"].reshape(3).contiguous(), "convs": []}
        for sl, i, cin, _ in VGG16_CONVS:
            w = sd[f"net.{sl}.{i}.weight"]
            W["convs"].append({"w": _pack_conv_padk(w, _kpad(9 * cin)) if cin % 64 else _pack_conv3(w),
                               "b": sd[f"net.{sl}.{i}.bias"].contiguous(), "pool": i in (5, 10, 17, 24),
                               "tap": i in (2, 7, 14, 21, 28)})
        W["lin"] = [sd[f"lin{k}.model.1.weight"].reshape(-1).contiguous() for k in range(5)]
        self.W = W

    @staticmethod
    def check_inputs(in0, in1):
        """Raises ValueError, before any launch, for inputs LPIPS cannot take."""
        _check_images(in0, in1, "LPIPS")
        h, w = in0.shape[2], in0.shape[3]
        if min(h, w) < LPIPS_MIN_SIDE:
            raise ValueError(f"LPIPS needs image sides of at least {LPIPS_MIN_SIDE} pixels (four 2x2 max-pools), "
                             f"got {h}x{w}")

    @torch.no_grad()
    def forward(self, in0, in1):
        self.check_inputs(in0, in1)
        assert self.W is not None, "sdb200.LPIPS: no weights (load a state dict and move it to CUDA)"
        W = self.W
        nb, _, H, Wd = in0.shape
        x = ops.lpips_scale(in0.contiguous().float(), in1.contiguous().float(), W["shift"], W["scale"])
        acc = torch.empty(nb, dtype=torch.float64, device=in0.device)
        out = torch.empty(nb, dtype=torch.float32, device=in0.device)
        h = None
        tap = 0
        for j, c in enumerate(W["convs"]):
            if j == 0:      # 3 input channels: explicit im2col into the padded-K operand
                col = ops.im2col3x3(x, 1, 1, H, Wd, c["w"].shape[1])
                h, _ = ops.gemm(col, c["w"], bias=c["b"], act=ACT_RELU, want_f16=True, splits=1)
                h = h.view(2 * nb, H, Wd, -1)
            else:
                if c["pool"]:
                    h = ops.maxpool2x2(h)
                n2, hh, ww, _ = h.shape
                # no split-K (splits=1, which also bypasses the autotuner): each output's K order is then fixed by
                # the layer alone, so a sample's LPIPS is the same bits alone and inside a batch
                h, _ = ops.gemm(h, c["w"], taps=9, bias=c["b"], act=ACT_RELU, want_f16=True, splits=1)
                h = h.view(n2, hh, ww, -1)
            if c["tap"]:
                ops.lpips_head(h, W["lin"][tap], acc, first=tap == 0, out=out if tap == 4 else None)
                tap += 1
        return out.view(nb, 1, 1, 1)


def discriminator_out_size(h, w, n_layers=3):
    """Logit map size of NLayerDiscriminator on an h x w image: n_layers stride-2 convs, then two stride-1 convs (4x4,
    pad 1)."""
    for _ in range(n_layers):
        h, w = (h + 2 - 4) // 2 + 1, (w + 2 - 4) // 2 + 1
    return h - 2, w - 2


class NLayerDiscriminator(PackedStage):
    """taming's PatchGAN discriminator (BatchNorm, eval: running statistics folded into the conv). forward(x) ->
    logits [B, 1, h', w']."""

    def __init__(self, input_nc=3, ndf=64, n_layers=3, use_actnorm=False):
        super().__init__()
        if use_actnorm:
            raise NotImplementedError("NLayerDiscriminator with ActNorm (use_actnorm=True)")
        self.layers = discriminator_layers(input_nc, ndf, n_layers)
        self.n_layers = n_layers
        self.shapes = discriminator_param_shapes(input_nc, ndf, n_layers)

    @torch.no_grad()
    def pack_weights(self, device):
        sd = {k: v.detach().to(device=device, dtype=torch.float32) for k, v in self._host_sd.items()
              if not k.endswith("num_batches_tracked")}
        convs = []
        for i, cin, cout, stride, has_bias, bn, lrelu in self.layers:
            w = sd[f"main.{i}.weight"]
            b = sd[f"main.{i}.bias"] if has_bias else torch.zeros(cout, device=device)
            if bn is not None:
                # eval BatchNorm folded into the conv: s = gamma / sqrt(var + eps), w' = s w, b' = beta + s (b - mean).
                # w' is rounded to fp16 once, as w would be, so the fold adds one fp32 rounding per weight and bias
                # (<= 2^-24 relative) to the fp16 operand rounding (2^-11) that the unfolded conv has anyway.
                s = sd[f"main.{bn}.weight"] / torch.sqrt(sd[f"main.{bn}.running_var"] + BN_EPS)
                w = w * s.view(-1, 1, 1, 1)
                b = sd[f"main.{bn}.bias"] + s * (b - sd[f"main.{bn}.running_mean"])
            if cout == 1:
                # the 512 -> 1 logit conv: the GEMM with its one output column padded to the narrowest tile (32);
                # the activation read dominates, and the padding only adds MMA work the tensor cores hide
                w = torch.cat([w, torch.zeros((31,) + tuple(w.shape[1:]), device=device)])
                b = torch.cat([b, torch.zeros(31, device=device)])
            convs.append({"w": _pack_conv_padk(w, _kpad(16 * cin)), "b": b.contiguous(), "stride": stride,
                          "act": ACT_LEAKY_RELU if lrelu else 0, "cout": cout})
        self.W = {"device": device, "convs": convs}

    def check_input(self, x, what="NLayerDiscriminator"):
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dim() == 4 and x.shape[1] == self.layers[0][1]):
            raise ValueError(f"{what}: need a CUDA NCHW tensor with {self.layers[0][1]} channels, got "
                             f"{tuple(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__}")
        ho, wo = discriminator_out_size(x.shape[2], x.shape[3], self.n_layers)
        if ho < 1 or wo < 1:
            raise ValueError(f"{what}: a {x.shape[2]}x{x.shape[3]} image leaves no logit after the discriminator's "
                             f"{self.n_layers + 2} 4x4 convs")

    @torch.no_grad()
    def logits_rows(self, x):
        """The logits as the GEMM writes them: fp32 [B * h' * w', 32], logit in column 0; and (h', w')."""
        self.check_input(x)
        assert self.W is not None, "sdb200.NLayerDiscriminator: no weights (load a state dict and move it to CUDA)"
        nb = x.shape[0]
        _, h = ops.nchw_to_nhwc(x.contiguous().float(), want_f32=False, want_f16=True)
        for c in self.W["convs"]:
            col, ho, wo = ops.im2col(h, 4, c["stride"], 1, c["w"].shape[1])
            if c["cout"] == 1:
                _, o = ops.gemm(col, c["w"], bias=c["b"], want_f32=True, splits=1)
                return o, (ho, wo)
            h, _ = ops.gemm(col, c["w"], bias=c["b"], act=c["act"], want_f16=True, splits=1)
            h = h.view(nb, ho, wo, c["cout"])

    def forward(self, x):
        o, (ho, wo) = self.logits_rows(x)
        return o[:, 0].reshape(x.shape[0], 1, ho, wo)


def adopt_weight(weight, global_step, threshold=0, value=0.0):
    return value if global_step < threshold else weight


class LPIPSWithDiscriminator(PackedStage):
    """ldm.modules.losses.contperceptual.LPIPSWithDiscriminator, forward only in eval mode. d_weight is 0, which is
    what the reference reaches under Lightning's no-grad validation (the autograd.grad RuntimeError branch)."""

    drop_prefixes = ("perceptual_loss.", "discriminator.")   # loaded by the two sub-stages

    def __init__(self, disc_start, logvar_init=0.0, kl_weight=1.0, pixelloss_weight=1.0, disc_num_layers=3,
                 disc_in_channels=3, disc_factor=1.0, disc_weight=1.0, perceptual_weight=1.0, use_actnorm=False,
                 disc_conditional=False, disc_loss="hinge"):
        super().__init__()
        assert disc_loss in ["hinge", "vanilla"]
        if use_actnorm:
            raise NotImplementedError("LPIPSWithDiscriminator with ActNorm (use_actnorm=True)")
        if disc_conditional:
            raise NotImplementedError("LPIPSWithDiscriminator with a conditional discriminator (disc_conditional=True)")
        self.kl_weight = kl_weight
        self.pixel_weight = pixelloss_weight
        self.perceptual_loss = LPIPS().eval()
        self.perceptual_weight = perceptual_weight
        self.logvar_init = float(logvar_init)
        self.discriminator = NLayerDiscriminator(input_nc=disc_in_channels, n_layers=disc_num_layers)
        self.discriminator_iter_start = disc_start
        self.disc_loss = disc_loss
        self.disc_factor = disc_factor
        self.discriminator_weight = disc_weight
        self.disc_conditional = disc_conditional
        self.shapes = {"logvar": ()}

    def pack_weights(self, device):
        self.W = {"device": device}

    @property
    def logvar(self):
        return float(self._host_sd["logvar"]) if self._host_sd is not None else None

    def missing_keys(self):
        """The state-dict keys this loss still lacks ([] once every weight is loaded)."""
        out = [] if self._host_sd is not None else ["logvar"]
        for pre, m in (("perceptual_loss.", self.perceptual_loss), ("discriminator.", self.discriminator)):
            if m._host_sd is None:
                out += [pre + k for k in m.shapes]
        return out

    def _check(self, inputs, reconstructions, posteriors, optimizer_idx, cond, weights):
        if self.training:
            raise NotImplementedError("LPIPSWithDiscriminator runs in eval mode only (no gradients, d_weight 0): "
                                      "call .eval()")
        if weights is not None:
            raise NotImplementedError("LPIPSWithDiscriminator with per-pixel weights")
        if cond is not None:
            raise NotImplementedError("LPIPSWithDiscriminator with a conditional discriminator (cond)")
        if optimizer_idx not in (0, 1):
            raise ValueError(f"optimizer_idx must be 0 or 1, got {optimizer_idx}")
        missing = self.missing_keys()
        if missing:
            raise RuntimeError(f"LPIPSWithDiscriminator has no weights for {len(missing)} keys, e.g. {missing[:4]}")
        _check_images(inputs, reconstructions, "LPIPSWithDiscriminator")
        if optimizer_idx == 0:
            if self.perceptual_weight > 0:
                LPIPS.check_inputs(inputs, reconstructions)
            if posteriors.nb != inputs.shape[0]:
                raise ValueError(f"posterior batch {posteriors.nb} != image batch {inputs.shape[0]}")
        self.discriminator.check_input(reconstructions, "LPIPSWithDiscriminator")

    @torch.no_grad()
    def terms(self, inputs, reconstructions, posteriors, want):
        """Per-sample fp64 sums on the host: "abs" sum |x - xrec|, "p" LPIPS (fp32 value), "kl", "fake" / "real" the
        five logit sums [5, B] of sdb_ae_loss_terms, and the logit count per sample "n_logits"."""
        x = inputs.contiguous().float()
        xr = reconstructions.contiguous().float()
        out = {}
        if "abs" in want:
            out["abs"] = ops.ae_loss_terms(x, "abs", b=xr)[0]
            out["p"] = (self.perceptual_loss(x, xr).view(-1).double() if self.perceptual_weight > 0
                        else torch.zeros(x.shape[0], dtype=torch.float64, device=x.device))
            out["kl"] = posteriors.kl_sums()
        for name, img in (("fake", xr), ("real", x)):
            if name in want:
                o, (ho, wo) = self.discriminator.logits_rows(img)
                out[name] = ops.ae_loss_terms(o, "logits", n=ho * wo, cc=o.shape[1])
                out["n_logits"] = ho * wo
        return {k: (v.cpu() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}, x

    def combine(self, t, x, optimizer_idx, global_step, split="train"):
        """The reference's (loss, log) from the per-sample sums `t` (contperceptual.py:47-119)."""
        dev = x.device
        nb, n = x.shape[0], x[0].numel()
        f32 = lambda v: torch.tensor(float(v), dtype=torch.float32, device=dev)
        disc_factor = adopt_weight(self.disc_factor, global_step, threshold=self.discriminator_iter_start)
        nl = nb * t["n_logits"]
        if optimizer_idx == 0:
            lv = self.logvar
            rec_sum = float(t["abs"].sum()) + self.perceptual_weight * n * float(t["p"].sum())
            nll = (rec_sum / math.exp(lv) + lv * nb * n) / nb
            kl = float(t["kl"].sum()) / nb
            g_loss = -float(t["fake"][0].sum()) / nl
            d_weight = 0.0
            loss = nll + self.kl_weight * kl + d_weight * disc_factor * g_loss
            log = {f"{split}/total_loss": f32(loss), f"{split}/logvar": f32(lv), f"{split}/kl_loss": f32(kl),
                   f"{split}/nll_loss": f32(nll), f"{split}/rec_loss": f32(rec_sum / (nb * n)),
                   f"{split}/d_weight": torch.tensor(d_weight), f"{split}/disc_factor": torch.tensor(disc_factor),
                   f"{split}/g_loss": f32(g_loss)}
            return f32(loss), log
        real, fake = t["real"], t["fake"]
        if self.disc_loss == "hinge":
            d = 0.5 * (float(real[1].sum()) / nl + float(fake[2].sum()) / nl)
        else:
            d = 0.5 * (float(real[3].sum()) / nl + float(fake[4].sum()) / nl)
        d_loss = disc_factor * d
        log = {f"{split}/disc_loss": f32(d_loss), f"{split}/logits_real": f32(float(real[0].sum()) / nl),
               f"{split}/logits_fake": f32(float(fake[0].sum()) / nl)}
        return f32(d_loss), log

    def forward(self, inputs, reconstructions, posteriors, optimizer_idx, global_step, last_layer=None, cond=None,
                split="train", weights=None):
        self._check(inputs, reconstructions, posteriors, optimizer_idx, cond, weights)
        want = ("abs", "fake") if optimizer_idx == 0 else ("real", "fake")
        t, x = self.terms(inputs, reconstructions, posteriors, want)
        return self.combine(t, x, optimizer_idx, global_step, split)
