"""ORACLE: a fresh restatement of the pieces of taming-transformers' `taming.modules.losses.vqperceptual` that the
reference's LPIPSWithDiscriminator (ldm/modules/losses/contperceptual.py) star-imports: LPIPS (over torchvision's own
vgg16 features, weights from the state dict instead of a download), ScalingLayer, NetLinLayer, NLayerDiscriminator
(BatchNorm variant), weights_init, hinge_d_loss, vanilla_d_loss and adopt_weight. taming is not part of the reference,
so these are not pinned against taming itself; the VGG16 trunk is torchvision's, and contperceptual.py /
autoencoder.py run unmodified on top of them.
"""
from collections import namedtuple

import torch
import torch.nn as nn
import torch.nn.functional as F


def adopt_weight(weight, global_step, threshold=0, value=0.):
    if global_step < threshold:
        weight = value
    return weight


def hinge_d_loss(logits_real, logits_fake):
    return 0.5 * (torch.mean(F.relu(1. - logits_real)) + torch.mean(F.relu(1. + logits_fake)))


def vanilla_d_loss(logits_real, logits_fake):
    return 0.5 * (torch.mean(F.softplus(-logits_real)) + torch.mean(F.softplus(logits_fake)))


def weights_init(m):
    name = m.__class__.__name__
    if "Conv" in name:
        nn.init.normal_(m.weight.data, 0.0, 0.02)
    elif "BatchNorm" in name:
        nn.init.normal_(m.weight.data, 1.0, 0.02)
        nn.init.constant_(m.bias.data, 0)


class ScalingLayer(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.Tensor([-.030, -.088, -.188])[None, :, None, None])
        self.register_buffer("scale", torch.Tensor([.458, .450, .450])[None, :, None, None])

    def forward(self, inp):
        return (inp - self.shift) / self.scale


class NetLinLayer(nn.Module):
    def __init__(self, chn_in, chn_out=1, use_dropout=False):
        super().__init__()
        layers = [nn.Dropout()] if use_dropout else []
        layers += [nn.Conv2d(chn_in, chn_out, 1, stride=1, padding=0, bias=False)]
        self.model = nn.Sequential(*layers)


class VGG16Slices(nn.Module):
    """torchvision vgg16().features cut after relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3."""

    def __init__(self):
        super().__init__()
        from torchvision.models import vgg16
        feats = vgg16(weights=None).features
        bounds = [(0, 4), (4, 9), (9, 16), (16, 23), (23, 30)]
        for s, (lo, hi) in enumerate(bounds, 1):
            sl = nn.Sequential()
            for i in range(lo, hi):
                sl.add_module(str(i), feats[i])
            setattr(self, f"slice{s}", sl)
        for p in self.parameters():
            p.requires_grad = False

    def forward(self, x):
        outs = []
        h = x
        for s in range(1, 6):
            h = getattr(self, f"slice{s}")(h)
            outs.append(h)
        return namedtuple("VggOutputs", ["relu1_2", "relu2_2", "relu3_3", "relu4_3", "relu5_3"])(*outs)


def normalize_tensor(x, eps=1e-10):
    norm_factor = torch.sqrt(torch.sum(x ** 2, dim=1, keepdim=True))
    return x / (norm_factor + eps)


def spatial_average(x, keepdim=True):
    return x.mean([2, 3], keepdim=keepdim)


class LPIPS(nn.Module):
    def __init__(self, use_dropout=True):
        super().__init__()
        self.scaling_layer = ScalingLayer()
        self.chns = [64, 128, 256, 512, 512]
        self.net = VGG16Slices()
        for k, c in enumerate(self.chns):
            setattr(self, f"lin{k}", NetLinLayer(c, use_dropout=use_dropout))
        for p in self.parameters():
            p.requires_grad = False

    def forward(self, input, target):
        outs0 = self.net(self.scaling_layer(input))
        outs1 = self.net(self.scaling_layer(target))
        val = None
        for k in range(len(self.chns)):
            d = (normalize_tensor(outs0[k]) - normalize_tensor(outs1[k])) ** 2
            r = spatial_average(getattr(self, f"lin{k}").model(d), keepdim=True)
            val = r if val is None else val + r
        return val


class NLayerDiscriminator(nn.Module):
    def __init__(self, input_nc=3, ndf=64, n_layers=3, use_actnorm=False):
        super().__init__()
        assert not use_actnorm, "ActNorm is not restated"
        norm_layer = nn.BatchNorm2d
        kw, padw = 4, 1
        seq = [nn.Conv2d(input_nc, ndf, kernel_size=kw, stride=2, padding=padw), nn.LeakyReLU(0.2, True)]
        mult = 1
        for n in range(1, n_layers):
            prev, mult = mult, min(2 ** n, 8)
            seq += [nn.Conv2d(ndf * prev, ndf * mult, kernel_size=kw, stride=2, padding=padw, bias=False),
                    norm_layer(ndf * mult), nn.LeakyReLU(0.2, True)]
        prev, mult = mult, min(2 ** n_layers, 8)
        seq += [nn.Conv2d(ndf * prev, ndf * mult, kernel_size=kw, stride=1, padding=padw, bias=False),
                norm_layer(ndf * mult), nn.LeakyReLU(0.2, True)]
        seq += [nn.Conv2d(ndf * mult, 1, kernel_size=kw, stride=1, padding=padw)]
        self.main = nn.Sequential(*seq)

    def forward(self, input):
        return self.main(input)


EXPORTS = dict(LPIPS=LPIPS, ScalingLayer=ScalingLayer, NetLinLayer=NetLinLayer, NLayerDiscriminator=NLayerDiscriminator,
               weights_init=weights_init, hinge_d_loss=hinge_d_loss, vanilla_d_loss=vanilla_d_loss,
               adopt_weight=adopt_weight)


def install():
    """Stub taming.modules.losses.vqperceptual with these restatements (ref_harness's _stub mechanism)."""
    import ref_harness as R
    R._stub("taming.modules.losses.vqperceptual", **EXPORTS)
