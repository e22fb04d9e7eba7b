"""ORACLE tooling (build container only): import the UNMODIFIED reference from /root/reference on CPU.

Nothing from the reference is copied or edited; third-party imports that are absent here are stubbed
(SURVEY.md Appendix E): omegaconf.listconfig.ListConfig (type check at openaimodel.py:476-478),
pytorch_lightning.LightningModule (= nn.Module + .device; ddpm.py:44, autoencoder.py:14), taming VectorQuantizer2
(autoencoder.py:6) and `clip` / `kornia` (imported by ldm/modules/encoders/modules.py, used only by the CLIP
embedders). The quantizer the reference imports (ldm.models.autoencoder.VectorQuantizer) is then set to
oracle/vq_oracle.py's restatement of taming's. The samplers' register_buffer forces .to("cuda")
(plms.py:18-22, ddim.py:19-23) and is patched to a plain setattr for CPU runs.

Also the pieces every golden generator shares: the reference's model builders, `gen` (seeded inputs), `rel` (the
oracle error they print) and `load_ema`.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys
import types

import torch
import torch.nn as nn

REF = os.environ.get("SD_REFERENCE", "/root/reference")


def available() -> bool:
    return os.path.isdir(os.path.join(REF, "ldm"))


def _stub(name, **attrs):
    parts = name.split(".")
    for i in range(1, len(parts) + 1):
        n = ".".join(parts[:i])
        if n not in sys.modules:
            m = types.ModuleType(n)
            m.__path__ = []
            sys.modules[n] = m
            if i > 1:
                setattr(sys.modules[".".join(parts[:i - 1])], parts[i - 1], m)
    for k, v in attrs.items():
        setattr(sys.modules[name], k, v)


_done = False


def install():
    global _done
    if _done:
        return
    if not available():
        raise RuntimeError(f"reference not found at {REF}")

    class ListConfig(list):
        pass

    class LightningModule(nn.Module):
        @property
        def device(self):
            return next(self.parameters()).device

        def log(self, *a, **k):
            pass

        def log_dict(self, *a, **k):
            pass

    _stub("omegaconf", ListConfig=ListConfig, OmegaConf=object)
    _stub("omegaconf.listconfig", ListConfig=ListConfig)
    _stub("pytorch_lightning", LightningModule=LightningModule, seed_everything=lambda s: torch.manual_seed(s))
    _stub("pytorch_lightning.utilities")
    _stub("pytorch_lightning.utilities.distributed", rank_zero_only=lambda f: f)
    _stub("taming")
    _stub("taming.modules")
    _stub("taming.modules.vqvae")
    _stub("taming.modules.vqvae.quantize", VectorQuantizer2=object)
    _stub("clip")
    _stub("kornia")
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import ldm.models.autoencoder as ae
    import vq_oracle
    ae.VectorQuantizer = vq_oracle.VectorQuantizer2
    _done = True


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def gen(shape, seed, scale=1.0):
    return scale * torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def build_unet(cfg):
    install()
    from ldm.modules.diffusionmodules.openaimodel import UNetModel
    return UNetModel(**cfg).eval()


def build_vae(cfg):
    install()
    from ldm.models.autoencoder import AutoencoderKL
    with contextlib.redirect_stdout(io.StringIO()):
        m = AutoencoderKL(ddconfig=cfg["ddconfig"], lossconfig={"target": "torch.nn.Identity"},
                          embed_dim=cfg["embed_dim"])
    return m.eval()


def build_vq(cfg):
    install()
    from ldm.models.autoencoder import VQModelInterface
    with contextlib.redirect_stdout(io.StringIO()):
        m = VQModelInterface(embed_dim=cfg["embed_dim"], n_embed=cfg["n_embed"], ddconfig=cfg["ddconfig"],
                             lossconfig={"target": "torch.nn.Identity"})
    return m.eval()


def build_samplers(model):
    install()
    from ldm.models.diffusion.ddim import DDIMSampler
    from ldm.models.diffusion.plms import PLMSSampler
    PLMSSampler.register_buffer = lambda s, n, a: setattr(s, n, a)
    DDIMSampler.register_buffer = lambda s, n, a: setattr(s, n, a)
    return PLMSSampler(model), DDIMSampler(model)


def build_ld(unet_cfg, first_stage_cfg, cond_stage_config, **params):
    """The reference's LatentDiffusion (ddpm.py:424-), assembled by its own instantiate_from_config from a config's
    `model.params`: `params` are the top-level keys (image_size and channels default to the UNet's image_size and
    in_channels), the UNet node is `unet_cfg`, and the first stage is VQModelInterface when the arch config
    `first_stage_cfg` has `n_embed`, AutoencoderKL otherwise, with the training loss replaced by torch.nn.Identity."""
    install()
    from ldm.models.diffusion.ddpm import LatentDiffusion
    kind = "VQModelInterface" if "n_embed" in first_stage_cfg else "AutoencoderKL"
    params = {"image_size": unet_cfg["image_size"], "channels": unet_cfg["in_channels"], **params}
    with contextlib.redirect_stdout(io.StringIO()):
        m = LatentDiffusion(
            first_stage_config={"target": "ldm.models.autoencoder." + kind,
                                "params": {**first_stage_cfg, "monitor": "val/rec_loss",
                                           "lossconfig": {"target": "torch.nn.Identity"}}},
            cond_stage_config=cond_stage_config,
            unet_config={"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": dict(unet_cfg)},
            **params)
    return m.eval()


def load_ema(ld, sd):
    """Copy a UNet state dict into `ld.model_ema`'s buffers (LitEma names them by the parameter path without dots,
    ema.py:19), so ema_scope() switches to these weights."""
    bufs = dict(ld.model_ema.named_buffers())
    for k, v in sd.items():
        bufs[("diffusion_model." + k).replace(".", "")].copy_(v)
