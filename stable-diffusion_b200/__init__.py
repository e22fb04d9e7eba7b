"""sdb200 — Hopper-native (sm_90a) kernels and host mirror for the CompVis/stable-diffusion denoising loop.

The directory name carries a hyphen (as the project layout prescribes); import it through the `sdb200`
alias module at the repo root, or `importlib.import_module("stable-diffusion_b200")`.
"""
__version__ = "0.1.0"

import sys as _sys

from . import ae_loss, arch, bert, checkpoint, clip, clip_image, diffusion, dist, encoders, lib, ops, pipeline, retrieval, safety, samplers, tokenizer, unet, util, vae, vq  # noqa: E402,F401
from .ae_loss import LPIPS, LPIPSWithDiscriminator, NLayerDiscriminator  # noqa: E402,F401
from .bert import BERTEmbedder  # noqa: E402,F401
from .clip import FrozenCLIPEmbedder, FrozenCLIPTextEmbedder  # noqa: E402,F401
from .clip_image import FrozenClipImageEmbedder  # noqa: E402,F401
from .diffusion import LatentDiffusion  # noqa: E402,F401
from .encoders import ClassEmbedder, SpatialRescaler  # noqa: E402,F401
from .safety import StableDiffusionSafetyChecker  # noqa: E402,F401
from .samplers import DDIMSampler, DPMSolverSampler, PLMSSampler  # noqa: E402,F401
from .unet import UNetModel  # noqa: E402,F401
from .vae import AutoencoderKL  # noqa: E402,F401
from .vq import VQModel, VQModelInterface  # noqa: E402,F401


def _alias_submodules():
    """Make `sdb200.X` and `stable-diffusion_b200.X` the same module objects."""
    pre = __name__ + "."
    for name, mod in list(_sys.modules.items()):
        if name.startswith(pre):
            _sys.modules.setdefault("sdb200." + name[len(pre):], mod)


_alias_submodules()
