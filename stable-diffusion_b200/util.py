"""Config plumbing with the reference's semantics (ldm/util.py:78-93): a node {target: "pkg.mod.Class",
params: {...}} is turned into an object. YAML files written for the reference work unchanged once the three
`target:` strings are pointed at sdb200 (see INTEGRATION.md). PackedStage is the weight plumbing every stage shares."""
import importlib

import torch
import torch.nn as nn


def get_obj_from_str(string, reload=False):
    module, cls = string.rsplit(".", 1)
    if reload:
        importlib.reload(importlib.import_module(module))
    return getattr(importlib.import_module(module, package=None), cls)


def instantiate_from_config(config):
    if "target" not in config:
        if config == "__is_first_stage__" or config == "__is_unconditional__":
            return None
        raise KeyError("Expected key `target` to instantiate.")
    return get_obj_from_str(config["target"])(**config.get("params", dict()))


# reference targets -> sdb200 engine classes (used by LatentDiffusion when handed an unmodified reference config)
TARGET_MAP = {
    "ldm.models.diffusion.ddpm.LatentDiffusion": "sdb200.diffusion.LatentDiffusion",
    "ldm.modules.diffusionmodules.openaimodel.UNetModel": "sdb200.unet.UNetModel",
    "ldm.models.autoencoder.AutoencoderKL": "sdb200.vae.AutoencoderKL",
    "ldm.models.autoencoder.VQModelInterface": "sdb200.vq.VQModelInterface",
    "ldm.models.autoencoder.VQModel": "sdb200.vq.VQModel",
    "ldm.modules.encoders.modules.FrozenCLIPEmbedder": "sdb200.clip.FrozenCLIPEmbedder",
    "ldm.modules.encoders.modules.FrozenCLIPTextEmbedder": "sdb200.clip.FrozenCLIPTextEmbedder",
    "ldm.modules.encoders.modules.FrozenClipImageEmbedder": "sdb200.clip_image.FrozenClipImageEmbedder",
    "ldm.modules.encoders.modules.ClassEmbedder": "sdb200.encoders.ClassEmbedder",
    "ldm.modules.encoders.modules.BERTEmbedder": "sdb200.bert.BERTEmbedder",
    "ldm.modules.encoders.modules.SpatialRescaler": "sdb200.encoders.SpatialRescaler",
    "ldm.modules.losses.LPIPSWithDiscriminator": "sdb200.ae_loss.LPIPSWithDiscriminator",
    "ldm.modules.losses.contperceptual.LPIPSWithDiscriminator": "sdb200.ae_loss.LPIPSWithDiscriminator",
}


def remap_config(config):
    """Return a copy of {target, params} with a reference target replaced by its sdb200 counterpart."""
    if isinstance(config, dict) and config.get("target") in TARGET_MAP:
        c = dict(config)
        c["target"] = TARGET_MAP[config["target"]]
        return c
    return config


class PackedStage(nn.Module):
    """Base of the engine's stages, which hold no nn parameters: the host tensors of the checkpoint keys in `shapes`
    ({name: shape}) are kept in `_host_sd` and packed into kernel-native layouts `W` ({"device": ..., ...}) on the
    device the stage is moved to. A subclass sets `shapes` and implements `pack_weights(device)`."""

    W = None
    _host_sd = None
    drop_prefixes = ()   # checkpoint keys under the stage that are not weights of the stage: dropped, not reported

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        self._adopt(state_dict, prefix, missing_keys, unexpected_keys, error_msgs)

    def _adopt(self, state_dict, prefix, missing_keys, unexpected_keys, error_msgs):
        """Take the tensors under `prefix` whose names are in `shapes`, with nn.Module's reporting conventions: missing
        and unexpected names are listed, a shape mismatch is an error message (raised by load_state_dict). Nothing is
        adopted when something required is absent; adopted weights are repacked when the stage is already packed."""
        sub = {k[len(prefix):]: v for k, v in state_dict.items() if k.startswith(prefix)}
        missing = [k for k in self.shapes if k not in sub]
        unexpected_keys.extend(prefix + k for k in sub if k not in self.shapes and not k.startswith(self.drop_prefixes))
        if missing:
            missing_keys.extend(prefix + k for k in missing)
            return
        bad = [k for k, shp in self.shapes.items() if tuple(sub[k].shape) != tuple(shp)]
        if bad:
            error_msgs.extend(f"size mismatch for {prefix + k}: copying a param with shape {tuple(sub[k].shape)} from "
                              f"checkpoint, the shape in current model is {tuple(self.shapes[k])}." for k in bad)
            return
        self._host_sd = {k: sub[k] for k in self.shapes}
        if self.W is not None:
            self.pack_weights(self.W["device"])

    def _checked(self, sd, what="weights"):
        """The tensors of `shapes` from the mapping sd; AssertionError if one is missing or misshapen."""
        for k, shape in self.shapes.items():
            assert k in sd and tuple(sd[k].shape) == tuple(shape), f"{what}: {k} missing or misshapen"
        return {k: sd[k] for k in self.shapes}

    def load_weights(self, sd, device):
        """sd: a state dict of the stage's own keys (reference names); packs on `device`."""
        self._host_sd = self._checked(sd)
        self.pack_weights(torch.device(device))
        return self

    def _apply(self, fn, *a, **k):  # .cuda() / .to(device) packs, like moving an nn.Module's parameters
        r = super()._apply(fn, *a, **k)
        probe = fn(torch.empty(0))
        if probe.is_cuda and self._host_sd is not None and (self.W is None or self.W["device"] != probe.device):
            self.pack_weights(probe.device)
        return r
