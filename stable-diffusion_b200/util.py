"""Config plumbing with the reference's semantics (ldm/util.py:78-93): a node {target: "pkg.mod.Class",
params: {...}} is turned into an object. YAML files written for the reference work unchanged once the three
`target:` strings are pointed at sdb200 (see INTEGRATION.md)."""
import importlib


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
    "ldm.modules.encoders.modules.FrozenCLIPEmbedder": "sdb200.clip.FrozenCLIPEmbedder",
    "ldm.modules.encoders.modules.ClassEmbedder": "sdb200.encoders.ClassEmbedder",
    "ldm.modules.encoders.modules.BERTEmbedder": "sdb200.bert.BERTEmbedder",
    "ldm.modules.encoders.modules.SpatialRescaler": "sdb200.encoders.SpatialRescaler",
}


def remap_config(config):
    """Return a copy of {target, params} with a reference target replaced by its sdb200 counterpart."""
    if isinstance(config, dict) and config.get("target") in TARGET_MAP:
        c = dict(config)
        c["target"] = TARGET_MAP[config["target"]]
        return c
    return config


def adopt_state_dict(owner, state_dict, prefix, missing_keys, unexpected_keys, error_msgs, ignore=()):
    """Shared body of the stages' `_load_from_state_dict` (what nn.Module.load_state_dict calls per sub-module):
    take the tensors under `prefix` whose names are in owner.shapes, with nn.Module's reporting conventions — missing
    and unexpected names are listed, a shape mismatch is an error message (raised by load_state_dict). Returns the
    adopted {name: tensor} or None when something required is absent."""
    sub = {k[len(prefix):]: v for k, v in state_dict.items() if k.startswith(prefix)}
    missing = [k for k in owner.shapes if k not in sub]
    unexpected_keys.extend(prefix + k for k in sub if k not in owner.shapes and not k.startswith(tuple(ignore) or ("\0",)))
    if missing:
        missing_keys.extend(prefix + k for k in missing)
        return None
    bad = [k for k, shp in owner.shapes.items() if tuple(sub[k].shape) != tuple(shp)]
    if bad:
        error_msgs.extend(f"size mismatch for {prefix + k}: copying a param with shape {tuple(sub[k].shape)} from "
                          f"checkpoint, the shape in current model is {tuple(owner.shapes[k])}." for k in bad)
        return None
    return {k: sub[k] for k in owner.shapes}
