"""Checkpoint ingest (SURVEY 8f-1): the reference's `load_model_from_config(config, ckpt)` (scripts/txt2img.py:49-66,
scripts/img2img.py:28-45) for the H100 engine — a `.ckpt` (pickled {"state_dict": ..., "global_step": ...}, what
`torch.save` of a Lightning checkpoint holds) or a `.safetensors` file with the reference key names goes through
`LatentDiffusion.load_state_dict(strict=False)`; `.cuda()` then packs the tensors into kernel-native fp16 layouts.

The config is the reference's YAML (`configs/stable-diffusion/v1-inference.yaml`) unchanged — its `target:` strings
are mapped onto sdb200 classes (util.TARGET_MAP) — given as a path, as a dict, or as anything with `.model`.
The safetensors container (8-byte little-endian header length, JSON header {name: {dtype, shape, data_offsets}},
raw little-endian tensor bytes) is parsed here directly; no third-party reader is needed.
"""
from __future__ import annotations

import json
import os
import struct

import numpy as np
import torch

from .util import instantiate_from_config, remap_config

_ST_DTYPES = {"F64": torch.float64, "F32": torch.float32, "F16": torch.float16, "BF16": torch.bfloat16,
              "I64": torch.int64, "I32": torch.int32, "I16": torch.int16, "I8": torch.int8, "U8": torch.uint8,
              "BOOL": torch.bool}
_ST_NAMES = {v: k for k, v in _ST_DTYPES.items()}


def read_safetensors(path):
    """{name: tensor} (host). Raises ValueError on a malformed container (bad header length, offsets out of range,
    byte count not matching dtype x shape)."""
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        head = f.read(8)
        if len(head) != 8:
            raise ValueError(f"{path}: not a safetensors file (shorter than 8 bytes)")
        (hlen,) = struct.unpack("<Q", head)
        if hlen > size - 8 or hlen > (100 << 20):
            raise ValueError(f"{path}: header length {hlen} exceeds the file")
        header = json.loads(f.read(hlen).decode("utf-8"))
    base = 8 + hlen
    raw = np.memmap(path, dtype=np.uint8, mode="r", offset=base) if size > base else np.zeros(0, np.uint8)
    out = {}
    for name, meta in header.items():
        if name == "__metadata__":
            continue
        if meta["dtype"] not in _ST_DTYPES:
            raise ValueError(f"{path}: tensor {name} has unsupported dtype {meta['dtype']}")
        dt = _ST_DTYPES[meta["dtype"]]
        lo, hi = meta["data_offsets"]
        shape = tuple(int(d) for d in meta["shape"])
        nbytes = int(np.prod(shape, dtype=np.int64)) * torch.empty(0, dtype=dt).element_size()
        if not (0 <= lo <= hi <= raw.shape[0]) or hi - lo != nbytes:
            raise ValueError(f"{path}: tensor {name}: offsets [{lo}, {hi}) do not hold {shape} x {meta['dtype']}")
        if nbytes == 0:
            out[name] = torch.empty(shape, dtype=dt)
            continue
        buf = torch.from_numpy(np.array(raw[lo:hi]))          # owned copy; the map is released with `raw`
        out[name] = buf.view(dt).reshape(shape)
    return out


def write_safetensors(path, tensors, metadata=None):
    """Inverse of read_safetensors (used by the tests and to convert a .ckpt once)."""
    header, blobs, off = {}, [], 0
    if metadata:
        header["__metadata__"] = {str(k): str(v) for k, v in metadata.items()}
    for name in sorted(tensors):
        t = tensors[name].detach().to("cpu").contiguous()
        b = t.reshape(-1).view(torch.uint8).numpy().tobytes() if t.numel() else b""
        header[name] = {"dtype": _ST_NAMES[t.dtype], "shape": list(t.shape), "data_offsets": [off, off + len(b)]}
        blobs.append(b)
        off += len(b)
    hjson = json.dumps(header, separators=(",", ":")).encode("utf-8")
    hjson += b" " * ((-len(hjson)) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(hjson)))
        f.write(hjson)
        for b in blobs:
            f.write(b)


def read_state_dict(path, allow_pickle=False):
    """(state_dict, info) from a .safetensors or a pickled .ckpt/.pt/.pth (txt2img.py:51-54).

    Pickled files are read with tensors-only unpickling (plus the few plain containers a Lightning checkpoint
    carries). Full unpickling executes arbitrary code from the file, so — unlike the reference's bare `torch.load` —
    it is an explicit opt-in: allow_pickle=True (CLI: --unsafe-ckpt), for files you trust."""
    if str(path).endswith(".safetensors"):
        return read_safetensors(path), {}
    try:
        pl_sd = torch.load(path, map_location="cpu", weights_only=True)
    except Exception as ex:   # noqa: BLE001
        if not allow_pickle:
            raise RuntimeError(
                f"{path} is not a tensors-only checkpoint ({type(ex).__name__}: {str(ex).splitlines()[0][:200]}). "
                "Full unpickling runs code from the file: pass allow_pickle=True / --unsafe-ckpt if you trust it, or "
                "convert it once with sdb200.checkpoint.write_safetensors.") from ex
        print(f"note: {path} is being fully unpickled (allow_pickle=True); load only checkpoints you trust")
        pl_sd = torch.load(path, map_location="cpu", weights_only=False)
    if isinstance(pl_sd, dict) and "state_dict" in pl_sd:
        return pl_sd["state_dict"], {k: pl_sd[k] for k in ("global_step", "epoch") if k in pl_sd}
    return pl_sd, {}


def load_config(config):
    """The `model:` node {target, params} of a reference YAML, from a path, a dict or an OmegaConf-like object."""
    if isinstance(config, (str, os.PathLike)):
        import yaml
        with open(config) as f:
            config = yaml.safe_load(f)
    node = config["model"] if (isinstance(config, dict) and "model" in config) else getattr(config, "model", config)
    if not isinstance(node, dict):
        try:
            from omegaconf import OmegaConf
            node = OmegaConf.to_container(node, resolve=True)
        except ImportError:
            node = dict(node)
    if "target" not in node:
        raise KeyError("Expected key `target` to instantiate.")
    return node


def load_model_from_config(config, ckpt, device="cuda", verbose=False, allow_pickle=False):
    """scripts/txt2img.py:49-66. Returns the model in eval mode on `device` (device=None: leave it on the host with the
    tensors adopted; `.cuda()` packs them later). Missing / unexpected keys are printed when verbose, as the
    reference does; EMA copies (`model_ema.*`) and training-only buffers in a full checkpoint are simply unexpected."""
    node = load_config(config)
    print(f"Loading model from {ckpt}")
    sd, info = read_state_dict(ckpt, allow_pickle=allow_pickle)
    if "global_step" in info:
        print(f"Global Step: {info['global_step']}")
    model = instantiate_from_config(remap_config(node))
    m, u = model.load_state_dict(sd, strict=False)
    schedule = ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod")
    hard = [k for k in m if k not in schedule]      # the schedule buffers are recomputed from the config
    if hard:
        raise RuntimeError(f"checkpoint {ckpt} lacks {len(hard)} tensors of the model, e.g. {hard[:3]}")
    if len(m) > 0 and verbose:
        print("missing keys:")
        print(m)
    if len(u) > 0 and verbose:
        print("unexpected keys:")
        print(u)
    if device is not None:
        model = model.to(device)
    model.eval()
    model.load_info = {"missing": list(m), "unexpected": list(u), **info}
    if "global_step" in info and hasattr(model, "global_step"):
        model.global_step = int(info["global_step"])
    return model


def load_first_stage_loss(model, config, ckpt, device="cuda", allow_pickle=False):
    """Build the training loss of a KL first stage from its YAML's `lossconfig` (ldm.modules.losses.
    LPIPSWithDiscriminator -> sdb200.ae_loss.LPIPSWithDiscriminator), load it from the checkpoint's `loss.*` tensors and
    attach it to `model` (an AutoencoderKL from load_model_from_config) for validation_step. A checkpoint without those
    tensors leaves the loss unloaded (`load_info["missing"]`), and validation_step then raises naming them. Returns the
    loss stage, in eval mode on `device`."""
    node = load_config(config)
    lc = node.get("params", {}).get("lossconfig")
    if not lc or "target" not in lc:
        raise KeyError(f"{node.get('target')}: the config has no lossconfig")
    loss = instantiate_from_config(remap_config(lc))
    sd, info = read_state_dict(ckpt, allow_pickle=allow_pickle)
    m, u = loss.load_state_dict({k[len("loss."):]: v for k, v in sd.items() if k.startswith("loss.")}, strict=False)
    if device is not None:
        loss = loss.to(device)
    loss.eval()
    loss.load_info = {"missing": ["loss." + k for k in m], "unexpected": ["loss." + k for k in u]}
    object.__setattr__(model, "loss", loss)    # not a submodule: the autoencoder's state dict is unchanged
    if "global_step" in info:
        model.global_step = int(info["global_step"])
    return loss
