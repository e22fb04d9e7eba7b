"""Golden data for the forward denoising objective (tests/golden/losses.pt): the unmodified reference's
LatentDiffusion.p_losses (ddpm.py:1012-1045), its lvlb_weights / logvar buffers (:158-169, :87-89) and get_input
(:654-705), on five tiny members that cover every conditioning path and both loss types:

  sd        crossattn on a given context, l2, KL first stage with 4 latent channels (v1-inference.yaml parameters)
  lsun      unconditional, l1, scale_by_std (lsun_churches-ldm-kl-8.yaml parameters)
  cin       class_label through ClassEmbedder (cond_stage_trainable), VQ first stage (cin256-v2.yaml parameters)
  semantic  segmentation through SpatialRescaler, concat, l1 (semantic_synthesis256.yaml parameters)
  bsr       LR_image concatenated as it is, l2 (bsr_sr.yaml parameters; no split path at the tiny size)

Per member: the model node (reference targets, so the engine builds the same model from it), the cond stage's
parameter shapes (its weights are arch.random_state_dict of them at COND_SEED), x_start, cond, one distinct t per
sample including 0 and T-1, noise, x_noisy, the model output, the loss_dict of p_losses in eval mode (val/ keys), the
two buffers, and get_input's z and encoded conditioning for a seeded batch dict, with the CPU generator seeded before
the call (the KL posterior draws its noise there). The batch is stored compactly and rebuilt by `batch_tensors`: the
images as uint8 (u / 127.5 - 1, as a data loader's [-1, 1] images) and the label map as its uint8 ids.
Run on the build machine: python oracle/make_golden_losses.py
"""
import contextlib
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import ref_harness as R  # noqa: E402
from ref_harness import gen  # noqa: E402
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "losses.pt")
UNET_SEED, FS_SEED, COND_SEED = 11, 12, 13
B = 4
T_VALUES = [0, 999, 381, 640]          # distinct, with both ends of the schedule
GET_INPUT_SEED = 77
UNET = "ldm.modules.diffusionmodules.openaimodel.UNetModel"


def _fs_node(cfg):
    kind = "VQModelInterface" if "n_embed" in cfg else "AutoencoderKL"
    return {"target": "ldm.models.autoencoder." + kind,
            "params": {**cfg, "monitor": "val/rec_loss", "lossconfig": {"target": "torch.nn.Identity"}}}


def _node(unet, fs, cond, **params):
    params = {"image_size": unet["image_size"], "channels": unet["in_channels"], "use_ema": False, **params}
    return {"target": "ldm.models.diffusion.ddpm.LatentDiffusion", "params": {
        **params, "unet_config": {"target": UNET, "params": dict(unet)}, "first_stage_config": _fs_node(fs),
        "cond_stage_config": cond}}


def _image_u8(seed, h, w, c=3):
    return torch.randint(0, 256, (B, h, w, c), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def batch_tensors(stored, n_labels):
    """The batch dict get_input reads, from its stored form: uint8 images to u / 127.5 - 1 in [-1, 1] and the uint8
    label map to its one-hot [B, H, W, n_labels]."""
    out = {}
    for k, v in stored.items():
        if k == "segmentation":
            out[k] = torch.nn.functional.one_hot(v.long(), n_labels).float()
        elif v.dtype == torch.uint8:
            out[k] = v.float() / 127.5 - 1.0
        else:
            out[k] = v
    return out


# member -> (unet, first stage, cond stage node, LatentDiffusion params)
MEMBERS = {
    "sd": (arch.TINY_UNET, arch.TINY_VAE, {"target": "torch.nn.Identity"},
           dict(linear_start=0.00085, linear_end=0.0120, num_timesteps_cond=1, timesteps=1000, first_stage_key="image",
                cond_stage_key="txt", cond_stage_trainable=False, conditioning_key="crossattn", scale_factor=0.18215,
                monitor="val/loss_simple_ema")),
    "lsun": (arch.TINY_ATTN_UNET, arch.TINY_VAE, "__is_unconditional__",
             dict(linear_start=0.0015, linear_end=0.0155, num_timesteps_cond=1, timesteps=1000, loss_type="l1",
                  first_stage_key="image", cond_stage_key="image", cond_stage_trainable=False, concat_mode=False,
                  scale_by_std=True, monitor="val/loss_simple_ema")),
    "cin": (arch.TINY_CIN_UNET, arch.TINY_VQ,
            {"target": "ldm.modules.encoders.modules.ClassEmbedder", "params": dict(arch.TINY_CIN_COND)},
            dict(linear_start=0.0015, linear_end=0.0195, num_timesteps_cond=1, timesteps=1000, first_stage_key="image",
                 cond_stage_key="class_label", cond_stage_trainable=True, conditioning_key="crossattn",
                 monitor="val/loss")),
    "semantic": (arch.TINY_SEMANTIC_UNET, arch.TINY_VQ_F4,
                 {"target": "ldm.modules.encoders.modules.SpatialRescaler", "params": dict(arch.TINY_SEMANTIC_COND)},
                 dict(linear_start=0.0015, linear_end=0.0205, timesteps=1000, loss_type="l1", first_stage_key="image",
                      cond_stage_key="segmentation", concat_mode=True, cond_stage_trainable=True)),
    "bsr": (arch.TINY_BSR_UNET, arch.TINY_VQ_F4, {"target": "torch.nn.Identity"},
            dict(linear_start=0.0015, linear_end=0.0155, timesteps=1000, loss_type="l2", first_stage_key="image",
                 cond_stage_key="LR_image", concat_mode=True, cond_stage_trainable=False)),
}
SCALE_BY_STD_FACTOR = 0.37     # the lsun member's scale_factor buffer (scale_by_std measures it on a training batch)


def _fs_shapes(cfg):
    return arch.vq_param_shapes(cfg) if "n_embed" in cfg else arch.vae_param_shapes(cfg)


def _build(name):
    R.install()
    from ldm.util import instantiate_from_config
    unet, fs, cond, params = MEMBERS[name]
    node = _node(unet, fs, cond, **params)
    with contextlib.redirect_stdout(io.StringIO()):
        ld = instantiate_from_config(node).eval()
    ld.model.diffusion_model.load_state_dict(arch.random_state_dict(arch.unet_param_shapes(unet), UNET_SEED),
                                             strict=True)
    ld.first_stage_model.load_state_dict(arch.random_state_dict(_fs_shapes(fs), FS_SEED), strict=True)
    shapes = {}
    if name in ("cin", "semantic"):
        shapes = {k: tuple(v.shape) for k, v in ld.cond_stage_model.state_dict().items()}
        ld.cond_stage_model.load_state_dict(arch.random_state_dict(shapes, COND_SEED), strict=True)
    if params.get("scale_by_std"):
        ld.scale_factor.fill_(SCALE_BY_STD_FACTOR)
    return ld, node, shapes


def _batch(name, ld):
    unet = MEMBERS[name][0]
    hw = unet["image_size"] * (2 ** (len(ld.first_stage_model.encoder.down) - 1))
    batch = {"image": _image_u8(501, hw, hw)}
    if name == "cin":
        batch["class_label"] = torch.tensor([3, 0, 999, 517])
    elif name == "semantic":
        n = arch.TINY_SEMANTIC_COND["in_channels"]
        batch["segmentation"] = torch.randint(0, n, (B, hw, hw), generator=torch.Generator().manual_seed(502),
                                              dtype=torch.uint8)
    elif name == "bsr":
        lr = unet["image_size"]
        batch["LR_image"] = _image_u8(503, lr, lr)
    return batch


@torch.no_grad()
def member(name):
    ld, node, cond_shapes = _build(name)
    stored = _batch(name, ld)
    batch = batch_tensors(stored, arch.TINY_SEMANTIC_COND["in_channels"])
    torch.manual_seed(GET_INPUT_SEED)
    if name == "sd":      # cond_stage_key txt has no get_input path in the reference (ddpm.py:672): the first stage only
        x = batch["image"].permute(0, 3, 1, 2).contiguous().float()
        z, c = ld.get_first_stage_encoding(ld.encode_first_stage(x)), None
    else:
        z, c = ld.get_input(batch, ld.first_stage_key)
    c_enc = ld.get_learned_conditioning(c) if (c is not None and ld.cond_stage_trainable) else c
    x_start = gen(tuple(z.shape), 601)
    if name == "sd":
        cond = gen((B, 77, arch.TINY_UNET["context_dim"]), 602)
    else:
        cond = c_enc
    t = torch.tensor(T_VALUES)
    noise = gen(tuple(z.shape), 603)
    x_noisy = ld.q_sample(x_start, t, noise)
    model_output = ld.apply_model(x_noisy, t, cond)
    loss, loss_dict = ld.p_losses(x_start, cond, t, noise=noise)
    assert torch.equal(loss, loss_dict["val/loss"])
    print(f"{name}: {', '.join(f'{k} {float(v):.6g}' for k, v in loss_dict.items())}; z {tuple(z.shape)}")
    return dict(node=node, cond_shapes=cond_shapes, scale_factor=float(ld.scale_factor), batch=stored,
                get_input_z=z, get_input_c_enc=c_enc,
                x_start=x_start, cond=cond, t=t, noise=noise, x_noisy=x_noisy, model_output=model_output,
                loss_dict={k: v.clone() for k, v in loss_dict.items()}, lvlb_weights=ld.lvlb_weights.clone(),
                logvar=ld.logvar.clone())


def published_params():
    """The LatentDiffusion `model.params` of every published YAML, without the three stage nodes: the loss fields
    (loss_type, l_simple_weight, original_elbo_weight, learn_logvar, logvar_init; absent = the reference default)
    and the schedule they are read with."""
    import glob
    import yaml
    out = {}
    paths = sorted(glob.glob(os.path.join(R.REF, "configs", "*", "*.yaml"))
                   + glob.glob(os.path.join(R.REF, "models", "ldm", "*", "config.yaml")))
    for path in paths:
        with open(path) as f:
            node = yaml.safe_load(f).get("model", {})
        if not node.get("target", "").endswith("ddpm.LatentDiffusion"):
            continue
        skip = ("unet_config", "first_stage_config", "cond_stage_config", "personalization_config", "scheduler_config",
                "ckpt_path", "ignore_keys")
        out[os.path.relpath(path, R.REF)] = {k: v for k, v in node["params"].items() if k not in skip}
    return out


def main():
    out = {"unet_seed": UNET_SEED, "fs_seed": FS_SEED, "cond_seed": COND_SEED, "get_input_seed": GET_INPUT_SEED,
           "members": {name: member(name) for name in MEMBERS}, "published_params": published_params()}
    torch.save(out, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
