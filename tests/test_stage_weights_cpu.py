"""Weight plumbing of every engine stage on the host: what `load_state_dict` adopts under a prefix, which checkpoint
leftovers are dropped silently, how missing, unexpected and misshapen tensors are reported, that host moves pack
nothing, that `load_weights` rejects an incomplete state dict, and which stages of a LatentDiffusion
`pipeline.load_random_weights` seeds with which seed. No GPU."""
import re

import pytest
import torch
import torch.nn as nn

import sdb200
from helpers import script
from sdb200 import arch, pipeline
from sdb200.util import PackedStage, instantiate_from_config, remap_config

# id -> (constructor, where the stage's keys sit below the stage, checkpoint keys the stage drops without reporting)
STAGES = {
    "unet": (lambda: sdb200.UNetModel(**arch.TINY_UNET), "", ()),
    "autoencoder_kl": (lambda: sdb200.AutoencoderKL(**arch.TINY_VAE), "", ("loss.logvar", "loss.discriminator.0.weight")),
    "vq": (lambda: sdb200.VQModelInterface(**arch.TINY_VQ), "", ("loss.logvar",)),
    "clip": (lambda: sdb200.FrozenCLIPEmbedder(config=arch.TINY_CLIP), "transformer.",
             ("text_model.embeddings.position_ids",)),
    "bert": (lambda: sdb200.BERTEmbedder(**arch.TINY_BERT), "",
             ("transformer.to_logits.weight", "transformer.to_logits.bias")),
    "safety": (lambda: sdb200.StableDiffusionSafetyChecker(config=arch.TINY_SAFETY), "",
               ("vision_model.vision_model.embeddings.position_ids",)),
    "class_embedder": (lambda: sdb200.ClassEmbedder(**arch.TINY_CIN_COND), "", ()),
    "rescaler_mapper": (lambda: sdb200.SpatialRescaler(**arch.TINY_SEMANTIC_COND), "", ()),
    "rescaler_mapper_bias": (lambda: sdb200.SpatialRescaler(**arch.TINY_SEMANTIC_COND, bias=True), "", ()),
    "rescaler_plain": (lambda: sdb200.SpatialRescaler(n_stages=2, in_channels=3), "", ()),
}
WITH_KEYS = [s for s in STAGES if s != "rescaler_plain"]


def _setup(name):
    """(holder, stage, state dict prefix of the stage's keys, state dict): the stage sits at `holder.stage`, as a
    first stage or cond stage sits inside a LatentDiffusion; every tensor has its own value."""
    make, below, _ = STAGES[name]
    stage = make()
    holder = nn.Module()
    holder.stage = stage
    prefix = "stage." + below
    sd = {prefix + k: torch.full(tuple(shp), float(i)) for i, (k, shp) in enumerate(stage.shapes.items())}
    return holder, stage, prefix, sd


def _nothing_adopted(stage):
    return getattr(stage, "_host_sd", None) is None and stage.W is None


def _dropped(name, prefix):
    return {prefix + k: torch.zeros(3) for k in STAGES[name][2]}


@pytest.mark.parametrize("name", list(STAGES))
def test_load_state_dict_adopts_exactly_shapes(name):
    holder, stage, prefix, sd = _setup(name)
    res = holder.load_state_dict({**sd, **_dropped(name, prefix)}, strict=False)
    assert res.missing_keys == [] and res.unexpected_keys == []
    assert list(stage._host_sd) == list(stage.shapes)
    for k, t in stage._host_sd.items():
        assert t is sd[prefix + k]
    # the dropped leftovers do not trip strict loading either
    holder2, stage2, _, _ = _setup(name)
    holder2.load_state_dict({**sd, **_dropped(name, prefix)}, strict=True)
    assert list(stage2._host_sd) == list(stage2.shapes)


@pytest.mark.parametrize("name", list(STAGES))
def test_other_extra_keys_are_unexpected(name):
    holder, stage, prefix, sd = _setup(name)
    extra = {prefix + "bogus.weight": torch.zeros(2), prefix + "loss_like": torch.zeros(1)}
    res = holder.load_state_dict({**sd, **extra}, strict=False)
    assert sorted(res.unexpected_keys) == sorted(extra) and res.missing_keys == []
    assert list(stage._host_sd) == list(stage.shapes)
    with pytest.raises(RuntimeError, match=re.escape(prefix + "bogus.weight")):
        _setup(name)[0].load_state_dict({**sd, **extra}, strict=True)


@pytest.mark.parametrize("name", WITH_KEYS)
def test_missing_key_is_reported_and_nothing_adopted(name):
    holder, stage, prefix, sd = _setup(name)
    gone = prefix + list(stage.shapes)[-1]
    del sd[gone]
    res = holder.load_state_dict(sd, strict=False)
    assert res.missing_keys == [gone] and res.unexpected_keys == []
    assert _nothing_adopted(stage)


@pytest.mark.parametrize("name", WITH_KEYS)
def test_wrong_shape_raises_size_mismatch(name):
    holder, stage, prefix, sd = _setup(name)
    k = prefix + list(stage.shapes)[0]
    sd[k] = torch.zeros((sd[k].shape[0] + 1,) + tuple(sd[k].shape[1:]))
    with pytest.raises(RuntimeError, match=re.escape(f"size mismatch for {k}")):
        holder.load_state_dict(sd, strict=False)
    assert _nothing_adopted(stage)


@pytest.mark.parametrize("name", list(STAGES))
def test_host_moves_pack_nothing(name):
    holder, stage, prefix, sd = _setup(name)
    holder.load_state_dict(sd)
    assert stage.to("cpu") is stage and stage.float() is stage and holder.cpu() is holder
    assert stage.W is None


@pytest.mark.parametrize("name", WITH_KEYS)
def test_load_weights_rejects_missing_or_misshapen(name):
    _, stage, prefix, sd = _setup(name)
    sd = {k[len(prefix):]: v for k, v in sd.items()}
    first = next(iter(sd))
    with pytest.raises(AssertionError):
        stage.load_weights({k: v for k, v in sd.items() if k != first}, "cpu")
    with pytest.raises(AssertionError):
        stage.load_weights({**sd, first: torch.zeros(tuple(sd[first].shape) + (1,))}, "cpu")
    assert _nothing_adopted(stage)


@pytest.mark.parametrize("name", list(STAGES))
def test_reload_repacks_on_the_packed_device(name):
    holder, stage, prefix, sd = _setup(name)
    stage.load_weights({k[len(prefix):]: v for k, v in sd.items()}, "cpu")
    packed = stage.W
    assert packed["device"] == torch.device("cpu")
    holder.load_state_dict({k: v + 1 for k, v in sd.items()})
    assert stage.W is not packed and stage.W["device"] == torch.device("cpu")
    assert all(torch.equal(stage._host_sd[k[len(prefix):]], v + 1) for k, v in sd.items())


def test_unet_weight_sets_checked_and_reset_by_a_reload():
    holder, unet, prefix, full = _setup("unet")
    sd = {k[len(prefix):]: v for k, v in full.items()}
    first = next(iter(sd))
    with pytest.raises(AssertionError):
        unet.set_weight_set("ema", {k: v for k, v in sd.items() if k != first})
    with pytest.raises(AssertionError):
        unet.set_weight_set("ema", {**sd, first: torch.zeros(1)})
    assert not unet.has_weight_set("ema")
    unet.set_weight_set("ema", {**sd, "extra": torch.zeros(1)})
    assert unet.has_weight_set("ema") and list(unet._alt_sd["ema"]) == list(unet.shapes)
    unet.load_weights(sd, "cpu")
    unet.use_weight_set("ema")
    assert unet._active == "ema" and set(unet._packed) == {"raw"}
    holder.load_state_dict(full)            # fresh weights: every packed set is stale
    assert unet._active == "raw" and unet._packed == {} and unet.has_weight_set("ema")


# one LDM of each kind: (script, its config function, the tiny members)
LDMS = {
    "cin_three_stages": ("sample_imagenet", "cin_config", (arch.TINY_CIN_UNET, arch.TINY_VQ, arch.TINY_CIN_COND)),
    "inpaint_first_stage_is_cond": ("inpaint", "inpaint_config", (arch.TINY_INPAINT_UNET, arch.TINY_VQ_NOATTN)),
    "superres_identity_cond": ("superres", "superres_config", (arch.TINY_BSR_UNET, arch.TINY_VQ_F4)),
    "lsun_unconditional": ("sample_diffusion", "lsun_churches_config", (arch.TINY_ATTN_UNET, arch.TINY_VAE)),
}


@pytest.mark.parametrize("name", list(LDMS))
def test_load_random_weights_seeds_each_weighted_stage_once(name, monkeypatch):
    """UNet, first stage and cond stage get seeds 11, 12 and 13; a cond stage that is the first stage is loaded once,
    with 12, and an Identity or absent cond stage is skipped."""
    mod, make, members = LDMS[name]
    m = instantiate_from_config(remap_config(getattr(script(mod), make)(*members)))
    loads = []
    load = PackedStage.load_weights
    monkeypatch.setattr(PackedStage, "load_weights", lambda self, sd, device: loads.append(self) or load(self, sd, device))
    assert pipeline.load_random_weights(m, "cpu") is m
    seeded = [m.model.diffusion_model, m.first_stage_model]
    if name == "cin_three_stages":
        seeded.append(m.cond_stage_model)
    elif name == "inpaint_first_stage_is_cond":
        assert m.cond_stage_model is m.first_stage_model
    elif name == "superres_identity_cond":
        assert isinstance(m.cond_stage_model, nn.Identity)
    else:
        assert m.cond_stage_model is None
    assert len(loads) == len(seeded) and all(a is b for a, b in zip(loads, seeded))
    for stage, seed in zip(seeded, (11, 12, 13)):
        want = arch.random_state_dict(stage.shapes, seed)
        assert list(stage._host_sd) == list(want) and all(torch.equal(stage._host_sd[k], t) for k, t in want.items())
