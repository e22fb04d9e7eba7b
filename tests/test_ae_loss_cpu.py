"""First-stage loss without a GPU: the ABI of include/sdb200_ae_loss.h, the lossconfig of every published KL YAML, the
loss stage's state dict against the oracle restatement, and inputs rejected before any launch."""
import glob
import os
import re

import pytest
import torch
import yaml

import helpers
import sdb200
from sdb200 import ae_loss, checkpoint, ops
from sdb200.util import instantiate_from_config, remap_config

REF = os.environ.get("SD_REFERENCE", "/root/reference")
HEADER = os.path.join(helpers.ROOT, "include", "sdb200_ae_loss.h")


def _declared():
    src = open(HEADER).read()
    return sorted(set(re.findall(r"^(?:int|int64_t)\s+(sdb_\w+)\(", src, re.M)))


def test_header_matches_ctypes_table():
    assert _declared() == sorted(sdb200.lib.AE_LOSS_SIGNATURES)
    # kept apart from the sampling and evaluation tables
    assert not set(sdb200.lib.AE_LOSS_SIGNATURES) & (set(sdb200.lib.SIGNATURES) | set(sdb200.lib.EVAL_SIGNATURES))


def test_symbols_resolve_with_their_argtypes():
    lib = sdb200.lib.load()
    for name, (argtypes, restype) in sdb200.lib.AE_LOSS_SIGNATURES.items():
        fn = getattr(lib, name)
        assert fn.argtypes == argtypes and fn.restype == restype


def test_activation_values():
    src = open(os.path.join(helpers.ROOT, "include", "sdb200.h")).read()
    assert "SDB_ACT_RELU = 6" in src and "SDB_ACT_LEAKY_RELU = 7" in src and "= 5" not in src
    assert (sdb200.lib.ACT_RELU, sdb200.lib.ACT_LEAKY_RELU) == (6, 7)


# the KL configs the reference publishes, with their lossconfig as the YAML states it
KL_YAMLS = {"configs/autoencoder/autoencoder_kl_16x16x16.yaml", "configs/autoencoder/autoencoder_kl_32x32x4.yaml",
            "configs/autoencoder/autoencoder_kl_64x64x3.yaml", "configs/autoencoder/autoencoder_kl_8x8x64.yaml",
            "models/first_stage_models/kl-f4/config.yaml", "models/first_stage_models/kl-f8/config.yaml",
            "models/first_stage_models/kl-f16/config.yaml", "models/first_stage_models/kl-f32/config.yaml"}
LOSS_NODE = {"target": "ldm.modules.losses.LPIPSWithDiscriminator",
             "params": {"disc_start": 50001, "kl_weight": 1.0e-6, "disc_weight": 0.5}}


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "configs")), reason="reference configs not present")
def test_published_kl_yamls_state_the_same_lossconfig():
    paths = sorted(glob.glob(os.path.join(REF, "configs", "autoencoder", "*.yaml"))
                   + glob.glob(os.path.join(REF, "models", "first_stage_models", "kl-*", "config.yaml")))
    assert {os.path.relpath(p, REF) for p in paths} == KL_YAMLS
    for p in paths:
        with open(p) as f:
            assert yaml.safe_load(f)["model"]["params"]["lossconfig"] == LOSS_NODE, p


def test_lossconfig_builds_the_loss_stage():
    m = instantiate_from_config(remap_config(LOSS_NODE))
    assert type(m) is sdb200.LPIPSWithDiscriminator
    assert (m.discriminator_iter_start, m.kl_weight, m.discriminator_weight) == (50001, 1.0e-6, 0.5)
    assert (m.disc_factor, m.perceptual_weight, m.disc_loss, m.logvar_init) == (1.0, 1.0, "hinge", 0.0)
    with pytest.raises(NotImplementedError):
        sdb200.LPIPSWithDiscriminator(disc_start=0, use_actnorm=True)
    with pytest.raises(NotImplementedError):
        sdb200.LPIPSWithDiscriminator(disc_start=0, disc_conditional=True)


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "ldm")), reason="reference not present")
def test_keys_and_shapes_equal_the_oracle_restatement():
    """The loss stage's state dict (taming's layout) is the reference LPIPSWithDiscriminator's over the oracle
    restatement of taming, key for key, in order."""
    import ref_harness as R
    import taming_loss_oracle
    taming_loss_oracle.install()
    R.install()
    from ldm.modules.losses import LPIPSWithDiscriminator
    ref = LPIPSWithDiscriminator(disc_start=1)
    assert [(k, tuple(v.shape)) for k, v in ref.state_dict().items()] == list(ae_loss.loss_param_shapes().items())
    sd = ae_loss.random_loss_state_dict(ae_loss.loss_param_shapes(), 5)
    ref.load_state_dict(sd, strict=True)
    m = sdb200.LPIPSWithDiscriminator(disc_start=1)
    res = m.load_state_dict(sd, strict=False)
    assert res.missing_keys == [] and res.unexpected_keys == [] and m.missing_keys() == []


def _stage_with_loss(tmp_path, with_loss):
    cfg = {"model": {"target": "ldm.models.autoencoder.AutoencoderKL",
                     "params": {**sdb200.arch.TINY_VAE, "lossconfig": LOSS_NODE}}}
    sd = dict(sdb200.arch.random_state_dict(sdb200.arch.vae_param_shapes(sdb200.arch.TINY_VAE), 3))
    if with_loss:
        sd.update({"loss." + k: v for k, v in
                   ae_loss.random_loss_state_dict(ae_loss.loss_param_shapes(), 4).items()})
    ck = tmp_path / "m.ckpt"
    torch.save({"state_dict": sd, "global_step": 60000}, ck)
    m = checkpoint.load_model_from_config(cfg, str(ck), device=None)
    loss = checkpoint.load_first_stage_loss(m, cfg, str(ck), device=None)
    return m, loss


def test_loss_loads_from_the_checkpoint_loss_tensors(tmp_path):
    m, loss = _stage_with_loss(tmp_path, True)
    assert m.load_info["unexpected"] == [] and m.global_step == 60000 and m.loss is loss
    assert loss.load_info["missing"] == [] and loss.missing_keys() == [] and not loss.training
    assert "loss.logvar" not in m.state_dict() and not any(k.startswith("loss") for k, _ in m.named_modules())


def test_checkpoint_without_loss_tensors(tmp_path):
    m, loss = _stage_with_loss(tmp_path, False)
    assert m.load_info["missing"] == [] and m._host_sd is not None
    assert "loss.logvar" in loss.load_info["missing"] and "logvar" in loss.missing_keys()
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match="loss.logvar"):
        m.validation_step({"image": torch.zeros(1, 32, 32, 3)}, 0)
    assert ops.launch_count() == n0


def _loaded_loss():
    m = sdb200.LPIPSWithDiscriminator(disc_start=1)
    m.load_state_dict(ae_loss.random_loss_state_dict(ae_loss.loss_param_shapes(), 6))
    return m.eval()


class _FakeCuda(torch.Tensor):
    """A host tensor that claims to live on the GPU, so the shape checks run without a device."""

    @property
    def is_cuda(self):
        return True


def _img(*shape):
    return torch.zeros(shape).as_subclass(_FakeCuda)


@pytest.mark.parametrize("a,b,exc", [
    ((2, 3, 15, 64), (2, 3, 15, 64), ValueError),     # LPIPS side below 16
    ((2, 3, 64, 64), (2, 3, 64, 32), ValueError),     # shapes differ
    ((2, 4, 64, 64), (2, 4, 64, 64), ValueError),     # not RGB
    ((2, 3, 64, 64), None, ValueError),               # not a tensor
])
def test_lpips_rejects_before_launch(a, b, exc):
    lp = _loaded_loss().perceptual_loss
    n0 = ops.launch_count()
    with pytest.raises(exc):
        lp.check_inputs(_img(*a), _img(*b) if b else "x")
    assert ops.launch_count() == n0


def test_loss_rejects_before_launch():
    m = _loaded_loss()
    x = _img(2, 3, 64, 64)
    n0 = ops.launch_count()
    with pytest.raises(NotImplementedError):
        m.train()._check(x, x, None, 0, None, None)
    m.eval()
    with pytest.raises(NotImplementedError):
        m._check(x, x, None, 0, None, torch.ones(1))
    with pytest.raises(NotImplementedError):
        m._check(x, x, None, 0, x, None)
    with pytest.raises(ValueError):
        m._check(x, x, None, 2, None, None)
    with pytest.raises(ValueError):   # 16 x 16 passes LPIPS but leaves the discriminator no logit
        m._check(_img(2, 3, 16, 16), _img(2, 3, 16, 16), None, 1, None, None)
    empty = sdb200.LPIPSWithDiscriminator(disc_start=1).eval()
    with pytest.raises(RuntimeError, match="logvar"):
        empty._check(x, x, None, 0, None, None)
    assert ops.launch_count() == n0


def test_discriminator_geometry():
    assert ae_loss.discriminator_out_size(256, 256) == (30, 30)
    assert ae_loss.discriminator_out_size(64, 96) == (6, 10)
    assert ae_loss.discriminator_out_size(23, 64)[0] < 1 <= ae_loss.discriminator_out_size(24, 64)[0]
    layers = ae_loss.discriminator_layers()
    assert [(i, cin, cout, s) for i, cin, cout, s, *_ in layers] == [
        (0, 3, 64, 2), (2, 64, 128, 2), (5, 128, 256, 2), (8, 256, 512, 1), (11, 512, 1, 1)]
