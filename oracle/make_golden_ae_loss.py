"""Golden data for the first-stage loss (tests/golden/ae_loss.pt): the unmodified reference's LPIPSWithDiscriminator
(ldm/modules/losses/contperceptual.py) and AutoencoderKL.validation_step (ldm/models/autoencoder.py:372-383), under
torch.no_grad() in eval mode as Lightning's validation runs them, on top of oracle/taming_loss_oracle.py's restatement
of the taming pieces the loss imports.

  lpips          LPIPS of two uint8 image pairs at 64x64 and 64x96 (B = 2), and the five per-layer terms
  logits         the discriminator's logits on the 64x64 reconstructions
  calls          both loss calls (optimizer_idx 0 and 1) with hinge and with vanilla, global_step on each side of
                 disc_start, on a seeded posterior (its NCHW moments are stored)
  validation     validation_step of a tiny 4-channel KL first stage (arch.TINY_VAE) on a 32x32 uint8 batch, the CPU
                 generator seeded with VAL_SEED before the call (the posterior draws its noise there)

Images are stored as uint8 (u / 127.5 - 1); weights as seeds: the loss's by ae_loss.random_loss_state_dict of
ae_loss.loss_param_shapes() at LOSS_SEED with logvar LOGVAR, the first stage's by arch.random_state_dict at FS_SEED.
Run on the build machine: python oracle/make_golden_ae_loss.py
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
import taming_loss_oracle  # noqa: E402
from sdb200 import ae_loss, arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ae_loss.pt")
LOSS_SEED, FS_SEED, VAL_SEED = 21, 22, 23
LOGVAR = 0.25
DISC_START = 10
B = 2
LOSS_PARAMS = dict(disc_start=DISC_START, kl_weight=1.0e-6, disc_weight=0.5)


def image_u8(seed, h, w, nb=B):
    return torch.randint(0, 256, (nb, h, w, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


def to_float(u8):
    return u8.permute(0, 3, 1, 2).float() / 127.5 - 1.0


def loss_state_dict():
    return ae_loss.random_loss_state_dict(ae_loss.loss_param_shapes(), LOSS_SEED, logvar=LOGVAR)


def _loss(disc_loss):
    taming_loss_oracle.install()
    R.install()
    from ldm.modules.losses import LPIPSWithDiscriminator
    m = LPIPSWithDiscriminator(**LOSS_PARAMS, disc_loss=disc_loss)
    m.load_state_dict(loss_state_dict(), strict=True)
    return m.eval()


def _f(d):
    return {k: float(v) for k, v in d.items()}


@torch.no_grad()
def main():
    hinge = _loss("hinge")
    from ldm.modules.distributions.distributions import DiagonalGaussianDistribution
    out = {"loss_seed": LOSS_SEED, "fs_seed": FS_SEED, "val_seed": VAL_SEED, "logvar": LOGVAR,
           "loss_params": LOSS_PARAMS}
    lp = hinge.perceptual_loss
    out["lpips"] = {}
    for h, w, s in ((64, 64, 301), (64, 96, 303)):
        a, b = image_u8(s, h, w), image_u8(s + 1, h, w)
        x0, x1 = to_float(a), to_float(b)
        f0, f1 = lp.net(lp.scaling_layer(x0)), lp.net(lp.scaling_layer(x1))
        taps = [taming_loss_oracle.spatial_average(getattr(lp, f"lin{k}").model(
            (taming_loss_oracle.normalize_tensor(f0[k]) - taming_loss_oracle.normalize_tensor(f1[k])) ** 2)).view(-1)
            for k in range(5)]
        val = lp(x0, x1)
        print(f"lpips {h}x{w}: {val.view(-1).tolist()}")
        out["lpips"][f"{h}x{w}"] = {"in0": a, "in1": b, "value": val.clone(), "taps": torch.stack(taps)}
    x_u8, xr_u8 = out["lpips"]["64x64"]["in0"], out["lpips"]["64x64"]["in1"]
    x, xr = to_float(x_u8), to_float(xr_u8)
    out["logits"] = hinge.discriminator(xr).clone()
    out["logits_real"] = hinge.discriminator(x).clone()
    moments = R.gen((B, 8, 8, 8), 305)
    moments[:, 4:] = moments[:, 4:].clamp(-3, 3) - 1.0
    out["moments"] = moments
    post = DiagonalGaussianDistribution(moments)
    out["kl"] = post.kl().clone()
    last = torch.zeros(1, requires_grad=True)    # autograd.grad fails under no_grad: d_weight 0, as in validation
    calls = {}
    for kind in ("hinge", "vanilla"):
        m = hinge if kind == "hinge" else _loss("vanilla")
        for gs in (DISC_START - 1, DISC_START):
            for idx in (0, 1):
                loss, log = m(x, xr, post, idx, gs, last_layer=last, split="val")
                calls[(kind, gs, idx)] = {"loss": float(loss), "log": _f(log)}
                print(kind, gs, idx, f"{float(loss):.6g}", {k: round(v, 6) for k, v in _f(log).items()})
    out["calls"] = calls

    # validation_step of a tiny KL first stage built with the loss from its lossconfig
    from ldm.models.autoencoder import AutoencoderKL
    with contextlib.redirect_stdout(io.StringIO()):
        ae = AutoencoderKL(ddconfig=arch.TINY_VAE["ddconfig"], embed_dim=arch.TINY_VAE["embed_dim"],
                           lossconfig={"target": "ldm.modules.losses.LPIPSWithDiscriminator", "params": LOSS_PARAMS})
    sd = dict(arch.random_state_dict(arch.vae_param_shapes(arch.TINY_VAE), FS_SEED))
    sd.update({"loss." + k: v for k, v in loss_state_dict().items()})
    ae.load_state_dict(sd, strict=True)
    ae.eval()
    val = {}
    for gs in (DISC_START - 1, DISC_START):
        logged = {}
        ae.log_dict = lambda d, **k: logged.update(_f(d))
        ae.global_step = gs
        batch_u8 = image_u8(307, 32, 32)
        torch.manual_seed(VAL_SEED)
        ae.validation_step({"image": batch_u8.float() / 127.5 - 1.0}, 0)
        val[gs] = logged
        print("validation", gs, {k: round(v, 6) for k, v in logged.items()})
    out["validation"] = {"batch": image_u8(307, 32, 32), "logs": val}
    torch.save(out, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1024:.0f} KiB)")


if __name__ == "__main__":
    main()
