"""Samplers and the LatentDiffusion facade on the H100 against the reference (golden) and the oracle."""
import numpy as np
import pytest
import torch

from helpers import golden, rel_l2, weights
from sdb200 import arch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


def _tiny_ld(dev):
    import sdb200
    m = sdb200.LatentDiffusion(
        first_stage_config={"target": "ldm.models.autoencoder.AutoencoderKL", "params": dict(arch.TINY_VAE)},
        cond_stage_config={"target": "ldm.modules.encoders.modules.FrozenCLIPEmbedder", "params": {"config": arch.TINY_CLIP}},
        unet_config={"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": dict(arch.TINY_UNET)},
        linear_start=0.00085, linear_end=0.0120, timesteps=1000, conditioning_key="crossattn", scale_factor=0.18215,
        image_size=64, channels=4)
    sd = {}
    sd.update({"model.diffusion_model." + k: v for k, v in weights("unet", "tiny", 11).items()})
    sd.update({"first_stage_model." + k: v for k, v in weights("vae", "tiny", 12).items()})
    sd.update({"cond_stage_model.transformer." + k: v for k, v in weights("clip", "tiny", 13).items()})
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.split(".")[0] in ("betas", "alphas_cumprod", "alphas_cumprod_prev",
                                                             "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod")
                                           for k in res.missing_keys)
    return m.to(dev)


class _ReplayModel:
    """Facade whose apply_model replays eps tensors recorded from an oracle run: isolates the sampler arithmetic."""

    def __init__(self, sched, eps_list, dev):
        self.num_timesteps = 1000
        self.alphas_cumprod = sched["alphas_cumprod"].to(dev)
        self.betas = sched["betas"].to(dev)
        self.device = dev
        self.eps = [e.to(dev) for e in eps_list]
        self.calls = []

    def apply_model(self, x, t, c):
        self.calls.append((tuple(x.shape), int(t[0])))
        return self.eps[len(self.calls) - 1]


@pytest.mark.parametrize("kind,scale", [("plms", 7.5), ("ddim", 7.5), ("plms", 1.0)])
def test_sampler_arithmetic_bit_exact(cuda_dev, kind, scale):
    """With identical eps inputs the fused step kernel reproduces the reference update sequence bit for bit."""
    import ldm_oracle as O
    import sdb200
    g = torch.Generator().manual_seed(5)
    B, shape = 2, (4, 8, 8)
    x_T = torch.randn(B, *shape, generator=g)
    c = torch.randn(B, 77, 64, generator=g)
    uc = torch.randn(B, 77, 64, generator=g) if scale != 1.0 else None
    rec = []

    def model_fn(x, t, cc):  # cheap deterministic stand-in for the UNet
        e = torch.tanh(0.7 * x + 0.01 * t.float()[:, None, None, None] * 0.01) + 0.05 * cc.mean(dim=(1, 2))[:, None, None, None]
        rec.append(e)
        return e

    fn = O.plms_sample if kind == "plms" else O.ddim_sample
    ref = fn(model_fn, x_T, c, uc, scale, S=10)
    model = _ReplayModel(O.register_schedule(), rec, cuda_dev)
    S = sdb200.PLMSSampler(model) if kind == "plms" else sdb200.DDIMSampler(model)
    out, inter = S.sample(S=10, conditioning=c.to(cuda_dev), batch_size=B, shape=list(shape), verbose=False,
                          unconditional_guidance_scale=scale,
                          unconditional_conditioning=None if uc is None else uc.to(cuda_dev), eta=0.0,
                          x_T=x_T.to(cuda_dev))
    nb = 2 * B if uc is not None else B
    assert len(model.calls) == (11 if kind == "plms" else 10) and all(s[0][0] == nb for s in model.calls)
    assert [s[1] for s in model.calls][:3] == ([901, 801, 801] if kind == "plms" else [901, 801, 701])
    assert torch.equal(out.cpu(), ref), float((out.cpu() - ref).abs().max())
    assert set(inter) == {"x_inter", "pred_x0"}


def test_schedule_matches_reference(cuda_dev):
    import sdb200
    g = golden("pipeline_tiny.pt")
    ld = _tiny_ld(cuda_dev)
    for k in ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod"):
        assert torch.equal(getattr(ld, k).cpu(), g["sched_" + k]), k
    for S in (50, 10):
        s = sdb200.PLMSSampler(ld)
        s.make_schedule(S, verbose=False)
        assert np.array_equal(s.ddim_timesteps, g[f"plms{S}_timesteps"].numpy())
        assert np.array_equal(s.ddim_alphas, g[f"plms{S}_alphas"].float().numpy())
        assert np.array_equal(s.ddim_alphas_prev, g[f"plms{S}_alphas_prev"].float().numpy())
        assert np.array_equal(s.ddim_sqrt_one_minus_alphas, g[f"plms{S}_sqrt_one_minus_alphas"].float().numpy())
    with pytest.raises(ValueError):
        sdb200.PLMSSampler(ld).make_schedule(10, ddim_eta=0.5, verbose=False)
    with pytest.raises(IndexError):
        sdb200.DDIMSampler(ld).make_schedule(3, verbose=False)   # the reference's S=3 IndexError (util.py:65)


def test_txt2img_and_img2img_vs_reference(cuda_dev):
    import sdb200
    g = golden("pipeline_tiny.pt")
    ld = _tiny_ld(cuda_dev)
    dev = cuda_dev
    c, uc, x_T = g["c"].to(dev), g["uc"].to(dev), g["x_T"].to(dev)
    eps = ld.apply_model(x_T, g["apply_model_t"].to(dev), c)
    assert rel_l2(eps, g["apply_model_eps"]) < 2e-3
    errs = {}
    for S in (10, 50):
        s, _ = sdb200.PLMSSampler(ld).sample(S=S, conditioning=c, batch_size=2, shape=[4, 16, 16], verbose=False,
                                             unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=0.0, x_T=x_T)
        errs[f"plms{S}"] = rel_l2(s, g[f"plms{S}"])
        d, _ = sdb200.DDIMSampler(ld).sample(S=S, conditioning=c, batch_size=2, shape=[4, 16, 16], verbose=False,
                                             unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=0.0, x_T=x_T)
        errs[f"ddim{S}"] = rel_l2(d, g[f"ddim{S}"])
    s1, _ = sdb200.PLMSSampler(ld).sample(S=10, conditioning=c, batch_size=2, shape=[4, 16, 16], verbose=False,
                                          unconditional_guidance_scale=1.0, unconditional_conditioning=None, eta=0.0, x_T=x_T)
    errs["plms10_noguidance"] = rel_l2(s1, g["plms10_noguidance"])
    # img2img (scripts/img2img.py:235-264)
    post = ld.encode_first_stage(g["img"].to(dev))
    z0 = ld.get_first_stage_encoding(post, noise=g["enc_noise"].to(dev))
    errs["z0"] = rel_l2(z0, g["z0"])
    ddim = sdb200.DDIMSampler(ld)
    ddim.make_schedule(ddim_num_steps=50, ddim_eta=0.0, verbose=False)
    z_enc = ddim.stochastic_encode(g["z0"].to(dev), torch.tensor([g["t_enc"]] * 2).to(dev), noise=g["se_noise"].to(dev))
    errs["z_enc"] = rel_l2(z_enc, g["z_enc"])
    z_dec = ddim.decode(g["z_enc"].to(dev), c, g["t_enc"], unconditional_guidance_scale=5.0, unconditional_conditioning=uc)
    errs["z_dec"] = rel_l2(z_dec, g["z_dec"])
    x_dec = ld.decode_first_stage(g["z_dec"].to(dev))
    errs["x_dec"] = rel_l2(x_dec, g["x_dec"])
    print({k: f"{v:.2e}" for k, v in errs.items()})
    assert errs["z_enc"] < 1e-6 and errs["z0"] < 2e-3 and errs["x_dec"] < 2e-3
    # trajectories accumulate the per-evaluation fp16 error over S(+1) guided steps with CFG 7.5 on random weights
    assert errs["plms10"] < 2e-2 and errs["ddim10"] < 2e-2 and errs["plms10_noguidance"] < 1e-2
    assert errs["plms50"] < 5e-2 and errs["ddim50"] < 5e-2 and errs["z_dec"] < 5e-2
