"""ORACLE tooling: generate tests/golden/lsun.pt by running the UNMODIFIED reference (located by ref_harness.py) on CPU fp32
for the unconditional attention-block LDM family (models/ldm/lsun_churches256/config.yaml, scripts/sample_diffusion.py).

Run in the build container:  python oracle/make_golden_lsun.py
Weights come from stable-diffusion_b200/arch.random_state_dict (seeded); only inputs, recorded noise draws and reference
outputs are stored. Every vector is also evaluated with oracle/uncond_oracle.py and the error printed.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import ref_harness as R  # noqa: E402
from ref_harness import gen, rel  # noqa: E402
import uncond_oracle as U  # noqa: E402
import ldm_oracle as O  # noqa: E402
import sdb200  # noqa: E402,F401
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_SEED, VAE_SEED, EMA_SEED = 11, 12, 31
CFGS = {"tiny_attn": arch.TINY_ATTN_UNET, "tiny_attn_plain": arch.TINY_ATTN_PLAIN_UNET, "lsun": arch.LSUN_CHURCHES_UNET}
SCALE_FACTOR = 0.37
# LatentDiffusion with the LSUN-Churches config parameters (unconditional, scale_by_std); each model built here then
# gets scale_factor = SCALE_FACTOR in place of the one scale_by_std would measure on the first training batch
LD_PARAMS = dict(linear_start=0.0015, linear_end=0.0155, num_timesteps_cond=1, log_every_t=200, timesteps=1000,
                 loss_type="l1", first_stage_key="image", cond_stage_key="image", channels=4,
                 cond_stage_trainable=False, concat_mode=False, scale_by_std=True, monitor="val/loss_simple_ema",
                 use_ema=False)


class Recorder:
    """Replaces a module's noise_like and keeps every draw."""

    def __init__(self, module):
        self.module, self.draws = module, []
        self.orig = module.noise_like

    def __enter__(self):
        def rec(shape, device, repeat=False):
            r = self.orig(shape, device, repeat)
            self.draws.append(r.clone())
            return r
        self.module.noise_like = rec
        return self

    def __exit__(self, *a):
        self.module.noise_like = self.orig


@torch.no_grad()
def main():
    out = {"unet": [], "scale_factor": SCALE_FACTOR, "unet_seed": UNET_SEED, "vae_seed": VAE_SEED, "ema_seed": EMA_SEED}
    for tag, cfg, shapes in (
        ("tiny_attn", arch.TINY_ATTN_UNET, [((2, 4, 16, 16), [981, 1]), ((2, 4, 16, 32), [500, 21])]),
        ("tiny_attn_plain", arch.TINY_ATTN_PLAIN_UNET, [((2, 4, 16, 16), [981, 1]), ((2, 4, 16, 32), [500, 21])]),
        ("lsun", arch.LSUN_CHURCHES_UNET, [((2, 4, 32, 32), [981, 1]), ((1, 4, 16, 48), [501])]),
    ):
        sd = arch.random_state_dict(arch.unet_param_shapes(cfg), UNET_SEED)
        net = R.build_unet(cfg)
        net.load_state_dict(sd, strict=True)
        for i, (xs, ts) in enumerate(shapes):
            x = gen(xs, 800 + i)
            t = torch.tensor(ts, dtype=torch.long)
            eps = net(x, t)
            mine = U.unet_forward(sd, cfg, x, t)
            print(f"unet {tag} {xs} t={ts}: eps std {float(eps.std()):.3f}  oracle rel-L2 {rel(mine, eps):.2e}")
            out["unet"].append(dict(cfg=tag, x=x, t=t, eps=eps))
        del net
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_ATTN_UNET), UNET_SEED)
    vsd = arch.random_state_dict(arch.vae_param_shapes(arch.TINY_VAE), VAE_SEED)
    model_fn = lambda x, t: U.unet_forward(usd, arch.TINY_ATTN_UNET, x, t)
    B, shape = 2, [4, 16, 16]

    # DDIM S=10, eta=1, unconditional (sample_diffusion.py convsample_ddim), then decode_first_stage
    ld = R.build_ld(arch.TINY_ATTN_UNET, arch.TINY_VAE, "__is_unconditional__", **LD_PARAMS)
    ld.scale_factor.fill_(SCALE_FACTOR)
    ld.model.diffusion_model.load_state_dict(usd, strict=True)
    ld.first_stage_model.load_state_dict(vsd, strict=True)
    _, ddim = R.build_samplers(ld)
    import ldm.models.diffusion.ddim as ddim_mod
    import ldm.models.diffusion.ddpm as ddpm_mod
    x_T = gen((B, *shape), 820)
    with Recorder(ddim_mod) as rec, contextlib.redirect_stdout(io.StringIO()):
        s_ddim, _ = ddim.sample(10, batch_size=B, shape=shape, eta=1.0, verbose=False, x_T=x_T)
    x_dec = ld.decode_first_stage(s_ddim)
    noises = torch.stack(rec.draws)
    mine = U.ddim_sample_uncond(model_fn, x_T, ld.alphas_cumprod, 10, 1.0, noises)
    print(f"ddim S=10 eta=1 uncond: sample std {float(s_ddim.std()):.3f}; oracle rel {rel(mine, s_ddim):.2e}; "
          f"decode oracle rel {rel(O.decode_first_stage(vsd, s_ddim, SCALE_FACTOR), x_dec):.2e}")
    out["ddim"] = dict(x_T=x_T, noise=noises, sample=s_ddim, x_dec=x_dec)
    for k in ("betas", "alphas_cumprod", "posterior_variance", "posterior_log_variance_clipped", "posterior_mean_coef1",
              "posterior_mean_coef2", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod"):
        out["sched_" + k] = getattr(ld, k).clone()

    # ancestral DDPM (progressive_denoising, sample_diffusion.py --vanilla) on a 20-step schedule
    ld20 = R.build_ld(arch.TINY_ATTN_UNET, arch.TINY_VAE, "__is_unconditional__", **dict(LD_PARAMS, timesteps=20))
    ld20.scale_factor.fill_(SCALE_FACTOR)
    ld20.model.diffusion_model.load_state_dict(usd, strict=True)
    ld20.first_stage_model.load_state_dict(vsd, strict=True)
    x_T = gen((B, *shape), 830)
    with Recorder(ddpm_mod) as rec:
        s_anc, inter = ld20.progressive_denoising(None, [B, *shape], verbose=False, x_T=x_T)
    noises = torch.stack(rec.draws)
    sched = U.ddpm_schedule(20)
    mine, mine_inter = U.progressive_denoising(model_fn, x_T, sched, noises)
    print(f"ancestral T=20: sample std {float(s_anc.std()):.3f}; oracle rel {rel(mine, s_anc):.2e}; "
          f"intermediates {len(inter)} rel {max(rel(a, b) for a, b in zip(mine_inter, inter)):.2e}")
    out["ancestral"] = dict(x_T=x_T, noise=noises, sample=s_anc, intermediates=torch.stack(inter),
                            x_dec=ld20.decode_first_stage(s_anc))

    # EMA: model_ema buffers (LitEma names) hold other weights; ema_scope() must switch to them
    lde = R.build_ld(arch.TINY_ATTN_UNET, arch.TINY_VAE, "__is_unconditional__", **dict(LD_PARAMS, use_ema=True))
    lde.scale_factor.fill_(SCALE_FACTOR)
    lde.model.diffusion_model.load_state_dict(usd, strict=True)
    esd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_ATTN_UNET), EMA_SEED)
    R.load_ema(lde, esd)
    x = gen((B, *shape), 840)
    t = torch.tensor([700, 3])
    raw = lde.apply_model(x, t, None)
    with contextlib.redirect_stdout(io.StringIO()):
        with lde.ema_scope("golden"):
            ema = lde.apply_model(x, t, None)
    after = lde.apply_model(x, t, None)
    assert torch.equal(raw, after) and rel(ema, raw) > 0.1
    print(f"ema: rel(ema, raw) {rel(ema, raw):.2f}; oracle rel {rel(U.unet_forward(esd, arch.TINY_ATTN_UNET, x, t), ema):.2e}")
    out["ema"] = dict(x=x, t=t, eps_raw=raw, eps_ema=ema,
                      ema_keys=sorted(k for k in lde.state_dict() if k.startswith("model_ema.")))
    path = os.path.join(OUT, "lsun.pt")
    torch.save(out, path)
    print(f"  wrote lsun.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
