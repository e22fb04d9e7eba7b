"""ORACLE tooling: generate tests/golden/rdm.pt by running the UNMODIFIED reference (located by ref_harness.py) on CPU
fp32 for the retrieval-augmented diffusion model (configs/retrieval-augmented-diffusion/768x768.yaml, scripts/knn2img.py).

Run in the build container:  python oracle/make_golden_rdm.py
clip / kornia are stubbed by ref_harness.install() (the model's cond stage is torch.nn.Identity; the CLIP text
embedder is checked against transformers on the GPU instead). LatentDiffusion, LitEma, UNetModel, AutoencoderKL (KL-f16,
with its level AttnBlocks), DDIMSampler and PLMSSampler are the reference's own code. Weights come from
stable-diffusion_b200/arch.random_state_dict (seeded; the tiny model's EMA copy from its own seed); inputs are regenerated
from the seeds stored next to the outputs. Conditioning is [text | neighbours]: unit-norm rows from a seed, as
FrozenCLIPTextEmbedder and the Searcher produce them. Decoded images are stored at every IMAGE_STRIDE-th pixel and UNet
outputs at every EPS_STRIDE-th latent pixel, in both directions, which keeps the file small; the tests compute in full
and compare the same pixels. Every vector is also evaluated with oracle/rdm_oracle.py and the error printed. The YAML's `model:` node is stored as parsed
data, so no test reads the reference.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys

import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import rdm_oracle as RO  # noqa: E402
import ref_harness as R  # noqa: E402
from ref_harness import gen, rel  # noqa: E402
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_SEED, VAE_SEED, EMA_SEED = 11, 12, 31
YAML = "configs/retrieval-augmented-diffusion/768x768.yaml"
SCALE_FACTOR = 0.22765929
IMAGE_STRIDE = 8
EPS_STRIDE = 2
GUIDANCE = 5.0
# LatentDiffusion with the 768x768.yaml parameters (use_ema left at its default, True); the cond stage is Identity
LD_PARAMS = dict(linear_start=0.0015, linear_end=0.015, num_timesteps_cond=1, log_every_t=200, timesteps=1000,
                 first_stage_key="jpg", cond_stage_key="nix", cond_stage_trainable=False, conditioning_key="crossattn",
                 monitor="val/loss_simple_ema", scale_by_std=False, scale_factor=SCALE_FACTOR)
LD_COND = {"target": "torch.nn.Identity"}


def sub(x):
    return x[..., ::IMAGE_STRIDE, ::IMAGE_STRIDE].contiguous()


def unit_rows(shape, seed):
    """Conditioning tokens as the embedder and the searcher give them: rows of unit L2 norm."""
    x = gen(shape, seed)
    return x / torch.linalg.norm(x, dim=-1, keepdim=True)


@torch.no_grad()
def main():
    out = {"unet_seed": UNET_SEED, "vae_seed": VAE_SEED, "ema_seed": EMA_SEED, "image_stride": IMAGE_STRIDE,
           "eps_stride": EPS_STRIDE,
           "scale_factor": SCALE_FACTOR, "guidance": GUIDANCE}
    with open(os.path.join(R.REF, YAML)) as f:
        out["yaml_node"] = yaml.safe_load(f)["model"]
    ld = R.build_ld(arch.RDM_UNET, arch.KL_F16, LD_COND, **LD_PARAMS)
    out["rdm_keys"] = [(k, tuple(v.shape)) for k, v in ld.state_dict().items()]
    out["alphas_cumprod"] = ld.alphas_cumprod.clone()
    del ld

    # UNet eps (apply_model with the crossattn context [text | neighbours])
    out["unet"] = []
    for tag, cfg, cases in (
        ("tiny", arch.TINY_RDM_UNET, [((2, 16, 16, 16), 3, [981, 1])]),
        ("rdm", arch.RDM_UNET, [((2, 16, 48, 48), 11, [981, 1]), ((2, 16, 48, 48), 1, [700, 11]),
                                ((1, 16, 24, 48), 11, [501])]),
    ):
        unet = R.build_unet(cfg)
        sd = arch.random_state_dict(arch.unet_param_shapes(cfg), UNET_SEED)
        unet.load_state_dict(sd, strict=True)
        for i, (xs, n_ctx, ts) in enumerate(cases):
            seed = 900 + 10 * len(out["unet"])
            x = gen(xs, seed)
            t = torch.tensor(ts, dtype=torch.long)
            c = unit_rows((xs[0], n_ctx, cfg["context_dim"]), seed + 1)
            eps = unet(x, t, context=c)
            mine = RO.unet_forward(sd, x, t, c)
            print(f"unet {tag} {xs} ctx {n_ctx} t={ts}: eps std {float(eps.std()):.3f}  oracle rel-L2 "
                  f"{rel(mine, eps):.2e}")
            out["unet"].append(dict(cfg=tag, seed=seed, shape=xs, n_ctx=n_ctx, t=t,
                                    eps=eps[..., ::EPS_STRIDE, ::EPS_STRIDE].contiguous()))
        del unet, sd

    # first stage: KL decode and encode (moments), reference AutoencoderKL
    out["decode"], out["encode"] = [], []
    for tag, cfg, decs, encs in (
        ("tiny", arch.TINY_KL_F16, [(2, 16, 8, 8), (1, 16, 4, 6)], [(1, 3, 64, 96)]),
        ("kl_f16", arch.KL_F16, [(1, 16, 48, 48)], []),
    ):
        sd = arch.random_state_dict(arch.vae_param_shapes(cfg), VAE_SEED)
        m = R.build_vae(cfg)
        m.load_state_dict(sd, strict=True)
        for j, ds in enumerate(decs):
            z = gen(ds, 920 + j)
            x = m.decode(z)
            print(f"decode {tag} {ds} -> {tuple(x.shape)}: oracle rel {rel(RO.kl_decode(sd, z), x):.2e}")
            out["decode"].append(dict(cfg=tag, seed=920 + j, shape=ds, x_shape=tuple(x.shape), x=sub(x)))
        for j, es in enumerate(encs):
            img = gen(es, 930 + j).clamp(-1, 1)
            moments = m.encode(img).parameters
            print(f"encode {tag} {es} -> {tuple(moments.shape)}: oracle rel "
                  f"{rel(RO.kl_encode_moments(sd, img), moments):.2e}")
            out["encode"].append(dict(cfg=tag, seed=930 + j, shape=es, moments=moments.clone()))
        del m

    # the tiny model, guided (uc = 0) inside ema_scope: DDIM-10 at eta 0 and 1, PLMS-10; c = [text | 2 neighbours]
    ld = R.build_ld(arch.TINY_RDM_UNET, arch.TINY_KL_F16, LD_COND, **LD_PARAMS)
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_RDM_UNET), UNET_SEED)
    esd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_RDM_UNET), EMA_SEED)
    vsd = arch.random_state_dict(arch.vae_param_shapes(arch.TINY_KL_F16), VAE_SEED)
    ld.model.diffusion_model.load_state_dict(usd, strict=True)
    ld.first_stage_model.load_state_dict(vsd, strict=True)
    R.load_ema(ld, esd)
    plms, ddim = R.build_samplers(ld)
    import ldm.models.diffusion.ddim as ddim_mod
    B, shape = 2, (16, 16, 16)
    c = unit_rows((B, 3, arch.TINY_RDM_UNET["context_dim"]), 950)
    uc = torch.zeros_like(c)
    out["sampling"] = dict(c_seed=950, x_T_seed=940, noise_seed=960)
    fn = lambda x, t, ctx: RO.unet_forward(esd, x, t, ctx)
    orig = ddim_mod.noise_like
    for name in ("ddim_eta0", "ddim_eta1", "plms"):
        x_T = gen((B, *shape), 940)
        draws = []
        ddim_mod.noise_like = lambda shp, device, repeat=False: draws.append(gen(shp, 960 + len(draws))) or draws[-1]
        try:
            with contextlib.redirect_stdout(io.StringIO()), ld.ema_scope():
                kw = dict(conditioning=c, batch_size=B, shape=shape, verbose=False, x_T=x_T,
                          unconditional_guidance_scale=GUIDANCE, unconditional_conditioning=uc)
                if name == "plms":
                    s, _ = plms.sample(10, eta=0.0, **kw)
                else:
                    s, _ = ddim.sample(10, eta=float(name[-1]), **kw)
        finally:
            ddim_mod.noise_like = orig
        x_dec = ld.decode_first_stage(s)
        if name == "plms":
            mine = RO.plms_sample(fn, x_T, c, uc, GUIDANCE, ld.alphas_cumprod, 10)
        else:
            eta = float(name[-1])
            mine = RO.ddim_sample(fn, x_T, c, uc, GUIDANCE, ld.alphas_cumprod, 10, eta,
                                  torch.stack(draws) if eta else torch.zeros(10, B, *shape))
        print(f"{name} S=10 (EMA weights, scale {GUIDANCE}): sample std {float(s.std()):.3f}, {len(draws)} draws; oracle "
              f"rel {rel(mine, s):.2e}; decode oracle rel {rel(RO.decode_first_stage(vsd, s), x_dec):.2e}")
        out["sampling"][name] = dict(sample=s, x_dec=sub(x_dec), n_noise=len(draws))
    path = os.path.join(OUT, "rdm.pt")
    torch.save(out, path)
    print(f"  wrote rdm.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
