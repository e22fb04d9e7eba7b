"""ORACLE tooling: generate tests/golden/cin_f8.pt by running the UNMODIFIED reference (located by ref_harness.py) on CPU
fp32 for the class-conditional ImageNet LDM-VQ-8 (models/ldm/cin256/config.yaml; configs/latent-diffusion/
cin-ldm-vq-f8.yaml has the same model node).

Run in the build container:  python oracle/make_golden_cin_f8.py
clip / kornia are stubbed and the VQ quantizer is oracle/vq_oracle.py's (ref_harness.install());
LatentDiffusion, LitEma, ClassEmbedder, UNetModel, VQModelInterface (with its level AttnBlocks) and DDIMSampler are the
reference's own code. Weights come from stable-diffusion_b200/arch.random_state_dict (seeded; the tiny model's EMA copy
from its own seed); inputs are regenerated from the seeds stored next to the outputs. Decoded images are stored at every
IMAGE_STRIDE-th pixel. Every vector is also evaluated with oracle/cin_f8_oracle.py and the error printed. Both YAMLs'
`model:` nodes are stored as parsed data, so no test reads the reference.
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

import cin_f8_oracle as F8  # noqa: E402
import cin_oracle as CO  # noqa: E402
import ref_harness as R  # noqa: E402
from ref_harness import gen, rel  # noqa: E402
import uncond_oracle as U  # noqa: E402
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_SEED, VQ_SEED, COND_SEED, EMA_SEED = 11, 12, 13, 31
LINEAR_START, LINEAR_END = 0.0015, 0.0195
# LatentDiffusion with the cin256/config.yaml parameters (use_ema left at its default, True); the cond stage is
# ClassEmbedder
COND_TARGET = "ldm.modules.encoders.modules.ClassEmbedder"
LD_PARAMS = dict(linear_start=LINEAR_START, linear_end=LINEAR_END, num_timesteps_cond=1, log_every_t=200,
                 timesteps=1000, first_stage_key="image", cond_stage_key="class_label", cond_stage_trainable=True,
                 conditioning_key="crossattn", monitor="val/loss_simple_ema")
YAMLS = ("models/ldm/cin256/config.yaml", "configs/latent-diffusion/cin-ldm-vq-f8.yaml")
# decoded images are stored at every IMAGE_STRIDE-th pixel in both directions (1/16 of the pixels, spread over the whole
# image), which keeps the file small; the tests decode in full and compare the same pixels
IMAGE_STRIDE = 4


def sub(x):
    return x[..., ::IMAGE_STRIDE, ::IMAGE_STRIDE].contiguous()


@torch.no_grad()
def main():
    out = {"unet_seed": UNET_SEED, "vq_seed": VQ_SEED, "cond_seed": COND_SEED, "ema_seed": EMA_SEED,
           "image_stride": IMAGE_STRIDE}
    out["yaml_nodes"] = {}
    for rel_path in YAMLS:
        with open(os.path.join(R.REF, rel_path)) as f:
            out["yaml_nodes"][rel_path] = yaml.safe_load(f)["model"]
    ld = R.build_ld(arch.CIN256_F8_UNET, arch.VQ_F8, {"target": COND_TARGET, "params": arch.CIN256_F8_COND},
                    **LD_PARAMS)
    out["cin256_keys"] = [(k, tuple(v.shape)) for k, v in ld.state_dict().items()]
    out["alphas_cumprod"] = ld.alphas_cumprod.clone()
    del ld

    # UNet eps (apply_model with the ClassEmbedder's context)
    out["unet"] = []
    for tag, cfg, ccfg, shapes in (
        ("tiny", arch.TINY_CIN_F8_UNET, arch.TINY_CIN_F8_COND, [((2, 4, 16, 16), [981, 1]), ((1, 4, 16, 24), [500])]),
        ("cin256", arch.CIN256_F8_UNET, arch.CIN256_F8_COND,
         [((2, 4, 32, 32), [981, 1]), ((2, 4, 64, 64), [700, 11]), ((1, 4, 16, 48), [501])]),
    ):
        ld = R.build_ld(cfg, arch.TINY_VQ_F8, {"target": COND_TARGET, "params": ccfg}, **LD_PARAMS)
        sd = arch.random_state_dict(arch.unet_param_shapes(cfg), UNET_SEED)
        csd = arch.random_state_dict(arch.class_embedder_param_shapes(ccfg), COND_SEED)
        ld.model.diffusion_model.load_state_dict(sd, strict=True)
        ld.cond_stage_model.load_state_dict(csd, strict=True)
        for i, (xs, ts) in enumerate(shapes):
            x = gen(xs, 900 + i)
            t = torch.tensor(ts, dtype=torch.long)
            labels = torch.tensor([25, 999][: xs[0]])
            c = ld.get_learned_conditioning({"class_label": labels})
            eps = ld.apply_model(x, t, c)
            mine = F8.unet_forward(sd, x, t, CO.class_embed(csd, labels))
            print(f"unet {tag} {xs} t={ts}: eps std {float(eps.std()):.3f}  oracle rel-L2 {rel(mine, eps):.2e}")
            out["unet"].append(dict(cfg=tag, x_seed=900 + i, shape=xs, t=t, labels=labels, c=c.clone(), eps=eps))
        del ld

    # first stage: decode (through the quantizer) and encode, reference VQModelInterface
    out["decode"], out["encode"] = [], []
    for tag, cfg, decs, encs in (
        ("tiny", arch.TINY_VQ_F8, [(2, 4, 8, 8), (1, 4, 8, 12)], [(1, 3, 64, 96)]),
        ("vq_f8", arch.VQ_F8, [(2, 4, 32, 32), (1, 4, 16, 48)], [(1, 3, 256, 256)]),
    ):
        sd = arch.random_state_dict(arch.vq_param_shapes(cfg), VQ_SEED)
        m = R.build_vq(cfg)
        m.load_state_dict(sd, strict=True)
        for j, ds in enumerate(decs):
            h = gen(ds, 920 + j)
            x = m.decode(h)
            print(f"decode {tag} {ds} -> {tuple(x.shape)}: oracle rel {rel(F8.vq_decode(sd, h), x):.2e}")
            out["decode"].append(dict(cfg=tag, seed=920 + j, shape=ds, x_shape=tuple(x.shape), x=sub(x)))
        for j, es in enumerate(encs):
            img = gen(es, 930 + j).clamp(-1, 1)
            h = m.encode(img)
            print(f"encode {tag} {es} -> {tuple(h.shape)}: oracle rel {rel(F8.vq_encode(sd, img), h):.2e}")
            out["encode"].append(dict(cfg=tag, seed=930 + j, shape=es, h=h))
        del m

    # the tiny model sampled unguided inside ema_scope (EMA weights from their own seed): DDIM-10 at eta 0 and 1, decode
    ld = R.build_ld(arch.TINY_CIN_F8_UNET, arch.TINY_VQ_F8, {"target": COND_TARGET, "params": arch.TINY_CIN_F8_COND},
                    **LD_PARAMS)
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_CIN_F8_UNET), UNET_SEED)
    esd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_CIN_F8_UNET), EMA_SEED)
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F8), VQ_SEED)
    csd = arch.random_state_dict(arch.class_embedder_param_shapes(arch.TINY_CIN_F8_COND), COND_SEED)
    ld.model.diffusion_model.load_state_dict(usd, strict=True)
    ld.first_stage_model.load_state_dict(vsd, strict=True)
    ld.cond_stage_model.load_state_dict(csd, strict=True)
    R.load_ema(ld, esd)
    out["ema_keys"] = sorted(k for k in ld.state_dict() if k.startswith("model_ema."))
    _, ddim = R.build_samplers(ld)
    import ldm.models.diffusion.ddim as ddim_mod
    classes = torch.tensor([25, 992])
    B, shape = 2, (4, 16, 16)
    c = ld.get_learned_conditioning({"class_label": classes})
    out["ddim"] = dict(classes=classes, x_T_seed=940, noise_seed=960)
    orig = ddim_mod.noise_like
    for eta in (0.0, 1.0):
        x_T = gen((B, *shape), 940)
        draws = []
        # draw i comes from seed noise_seed + i, so the tests regenerate the draws
        ddim_mod.noise_like = lambda shp, device, repeat=False: draws.append(gen(shp, 960 + len(draws))) or draws[-1]
        try:
            with contextlib.redirect_stdout(io.StringIO()), ld.ema_scope():
                s, _ = ddim.sample(10, conditioning=c, batch_size=B, shape=shape, eta=eta, verbose=False, x_T=x_T)
        finally:
            ddim_mod.noise_like = orig
        x_dec = ld.decode_first_stage(s)
        fn = lambda x, t: F8.unet_forward(esd, x, t, CO.class_embed(csd, classes))
        mine = U.ddim_sample_uncond(fn, x_T, ld.alphas_cumprod, 10, eta, torch.stack(draws) if eta else
                                    torch.zeros(10, B, *shape))
        print(f"ddim S=10 eta={eta} (EMA weights): sample std {float(s.std()):.3f}, {len(draws)} draws; oracle rel "
              f"{rel(mine, s):.2e}; decode oracle rel {rel(F8.decode_first_stage(vsd, s), x_dec):.2e}")
        out["ddim"][f"eta{int(eta)}"] = dict(sample=s, x_dec=sub(x_dec), n_noise=len(draws))
    path = os.path.join(OUT, "cin_f8.pt")
    torch.save(out, path)
    print(f"  wrote cin_f8.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
