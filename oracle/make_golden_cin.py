"""ORACLE tooling: generate tests/golden/cin.pt by running the UNMODIFIED reference (located by ref_harness.py) on CPU fp32
for the class-conditional ImageNet LDM (configs/latent-diffusion/cin256-v2.yaml; scripts/latent_imagenet_diffusion.ipynb).

Run in the build container:  python oracle/make_golden_cin.py
ldm/modules/encoders/modules.py imports `clip` and `kornia`, which are not installed and which ClassEmbedder does not use:
ref_harness.install() stubs them, and sets the VQ quantizer to oracle/vq_oracle.py's; LatentDiffusion, ClassEmbedder,
UNetModel, VQModelInterface and DDIMSampler are the reference's own code. Weights come from
stable-diffusion_b200/arch.random_state_dict (seeded); every vector is also evaluated with the oracle and the error
printed.
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

import cin_oracle as CO  # noqa: E402
import ldm_oracle as O  # noqa: E402
import ref_harness as R  # noqa: E402
from ref_harness import gen, rel  # noqa: E402
import vq_oracle as V  # noqa: E402
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_SEED, VQ_SEED, COND_SEED = 11, 12, 13
LINEAR_START, LINEAR_END = 0.0015, 0.0195
# LatentDiffusion with the cin256-v2.yaml parameters; the cond stage is ClassEmbedder
COND_TARGET = "ldm.modules.encoders.modules.ClassEmbedder"
LD_PARAMS = dict(linear_start=LINEAR_START, linear_end=LINEAR_END, num_timesteps_cond=1, log_every_t=200,
                 timesteps=1000, first_stage_key="image", cond_stage_key="class_label", cond_stage_trainable=True,
                 conditioning_key="crossattn", monitor="val/loss", use_ema=False)


@torch.no_grad()
def main():
    out = {"unet_seed": UNET_SEED, "vq_seed": VQ_SEED, "cond_seed": COND_SEED, "linear_end": LINEAR_END}
    # the reference's key / shape list of the whole cin256-v2 model, so the CPU tests need no reference
    ld = R.build_ld(arch.CIN256_V2_UNET, arch.VQ_F4, {"target": COND_TARGET, "params": arch.CIN256_V2_COND},
                    **LD_PARAMS)
    out["cin256_keys"] = [(k, tuple(v.shape)) for k, v in ld.state_dict().items()]
    del ld

    out["unet"] = []
    for tag, cfg, ccfg, shapes in (
        ("tiny_cin", arch.TINY_CIN_UNET, arch.TINY_CIN_COND, [((2, 3, 16, 16), [981, 1]), ((2, 3, 16, 24), [500, 21])]),
        ("cin256", arch.CIN256_V2_UNET, arch.CIN256_V2_COND,
         [((2, 3, 32, 32), [981, 1]), ((2, 3, 64, 64), [700, 11]), ((1, 3, 16, 48), [501])]),
    ):
        ld = R.build_ld(cfg, arch.TINY_VQ, {"target": COND_TARGET, "params": ccfg}, **LD_PARAMS)
        sd = arch.random_state_dict(arch.unet_param_shapes(cfg), UNET_SEED)
        csd = arch.random_state_dict(arch.class_embedder_param_shapes(ccfg), COND_SEED)
        ld.model.diffusion_model.load_state_dict(sd, strict=True)
        ld.cond_stage_model.load_state_dict(csd, strict=True)
        for i, (xs, ts) in enumerate(shapes):
            x = gen(xs, 900 + i)
            t = torch.tensor(ts, dtype=torch.long)
            labels = torch.tensor([25, 1000][: xs[0]])
            c = ld.get_learned_conditioning({"class_label": labels})
            eps = ld.apply_model(x, t, c)
            mine = O.unet_forward(sd, x, t, CO.class_embed(csd, labels), num_heads=1)
            print(f"unet {tag} {xs} t={ts}: eps std {float(eps.std()):.3f}  oracle rel-L2 {rel(mine, eps):.2e}")
            out["unet"].append(dict(cfg=tag, x=x, t=t, labels=labels, c=c.clone(), eps=eps))
        del ld

    # the notebook's sampling cell on the tiny model: DDIM-10, eta 0, scale 3.0, uc from label 1000, then decode
    ld = R.build_ld(arch.TINY_CIN_UNET, arch.TINY_VQ, {"target": COND_TARGET, "params": arch.TINY_CIN_COND},
                    **LD_PARAMS)
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_CIN_UNET), UNET_SEED)
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ), VQ_SEED)
    csd = arch.random_state_dict(arch.class_embedder_param_shapes(arch.TINY_CIN_COND), COND_SEED)
    ld.model.diffusion_model.load_state_dict(usd, strict=True)
    ld.first_stage_model.load_state_dict(vsd, strict=True)
    ld.cond_stage_model.load_state_dict(csd, strict=True)
    _, ddim = R.build_samplers(ld)
    classes = torch.tensor([25, 187, 448, 992])
    B, shape = 4, [3, 16, 16]
    x_T = gen((B, *shape), 940)
    with contextlib.redirect_stdout(io.StringIO()):
        with ld.ema_scope():
            uc = ld.get_learned_conditioning({"class_label": torch.full((B,), 1000)})
            c = ld.get_learned_conditioning({"class_label": classes})
            s, _ = ddim.sample(10, conditioning=c, batch_size=B, shape=shape, verbose=False,
                               unconditional_guidance_scale=3.0, unconditional_conditioning=uc, eta=0.0, x_T=x_T)
    x_dec = ld.decode_first_stage(s)
    fn = lambda x, t, ctx: O.unet_forward(usd, x, t, ctx, num_heads=1)
    mine = CO.ddim_sample_guided(fn, x_T, CO.class_embed(csd, classes), CO.class_embed(csd, torch.full((B,), 1000)), 3.0,
                                 ld.alphas_cumprod, 10)
    print(f"guided ddim S=10 eta=0: sample std {float(s.std()):.3f}; oracle rel {rel(mine, s):.2e}; "
          f"decode oracle rel {rel(V.decode_first_stage(vsd, s), x_dec):.2e}")
    out["ddim"] = dict(classes=classes, x_T=x_T, sample=s, x_dec=x_dec, alphas_cumprod=ld.alphas_cumprod.clone())
    path = os.path.join(OUT, "cin.pt")
    torch.save(out, path)
    print(f"  wrote cin.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
