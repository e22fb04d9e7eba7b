"""ORACLE tooling: generate tests/golden/vq.pt by running the UNMODIFIED reference (located by ref_harness.py) on CPU fp32
for the VQ-f4 latent diffusion models (configs/latent-diffusion/celebahq-ldm-vq-4.yaml, ffhq- and lsun_bedrooms-, which
share the UNet and the first stage).

Run in the build container:  python oracle/make_golden_vq.py
taming's VectorQuantizer2 is not part of the reference checkout: after ref_harness.install() the quantizer class the
reference imports (ldm.models.autoencoder.VectorQuantizer) is set to oracle/vq_oracle.py's restatement, and everything
around it (VQModelInterface, Encoder / Decoder, UNetModel, LatentDiffusion, DDIMSampler) is the reference's own code.
Weights come from stable-diffusion_b200/arch.random_state_dict (seeded); every vector is also evaluated with the oracle
and the error printed.
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
import vq_oracle as V  # noqa: E402
import sdb200  # noqa: E402,F401
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_SEED, VQ_SEED, EMA_SEED = 11, 12, 31
LINEAR_START, LINEAR_END = 0.0015, 0.0195
# LatentDiffusion with the celebahq-ldm-vq-4.yaml parameters
LD_PARAMS = dict(linear_start=LINEAR_START, linear_end=LINEAR_END, num_timesteps_cond=1, log_every_t=200,
                 timesteps=1000, first_stage_key="image", monitor="val/loss_simple_ema", use_ema=True)


@torch.no_grad()
def main():
    out = {"unet_seed": UNET_SEED, "vq_seed": VQ_SEED, "ema_seed": EMA_SEED, "linear_end": LINEAR_END}
    # the reference's key / shape lists, so the CPU tests need no reference
    net = R.build_unet(arch.CELEBAHQ_UNET)
    out["celebahq_unet_keys"] = [(k, tuple(v.shape)) for k, v in net.state_dict().items()]
    del net
    out["vq_f4_keys"] = [(k, tuple(v.shape)) for k, v in R.build_vq(arch.VQ_F4).state_dict().items()]

    out["unet"] = []
    for tag, cfg, shapes in (
        ("tiny_vq", arch.TINY_VQ_UNET, [((2, 3, 16, 16), [981, 1]), ((2, 3, 16, 24), [500, 21])]),
        ("celebahq", arch.CELEBAHQ_UNET, [((2, 3, 32, 32), [981, 1]), ((1, 3, 16, 48), [501])]),
    ):
        sd = arch.random_state_dict(arch.unet_param_shapes(cfg), UNET_SEED)
        net = R.build_unet(cfg)
        net.load_state_dict(sd, strict=True)
        for i, (xs, ts) in enumerate(shapes):
            x = gen(xs, 900 + i)
            t = torch.tensor(ts, dtype=torch.long)
            eps = net(x, t)
            mine = V.unet_forward(sd, cfg, x, t)
            print(f"unet {tag} {xs} t={ts}: eps std {float(eps.std()):.3f}  oracle rel-L2 {rel(mine, eps):.2e}")
            out["unet"].append(dict(cfg=tag, x=x, t=t, eps=eps))
        del net

    # quantizer, decode and encode through the reference's VQModelInterface
    out["quantize"], out["decode"] = [], []
    for tag, cfg, zs, decs in (
        ("tiny_vq", arch.TINY_VQ, (2, 3, 8, 12), [(2, 3, 8, 12)]),
        ("vq_f4", arch.VQ_F4, (2, 3, 16, 24), [(1, 3, 16, 16), (1, 3, 16, 24)]),
    ):
        sd = arch.random_state_dict(arch.vq_param_shapes(cfg), VQ_SEED)
        m = R.build_vq(cfg)
        m.load_state_dict(sd, strict=True)
        z = gen(zs, 910)
        z_q, _, (_, _, idx) = m.quantize(z)
        mine_q, mine_i = V.quantize(z, sd["quantize.embedding.weight"])
        print(f"quantize {tag} {zs}: oracle indices equal {torch.equal(mine_i, idx)}, z_q equal {torch.equal(mine_q, z_q)}")
        out["quantize"].append(dict(cfg=tag, z=z, indices=idx, z_q=z_q))
        for j, ds in enumerate(decs):
            h = gen(ds, 920 + j)
            for fnq in (False, True):
                x = m.decode(h, force_not_quantize=fnq)
                print(f"decode {tag} {ds} force_not_quantize={fnq}: -> {tuple(x.shape)} oracle rel "
                      f"{rel(V.vq_decode(sd, h, fnq), x):.2e}")
                out["decode"].append(dict(cfg=tag, h=h, force_not_quantize=fnq, x=x))
        if tag == "vq_f4":
            img = gen((1, 3, 64, 96), 930).clamp(-1, 1)
            h = m.encode(img)
            print(f"encode {tag} 64x96 -> {tuple(h.shape)} oracle rel {rel(V.vq_encode(sd, img), h):.2e}")
            out["encode"] = dict(cfg=tag, x=img, h=h)

    # DDIM S=10, eta 0 (sample_diffusion.py -e 0) of the tiny VQ LDM inside ema_scope, then decode_first_stage
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_VQ_UNET), UNET_SEED)
    esd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_VQ_UNET), EMA_SEED)
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ), VQ_SEED)
    ld = R.build_ld(arch.TINY_VQ_UNET, arch.TINY_VQ, "__is_unconditional__", **LD_PARAMS)
    ld.model.diffusion_model.load_state_dict(usd, strict=True)
    ld.first_stage_model.load_state_dict(vsd, strict=True)
    R.load_ema(ld, esd)
    _, ddim = R.build_samplers(ld)
    B, shape = 2, [3, 16, 16]
    x_T = gen((B, *shape), 940)
    with contextlib.redirect_stdout(io.StringIO()):
        with ld.ema_scope("golden"):
            s, _ = ddim.sample(10, batch_size=B, shape=shape, eta=0.0, verbose=False, x_T=x_T)
    x_dec = ld.decode_first_stage(s)
    model_fn = lambda x, t: V.unet_forward(esd, arch.TINY_VQ_UNET, x, t)
    mine = U.ddim_sample_uncond(model_fn, x_T, ld.alphas_cumprod, 10, 0.0, torch.zeros(10, B, *shape))
    print(f"ddim S=10 eta=0 (EMA weights): sample std {float(s.std()):.3f}; oracle rel {rel(mine, s):.2e}; "
          f"decode oracle rel {rel(V.decode_first_stage(vsd, s), x_dec):.2e}")
    out["ddim"] = dict(x_T=x_T, sample=s, x_dec=x_dec, alphas_cumprod=ld.alphas_cumprod.clone(),
                       ema_keys=sorted(k for k in ld.state_dict() if k.startswith("model_ema.")))
    path = os.path.join(OUT, "vq.pt")
    torch.save(out, path)
    print(f"  wrote vq.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
