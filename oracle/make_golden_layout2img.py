"""ORACLE tooling: generate tests/golden/layout2img.pt by running the UNMODIFIED reference (located by ref_harness.py) on
CPU fp32 for the layout-to-image LDM (models/ldm/layout2img-openimages256/config.yaml: spatial transformers of depth 3
with heads of num_head_channels 32 on a 512-wide context, BERTEmbedder(n_embed=512, n_layer=16, vocab_size=8192,
max_seq_len=92) fed token ids, VQ-f4 first stage, use_ema left at its default, True).

Run in the build container:  python oracle/make_golden_layout2img.py
clip / kornia are stubbed and the VQ quantizer is oracle/vq_oracle.py's (ref_harness.install()). LatentDiffusion, LitEma,
BERTEmbedder, UNetModel, VQModelInterface and DDIMSampler are the reference's own code. Weights come from
stable-diffusion_b200/arch.random_state_dict (seeded); inputs are stored or regenerated from stored seeds. Every vector
is also evaluated with the oracles (bert_oracle, layout2img_oracle's UNet with heads of num_head_channels and every
block of each spatial transformer, vq_oracle's decode, uncond_oracle's DDIM loop) and the error printed.

Contents: the YAML's `model:` node as parsed data, the reference's key / shape list of the whole model (model_ema.*
included); alphas_cumprod; the full-size BERT output for 2 x 92 ids (stored as fp16); the full-size UNet's eps at
(2, 3, 64, 64) with two different 92 x 512 contexts at two timesteps; a tiny unguided trajectory (10 steps) for DDIM at
eta 0 and 1 (the eta 1 noise draws from stored seeds) as LatentDiffusion.log_images samples it - inside ema_scope(), on
an EMA weight set that differs from the raw one - each with decode_first_stage (VQ re-quantization).
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

import bert_oracle as BO  # noqa: E402
import layout2img_oracle as L  # noqa: E402
import ref_harness as R  # noqa: E402
import uncond_oracle as U  # noqa: E402
import vq_oracle as VO  # noqa: E402
from ref_harness import gen, rel  # noqa: E402
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
YAML = "models/ldm/layout2img-openimages256/config.yaml"
UNET_SEED, VQ_SEED, BERT_SEED, EMA_SEED = 11, 12, 13, 31
LINEAR_START, LINEAR_END = 0.0015, 0.0205
# LatentDiffusion with the layout2img-openimages256/config.yaml parameters (scale_factor and use_ema at their defaults)
LD_PARAMS = dict(linear_start=LINEAR_START, linear_end=LINEAR_END, log_every_t=100, timesteps=1000, loss_type="l1",
                 first_stage_key="image", cond_stage_key="coordinates_bbox", cond_stage_trainable=True,
                 conditioning_key="crossattn", monitor="val/loss_simple_ema")
STEPS = 10


def bert_cond(cfg):
    """The cond stage node: BERTEmbedder fed token ids, as in the YAML."""
    return {"target": "ldm.modules.encoders.modules.BERTEmbedder",
            "params": {**cfg, "use_tokenizer": False}}


def layout_ids(B, seed, vocab_size=8192, n=92):
    """Seeded stand-ins for the bounding-box token ids: B rows of n ids in [0, vocab_size)."""
    return torch.randint(0, vocab_size, (B, n), generator=torch.Generator().manual_seed(seed))


@torch.no_grad()
def main():
    out = {"unet_seed": UNET_SEED, "vq_seed": VQ_SEED, "bert_seed": BERT_SEED, "ema_seed": EMA_SEED, "steps": STEPS}
    with open(os.path.join(R.REF, YAML)) as f:
        out["yaml_node"] = yaml.safe_load(f)["model"]
    node = out["yaml_node"]["params"]
    assert node["unet_config"]["params"] == arch.LAYOUT2IMG_UNET
    assert node["cond_stage_config"]["params"] == {**arch.LAYOUT2IMG_BERT, "use_tokenizer": False}
    assert {k: v for k, v in node["first_stage_config"]["params"].items() if k not in ("lossconfig", "monitor")} == \
        arch.VQ_F4
    ld = R.build_ld(arch.LAYOUT2IMG_UNET, arch.VQ_F4, bert_cond(arch.LAYOUT2IMG_BERT), **LD_PARAMS)
    assert ld.use_ema and ld.bbox_tokenizer is None
    out["keys"] = [(k, tuple(v.shape)) for k, v in ld.state_dict().items()]
    out["alphas_cumprod"] = ld.alphas_cumprod.clone()
    del ld

    # full-size BERT-512 x 16 on 92 ids
    R.install()
    from ldm.modules.encoders.modules import BERTEmbedder
    cfg = arch.LAYOUT2IMG_BERT
    ref = BERTEmbedder(**cfg, use_tokenizer=False).eval()
    bsd = arch.random_state_dict(arch.bert_param_shapes(cfg), BERT_SEED)
    ref.load_state_dict(bsd, strict=True)
    ids = layout_ids(2, 520)
    z = ref.encode(ids)
    print(f"bert full {tuple(z.shape)}: std {float(z.std()):.3f}  oracle rel-L2 {rel(BO.bert_embed(bsd, ids), z):.2e}")
    out["bert"] = dict(ids=ids, z=z.half())
    del ref, bsd

    # full-size UNet: two samples with different contexts at two timesteps
    unet = R.build_unet(arch.LAYOUT2IMG_UNET)
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.LAYOUT2IMG_UNET), UNET_SEED)
    unet.load_state_dict(usd, strict=True)
    out["unet"] = []
    for i, ts in enumerate((981, 1)):
        x = gen((2, 3, 64, 64), 900 + i)
        t = torch.tensor([ts, ts], dtype=torch.long)
        ctx_seed = 950 + i
        ctx = gen((2, 92, 512), ctx_seed)
        eps = unet(x, t, context=ctx)
        mine = L.unet_forward(usd, x, t, ctx)
        print(f"unet full (2, 3, 64, 64) t={ts}: eps std {float(eps.std()):.3f}  oracle rel-L2 {rel(mine, eps):.2e}")
        out["unet"].append(dict(x_seed=900 + i, t=t, ctx_seed=ctx_seed, eps=eps))
    del unet, usd

    # the tiny model through log_images' call sequence: c of the ids, ema_scope(), unguided DDIM, decode_first_stage
    ld = R.build_ld(arch.TINY_LAYOUT2IMG_UNET, arch.TINY_VQ_F4, bert_cond(arch.TINY_LAYOUT2IMG_BERT), **LD_PARAMS)
    ushapes = arch.unet_param_shapes(arch.TINY_LAYOUT2IMG_UNET)
    usd = arch.random_state_dict(ushapes, UNET_SEED)
    esd = arch.random_state_dict(ushapes, EMA_SEED)
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F4), VQ_SEED)
    bsd = arch.random_state_dict(arch.bert_param_shapes(arch.TINY_LAYOUT2IMG_BERT), BERT_SEED)
    ld.model.diffusion_model.load_state_dict(usd, strict=True)
    R.load_ema(ld, esd)
    ld.first_stage_model.load_state_dict(vsd, strict=True)
    ld.cond_stage_model.load_state_dict(bsd, strict=True)
    _, ddim = R.build_samplers(ld)
    import ldm.models.diffusion.ddim as ddim_mod
    B, shape = 2, [3, 16, 16]
    ids = layout_ids(B, 530)
    x_T = gen((B, *shape), 940)
    c = ld.get_learned_conditioning(ids)
    out["tiny"] = dict(ids=ids, x_T=x_T, noise_seed=960)
    unet_fn = lambda x, t: L.unet_forward(esd, x, t, BO.bert_embed(bsd, ids))
    orig = ddim_mod.noise_like
    for eta in (0, 1):
        draws = []
        # DDIM at eta 1: draw i comes from seed noise_seed + i, so the tests regenerate the draws
        ddim_mod.noise_like = lambda shp, device, repeat=False: draws.append(gen(shp, 960 + len(draws))) or draws[-1]
        try:
            with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
                with ld.ema_scope("Plotting"):
                    s, _ = ddim.sample(STEPS, batch_size=B, shape=shape, conditioning=c, verbose=False,
                                       eta=float(eta), x_T=x_T)
        finally:
            ddim_mod.noise_like = orig
        x_dec = ld.decode_first_stage(s)
        mine = U.ddim_sample_uncond(unet_fn, x_T, out["alphas_cumprod"], STEPS, float(eta),
                                    torch.stack(draws) if eta else torch.zeros(STEPS, B, *shape))
        print(f"ddim eta {eta} S={STEPS}: sample std {float(s.std()):.3f}, {len(draws)} draws; oracle rel "
              f"{rel(mine, s):.2e}; decode oracle rel {rel(VO.decode_first_stage(vsd, s), x_dec):.2e}")
        out["tiny"][f"ddim_eta{eta}"] = dict(sample=s, x_dec=x_dec, n_noise=len(draws))
    path = os.path.join(OUT, "layout2img.pt")
    torch.save(out, path)
    print(f"  wrote layout2img.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
