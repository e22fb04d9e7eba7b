"""ORACLE tooling: generate tests/golden/text2img256.pt by running the UNMODIFIED reference (located by ref_harness.py) on
CPU fp32 for the text-conditional LDM-VQ-4 (models/ldm/text2img256/config.yaml: BERTEmbedder(n_embed=640, n_layer=32),
spatial transformers with heads of num_head_channels 32 on a 640-wide context, VQ-f4 first stage, use_ema left at its
default, True).

Run in the build container:  python oracle/make_golden_text2img256.py
clip / kornia are stubbed and the VQ quantizer is oracle/vq_oracle.py's (ref_harness.install()). BERTEmbedder is built
with use_tokenizer=False and fed token ids, as in make_golden_laion.py. LatentDiffusion, LitEma, BERTEmbedder,
UNetModel, VQModelInterface, DDIMSampler, PLMSSampler and DPMSolverSampler are the reference's own code. Weights come
from stable-diffusion_b200/arch.random_state_dict (seeded); inputs are stored or regenerated from stored seeds. Every
vector is also evaluated with the oracles (bert_oracle, cin_f8_oracle's UNet with heads of num_head_channels,
vq_oracle's decode, ldm_oracle's / uncond_oracle's samplers) and the error printed.

Contents: the YAML's `model:` node as parsed data, the reference's key / shape list of the whole model (model_ema.*
included); the full-size UNet's eps of a guidance batch [uncond; cond] at (2, 3, 64, 64) at two timesteps; the full-size
BERT output for 2 x 77 ids (stored as fp16); a tiny guided trajectory (scale 5.0, 10 steps) for DDIM at eta 0 and 1
(the eta 1 noise draws from stored seeds), PLMS and DPM-Solver, each with decode_first_stage (VQ re-quantization).
"""
from __future__ import annotations

import contextlib
import functools
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
import cin_f8_oracle as F8  # noqa: E402
import ldm_oracle as O  # noqa: E402
import ref_harness as R  # noqa: E402
import uncond_oracle as U  # noqa: E402
import vq_oracle as VO  # noqa: E402
from ref_harness import gen, rel  # noqa: E402
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
YAML = "models/ldm/text2img256/config.yaml"
UNET_SEED, VQ_SEED, BERT_SEED = 11, 12, 13
LINEAR_START, LINEAR_END = 0.0015, 0.0195
# LatentDiffusion with the text2img256/config.yaml parameters (scale_factor and use_ema at their defaults, 1.0 / True)
LD_PARAMS = dict(linear_start=LINEAR_START, linear_end=LINEAR_END, num_timesteps_cond=1, log_every_t=200,
                 timesteps=1000, first_stage_key="image", cond_stage_key="caption", cond_stage_trainable=True,
                 conditioning_key="crossattn", monitor="val/loss_simple_ema")
SCALE, STEPS = 5.0, 10


def bert_cond(cfg):
    """The cond stage node: BERTEmbedder without tokenizer."""
    return {"target": "ldm.modules.encoders.modules.BERTEmbedder",
            "params": {"n_embed": cfg["n_embed"], "n_layer": cfg["n_layer"], "vocab_size": cfg["vocab_size"],
                       "use_tokenizer": False}}


def prompt_ids(vocab_size, seed, B=2, n_tok=20):
    """Rows 0 .. B-2: [CLS] + n_tok seeded ids + [SEP] + [PAD]...; the last row: the empty prompt [CLS] [SEP] [PAD]..."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros((B, 77), dtype=torch.long)
    ids[:, 0] = 101
    lo = 999 if vocab_size > 2000 else 103
    for b in range(B - 1):
        ids[b, 1:1 + n_tok] = torch.randint(lo, vocab_size, (n_tok,), generator=g)
        ids[b, 1 + n_tok] = 102
    ids[B - 1, 1] = 102
    return ids


@torch.no_grad()
def main():
    out = {"unet_seed": UNET_SEED, "vq_seed": VQ_SEED, "bert_seed": BERT_SEED, "scale": SCALE, "steps": STEPS}
    with open(os.path.join(R.REF, YAML)) as f:
        out["yaml_node"] = yaml.safe_load(f)["model"]
    node = out["yaml_node"]["params"]
    assert node["unet_config"]["params"] == arch.TEXT2IMG256_UNET
    assert node["cond_stage_config"]["params"] == {k: arch.TEXT2IMG256_BERT[k] for k in ("n_embed", "n_layer")}
    assert {k: v for k, v in node["first_stage_config"]["params"].items() if k != "lossconfig"} == arch.VQ_F4
    ld = R.build_ld(arch.TEXT2IMG256_UNET, arch.VQ_F4, bert_cond(arch.TEXT2IMG256_BERT), **LD_PARAMS)
    out["keys"] = [(k, tuple(v.shape)) for k, v in ld.state_dict().items()]
    out["alphas_cumprod"] = ld.alphas_cumprod.clone()
    del ld

    # full-size BERT-640 x 32: a prompt row and the empty-prompt row
    R.install()
    from ldm.modules.encoders.modules import BERTEmbedder
    cfg = arch.TEXT2IMG256_BERT
    ref = BERTEmbedder(n_embed=cfg["n_embed"], n_layer=cfg["n_layer"], use_tokenizer=False).eval()
    bsd = arch.random_state_dict(arch.bert_param_shapes(cfg), BERT_SEED)
    ref.load_state_dict(bsd, strict=True)
    ids = prompt_ids(cfg["vocab_size"], 520)
    z = ref.encode(ids)
    print(f"bert full {tuple(z.shape)}: std {float(z.std()):.3f}  oracle rel-L2 {rel(BO.bert_embed(bsd, ids), z):.2e}")
    out["bert"] = dict(ids=ids, z=z.half())
    del ref, bsd

    # full-size UNet: a guidance batch (the same x_t twice, the uncond and the cond context) at two timesteps
    unet = R.build_unet(arch.TEXT2IMG256_UNET)
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TEXT2IMG256_UNET), UNET_SEED)
    unet.load_state_dict(usd, strict=True)
    out["unet"] = []
    for i, ts in enumerate((981, 1)):
        x = gen((1, 3, 64, 64), 900 + i).repeat(2, 1, 1, 1)
        t = torch.tensor([ts, ts], dtype=torch.long)
        ctx_seed = 950 + i
        ctx = gen((2, 77, 640), ctx_seed)
        eps = unet(x, t, context=ctx)
        mine = F8.unet_forward(usd, x, t, ctx)
        print(f"unet full (2, 3, 64, 64) t={ts}: eps std {float(eps.std()):.3f}  oracle rel-L2 {rel(mine, eps):.2e}")
        out["unet"].append(dict(x_seed=900 + i, t=t, ctx_seed=ctx_seed, eps=eps))
    del unet, usd

    # the tiny model through txt2img's call sequence: uc from the empty prompt, guided sampling, decode_first_stage
    ld = R.build_ld(arch.TINY_TEXT2IMG256_UNET, arch.TINY_VQ_F4, bert_cond(arch.TINY_BERT), **LD_PARAMS)
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_TEXT2IMG256_UNET), UNET_SEED)
    vsd = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F4), VQ_SEED)
    bsd = arch.random_state_dict(arch.bert_param_shapes(arch.TINY_BERT), BERT_SEED)
    ld.model.diffusion_model.load_state_dict(usd, strict=True)
    ld.first_stage_model.load_state_dict(vsd, strict=True)
    ld.cond_stage_model.load_state_dict(bsd, strict=True)
    plms, ddim = R.build_samplers(ld)
    from ldm.models.diffusion.dpm_solver import DPMSolverSampler
    import ldm.models.diffusion.ddim as ddim_mod
    DPMSolverSampler.register_buffer = lambda s, n, a: setattr(s, n, a)
    dpm = DPMSolverSampler(ld)
    B, shape = 2, [3, 16, 16]
    rows = prompt_ids(arch.TINY_BERT["vocab_size"], 530, B=B + 1)
    ids, uc_ids = rows[:B], rows[B:].repeat(B, 1)
    x_T = gen((B, *shape), 940)
    with contextlib.redirect_stdout(io.StringIO()):
        uc = ld.get_learned_conditioning(uc_ids)
        c = ld.get_learned_conditioning(ids)
    out["tiny"] = dict(ids=ids, uc_ids=uc_ids, x_T=x_T, noise_seed=960)
    sched = O.register_schedule(linear_start=LINEAR_START, linear_end=LINEAR_END)
    unet_fn = lambda x, t, ctx: F8.unet_forward(usd, x, t, ctx)
    guided = lambda x, t: O._guided_eps(unet_fn, x, t, BO.bert_embed(bsd, ids), BO.bert_embed(bsd, uc_ids), SCALE)
    kw = dict(conditioning=c, batch_size=B, shape=shape, verbose=False, unconditional_guidance_scale=SCALE,
              unconditional_conditioning=uc, x_T=x_T)
    orig = ddim_mod.noise_like
    for name in ("ddim_eta0", "ddim_eta1", "plms", "dpm_solver"):
        draws = []
        # DDIM at eta 1: draw i comes from seed noise_seed + i, so the tests regenerate the draws
        ddim_mod.noise_like = lambda shp, device, repeat=False: draws.append(gen(shp, 960 + len(draws))) or draws[-1]
        try:
            with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
                if name.startswith("ddim"):
                    s, _ = ddim.sample(STEPS, eta=float(name[-1]), **kw)
                elif name == "plms":
                    s, _ = plms.sample(STEPS, eta=0.0, **kw)
                else:
                    s, _ = dpm.sample(STEPS, eta=0.0, **kw)
        finally:
            ddim_mod.noise_like = orig
        x_dec = ld.decode_first_stage(s)
        if name.startswith("ddim"):
            eta = float(name[-1])
            mine = U.ddim_sample_uncond(guided, x_T, sched["alphas_cumprod"], STEPS, eta,
                                        torch.stack(draws) if eta else torch.zeros(STEPS, B, *shape))
        elif name == "plms":
            with _schedule(O):
                mine = O.plms_sample(unet_fn, x_T, BO.bert_embed(bsd, ids), BO.bert_embed(bsd, uc_ids), SCALE, S=STEPS)
        else:
            mine = O.dpm_solver_sample(unet_fn, x_T, BO.bert_embed(bsd, ids), BO.bert_embed(bsd, uc_ids), SCALE,
                                       S=STEPS, sched=sched)
        print(f"{name} S={STEPS} scale {SCALE}: sample std {float(s.std()):.3f}, {len(draws)} draws; oracle rel "
              f"{rel(mine, s):.2e}; decode oracle rel {rel(VO.decode_first_stage(vsd, s), x_dec):.2e}")
        out["tiny"][name] = dict(sample=s, x_dec=x_dec, n_noise=len(draws))
    path = os.path.join(OUT, "text2img256.pt")
    torch.save(out, path)
    print(f"  wrote text2img256.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


@contextlib.contextmanager
def _schedule(oracle):
    """ldm_oracle's PLMS reads SD-v1's schedule from register_schedule(); text2img256 has its own linear_start / end."""
    orig = oracle.register_schedule
    oracle.register_schedule = functools.partial(orig, linear_start=LINEAR_START, linear_end=LINEAR_END)
    try:
        yield
    finally:
        oracle.register_schedule = orig


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
