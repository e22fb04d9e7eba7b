"""ORACLE tooling: generate tests/golden/laion.pt by running the UNMODIFIED reference (located by ref_harness.py) on CPU
fp32 for the LAION-400M text-to-image LDM (configs/latent-diffusion/txt2img-1p4B-eval.yaml; scripts/txt2img.py
--laion400m).

Run in the build container:  python oracle/make_golden_laion.py
ldm/modules/encoders/modules.py imports `clip` and `kornia`, which are not installed and which BERTEmbedder does not use:
ref_harness.install() stubs them. BERTEmbedder is always built with use_tokenizer=False and fed token ids
(use_tokenizer=True would fetch the bert-base-uncased tokenizer). LatentDiffusion, BERTEmbedder, UNetModel,
AutoencoderKL and PLMSSampler are the reference's own code. Weights come from stable-diffusion_b200/arch.random_state_dict
(seeded); every vector is also evaluated with the oracle and the error printed.

Contents: the reference's key / shape list of the whole LAION model; BERT outputs of a prompt row and the empty-prompt
row ([CLS] [SEP] [PAD]...) for the tiny and the full-size encoder (the full-size output stored as fp16 to keep the file
small: that rounding is below 2e-4 rel-L2); UNet eps of the tiny and the full-size UNet (contexts regenerated from their
seeds by the tests); a tiny guided PLMS-10 run from token ids to the decoded image.
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

import bert_oracle as BO  # noqa: E402
import ldm_oracle as O  # noqa: E402
import ref_harness as R  # noqa: E402
from ref_harness import gen, rel  # noqa: E402
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_SEED, VAE_SEED, BERT_SEED = 11, 12, 13
# LatentDiffusion with the txt2img-1p4B-eval.yaml parameters
LD_PARAMS = dict(linear_start=0.00085, linear_end=0.012, num_timesteps_cond=1, log_every_t=200, timesteps=1000,
                 first_stage_key="image", cond_stage_key="caption", image_size=32, channels=4,
                 cond_stage_trainable=True, conditioning_key="crossattn", monitor="val/loss_simple_ema",
                 scale_factor=0.18215, use_ema=False)


def bert_cond(cfg):
    """The cond stage node: BERTEmbedder without tokenizer."""
    return {"target": "ldm.modules.encoders.modules.BERTEmbedder",
            "params": {"n_embed": cfg["n_embed"], "n_layer": cfg["n_layer"], "vocab_size": cfg["vocab_size"],
                       "use_tokenizer": False}}


def prompt_ids(vocab_size, seed, n_tok=20, B=2):
    """Row 0: [CLS] + n_tok seeded ids + [SEP] + [PAD]...; the last row: the empty prompt [CLS] [SEP] [PAD]..."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros((B, 77), dtype=torch.long)
    ids[:, 0] = 101
    for b in range(B - 1):
        ids[b, 1:1 + n_tok] = torch.randint(999, vocab_size, (n_tok,), generator=g) if vocab_size > 2000 else \
            torch.randint(103, vocab_size, (n_tok,), generator=g)
        ids[b, 1 + n_tok] = 102
    ids[B - 1, 1] = 102
    return ids


@torch.no_grad()
def main():
    out = {"unet_seed": UNET_SEED, "vae_seed": VAE_SEED, "bert_seed": BERT_SEED}
    ld = R.build_ld(arch.LAION_UNET, arch.SD_V1_VAE, bert_cond(arch.LAION_BERT), **LD_PARAMS)
    out["laion_keys"] = [(k, tuple(v.shape)) for k, v in ld.state_dict().items()]
    del ld

    out["bert"] = []
    for tag, cfg, seed in (("tiny", arch.TINY_BERT, 500), ("full", arch.LAION_BERT, 501)):
        R.install()
        from ldm.modules.encoders.modules import BERTEmbedder
        ref = BERTEmbedder(n_embed=cfg["n_embed"], n_layer=cfg["n_layer"], vocab_size=cfg["vocab_size"],
                           use_tokenizer=False).eval()
        sd = arch.random_state_dict(arch.bert_param_shapes(cfg), BERT_SEED)
        ref.load_state_dict(sd, strict=True)
        ids = prompt_ids(cfg["vocab_size"], seed)
        z = ref.encode(ids)
        print(f"bert {tag} {tuple(z.shape)}: std {float(z.std()):.3f}  oracle rel-L2 {rel(BO.bert_embed(sd, ids), z):.2e}")
        out["bert"].append(dict(cfg=tag, ids=ids, z=z.half() if tag == "full" else z.clone()))
        del ref, sd

    out["unet"] = []
    for tag, cfg, shapes in (
        ("tiny", arch.TINY_LAION_UNET, [((2, 4, 16, 16), [981, 1]), ((1, 4, 16, 24), [500])]),
        ("full", arch.LAION_UNET, [((2, 4, 32, 32), [981, 1]), ((1, 4, 16, 48), [501])]),
    ):
        unet = R.build_unet(cfg)
        sd = arch.random_state_dict(arch.unet_param_shapes(cfg), UNET_SEED)
        unet.load_state_dict(sd, strict=True)
        for i, (xs, ts) in enumerate(shapes):
            x = gen(xs, 900 + i)
            t = torch.tensor(ts, dtype=torch.long)
            ctx_seed = 950 + i
            ctx = gen((xs[0], 77, cfg["context_dim"]), ctx_seed)
            eps = unet(x, t, context=ctx)
            mine = O.unet_forward(sd, x, t, ctx, num_heads=cfg["num_heads"])
            print(f"unet {tag} {xs} t={ts}: eps std {float(eps.std()):.3f}  oracle rel-L2 {rel(mine, eps):.2e}")
            out["unet"].append(dict(cfg=tag, x=x, t=t, ctx_seed=ctx_seed, eps=eps))
        del unet, sd

    # scripts/txt2img.py --laion400m on the tiny model: uc from the empty prompt, guided PLMS-10, decode
    ld = R.build_ld(arch.TINY_LAION_UNET, arch.TINY_VAE, bert_cond(arch.TINY_BERT), **LD_PARAMS)
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_LAION_UNET), UNET_SEED)
    vsd = arch.random_state_dict(arch.vae_param_shapes(arch.TINY_VAE), VAE_SEED)
    bsd = arch.random_state_dict(arch.bert_param_shapes(arch.TINY_BERT), BERT_SEED)
    ld.model.diffusion_model.load_state_dict(usd, strict=True)
    ld.first_stage_model.load_state_dict(vsd, strict=True)
    ld.cond_stage_model.load_state_dict(bsd, strict=True)
    plms, _ = R.build_samplers(ld)
    B, shape = 2, [4, 16, 16]
    ids = prompt_ids(arch.TINY_BERT["vocab_size"], 510, B=B + 1)[:B]
    uc_ids = prompt_ids(arch.TINY_BERT["vocab_size"], 510, B=B + 1)[B:].repeat(B, 1)
    x_T = gen((B, *shape), 940)
    with contextlib.redirect_stdout(io.StringIO()):
        uc = ld.get_learned_conditioning(uc_ids)
        c = ld.get_learned_conditioning(ids)
        s, _ = plms.sample(S=10, conditioning=c, batch_size=B, shape=shape, verbose=False,
                           unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=0.0, x_T=x_T)
    x_dec = ld.decode_first_stage(s)
    fn = lambda x, t, ctx: O.unet_forward(usd, x, t, ctx, num_heads=arch.TINY_LAION_UNET["num_heads"])
    mine = O.plms_sample(fn, x_T, BO.bert_embed(bsd, ids), BO.bert_embed(bsd, uc_ids), 7.5, S=10)
    print(f"guided plms S=10: sample std {float(s.std()):.3f}; oracle rel {rel(mine, s):.2e}; "
          f"decode oracle rel {rel(O.decode_first_stage(vsd, s), x_dec):.2e}")
    out["plms"] = dict(ids=ids, uc_ids=uc_ids, x_T=x_T, sample=s, x_dec=x_dec)
    path = os.path.join(OUT, "laion.pt")
    torch.save(out, path)
    print(f"  wrote laion.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
