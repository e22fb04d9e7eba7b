"""ORACLE tooling: generate tests/golden/semantic.pt by running the UNMODIFIED reference (located by ref_harness.py) on
CPU fp32 for the LDM semantic-synthesis models (models/ldm/semantic_synthesis256 / semantic_synthesis512 config.yaml).

Run in the build container:  python oracle/make_golden_semantic.py
The cond stage is the reference's SpatialRescaler, fed as DDPM.get_input feeds it (np.eye(182)[labels] -> NCHW float).
clip / kornia are stubbed and the VQ quantizer is oracle/vq_oracle.py's (ref_harness.install());
LatentDiffusion, SpatialRescaler, UNetModel, VQModelInterface and DDIMSampler are the reference's own code. Weights come
from stable-diffusion_b200/arch.random_state_dict (seeded); label maps and soft maps are regenerated from seeds
(oracle/semantic_oracle.py), so only outputs are stored. Every cond output is also computed by the oracle and must equal
the reference's bit for bit.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import ref_harness as R  # noqa: E402
from ref_harness import gen  # noqa: E402
import semantic_oracle as SO  # noqa: E402
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_SEED, VQ_SEED, COND_SEED = 11, 12, 13
LINEAR_START, LINEAR_END = 0.0015, 0.0205
TINY_BIAS_COND = dict(n_stages=1, in_channels=20, out_channels=3, bias=True)
# (tag, cond config name, kind, h, w, seed): label maps are Voronoi partitions or all ids; "soft" is a softmax map
COND_CASES = [
    ("voronoi64", "full", "voronoi", 64, 64, 21),
    ("voronoi256", "full", "voronoi", 256, 256, 22),
    ("voronoi30x46", "full", "voronoi", 30, 46, 23),
    ("all_ids", "full", "all_ids", 56, 64, 24),
    ("soft", "full", "soft", 32, 48, 25),
    ("tiny_bias", "tiny_bias", "voronoi", 30, 46, 26),
    ("tiny", "tiny", "voronoi", 64, 64, 27),
]
# LatentDiffusion with the semantic_synthesis config's parameters; the cond stage is SpatialRescaler
COND_TARGET = "ldm.modules.encoders.modules.SpatialRescaler"
LD_PARAMS = dict(linear_start=LINEAR_START, linear_end=LINEAR_END, log_every_t=100, timesteps=1000, loss_type="l1",
                 first_stage_key="image", cond_stage_key="segmentation", channels=3, concat_mode=True,
                 cond_stage_trainable=True)
COND_CFGS = {"full": arch.SEMANTIC_SYNTHESIS_COND, "tiny": arch.TINY_SEMANTIC_COND, "tiny_bias": TINY_BIAS_COND}


def case_input(kind, h, w, seed, n_classes):
    """(labels uint8 [1, h, w] or None, float NCHW input of the cond stage)."""
    if kind == "soft":
        return None, SO.soft_map((1, n_classes, h, w), seed)
    lab = SO.voronoi_labels(h, w, n_classes, seed) if kind == "voronoi" else SO.all_ids_labels(h, w, n_classes, seed)
    return torch.from_numpy(lab)[None], None


def ref_cond(ld, labels=None, soft=None):
    """get_input on the dataset's one-hot (np.eye(n)[labels], [B, H, W, n]) or on a float map, then
    get_learned_conditioning."""
    from ldm.models.diffusion.ddpm import DDPM
    n = ld.cond_stage_model.channel_mapper.in_channels
    if labels is not None:
        batch = {"segmentation": torch.from_numpy(np.eye(n)[labels.numpy()])}
    else:
        batch = {"segmentation": soft.permute(0, 2, 3, 1)}
    x = DDPM.get_input(ld, batch, "segmentation")
    return ld.get_learned_conditioning(x)


@torch.no_grad()
def main():
    out = {"unet_seed": UNET_SEED, "vq_seed": VQ_SEED, "cond_seed": COND_SEED, "linear_start": LINEAR_START,
           "linear_end": LINEAR_END, "tiny_bias_cond": TINY_BIAS_COND}
    # the reference's key / shape list of the whole model (both checkpoints share it) and its schedule
    cond = {"target": COND_TARGET, "params": arch.SEMANTIC_SYNTHESIS_COND}
    ld = R.build_ld(arch.SEMANTIC_SYNTHESIS_UNET, arch.VQ_F4, cond, **LD_PARAMS)
    out["ld_keys"] = [(k, tuple(v.shape)) for k, v in ld.state_dict().items()]
    out["alphas_cumprod"] = ld.alphas_cumprod.clone()
    ld512 = R.build_ld(arch.SEMANTIC_SYNTHESIS_UNET, arch.VQ_F4, cond, image_size=128, **LD_PARAMS)
    assert [(k, tuple(v.shape)) for k, v in ld512.state_dict().items()] == out["ld_keys"]
    del ld, ld512

    # cond stage outputs
    out["cond"] = []
    cond_lds = {}
    for tag, cname, kind, h, w, seed in COND_CASES:
        cfg = COND_CFGS[cname]
        if cname not in cond_lds:
            ld = R.build_ld(arch.TINY_SEMANTIC_UNET, arch.TINY_VQ_F4, {"target": COND_TARGET, "params": cfg},
                            use_ema=False, **LD_PARAMS)
            sd = arch.random_state_dict(arch.spatial_rescaler_param_shapes(cfg), COND_SEED)
            ld.cond_stage_model.load_state_dict(sd, strict=True)
            cond_lds[cname] = (ld, sd)
        ld, sd = cond_lds[cname]
        labels, soft = case_input(kind, h, w, seed, cfg["in_channels"])
        c = ref_cond(ld, labels, soft)
        x = SO.one_hot(labels, cfg["in_channels"]) if soft is None else soft
        o = SO.spatial_rescale(x, cfg["n_stages"], sd["channel_mapper.weight"], sd.get("channel_mapper.bias"))
        assert torch.equal(o, c), tag
        print(f"cond {tag} ({cname}, {kind} {h}x{w}) -> {tuple(c.shape)}: oracle equal True")
        out["cond"].append(dict(tag=tag, cfg=cname, kind=kind, h=h, w=w, seed=seed, c=c))
    del cond_lds

    # UNet eps
    out["unet"] = []
    for tag, cfg, shapes in (
        ("tiny", arch.TINY_SEMANTIC_UNET, [((2, 6, 16, 16), [981, 1])]),
        ("big", arch.SEMANTIC_SYNTHESIS_UNET, [((1, 6, 64, 64), [981]), ((1, 6, 16, 48), [501])]),
    ):
        net = R.build_unet(cfg)
        net.load_state_dict(arch.random_state_dict(arch.unet_param_shapes(cfg), UNET_SEED), strict=True)
        for i, (xs, ts) in enumerate(shapes):
            x = gen(xs, 900 + i)
            eps = net(x, torch.tensor(ts, dtype=torch.long))
            print(f"unet {tag} {xs} t={ts}: eps std {float(eps.std()):.3f}")
            out["unet"].append(dict(cfg=tag, x_seed=900 + i, shape=xs, t=torch.tensor(ts), eps=eps))
        del net

    # log_images' sampling on the tiny model: conditioning from a 64x64 label map, DDIM-10 at eta 0 and 1, decode
    cond = {"target": COND_TARGET, "params": arch.TINY_SEMANTIC_COND}
    ld = R.build_ld(arch.TINY_SEMANTIC_UNET, arch.TINY_VQ_F4, cond, use_ema=False, **LD_PARAMS)
    ld.model.diffusion_model.load_state_dict(arch.random_state_dict(arch.unet_param_shapes(arch.TINY_SEMANTIC_UNET),
                                                                    UNET_SEED), strict=True)
    ld.first_stage_model.load_state_dict(arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F4), VQ_SEED),
                                         strict=True)
    ld.cond_stage_model.load_state_dict(arch.random_state_dict(
        arch.spatial_rescaler_param_shapes(arch.TINY_SEMANTIC_COND), COND_SEED), strict=True)
    _, ddim = R.build_samplers(ld)
    import ldm.models.diffusion.ddim as ddim_mod
    lab_seed = 30
    labels = torch.from_numpy(SO.voronoi_labels(64, 64, arch.TINY_SEMANTIC_COND["in_channels"], lab_seed))[None]
    c = ref_cond(ld, labels)
    out["e2e"] = dict(labels_seed=lab_seed, h=64, w=64, c=c, x_T_seed=940, noise_seed=960)
    orig = ddim_mod.noise_like
    for eta in (0.0, 1.0):
        x_T = gen((1, 3, 16, 16), 940)
        draws = []
        # the DDIM noise draws come from seeds (draw i: noise_seed + i), so the tests regenerate them
        ddim_mod.noise_like = lambda shape, device, repeat=False: draws.append(gen(shape, 960 + len(draws))) or draws[-1]
        try:
            with contextlib.redirect_stdout(io.StringIO()), ld.ema_scope():
                s, _ = ddim.sample(S=10, conditioning=c, batch_size=1, shape=(3, 16, 16), eta=eta, verbose=False,
                                   x_T=x_T)
                x_dec = ld.decode_first_stage(s)
        finally:
            ddim_mod.noise_like = orig
        print(f"e2e eta {eta}: sample std {float(s.std()):.3f}, image {tuple(x_dec.shape)}, {len(draws)} noise draws")
        out["e2e"][f"eta{int(eta)}"] = dict(sample=s, x_dec=x_dec, n_noise=len(draws))
    path = os.path.join(OUT, "semantic.pt")
    torch.save(out, path)
    print(f"  wrote semantic.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
