"""ORACLE tooling: generate tests/golden/superres.pt by running the UNMODIFIED reference (located by ref_harness.py) on
CPU fp32 for the LDM super-resolution model (models/ldm/bsr_sr/config.yaml, notebook_helpers.py).

Run in the build container:  python oracle/make_golden_superres.py
notebook_helpers.py is imported as it is; its notebook-only imports (google.colab, IPython.display, ipywidgets) and the
bare `display` that get_cond calls are stubbed here. taming's quantizer is oracle/vq_oracle.py's restatement (set by
ref_harness.install()). Weights come from stable-diffusion_b200/arch.random_state_dict (seeded); large tables are stored
as the SHA-256 of their bytes, inputs are regenerated from seeds.
"""
from __future__ import annotations

import contextlib
import hashlib
import importlib.util
import io
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import ref_harness as R  # noqa: E402
from ref_harness import gen  # noqa: E402
import superres_oracle as S  # noqa: E402
import sdb200  # noqa: E402,F401
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_SEED, VQ_SEED = 11, 12
LINEAR_START, LINEAR_END = 0.0015, 0.0155
# (tag, latent h, w, params, uf): the notebook's geometry at the 256x256 and 192x192 latents, and small test geometries
TABLES = [
    ("nb256_uf1", 256, 256, S.notebook_params(), 1), ("nb256_uf4", 256, 256, S.notebook_params(), 4),
    ("nb192_uf1", 192, 192, S.notebook_params(), 1), ("nb192_uf4", 192, 192, S.notebook_params(), 4),
    ("tiny_uf1", 24, 40, S.notebook_params(16, 8), 1), ("tiny_uf4", 24, 40, S.notebook_params(16, 8), 4),
    ("tiny_tie_uf1", 24, 40, S.notebook_params(16, 8, tie_braker=True), 1),
    ("tiny_tie_uf4", 24, 40, S.notebook_params(16, 8, tie_braker=True), 4),
    ("tiny_stride4_uf1", 20, 28, S.notebook_params(12, 4), 1),
]
# LatentDiffusion with the bsr_sr config's parameters; the cond stage is Identity: the LR image is concatenated as it is
LD_PARAMS = dict(linear_start=LINEAR_START, linear_end=LINEAR_END, log_every_t=100, timesteps=1000, loss_type="l2",
                 first_stage_key="image", cond_stage_key="LR_image", channels=3, concat_mode=True,
                 cond_stage_trainable=False)
LD_COND = {"target": "torch.nn.Identity"}
BIG = 64 * 1024            # tables larger than this many bytes are stored as their SHA-256


def sha(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def notebook_module():
    R.install()
    for name, attrs in (("google.colab", dict(files=None)), ("IPython.display", dict(Image=lambda **k: None)),
                        ("ipywidgets", {})):
        R._stub(name, **attrs)
    spec = importlib.util.spec_from_file_location("ref_notebook_helpers", os.path.join(R.REF, "notebook_helpers.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.display = lambda *a, **k: None

    class CpuTorch:        # get_cond moves the conditioning to torch.device("cuda"): keep it on the CPU
        device = staticmethod(lambda *a, **k: torch.device("cpu"))

        def __getattr__(self, name):
            return getattr(torch, name)
    mod.torch = CpuTorch()
    return mod


def lr_png(h, w, seed):
    g = np.random.default_rng(seed)
    img = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
    img.reshape(-1)[:256] = np.arange(256, dtype=np.uint8)         # every byte value once
    return img


@torch.no_grad()
def main():
    nb = notebook_module()
    out = {"unet_seed": UNET_SEED, "vq_seed": VQ_SEED, "linear_start": LINEAR_START, "linear_end": LINEAR_END}
    ld = R.build_ld(arch.BSR_SR_UNET, arch.VQ_F4, LD_COND, **LD_PARAMS)
    out["ld_keys"] = [(k, tuple(v.shape)) for k, v in ld.state_dict().items()]
    assert not [k for k in out["ld_keys"] if k[0].startswith("cond_stage_model.")]

    # weighting / normalization tables through the reference's own get_fold_unfold
    out["tables"] = []
    for tag, h, w, p, uf in TABLES:
        ld.split_input_params = p
        _, _, norm, weighting = ld.get_fold_unfold(torch.zeros(1, 3, h, w), p["ks"], p["stride"], uf=uf)
        o_fold, _, o_norm, o_w = S.get_fold_unfold((1, 3, h, w), p["ks"], p["stride"], p, uf=uf)
        same = torch.equal(o_norm, norm) and torch.equal(o_w, weighting)
        print(f"tables {tag}: weighting {tuple(weighting.shape)}, norm {tuple(norm.shape)}, oracle equal {same}")
        assert same
        e = dict(tag=tag, h=h, w=w, params=p, uf=uf, weighting_shape=tuple(weighting.shape),
                 norm_shape=tuple(norm.shape))
        for k, v in (("weighting", weighting), ("norm", norm)):
            if v.numel() * 4 > BIG:
                e[k + "_sha256"] = sha(v)
            else:
                e[k] = v.clone()
        out["tables"].append(e)
    del ld.split_input_params
    del ld

    # get_cond's conversion of a PNG the reference reads with PIL
    out["lr"] = []
    with tempfile.TemporaryDirectory() as tmp:
        from PIL import Image
        for i, (h, w) in enumerate(((24, 40), (32, 32))):
            img = lr_png(h, w, 60 + i)
            path = os.path.join(tmp, f"lr{i}.png")
            Image.fromarray(img).save(path)
            ex = nb.get_cond("superresolution", path)
            c = ex["LR_image"].permute(0, 3, 1, 2).contiguous()        # get_input's rearrange to NCHW
            assert torch.equal(c, S.lr_image(img))
            assert tuple(ex["image"].shape) == (1, 4 * h, 4 * w, 3)
            out["lr"].append(dict(image=torch.from_numpy(img), c=c))
            print(f"get_cond {h}x{w}: oracle equal True, range [{float(c.min())}, {float(c.max())}]")

    # UNet eps
    out["unet"] = []
    for tag, cfg, shapes in (
        ("tiny", arch.TINY_BSR_UNET, [((2, 6, 16, 16), [981, 1])]),
        ("big", arch.BSR_SR_UNET, [((2, 6, 32, 32), [981, 1]), ((1, 6, 16, 48), [501]), ((1, 6, 128, 128), [999])]),
    ):
        net = R.build_unet(cfg)
        net.load_state_dict(arch.random_state_dict(arch.unet_param_shapes(cfg), UNET_SEED), strict=True)
        for i, (xs, ts) in enumerate(shapes):
            x = gen(xs, 900 + i)
            eps = net(x, torch.tensor(ts, dtype=torch.long))
            print(f"unet {tag} {xs} t={ts}: eps std {float(eps.std()):.3f}")
            out["unet"].append(dict(cfg=tag, x_seed=900 + i, shape=xs, t=torch.tensor(ts), eps=eps))
        del net

    # VQ-f4 decode (mid-block attention) of one small latent
    m = R.build_vq(arch.VQ_F4)
    m.load_state_dict(arch.random_state_dict(arch.vq_param_shapes(arch.VQ_F4), VQ_SEED), strict=True)
    h = gen((1, 3, 16, 24), 931)
    out["vq_f4"] = dict(h=h, dec=m.decode(h))
    print(f"vq_f4 decode {tuple(h.shape)} -> {tuple(out['vq_f4']['dec'].shape)}")
    del m

    # make_convolutional_sample end to end on the tiny model, split at ks 16 / stride 8 / vqf 4, DDIM-10 at eta 0 and 1
    ld = R.build_ld(arch.TINY_BSR_UNET, arch.TINY_VQ_F4, LD_COND, use_ema=False, **LD_PARAMS)
    ld.model.diffusion_model.load_state_dict(arch.random_state_dict(arch.unet_param_shapes(arch.TINY_BSR_UNET),
                                                                    UNET_SEED), strict=True)
    ld.first_stage_model.load_state_dict(arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_F4), VQ_SEED),
                                         strict=True)
    R.build_samplers(ld)      # the samplers' register_buffer runs on the CPU
    import ldm.models.diffusion.ddim as ddim_mod
    p = S.notebook_params(16, 8)
    ld.split_input_params = p
    lr = lr_png(24, 24, 70)
    with tempfile.TemporaryDirectory() as tmp:
        from PIL import Image
        path = os.path.join(tmp, "e2e.png")
        Image.fromarray(lr).save(path)
        batch = nb.get_cond("superresolution", path)
    out["e2e"] = dict(image=torch.from_numpy(lr), params=p, alphas_cumprod=ld.alphas_cumprod.clone(), x_T_seed=940,
                      noise_seed=960)
    orig = ddim_mod.noise_like
    for eta in (0.0, 1.0):
        x_T = gen((1, 3, 24, 24), 940)
        # the DDIM noise draws come from seeds (draw i: noise_seed + i), so the tests regenerate them
        for pass_ in range(2):
            draws = []
            ddim_mod.noise_like = lambda shape, device, repeat=False: draws.append(gen(shape, 960 + len(draws))) or draws[-1]
            try:
                with contextlib.redirect_stdout(io.StringIO()):
                    if pass_ == 0:
                        logs = nb.make_convolutional_sample(batch, ld, mode="ddim", custom_steps=10, eta=eta,
                                                            quantize_x0=False, custom_shape=None, x_T=x_T)
                    else:    # the sample latent, which the notebook does not log: DDIM again on the same draws
                        c = ld.get_learned_conditioning(batch["LR_image"].permute(0, 3, 1, 2).contiguous().float())
                        s, _ = nb.convsample_ddim(ld, c, steps=10, shape=(1, 3, 24, 24), eta=eta, x_T=x_T)
            finally:
                ddim_mod.noise_like = orig
        assert torch.equal(ld.decode_first_stage(s), logs["sample"])
        print(f"e2e eta {eta}: sample std {float(s.std()):.3f}, image {tuple(logs['sample'].shape)}, "
              f"{len(draws)} noise draws")
        out["e2e"][f"eta{int(eta)}"] = dict(sample=s, x_dec=logs["sample"], n_noise=len(draws))
    # the split apply_model and decode on one state, with the per-tile outputs, for the oracle's restatement
    t = torch.tensor([901])
    xs = gen((1, 3, 24, 40), 941)
    cl = S.lr_image(lr_png(24, 40, 71))
    eps = ld.apply_model(xs, t, cl)
    eps_tiles = []
    fn = lambda xt, tt, ct: eps_tiles.append(ld.model(xt, tt, c_concat=[ct])) or eps_tiles[-1]
    assert torch.equal(S.split_apply(fn, xs, t, cl, p), eps)
    pd = S.notebook_params(8, 4)
    ld.split_input_params = pd
    zs = gen((1, 3, 12, 20), 942)
    dec = ld.decode_first_stage(zs)
    dec_tiles = []
    dfn = lambda zt: dec_tiles.append(ld.first_stage_model.decode(zt)) or dec_tiles[-1]
    assert torch.equal(S.split_decode(dfn, zs, pd), dec)
    out["e2e"]["apply"] = dict(x_seed=941, lr_seed=71, t=t, eps=eps, eps_tiles=torch.stack(eps_tiles))
    out["e2e"]["decode"] = dict(z_seed=942, params=pd, dec=dec, dec_tiles=torch.stack(dec_tiles))
    print(f"split apply_model ({len(eps_tiles)} tiles) / decode ({len(dec_tiles)} tiles): oracle equal True")
    path = os.path.join(OUT, "superres.pt")
    torch.save(out, path)
    print(f"  wrote superres.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
