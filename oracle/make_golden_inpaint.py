"""ORACLE tooling: generate tests/golden/inpaint.pt by running the UNMODIFIED reference (located by ref_harness.py) on CPU
fp32 for the LDM inpainting model (models/ldm/inpainting_big/config.yaml, scripts/inpaint.py).

Run in the build container:  python oracle/make_golden_inpaint.py
taming's quantizer is oracle/vq_oracle.py's restatement (set by ref_harness.install()) and the training loss is
torch.nn.Identity (the config's DummyLoss only exists through taming). `make_batch` is the reference script's own
function, called on PNG files written here; its `main` import (the training entry point) is stubbed with ldm.util's
instantiate_from_config. The composite is the script's inline code, restated in oracle/inpaint_oracle.py.
Weights come from stable-diffusion_b200/arch.random_state_dict (seeded).
"""
from __future__ import annotations

import contextlib
import importlib.util
import io
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import inpaint_oracle as P  # noqa: E402
import ref_harness as R  # noqa: E402
from ref_harness import gen  # noqa: E402
import sdb200  # noqa: E402,F401
from sdb200 import arch  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_SEED, VQ_SEED = 11, 12
LINEAR_START, LINEAR_END = 0.0015, 0.0205
# LatentDiffusion with the inpainting_big config's parameters; the first stage is also the cond stage
LD_PARAMS = dict(linear_start=LINEAR_START, linear_end=LINEAR_END, log_every_t=100, timesteps=1000, loss_type="l1",
                 first_stage_key="image", cond_stage_key="masked_image", channels=3, concat_mode=True,
                 monitor="val/loss")


def ref_inpaint_module():
    R.install()
    from ldm.util import instantiate_from_config
    sys.modules.setdefault("main", types.SimpleNamespace(instantiate_from_config=instantiate_from_config))
    spec = importlib.util.spec_from_file_location("ref_inpaint_script", os.path.join(R.REF, "scripts", "inpaint.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def synthetic_pair(h, w, seed, threshold=False):
    g = np.random.default_rng(seed)
    image = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if threshold:      # values at the 0.5 threshold: 127 -> 0, 128 -> 1
        mask = g.choice(np.array([0, 127, 128, 255], dtype=np.uint8), size=(h, w))
    else:              # a rectangle plus noise
        mask = (g.random((h, w)) < 0.1).astype(np.uint8) * 255
        mask[h // 4: h // 2, w // 3: (2 * w) // 3] = 255
    return image, mask


def example_pair(name, size):
    """A downscaled (nearest) copy of one of the reference's data/inpainting_examples pairs: image RGB, mask as stored."""
    from PIL import Image
    d = os.path.join(R.REF, "data", "inpainting_examples")
    im = Image.open(os.path.join(d, name + ".png")).resize(size, Image.NEAREST)
    mk = Image.open(os.path.join(d, name + "_mask.png")).resize(size, Image.NEAREST)
    return np.array(im.convert("RGB")), np.array(mk)


def run_make_batch(mod, tmp, image_u8, mask_raw, tag):
    """The reference's make_batch on PNGs of the given arrays (mask_raw: L [h, w] or RGB [h, w, 3])."""
    from PIL import Image
    ip, mp = os.path.join(tmp, tag + ".png"), os.path.join(tmp, tag + "_mask.png")
    Image.fromarray(image_u8).save(ip)
    Image.fromarray(mask_raw).save(mp)
    mask_l = np.array(Image.open(mp).convert("L"))
    return mod.make_batch(ip, mp, device=torch.device("cpu")), mask_l


@torch.no_grad()
def main():
    mod = ref_inpaint_module()
    out = {"unet_seed": UNET_SEED, "vq_seed": VQ_SEED, "linear_start": LINEAR_START, "linear_end": LINEAR_END}
    # the reference model's state-dict keys: cond_stage_model.* repeats first_stage_model.*
    ld = R.build_ld(arch.INPAINTING_BIG_UNET, arch.VQ_F4_NOATTN, "__is_first_stage__", **LD_PARAMS)
    out["ld_keys"] = [(k, tuple(v.shape)) for k, v in ld.state_dict().items()]
    del ld

    # make_batch + the interpolated mask channel + composite
    out["prepare"] = []
    with tempfile.TemporaryDirectory() as tmp:
        cases = [("64x64", *synthetic_pair(64, 64, 1)), ("64x96", *synthetic_pair(64, 96, 2)),
                 ("threshold", *synthetic_pair(48, 64, 3, threshold=True)),
                 ("rgb_mask", *example_pair("bench2", (64, 64)))]
        for i, (tag, image, mask_raw) in enumerate(cases):
            b, mask_l = run_make_batch(mod, tmp, image, mask_raw, tag)
            o = P.make_batch(image, mask_l)
            same = all(torch.equal(o[k], b[k]) for k in b)
            h, w = image.shape[:2]
            sizes = [(h // 4, w // 4)] + ([(21, 27)] if tag == "64x96" else [])
            cc = {s: torch.nn.functional.interpolate(b["mask"], size=s) for s in sizes}
            x_dec = gen((1, 3, h, w), 950 + i, 0.6)
            comp = P.composite(b, x_dec)
            print(f"make_batch {tag} ({mask_raw.ndim == 3 and 'RGB' or 'L'} mask): oracle equal {same}; "
                  f"mask mean {float(b['mask'].mean()):.3f}")
            # batch["image"] is a function of `image`, and the decoded image is regenerated from its seed
            out["prepare"].append(dict(tag=tag, image=torch.from_numpy(image), mask_raw=torch.from_numpy(mask_raw),
                                       mask=torch.from_numpy(mask_l), masked_image=b["masked_image"],
                                       batch_mask=b["mask"], cc=[(s, v) for s, v in cc.items()], x_dec_seed=950 + i,
                                       composite=torch.from_numpy(comp)))

    # UNet eps
    out["unet"] = []
    for tag, cfg, shapes in (
        ("tiny", arch.TINY_INPAINT_UNET, [((2, 7, 16, 16), [981, 1])]),
        ("big", arch.INPAINTING_BIG_UNET, [((1, 7, 32, 32), [981]), ((1, 7, 16, 48), [501])]),
    ):
        sd = arch.random_state_dict(arch.unet_param_shapes(cfg), UNET_SEED)
        net = R.build_unet(cfg)
        net.load_state_dict(sd, strict=True)
        for i, (xs, ts) in enumerate(shapes):
            x = gen(xs, 900 + i)
            t = torch.tensor(ts, dtype=torch.long)
            eps = net(x, t)
            print(f"unet {tag} {xs} t={ts}: eps std {float(eps.std()):.3f}")
            out["unet"].append(dict(cfg=tag, x=x, t=t, eps=eps))
        del net

    # VQ without mid attention: encode / decode
    out["vq"] = []
    for tag, cfg, size in (("tiny", arch.TINY_VQ_NOATTN, (2, 3, 32, 48)), ("big", arch.VQ_F4_NOATTN, (1, 3, 32, 48))):
        sd = arch.random_state_dict(arch.vq_param_shapes(cfg), VQ_SEED)
        m = R.build_vq(cfg)
        m.load_state_dict(sd, strict=True)
        img = gen(size, 930).clamp(-1, 1)
        h = m.encode(img)
        x = m.decode(h)
        print(f"vq {tag} {size}: encode -> {tuple(h.shape)}, decode -> {tuple(x.shape)}")
        out["vq"].append(dict(cfg=tag, x=img, h=h, dec=x))

    # the script end to end on the tiny model: DDIM-10 from a recorded x_T, decode, composite
    ld = R.build_ld(arch.TINY_INPAINT_UNET, arch.TINY_VQ_NOATTN, "__is_first_stage__", use_ema=False, **LD_PARAMS)
    ld.model.diffusion_model.load_state_dict(arch.random_state_dict(arch.unet_param_shapes(arch.TINY_INPAINT_UNET),
                                                                    UNET_SEED), strict=True)
    ld.first_stage_model.load_state_dict(arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_NOATTN), VQ_SEED),
                                         strict=True)
    assert ld.cond_stage_model is ld.first_stage_model
    _, ddim = R.build_samplers(ld)
    with tempfile.TemporaryDirectory() as tmp:
        image, mask = synthetic_pair(32, 32, 4)
        batch, _ = run_make_batch(mod, tmp, image, mask, "e2e")
    with contextlib.redirect_stdout(io.StringIO()):
        with ld.ema_scope():
            c = ld.cond_stage_model.encode(batch["masked_image"])
            cc = torch.nn.functional.interpolate(batch["mask"], size=c.shape[-2:])
            c = torch.cat((c, cc), dim=1)
            shape = (c.shape[1] - 1,) + c.shape[2:]
            x_T = gen((1, *shape), 940)
            s, _ = ddim.sample(S=10, conditioning=c, batch_size=c.shape[0], shape=shape, verbose=False, x_T=x_T)
            x_dec = ld.decode_first_stage(s)
    result = P.composite(batch, x_dec)
    print(f"e2e DDIM-10: sample std {float(s.std()):.3f}, decoded {tuple(x_dec.shape)}")
    out["e2e"] = dict(image=torch.from_numpy(image), mask=torch.from_numpy(mask), c=c, x_T=x_T, sample=s,
                      x_dec=x_dec, result=torch.from_numpy(result), alphas_cumprod=ld.alphas_cumprod.clone())
    path = os.path.join(OUT, "inpaint.pt")
    torch.save(out, path)
    print(f"  wrote inpaint.pt ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    main()
