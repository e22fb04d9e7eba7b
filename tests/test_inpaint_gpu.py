"""The LDM inpainting model on the H100: the prepare / composite kernels bit-exact against the reference's make_batch,
interpolate and composite (tests/golden/inpaint.pt), the two-source conv_in im2col and the UNet's concat route
bit-identical to the 7-channel input, UNet / VQ / DDIM parity with the reference, and scripts/inpaint.py end to end."""
import os

import numpy as np
import pytest
import torch

import helpers  # noqa: F401
from helpers import golden, rel_l2, script
from sdb200 import arch, ops, pipeline

pytestmark = pytest.mark.gpu
UCFG = {"tiny": arch.TINY_INPAINT_UNET, "big": arch.INPAINTING_BIG_UNET}
VCFG = {"tiny": arch.TINY_VQ_NOATTN, "big": arch.VQ_F4_NOATTN}


_UNETS = {}


def _unet(tag, dev):
    if tag not in _UNETS:
        import sdb200
        sd = arch.random_state_dict(arch.unet_param_shapes(UCFG[tag]), golden("inpaint.pt")["unet_seed"])
        _UNETS[tag] = sdb200.UNetModel(**UCFG[tag]).load_weights(sd, dev)
    return _UNETS[tag]


@pytest.mark.parametrize("idx", range(4))
def test_prepare_bit_exact(cuda_dev, idx):
    case = golden("inpaint.pt")["prepare"][idx]
    img, mk = case["image"][None].to(cuda_dev), case["mask"][None].to(cuda_dev)
    for size, cc in case["cc"]:
        cond = torch.full((1, 4, *size), float("nan"), device=cuda_dev)
        masked = ops.inpaint_prepare(img, mk, cond, 3)
        assert torch.equal(masked.cpu(), case["masked_image"]), case["tag"]
        assert torch.equal(cond[:, 3:].cpu(), cc), (case["tag"], size)
        assert bool(cond[:, :3].isnan().all())        # the encoder's channels are left alone


@pytest.mark.parametrize("idx", range(4))
def test_composite_byte_exact(cuda_dev, idx):
    case = golden("inpaint.pt")["prepare"][idx]
    h, w = case["image"].shape[:2]
    x = torch.randn((1, 3, h, w), generator=torch.Generator().manual_seed(case["x_dec_seed"])) * 0.6
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().to(cuda_dev)
    img, mk = case["image"][None].to(cuda_dev), case["mask"][None].to(cuda_dev)
    out = ops.inpaint_composite(x_nhwc, img, mk)
    assert torch.equal(out[0].cpu(), case["composite"])
    # outside the mask the output depends on the input image only, whatever was decoded
    other = ops.inpaint_composite(torch.randn_like(x_nhwc) * 3, img, mk)
    keep = (case["mask"] < 128)[None, :, :, None].expand_as(out).to(cuda_dev)
    assert torch.equal(out[keep], other[keep]) and not torch.equal(out, other)


def test_two_source_im2col_matches_cat(cuda_dev):
    g = torch.Generator(device=cuda_dev).manual_seed(3)
    x = torch.randn(2, 3, 12, 20, device=cuda_dev, generator=g)
    c = torch.randn(2, 4, 12, 20, device=cuda_dev, generator=g)
    ref = ops.im2col3x3(ops.nchw_to_nhwc(torch.cat([x, c], 1))[0], 1, 1, 12, 20, 64)
    assert torch.equal(ops.im2col3x3_concat(x, c, 64), ref)
    with pytest.raises(RuntimeError, match="exceed kpad"):
        ops.im2col3x3_concat(x, torch.randn(2, 5, 12, 20, device=cuda_dev), 64)
    with pytest.raises(RuntimeError, match="does not match"):
        ops.im2col3x3_concat(x, c[:1], 64)
    with pytest.raises(RuntimeError, match="does not match"):
        ops.im2col3x3_concat(x, c[:, :, :, :16].contiguous(), 64)


def test_concat_route_bit_identical_to_seven_channels(cuda_dev):
    """Eager, graph replay with autotuning (each route captures its own graph) and after switching the conditioning."""
    u = _unet("tiny", cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(5)
    x = torch.randn(2, 3, 16, 16, device=cuda_dev, generator=g)
    c1, c2 = (torch.randn(2, 4, 16, 16, device=cuda_dev, generator=g) for _ in range(2))
    t = torch.tensor([981, 1], device=cuda_dev)
    try:
        for graph in (False, True):
            u.use_cuda_graph = graph
            for c in (c1, c2, c1):
                seven = u(torch.cat([x, c], 1), t)
                assert torch.equal(u(x, t, concat=c), seven), (graph, c is c2)
    finally:
        u.use_cuda_graph = False


@pytest.mark.parametrize("idx", range(3))
def test_unet_eps_matches_reference(cuda_dev, idx):
    case = golden("inpaint.pt")["unet"][idx]
    u = _unet(case["cfg"], cuda_dev)
    x, t = case["x"].to(cuda_dev), case["t"].to(cuda_dev)
    eps = u(x[:, :3].contiguous(), t, concat=x[:, 3:].contiguous())
    err = rel_l2(eps, case["eps"])
    print(f"unet {case['cfg']} {tuple(x.shape)}: eps rel-L2 {err:.2e}")
    assert err < 1e-3, (case["cfg"], tuple(x.shape), err)
    assert torch.equal(eps, u(x, t))


@pytest.mark.parametrize("idx", range(2))
def test_vq_noattn_encode_decode(cuda_dev, idx):
    import sdb200
    case = golden("inpaint.pt")["vq"][idx]
    cfg = VCFG[case["cfg"]]
    m = sdb200.VQModelInterface(**cfg).load_weights(
        arch.random_state_dict(arch.vq_param_shapes(cfg), golden("inpaint.pt")["vq_seed"]), cuda_dev)
    assert m.W["encoder"]["attn"] is None and m.W["decoder"]["attn"] is None
    e_enc = rel_l2(m.encode(case["x"].to(cuda_dev)), case["h"])
    e_dec = rel_l2(m.decode(case["h"].to(cuda_dev)), case["dec"])
    print(f"vq {case['cfg']}: encode rel-L2 {e_enc:.2e}, decode {e_dec:.2e}")
    assert e_enc < 2e-3 and e_dec < 2e-3           # the VQ-f4 tests' tolerance (test_vq_ldm_gpu.py)


def _tiny_model(dev):
    S = script("inpaint")
    return S, S.load_model(random_init=True, tiny=True, device=dev)


def test_tiny_end_to_end_ddim10(cuda_dev):
    from sdb200.samplers import DDIMSampler
    g = golden("inpaint.pt")
    e = g["e2e"]
    S, m = _tiny_model(cuda_dev)
    assert torch.equal(m.alphas_cumprod.cpu(), e["alphas_cumprod"])
    # load_model(random_init) draws on the device generator: load the CPU-drawn golden weights instead
    pipeline.load_random_weights(m, cuda_dev, seeds=(g["unet_seed"], g["vq_seed"]))
    img, mk = e["image"][None].to(cuda_dev), e["mask"][None].to(cuda_dev)
    with m.ema_scope():
        out, c, s, x = S.inpaint(m, DDIMSampler(m), img, mk, steps=10, x_T=e["x_T"].to(cuda_dev), return_latents=True)
    e_c, e_s, e_x = rel_l2(c[:, :3], e["c"][:, :3]), rel_l2(s, e["sample"]), rel_l2(x.permute(0, 3, 1, 2), e["x_dec"])
    print(f"e2e: conditioning rel-L2 {e_c:.2e}, DDIM-10 latent {e_s:.2e}, decoded {e_x:.2e}")
    assert torch.equal(c[:, 3:].cpu(), e["c"][:, 3:])
    assert e_c < 1e-3 and e_s < 1e-3 and e_x < 1e-3
    keep = (e["mask"] < 128)[:, :, None].expand(*e["mask"].shape, 3)
    assert torch.equal(out[0].cpu()[keep], e["result"][keep])


def test_guided_and_plms_sampling_of_a_concat_model(cuda_dev):
    """Guidance runs on the doubled batch with no extra branch: with uc = c it equals the unguided trajectory; PLMS
    samples a concat model too."""
    from sdb200.samplers import DDIMSampler, PLMSSampler
    _, m = _tiny_model(cuda_dev)
    g = torch.Generator(device=cuda_dev).manual_seed(7)
    c = torch.randn(2, 4, 16, 16, device=cuda_dev, generator=g)
    x_T = torch.randn(2, 3, 16, 16, device=cuda_dev, generator=g)
    kw = dict(S=5, conditioning=c, batch_size=2, shape=(3, 16, 16), verbose=False, x_T=x_T)
    plain, _ = DDIMSampler(m).sample(**kw)
    guided, _ = DDIMSampler(m).sample(**kw, unconditional_guidance_scale=3.0, unconditional_conditioning=c.clone())
    err = rel_l2(guided, plain)
    print(f"guided (uc = c) vs unguided DDIM-5: rel-L2 {err:.2e}")
    assert err < 1e-3          # batch 4 against batch 2: GEMM tiles differ, not the math
    p, _ = PLMSSampler(m).sample(**kw)
    assert p.shape == plain.shape and bool(torch.isfinite(p).all())


def _write_pair(d, name, h, w, seed):
    from PIL import Image
    r = np.random.default_rng(seed)
    Image.fromarray(r.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(os.path.join(d, name + ".png"))
    mask = np.zeros((h, w), dtype=np.uint8)
    mask[h // 4: h // 2, w // 4: w // 2] = 255
    Image.fromarray(mask).save(os.path.join(d, name + "_mask.png"))


def test_script_tiny_writes_one_png_per_pair(cuda_dev, tmp_path):
    from PIL import Image
    indir, outdir = tmp_path / "in", tmp_path / "out"
    indir.mkdir()
    _write_pair(str(indir), "a", 32, 48, 0)
    _write_pair(str(indir), "b", 40, 32, 1)
    written = script("inpaint").main(["--indir", str(indir), "--outdir", str(outdir), "--steps", "5", "--random_init",
                                      "--tiny"])
    assert sorted(os.path.basename(p) for p in written) == ["a.png", "b.png"]
    assert Image.open(outdir / "a.png").size == (48, 32) and Image.open(outdir / "b.png").size == (32, 40)


def test_script_full_size_512(cuda_dev, tmp_path):
    """The full model at 512x512: a 128x128 latent, 4096-token attention at level 1."""
    from PIL import Image
    indir, outdir = tmp_path / "in", tmp_path / "out"
    indir.mkdir()
    _write_pair(str(indir), "x", 512, 512, 2)
    written = script("inpaint").main(["--indir", str(indir), "--outdir", str(outdir), "--steps", "5", "--random_init"])
    assert len(written) == 1 and Image.open(written[0]).size == (512, 512)
