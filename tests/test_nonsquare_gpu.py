"""Non-square latents end to end on the H100 against the unmodified reference (tests/golden/nonsquare.pt).

Every other model fixture is square, and in a square problem an H/W mix-up (a swapped axis in the conv tile geometry,
a transposed tile walk, a transposed store box) can cancel out. The SD-v1 case (2,4,24,40) walks the UNet through
24x40 -> 12x20 -> 6x10 -> 3x5, i.e. conv tile classes TN = 2, 8, 32 and 128 and ragged token counts (60, 15); the
(1,4,8,64) case reaches a 1x8 deepest level (h = 1). Tolerances are those of the square tests."""
import pytest
import torch

from helpers import CFGS, golden, rel_l2, weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
TOL = 1e-3          # SD-v1 UNet eps (test_unet_gpu.py)
TOL_TINY = 1.5e-3   # tiny UNet eps
TOL_VAE = 2e-3      # VAE decode / encode moments (test_vae_clip_gpu.py)
_models = {}


def _ctx(case):
    n = case["x"].shape[0]
    cd = CFGS["unet"][case["cfg"]]["context_dim"]
    return torch.randn((n, 77, cd), generator=torch.Generator().manual_seed(case["ctx_seed"]))


def _unet(tag, seed, dev):
    import sdb200
    key = (tag, seed)
    if key not in _models:
        _models[key] = sdb200.UNetModel(**CFGS["unet"][tag]).load_weights(weights("unet", tag, seed), dev)
    return _models[key]


def _sdv1_case():
    case = golden("nonsquare.pt")["unet"][2]
    assert case["cfg"] == "sdv1" and tuple(case["x"].shape) == (2, 4, 24, 40)
    return case


@pytest.mark.parametrize("idx", range(4))
def test_unet_nonsquare_vs_reference(cuda_dev, idx):
    case = golden("nonsquare.pt")["unet"][idx]
    m = _unet(case["cfg"], case["seed"], cuda_dev)
    x = case["x"].to(cuda_dev)
    eps = m(x, case["t"].to(cuda_dev), context=_ctx(case).to(cuda_dev))
    torch.cuda.synchronize()
    assert eps.shape == case["eps"].shape
    err = rel_l2(eps, case["eps"])
    # the same output with H and W exchanged is nowhere near the reference: the comparison can tell the axes apart
    swapped = eps.cpu().transpose(2, 3).reshape(eps.shape)
    print(f"nonsquare unet {case['cfg']} {tuple(x.shape)} rel-L2 {err:.3e}")
    assert err < (TOL if case["cfg"] == "sdv1" else TOL_TINY), err
    assert rel_l2(swapped, case["eps"]) > 0.1


@pytest.mark.parametrize("idx", range(2))
def test_vae_nonsquare_vs_reference(cuda_dev, idx):
    import sdb200
    case = golden("nonsquare.pt")["vae"][idx]
    vae = sdb200.AutoencoderKL(**CFGS["vae"][case["cfg"]]).load_weights(weights("vae", case["cfg"], case["seed"]), cuda_dev)
    dec = vae.decode(case["z"].to(cuda_dev))
    post = vae.encode(case["img"].to(cuda_dev))
    torch.cuda.synchronize()
    assert dec.shape == case["dec"].shape and post.mean.shape == case["moments"][:, :4].shape
    e_dec = rel_l2(dec, case["dec"])
    e_mean = rel_l2(post.mean, case["moments"][:, :4])
    e_lv = rel_l2(post.logvar, case["moments"][:, 4:].clamp(-30.0, 20.0))
    print(f"nonsquare vae {case['cfg']} z {tuple(case['z'].shape)} img {tuple(case['img'].shape)}: "
          f"decode {e_dec:.2e} mean {e_mean:.2e} logvar {e_lv:.2e}")
    assert e_dec < TOL_VAE and e_mean < TOL_VAE and e_lv < TOL_VAE


def test_vae_attention_rejects_token_counts_not_multiple_of_8(cuda_dev):
    """The VAE mid-block attention needs h*w % 8 == 0 (a 5x7 latent has 35 tokens): a clear error, not a wrong image."""
    import sdb200
    vae = sdb200.AutoencoderKL(**CFGS["vae"]["tiny"]).load_weights(weights("vae", "tiny", 12), cuda_dev)
    with pytest.raises(NotImplementedError, match="h\\*w % 8"):
        vae.decode(torch.randn(1, 4, 5, 7, device=cuda_dev))


def test_unet_rejects_latent_sides_not_divisible_by_the_level_count(cuda_dev):
    m = _unet("tiny", 11, cuda_dev)
    with pytest.raises(AssertionError, match="divisible"):
        m(torch.zeros(1, 4, 9, 16, device=cuda_dev), torch.zeros(1, device=cuda_dev),
          context=torch.zeros(1, 77, 64, device=cuda_dev))


def test_pipeline_plms_nonsquare_vs_reference(cuda_dev):
    """PLMS S=10, CFG 7.5 at a 8x24 latent through the LatentDiffusion facade, and decode_first_stage."""
    import sdb200
    from test_pipeline_gpu import _tiny_ld
    g = golden("nonsquare.pt")["pipeline"]
    ld = _tiny_ld(cuda_dev)
    c, uc, x_T = g["c"].to(cuda_dev), g["uc"].to(cuda_dev), g["x_T"].to(cuda_dev)
    s, _ = sdb200.PLMSSampler(ld).sample(S=10, conditioning=c, batch_size=2, shape=[4, 8, 24], verbose=False,
                                         unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=0.0, x_T=x_T)
    x_dec = ld.decode_first_stage(g["plms10"].to(cuda_dev))
    e_s, e_dec = rel_l2(s, g["plms10"]), rel_l2(x_dec, g["x_dec"])
    print(f"nonsquare plms10 (2,4,8,24): trajectory {e_s:.2e} decode_first_stage {e_dec:.2e}")
    assert s.shape == g["plms10"].shape and x_dec.shape == g["x_dec"].shape
    assert e_s < 2e-2 and e_dec < 2e-3


def test_unet_nonsquare_cuda_graph_and_autotune(cuda_dev):
    """Graph mode at (2,4,24,40): the first call autotunes every GEMM problem (tile shapes picked by timing alone) and
    captures; the replay must reproduce it, and both must match the reference."""
    import sdb200
    case = _sdv1_case()
    sd = weights("unet", "sdv1", case["seed"])
    graphed = sdb200.UNetModel(**CFGS["unet"]["sdv1"]).load_weights(sd, cuda_dev)
    graphed.use_cuda_graph = True
    x, t, ctx = case["x"].to(cuda_dev), case["t"].to(cuda_dev), _ctx(case).to(cuda_dev)
    first = graphed(x, t, context=ctx).clone()
    replay = graphed(x, t, context=ctx)
    torch.cuda.synchronize()
    e_first, e_replay = rel_l2(first, case["eps"]), rel_l2(replay, case["eps"])
    print(f"nonsquare unet sdv1 graph: first {e_first:.3e} replay {e_replay:.3e}")
    assert len(graphed._graphs) == 1
    assert e_first < TOL and e_replay < TOL
    assert rel_l2(replay, first) < 1e-4
    del graphed


def test_unet_nonsquare_c_handle_matches_python_forward(cuda_dev):
    """sdb_unet_create with h != w: the C plan reproduces the Python-sequenced evaluation bit for bit."""
    case = _sdv1_case()
    net = _unet("sdv1", case["seed"], cuda_dev)
    ctx = _ctx(case).to(cuda_dev)
    x, t = case["x"].to(cuda_dev), case["t"].to(cuda_dev).float()
    h = net.c_handle(tuple(x.shape), ctx)
    try:
        ref = net(x, t, context=ctx)
        out = h.forward(x, t)
        torch.cuda.synchronize()
        assert out.shape == (2, 4, 24, 40)
        assert torch.equal(out, ref), rel_l2(out, ref)
        err = rel_l2(out, case["eps"])
        print(f"nonsquare C-handle sdv1 (2,4,24,40) rel-L2 {err:.3e}")
        assert err < TOL
    finally:
        h.close()


def test_txt2img_nonsquare_image_shape(cuda_dev):
    """Txt2Img(height=64, width=192) on the tiny model (first-stage factor 2: a 32x96 latent, CUDA-graph UNet):
    [B, 64, 192, 3] uint8, not a transposed image. The text encoder is the tiny CLIP at the tiny UNet's context width."""
    import sdb200
    from sdb200 import arch
    from sdb200.pipeline import Txt2Img
    clip = {**arch.TINY_CLIP, "hidden_size": arch.TINY_UNET["context_dim"], "intermediate_size": 256,
            "num_attention_heads": 1}
    ld = sdb200.LatentDiffusion(
        first_stage_config={"target": "ldm.models.autoencoder.AutoencoderKL", "params": dict(arch.TINY_VAE)},
        cond_stage_config={"target": "ldm.modules.encoders.modules.FrozenCLIPEmbedder", "params": {"config": clip}},
        unet_config={"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": dict(arch.TINY_UNET)},
        linear_start=0.00085, linear_end=0.0120, timesteps=1000, conditioning_key="crossattn", scale_factor=0.18215,
        image_size=64, channels=4)
    sd = {"model.diffusion_model." + k: v for k, v in weights("unet", "tiny", 11).items()}
    sd.update({"first_stage_model." + k: v for k, v in weights("vae", "tiny", 12).items()})
    sd.update({"cond_stage_model.transformer." + k: v
               for k, v in arch.random_state_dict(arch.clip_param_shapes(clip), 13).items()})
    res = ld.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys
    ld = ld.to(cuda_dev)
    pipe = Txt2Img(ld, steps=5, height=64, width=192, f=2)
    assert pipe.shape == [4, 32, 96]
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 998, (2, 77), generator=g).to(cuda_dev)
    uids = torch.randint(0, 998, (2, 77), generator=g).to(cuda_dev)
    img = pipe(ids, uncond_ids=uids, x_T=torch.randn(2, 4, 32, 96, generator=g).to(cuda_dev))
    torch.cuda.synchronize()
    assert img.shape == (2, 64, 192, 3) and img.dtype == torch.uint8
    assert int(img.max()) > int(img.min())
