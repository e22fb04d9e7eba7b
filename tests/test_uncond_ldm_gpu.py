"""The unconditional attention-block LDM family (LSUN-Churches, scripts/sample_diffusion.py) on the H100.

Kernels against fp64 torch: sdb_groupnorm_mod (modulation x resample, non-square, 192 channels = 6 per group, strided
FiLM slices, fused and computed statistics), sdb_resample_f32 (exact), sdb_ddpm_step (bit-equal to the oracle). The
UNet, the DDIM (eta = 1) and ancestral trajectories and the EMA scope against the unmodified reference
(tests/golden/lsun.pt), the graph / autotune path and the C handle against the Python forward, argument checks, and the
sampling script end to end."""
import os

import pytest
import torch
import torch.nn.functional as F
import yaml

import helpers  # noqa: F401
import uncond_oracle as U
from helpers import golden, rel_l2, script
from sdb200 import arch, pipeline

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
CFG = {"tiny_attn": arch.TINY_ATTN_UNET, "tiny_attn_plain": arch.TINY_ATTN_PLAIN_UNET, "lsun": arch.LSUN_CHURCHES_UNET}
TOL = 1e-3
_models = {}


def _sd(tag, seed=11):
    return arch.random_state_dict(arch.unet_param_shapes(CFG[tag]), seed)


def _unet(tag, dev):
    import sdb200
    if tag not in _models:
        _models[tag] = sdb200.UNetModel(**CFG[tag]).load_weights(_sd(tag), dev)
    return _models[tag]


def _gn_ref(x, gamma, beta, scale, shift, resample):
    """fp64 torch: NHWC in, NHWC out."""
    h = x.double().permute(0, 3, 1, 2)
    y = F.group_norm(h, 32, gamma.double(), beta.double(), 1e-5)
    if scale is not None:
        y = y * (1 + scale.double()[:, :, None, None]) + shift.double()[:, :, None, None]
    y = F.silu(y)
    if resample == 1:
        y = F.avg_pool2d(y, 2)
    elif resample == 2:
        y = F.interpolate(y, scale_factor=2, mode="nearest")
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("resample", [0, 1, 2])
@pytest.mark.parametrize("mod", [False, True])
@pytest.mark.parametrize("shape", [(2, 6, 10, 192), (3, 12, 4, 64)])
def test_groupnorm_mod_vs_fp64(cuda_dev, shape, mod, resample):
    from sdb200 import ops
    g = torch.Generator(device="cpu").manual_seed(5)
    nb, h, w, c = shape
    x = (torch.randn(shape, generator=g) * 2 + 0.5).to(cuda_dev)
    gamma = (1 + 0.1 * torch.randn(c, generator=g)).to(cuda_dev)
    beta = (0.1 * torch.randn(c, generator=g)).to(cuda_dev)
    film = torch.randn(nb, 3 * c + 32, generator=g).to(cuda_dev) * 0.5     # scale / shift are strided column slices
    scale, shift = (film[:, 16: 16 + c], film[:, 16 + c: 16 + 2 * c]) if mod else (None, None)
    out = ops.groupnorm_mod(x, gamma, beta, scale=scale, shift=shift, resample=resample)
    ref = _gn_ref(x, gamma, beta, scale, shift, resample)
    assert out.shape == ref.shape
    err = rel_l2(out, ref)
    assert err < 1e-3, err
    if resample:     # the same buffer read as [nb, w, h, c] resamples different pixel pairs: far from the result
        far = _gn_ref(x.reshape(nb, w, h, c), gamma, beta, scale, shift, resample).reshape(out.shape)
        assert rel_l2(out, far) > 0.1


def test_groupnorm_mod_fused_statistics(cuda_dev):
    """Statistics from the producing GEMM's epilogue (entries of 2 channels, 6 per group) give the same result."""
    from sdb200 import ops
    g = torch.Generator(device="cpu").manual_seed(6)
    nb, h, w, k, c = 2, 8, 12, 64, 192
    a = (torch.randn(nb, h, w, k, generator=g)).half().to(cuda_dev)
    b = (torch.randn(c, 9 * k, generator=g) * (9 * k) ** -0.5).half().to(cuda_dev)
    _, y = ops.gemm(a, b, taps=9, want_f32=True, splits=-1, want_stats=True, stats_group=2)    # a 3x3 conv, as the UNet
    y = y.view(nb, h, w, c)
    assert ops.channel_stats(y) is not None
    gamma = (1 + 0.1 * torch.randn(c, generator=g)).to(cuda_dev)
    beta = (0.1 * torch.randn(c, generator=g)).to(cuda_dev)
    film = torch.randn(nb, 2 * c, generator=g).to(cuda_dev) * 0.5
    for resample in (0, 1, 2):
        out = ops.groupnorm_mod(y, gamma, beta, scale=film[:, :c], shift=film[:, c:], resample=resample)
        assert rel_l2(out, _gn_ref(y, gamma, beta, film[:, :c], film[:, c:], resample)) < 1e-3


@pytest.mark.parametrize("shape", [(2, 6, 10, 192), (1, 4, 2, 64)])
def test_resample_f32_exact(cuda_dev, shape):
    from sdb200 import ops
    x = torch.randn(shape, generator=torch.Generator().manual_seed(7)).to(cuda_dev)
    down = ops.resample_f32(x, 1)
    s = x[:, 0::2, 0::2] + x[:, 0::2, 1::2]
    s = s + x[:, 1::2, 0::2]
    s = s + x[:, 1::2, 1::2]
    assert torch.equal(down, s / 4)
    up = ops.resample_f32(x, 2)
    assert torch.equal(up, x.repeat_interleave(2, 1).repeat_interleave(2, 2))


@pytest.mark.parametrize("t", [0, 1, 13, 19])
def test_ddpm_step_bit_exact(cuda_dev, t):
    from sdb200 import ops
    g = torch.Generator().manual_seed(8 + t)
    x, eps, noise = (torch.randn(2, 4, 16, 24, generator=g) for _ in range(3))
    sched = U.ddpm_schedule(20)
    ref, ref_x0 = U.p_sample(x, eps, t, sched, noise)
    f = lambda k: float(sched[k][t])
    sigma = float(torch.tensor(1.0 if t else 0.0) * (0.5 * sched["posterior_log_variance_clipped"][t]).exp())
    out, x0 = ops.ddpm_step(x.to(cuda_dev), eps.to(cuda_dev), noise.to(cuda_dev),
                            sqrt_recip_ac=f("sqrt_recip_alphas_cumprod"), sqrt_recipm1_ac=f("sqrt_recipm1_alphas_cumprod"),
                            coef1=f("posterior_mean_coef1"), coef2=f("posterior_mean_coef2"), sigma=sigma)
    assert torch.equal(out.cpu(), ref) and torch.equal(x0.cpu(), ref_x0)


@pytest.mark.parametrize("idx", range(6))
def test_unet_vs_reference(cuda_dev, idx):
    case = golden("lsun.pt")["unet"][idx]
    net = _unet(case["cfg"], cuda_dev)
    eps = net(case["x"].to(cuda_dev), case["t"].to(cuda_dev))
    err = rel_l2(eps, case["eps"])
    print(f"unet {case['cfg']} {tuple(case['x'].shape)} rel-L2 {err:.3e}")
    assert eps.shape == case["eps"].shape and err < TOL


def test_lsun_graph_autotune_and_c_handle(cuda_dev):
    """(2,4,32,32), the real LSUN latent: the graph path (autotuned, first call and replay) and the C handle are
    bit-equal to the Python forward with the same tile choices."""
    import sdb200
    case = golden("lsun.pt")["unet"][4]
    assert tuple(case["x"].shape) == (2, 4, 32, 32)
    graphed = sdb200.UNetModel(**CFG["lsun"]).load_weights(_sd("lsun"), cuda_dev)
    graphed.use_cuda_graph = True
    x, t = case["x"].to(cuda_dev), case["t"].to(cuda_dev).float()
    first = graphed(x, t).clone()
    replay = graphed(x, t)
    graphed.use_cuda_graph = False
    eager = graphed(x, t)
    h = graphed.c_handle(tuple(x.shape))
    try:
        out = h.forward(x, t)
        torch.cuda.synchronize()
        print(f"lsun graph first {rel_l2(first, case['eps']):.3e} replay {rel_l2(replay, case['eps']):.3e} "
              f"C handle {rel_l2(out, case['eps']):.3e}")
        assert torch.equal(first, replay) and torch.equal(replay, eager) and torch.equal(out, eager)
        assert rel_l2(replay, case["eps"]) < TOL
    finally:
        h.close()


def test_rejections(cuda_dev):
    import sdb200
    net = _unet("tiny_attn", cuda_dev)
    x, t = torch.zeros(1, 4, 16, 16, device=cuda_dev), torch.zeros(1, device=cuda_dev)
    with pytest.raises(ValueError, match="unconditional"):
        net(x, t, context=torch.zeros(1, 77, 64, device=cuda_dev))
    with pytest.raises(AssertionError):
        net(torch.zeros(1, 4, 14, 16, device=cuda_dev), t)          # sides must divide by 2^(levels-1)
    sdt = sdb200.UNetModel(**arch.TINY_UNET).load_weights(arch.random_state_dict(arch.unet_param_shapes(arch.TINY_UNET), 11),
                                                         cuda_dev)
    with pytest.raises(AssertionError):
        sdt(x, t)                                                   # the transformer UNet needs a context


def _model(dev, timesteps=1000, use_ema=False):
    from sdb200.util import instantiate_from_config, remap_config
    g = golden("lsun.pt")
    mod = script("sample_diffusion")
    node = mod.lsun_churches_config(arch.TINY_ATTN_UNET, arch.TINY_VAE)
    node["params"].update(timesteps=timesteps, use_ema=use_ema)
    m = instantiate_from_config(remap_config(node))
    m = pipeline.load_random_weights(m, dev, seeds=(g["unet_seed"], g["vae_seed"])).eval()
    m.scale_factor.fill_(g["scale_factor"])
    return m, mod


def test_ddim_eta1_unconditional_trajectory(cuda_dev, monkeypatch):
    from sdb200.samplers import DDIMSampler
    g = golden("lsun.pt")
    d = g["ddim"]
    m, _ = _model(cuda_dev)
    draws = list(d["noise"])
    monkeypatch.setattr(torch, "randn_like", lambda t, *a, **k: draws.pop(0).to(t.device))
    s, _ = DDIMSampler(m).sample(10, batch_size=2, shape=[4, 16, 16], eta=1.0, verbose=False, x_T=d["x_T"].to(cuda_dev))
    monkeypatch.undo()
    assert not draws
    e_s = rel_l2(s, d["sample"])
    x_dec = m.decode_first_stage(d["sample"].to(cuda_dev))
    e_dec = rel_l2(x_dec, d["x_dec"])
    print(f"ddim eta=1 S=10 trajectory {e_s:.2e}; decode_first_stage {e_dec:.2e}")
    assert e_s < 5e-2 and e_dec < 2e-3


def test_ancestral_trajectory(cuda_dev, monkeypatch):
    a = golden("lsun.pt")["ancestral"]
    m, _ = _model(cuda_dev, timesteps=20)
    for k in ("posterior_mean_coef1", "posterior_log_variance_clipped", "sqrt_recipm1_alphas_cumprod"):
        assert torch.equal(getattr(m, k).cpu(), U.ddpm_schedule(20)[k])
    draws = list(a["noise"])
    real = torch.randn
    monkeypatch.setattr(torch, "randn", lambda *s, **k: draws.pop(0).to(k.get("device", "cpu")) if draws else real(*s, **k))
    s, inter = m.progressive_denoising(None, [2, 4, 16, 16], verbose=False, x_T=a["x_T"].to(cuda_dev))
    monkeypatch.undo()
    assert not draws and len(inter) == a["intermediates"].shape[0]
    e_s = rel_l2(s, a["sample"])
    e_dec = rel_l2(m.decode_first_stage(a["sample"].to(cuda_dev)), a["x_dec"])
    print(f"ancestral T=20 trajectory {e_s:.2e}; x0 intermediates {rel_l2(torch.stack(inter), a['intermediates']):.2e}; "
          f"decode {e_dec:.2e}")
    assert e_s < 5e-2 and e_dec < 2e-3


def test_ema_scope_switches_weights(cuda_dev):
    e = golden("lsun.pt")["ema"]
    m, _ = _model(cuda_dev, use_ema=True)
    unet = m.model.diffusion_model
    unet.set_weight_set("ema", _sd("tiny_attn", golden("lsun.pt")["ema_seed"]))
    x, t = e["x"].to(cuda_dev), e["t"].to(cuda_dev)
    raw = m.apply_model(x, t, None)
    with m.ema_scope():
        ema = m.apply_model(x, t, None)
    after = m.apply_model(x, t, None)
    print(f"ema scope: raw {rel_l2(raw, e['eps_raw']):.2e} ema {rel_l2(ema, e['eps_ema']):.2e}")
    assert rel_l2(raw, e["eps_raw"]) < TOL and rel_l2(ema, e["eps_ema"]) < TOL and torch.equal(raw, after)


def test_sample_diffusion_script_random_init(cuda_dev, tmp_path):
    import glob
    import numpy as np
    _, mod = _model(cuda_dev)
    node = mod.lsun_churches_config(arch.TINY_ATTN_UNET, arch.TINY_VAE)
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": node}))
    logdir = mod.main(["--random_init", "--config", str(cfg), "-n", "4", "--batch_size", "2", "-c", "5",
                       "-l", str(tmp_path / "out"), "--seed", "0"])
    pngs = sorted(glob.glob(os.path.join(logdir, "img", "*.png")))
    assert len(pngs) == 4      # numbered from len(existing pngs) - 1, as the reference script does
    npz = glob.glob(os.path.join(logdir, "numpy", "*.npz"))
    assert len(npz) == 1 and os.path.basename(npz[0]) == "4x32x32x3-samples.npz"     # tiny VAE: f = 2
    arr = np.load(npz[0])["arr_0"]
    assert arr.shape == (4, 32, 32, 3) and arr.dtype == np.uint8
