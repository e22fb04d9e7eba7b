"""First-stage loss on the GPU: every entry point of include/sdb200_ae_loss.h and the ReLU / LeakyReLU GEMM epilogues
elementwise against fp64, determinism, and LPIPS / the discriminator / both loss calls / validation_step against the
unmodified reference (tests/golden/ae_loss.pt)."""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import helpers
import sdb200
from sdb200 import ae_loss, arch, ops
from sdb200.vae import DiagonalGaussianDistribution

pytestmark = pytest.mark.gpu
TAU = 1e-5    # the GEMM plan test's elementwise bound of the fp32 accumulation, relative to the abs-value reference
U = 2.0 ** -24


def _g():
    return helpers.golden("ae_loss.pt")


def _u8(u8, dev):
    return (u8.permute(0, 3, 1, 2).float() / 127.5 - 1.0).contiguous().to(dev)


def ulp16(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return 2.0 ** (e - 10)


def _loss(dev, disc_loss="hinge", seed=None, logvar=None):
    g = _g()
    m = sdb200.LPIPSWithDiscriminator(**g["loss_params"], disc_loss=disc_loss)
    m.load_state_dict(ae_loss.random_loss_state_dict(ae_loss.loss_param_shapes(), seed or g["loss_seed"],
                                                     logvar=g["logvar"] if logvar is None else logvar))
    return m.to(dev).eval()


# ---------------------------------------------------------------- kernels against fp64
def test_maxpool_exact(cuda_dev):
    for nb, h, w, c in ((2, 64, 64, 64), (1, 17, 9, 512), (3, 2, 2, 8)):
        x = torch.randn(nb, h, w, c, device=cuda_dev).half()
        x[0, 0, 0, 0] = float("nan")
        ref = F.max_pool2d(x.float().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
        out = ops.maxpool2x2(x)
        assert out.shape == ref.shape
        assert torch.equal(out.float().nan_to_num(7.0), ref.nan_to_num(7.0)) and out.float()[0, 0, 0, 0].isnan()


@pytest.mark.parametrize("c,h,w,k,stride,pad", [(3, 64, 64, 4, 2, 1), (64, 32, 32, 4, 2, 1), (256, 8, 8, 4, 1, 1),
                                                (8, 9, 7, 3, 1, 1), (512, 5, 6, 4, 1, 1)])
def test_im2col_exact(cuda_dev, c, h, w, k, stride, pad):
    x = torch.randn(2, h, w, c, device=cuda_dev).half()
    kpad = (k * k * c + 63) // 64 * 64
    col, ho, wo = ops.im2col(x, k, stride, pad, kpad)
    u = F.unfold(x.float().permute(0, 3, 1, 2), k, padding=pad, stride=stride)        # [n, c*k*k, L], (c, ky, kx)
    u = u.view(2, c, k * k, ho * wo).permute(0, 3, 2, 1).reshape(2 * ho * wo, k * k * c)
    assert torch.equal(col[:, : k * k * c].float(), u) and not col[:, k * k * c:].any()


def _conv_ref(x16, w, b, stride, pad, act):
    """fp64 conv of the fp16 operands + bias and activation, and the abs-value bound reference."""
    xd = x16.double().permute(0, 3, 1, 2)
    wd = w.double()
    v = F.conv2d(xd, wd, b.double(), stride=stride, padding=pad)
    av = F.conv2d(xd.abs(), wd.abs(), b.double().abs(), stride=stride, padding=pad)
    ref = v.clamp_min(0) if act == sdb200.lib.ACT_RELU else torch.where(v > 0, v, 0.2 * v)
    return ref.permute(0, 2, 3, 1), av.permute(0, 2, 3, 1)


def test_vgg_and_discriminator_gemms_at_256(cuda_dev):
    """Every GEMM problem LPIPS and the discriminator run at 256^2 (one image pair), with its ReLU / LeakyReLU epilogue,
    elementwise: |out - ref| <= ulp16(ref) + TAU * (|A| |B| + |bias|)."""
    lp = _loss(cuda_dev).perceptual_loss
    torch.manual_seed(0)
    h = 256
    worst = 0.0
    for j, (sl, i, cin, cout) in enumerate(ae_loss.VGG16_CONVS):
        if i in (5, 10, 17, 24):
            h //= 2
        w = lp._host_sd[f"net.{sl}.{i}.weight"].to(cuda_dev).half().float()
        b = lp._host_sd[f"net.{sl}.{i}.bias"].to(cuda_dev).float()
        x = torch.rand(2, h, h, cin, device=cuda_dev).half()
        c = lp.W["convs"][j]
        if j == 0:
            col = ops.im2col3x3(x.float().contiguous(), 1, 1, h, h, c["w"].shape[1])
            o, _ = ops.gemm(col, c["w"], bias=c["b"], act=sdb200.lib.ACT_RELU, want_f16=True)
        else:
            o, _ = ops.gemm(x, c["w"], taps=9, bias=c["b"], act=sdb200.lib.ACT_RELU, want_f16=True, splits=-1)
        ref, av = _conv_ref(x, w, b, 1, 1, sdb200.lib.ACT_RELU)
        e = ((o.view_as(ref).double() - ref).abs() / (ulp16(ref) + TAU * av)).max().item()
        worst = max(worst, e)
        assert e <= 1.0, (sl, i, h, e)
    d = _loss(cuda_dev).discriminator
    h = 256
    for li, (i, cin, cout, stride, _, bn, lrelu) in enumerate(d.layers):
        c = d.W["convs"][li]
        x = torch.randn(1, h, h, cin, device=cuda_dev).half()
        col, ho, wo = ops.im2col(x, 4, stride, 1, c["w"].shape[1])
        wf = c["w"][:, : 16 * cin].contiguous().float().view(-1, 4, 4, cin).permute(0, 3, 1, 2)   # the folded, packed weights
        if lrelu:
            o, _ = ops.gemm(col, c["w"], bias=c["b"], act=c["act"], want_f16=True)
            ref, av = _conv_ref(x, wf, c["b"], stride, 1, sdb200.lib.ACT_LEAKY_RELU)
            e = ((o.view_as(ref).double() - ref).abs() / (ulp16(ref) + TAU * av)).max().item()
        else:
            _, o = ops.gemm(col, c["w"], bias=c["b"], want_f32=True)
            xd = x.double().permute(0, 3, 1, 2)
            ref = F.conv2d(xd, wf.double(), c["b"].double(), stride=stride, padding=1).permute(0, 2, 3, 1)
            av = F.conv2d(xd.abs(), wf.double().abs(), c["b"].double().abs(), stride=stride, padding=1).permute(0, 2, 3, 1)
            e = ((o.view_as(ref).double() - ref).abs() / (TAU * av + 1e-30)).max().item()
        worst = max(worst, e)
        assert e <= 1.0, (i, h, e)
        h = ho
    print(f"largest share of the bound used: {worst:.3f}")


@pytest.mark.parametrize("act", [sdb200.lib.ACT_RELU, sdb200.lib.ACT_LEAKY_RELU])
def test_relu_family_runs_unsplit(cuda_dev, act):
    """A split-K request with a ReLU activation resolves to one split (the split-K second pass has no ReLU): the plan
    says so and the output equals the unsplit launch bit for bit; value 5, between GELU and ReLU, stays rejected."""
    g = torch.Generator(device=cuda_dev).manual_seed(3)
    a = torch.randn(256, 4608, generator=g, device=cuda_dev).half()
    b = torch.randn(512, 4608, generator=g, device=cuda_dev).half()
    d = ops.GemmDesc()
    d.a0, d.c0, d.nb, d.h, d.w, d.taps = a.data_ptr(), 4608, 1, 1, 256, 1
    d.b, d.n, d.alpha, d.act, d.splits = b.data_ptr(), 512, 1.0, act, 8
    d.out_f32 = torch.empty(1, device=cuda_dev).data_ptr()
    plan = (ctypes.c_int32 * 5)()
    assert sdb200.lib.load().sdb_gemm_plan(ctypes.byref(d), plan) == 0 and plan[2] == 1
    _, o8 = ops.gemm(a, b, act=act, want_f32=True, splits=8)
    _, o1 = ops.gemm(a, b, act=act, want_f32=True, splits=1)
    assert torch.equal(o8, o1) and (o1 >= 0).all() == (act == sdb200.lib.ACT_RELU)
    with pytest.raises(RuntimeError, match="unknown activation"):
        ops.gemm(a, b, act=5, want_f32=True)


def test_batchnorm_fold(cuda_dev):
    """The folded conv equals conv -> eval BatchNorm in fp64 to the fold's fp32 roundings."""
    d = _loss(cuda_dev).discriminator
    sd = {k: v.double() for k, v in d._host_sd.items() if not k.endswith("num_batches_tracked")}
    i, cin, cout, _, _, bn, _ = d.layers[1]
    x = torch.randn(1, cin, 8, 8, dtype=torch.float64)
    ref = F.batch_norm(F.conv2d(x, sd[f"main.{i}.weight"], padding=1), sd[f"main.{bn}.running_mean"],
                       sd[f"main.{bn}.running_var"], sd[f"main.{bn}.weight"], sd[f"main.{bn}.bias"], eps=1e-5)
    s = sd[f"main.{bn}.weight"] / torch.sqrt(sd[f"main.{bn}.running_var"] + 1e-5)
    wf = (d._host_sd[f"main.{i}.weight"] * s.float().view(-1, 1, 1, 1)).double()
    bf = d.W["convs"][1]["b"].cpu().double()
    out = F.conv2d(x, wf, bf, padding=1)
    av = F.conv2d(x.abs(), wf.abs(), bf.abs(), padding=1)
    assert ((out - ref).abs() <= 8 * U * (av + 1.0)).all()


def _head_ref(f, lin_w, nb):
    x = f.double()
    n = (x * x).sum(-1, keepdim=True).sqrt().float() + 1e-10
    a, b = (f.float() / n)[:nb].double(), (f.float() / n)[nb:].double()
    d = (a - b) ** 2
    return (d * lin_w.double()).sum(-1).mean((1, 2)), (lin_w.double().abs() * (a.abs() + b.abs()) ** 2).sum(-1).mean((1, 2))


@pytest.mark.parametrize("c,h,w", [(64, 64, 64), (128, 17, 33), (256, 16, 16), (512, 1, 1), (512, 4, 6)])
def test_lpips_head_vs_fp64(cuda_dev, c, h, w):
    """Within 2^-20 of the abs-value reference: the normalised features and their difference carry a few fp32
    roundings (each <= 2^-24 of |a| + |b|), squared (x 2) and summed with non-negative weights in fp64."""
    nb = 3
    f = torch.randn(2 * nb, h, w, c, device=cuda_dev).abs().half()
    lin_w = torch.rand(c, device=cuda_dev)
    acc = torch.empty(nb, dtype=torch.float64, device=cuda_dev)
    ops.lpips_head(f, lin_w, acc, first=True)
    ref, absref = _head_ref(f, lin_w, nb)
    assert ((acc - ref).abs() <= 2.0 ** -20 * absref).all(), ((acc - ref).abs() / absref).max()
    out = torch.empty(nb, device=cuda_dev)
    ops.lpips_head(f, lin_w, acc, first=False, out=out)
    assert torch.allclose(acc, 2 * ref, rtol=2.0 ** -19) and torch.equal(out, acc.float())


def test_loss_terms_vs_fp64(cuda_dev):
    """fp64 sums of fp32 element values: within n * 2^-52 of the exact sum of those values (the element value's own
    fp32 roundings are the reference's); KL within 4 ulp of expf per element."""
    nb = 3
    a = torch.randn(nb, 3, 40, 24, device=cuda_dev)
    b = torch.randn(nb, 3, 40, 24, device=cuda_dev)
    s = ops.ae_loss_terms(a, "abs", b=b)[0]
    ref = (a - b).abs().double().sum((1, 2, 3))
    assert torch.allclose(s, ref, rtol=a[0].numel() * 2.0 ** -52, atol=0)
    m = torch.randn(nb, 5, 7, 8, device=cuda_dev) * 4
    kl = ops.ae_loss_terms(m, "kl", cc=4)[0]
    mu, lv = m[..., :4].double(), m[..., 4:].double().clamp(-30, 20)
    ref = 0.5 * (mu * mu + lv.exp() - 1 - lv).sum((1, 2, 3))
    absref = 0.5 * (mu * mu + lv.exp() + 1 + lv.abs()).sum((1, 2, 3))
    assert ((kl - ref).abs() <= 8 * U * absref).all()
    lg = torch.randn(nb * 10, 32, device=cuda_dev) * 10
    t = ops.ae_loss_terms(lg, "logits", n=10, cc=32)
    l0 = lg[:, 0].double().view(nb, 10)
    refs = [l0.sum(1), (1 - l0).clamp_min(0).sum(1), (1 + l0).clamp_min(0).sum(1), F.softplus(-l0).sum(1),
            F.softplus(l0).sum(1)]
    for r in range(5):
        assert torch.allclose(t[r], refs[r], rtol=1e-6, atol=1e-5), (r, t[r], refs[r])


def test_determinism_and_batch_of_one(cuda_dev):
    """A sample's LPIPS, loss terms and logit sums are the same bits on a rerun and alone as inside the batch."""
    lp = _loss(cuda_dev)
    g = torch.Generator().manual_seed(5)
    x0 = (torch.rand(3, 3, 48, 40, generator=g) * 2 - 1).to(cuda_dev)
    x1 = (torch.rand(3, 3, 48, 40, generator=g) * 2 - 1).to(cuda_dev)
    v = lp.perceptual_loss(x0, x1)
    assert torch.equal(v, lp.perceptual_loss(x0, x1))
    for i in range(3):
        assert torch.equal(lp.perceptual_loss(x0[i:i + 1], x1[i:i + 1]).view(-1), v.view(-1)[i:i + 1])
    s = ops.ae_loss_terms(x0, "abs", b=x1)[0]
    o, (ho, wo) = lp.discriminator.logits_rows(x1)
    t = ops.ae_loss_terms(o, "logits", n=ho * wo, cc=o.shape[1])
    for i in range(3):
        assert torch.equal(ops.ae_loss_terms(x0[i:i + 1].contiguous(), "abs", b=x1[i:i + 1].contiguous())[0], s[i:i + 1])
        oi, _ = lp.discriminator.logits_rows(x1[i:i + 1])
        assert torch.equal(ops.ae_loss_terms(oi, "logits", n=ho * wo, cc=o.shape[1]), t[:, i:i + 1])


# ---------------------------------------------------------------- against the reference
def _feature_error(cuda_dev, lp, x0):
    """Measured rel-L2 of the engine's relu1_2 features against fp32 CPU convs of the same input."""
    sd = lp._host_sd
    W = lp.W
    xs = ops.lpips_scale(x0, x0, W["shift"], W["scale"])
    col = ops.im2col3x3(xs, 1, 1, x0.shape[2], x0.shape[3], W["convs"][0]["w"].shape[1])
    h, _ = ops.gemm(col, W["convs"][0]["w"], bias=W["convs"][0]["b"], act=sdb200.lib.ACT_RELU, want_f16=True)
    h = h.view(2 * x0.shape[0], x0.shape[2], x0.shape[3], -1)
    h, _ = ops.gemm(h, W["convs"][1]["w"], taps=9, bias=W["convs"][1]["b"], act=sdb200.lib.ACT_RELU, want_f16=True)
    h = h.view(2 * x0.shape[0], x0.shape[2], x0.shape[3], -1)
    sc = (x0.cpu() - sd["scaling_layer.shift"]) / sd["scaling_layer.scale"]
    r = F.relu(F.conv2d(sc, sd["net.slice1.0.weight"], sd["net.slice1.0.bias"], padding=1))
    r = F.relu(F.conv2d(r, sd["net.slice1.2.weight"], sd["net.slice1.2.bias"], padding=1))
    return helpers.rel_l2(h[: x0.shape[0]].permute(0, 3, 1, 2), r)


@pytest.mark.parametrize("size", ["64x64", "64x96"])
def test_lpips_vs_reference(cuda_dev, size):
    """LPIPS within 2 * 13 * e of the reference's value (relative), e the measured relu1_2 feature error: the error
    carried through 13 convs grows at most linearly with depth, and LPIPS is quadratic in the feature difference."""
    g = _g()["lpips"][size]
    lp = _loss(cuda_dev).perceptual_loss
    x0, x1 = _u8(g["in0"], cuda_dev), _u8(g["in1"], cuda_dev)
    e = _feature_error(cuda_dev, lp, x0)
    v = lp(x0, x1)
    assert v.shape == (2, 1, 1, 1)
    err = ((v.cpu().double() - g["value"].double()).abs() / g["value"].double().abs()).max().item()
    print(f"LPIPS {size}: feature error {e:.2e}, value error {err:.2e}")
    assert e < 2e-3 and err <= 26 * e


def test_discriminator_logits_vs_reference(cuda_dev):
    """Logits within 5 layers x 2 fp16 roundings of the activations (2^-11 each) of the reference's, rel-L2."""
    g = _g()
    d = _loss(cuda_dev).discriminator
    xr = _u8(g["lpips"]["64x64"]["in1"], cuda_dev)
    lg = d(xr)
    assert lg.shape == g["logits"].shape
    err = helpers.rel_l2(lg, g["logits"])
    print(f"logits rel-L2 {err:.2e}")
    assert err < 10 * 2.0 ** -11


# LPIPS enters rec / nll / total with its 26 e bound (about 1.3e-2 at the measured e) times its share of rec_loss
# (0.1 of 0.77 here); the logit means carry the logits' error, against means near -0.15 that are averages of both signs
TOL = {"rec_loss": 5e-3, "nll_loss": 5e-3, "total_loss": 5e-3, "g_loss": 5e-2, "disc_loss": 5e-2, "logits_real": 5e-2,
       "logits_fake": 5e-2}


def _close(a, b, rel):
    return abs(a - b) <= rel * max(abs(b), 1e-3)


@pytest.mark.parametrize("kind", ["hinge", "vanilla"])
def test_loss_calls_vs_reference(cuda_dev, kind):
    """Both calls on each side of disc_start. Terms from the images and posterior: within 1e-5; LPIPS- and
    logit-derived entries within the LPIPS / logit bounds above."""
    g = _g()
    m = _loss(cuda_dev, kind)
    x = _u8(g["lpips"]["64x64"]["in0"], cuda_dev)
    xr = _u8(g["lpips"]["64x64"]["in1"], cuda_dev)
    mom = g["moments"]
    post = DiagonalGaussianDistribution(mom.permute(0, 2, 3, 1).reshape(-1, mom.shape[1]).contiguous().to(cuda_dev),
                                        mom.shape[0], mom.shape[2], mom.shape[3], mom.shape[1] // 2)
    assert torch.allclose(post.kl().cpu(), g["kl"], rtol=1e-5)
    for (k, gs, idx), ref in g["calls"].items():
        if k != kind:
            continue
        loss, log = m(x, xr, post, idx, gs, split="val")
        assert set(log) == set(ref["log"])
        for name, r in ref["log"].items():
            assert _close(float(log[name]), r, TOL.get(name.split("/")[1], 1e-5)), (kind, gs, idx, name, float(log[name]), r)
        assert _close(float(loss), ref["loss"], TOL["total_loss"])


def test_validation_step_vs_reference(cuda_dev, tmp_path):
    g = _g()
    vae = sdb200.AutoencoderKL(**arch.TINY_VAE)
    vae.load_weights(arch.random_state_dict(arch.vae_param_shapes(arch.TINY_VAE), g["fs_seed"]), cuda_dev)
    object.__setattr__(vae, "loss", _loss(cuda_dev))
    batch = {"image": g["validation"]["batch"].float() / 127.5 - 1.0}
    for gs, ref in g["validation"]["logs"].items():
        vae.global_step = gs
        torch.manual_seed(g["val_seed"])
        log = vae.validation_step(batch, 0)
        assert set(log) == set(ref)
        for name, r in ref.items():
            assert _close(float(log[name]), r, TOL.get(name.split("/")[1], 1e-3)), (gs, name, float(log[name]), r)


@pytest.mark.parametrize("zc", [3, 16])
def test_validation_step_refuses_non_4_channel_posteriors(cuda_dev, zc):
    """KL-f4 (3 channels) and KL-f16 (16): validation_step samples through forward(), which refuses these widths."""
    cfg = dict(arch.TINY_VAE, embed_dim=zc, ddconfig=dict(arch.TINY_VAE["ddconfig"], z_channels=zc))
    vae = sdb200.AutoencoderKL(**cfg)
    vae.load_weights(arch.random_state_dict(vae.shapes, 3), cuda_dev)
    object.__setattr__(vae, "loss", _loss(cuda_dev))
    x = torch.zeros(1, 3, 32, 32, device=cuda_dev)
    with pytest.raises(NotImplementedError) as fwd:
        vae(x)
    with pytest.raises(NotImplementedError) as val:
        vae.validation_step({"image": torch.zeros(1, 32, 32, 3)}, 0)
    assert str(val.value) == str(fwd.value)


def test_eval_autoencoder_script_random_init(cuda_dev, tmp_path):
    import yaml
    cfg = {"model": {"target": "ldm.models.autoencoder.AutoencoderKL",
                     "params": {**arch.TINY_VAE, "lossconfig": {"target": "ldm.modules.losses.LPIPSWithDiscriminator",
                                                                "params": {"disc_start": 5, "kl_weight": 1e-6,
                                                                           "disc_weight": 0.5}}}}}
    path = tmp_path / "tiny.yaml"
    path.write_text(yaml.safe_dump(cfg))
    r = subprocess.run([sys.executable, os.path.join(helpers.ROOT, "scripts", "eval_autoencoder.py"), "--config",
                        str(path), "--random_init", "--size", "32", "--batch_size", "2", "--n_batches", "2",
                        "--global_step", "7"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    import json
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["batches"] == 2 and res["global_step"] == 7 and res["val/disc_factor"] == 1.0
    assert all(math.isfinite(res[k]) for k in ("val/rec_loss", "val/nll_loss", "val/kl_loss", "val/disc_loss"))
