"""The first-stage autoencoders of models/first_stage_models/* on the H100: KL-f4, KL-f32, VQ-f8-n256 and VQ-f16 against
the unmodified reference (tests/golden/first_stage.pt) at full width, their small members against the oracle, the index
decisions of the quantizer, VQModel against VQModelInterface, the 1x1 latent heads up to 128 channels against fp64, and
scripts/autoencode.py end to end for all nine configs."""

import numpy as np
import pytest
import torch
import yaml

import helpers  # noqa: F401
import cin_f8_oracle as F8
import rdm_oracle as RO
from helpers import golden, rel_l2, script
import sdb200
from sdb200 import arch, ops

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
TOL = 2e-3
LS_REL = 1e-5     # the elementwise sweep's bound for sdb_pointwise_small: 1e-5 * sum_c |alpha x w| + |b|
_models = {}


def _shapes(cfg):
    return arch.vq_param_shapes(cfg) if "n_embed" in cfg else arch.vae_param_shapes(cfg)


def _model(cfg, seed, dev, cls=None):
    cls = cls or (sdb200.VQModel if "n_embed" in cfg else sdb200.AutoencoderKL)
    return cls(**cfg).load_weights(arch.random_state_dict(_shapes(cfg), seed), dev)


def _golden_model(name, dev):
    if name not in _models:
        _models.clear()
        _models[name] = _model(arch.FIRST_STAGES[name], golden("first_stage.pt")["weight_seed"], dev)
    return _models[name]


def _input(case):
    return torch.randn(case["shape"], generator=torch.Generator().manual_seed(case["seed"])).clamp(-1, 1)


# ------------------------------------------------------------------------------------------------ against the reference
@pytest.mark.parametrize("name", ["kl-f4", "kl-f32"])
def test_kl_vs_reference(cuda_dev, name):
    case = golden("first_stage.pt")["cases"][name]
    m = _golden_model(name, cuda_dev)
    x = _input(case).to(cuda_dev)
    post = m.encode(x)
    e_mom = rel_l2(post.parameters, case["moments"])
    zc = arch.FIRST_STAGES[name]["embed_dim"]
    assert torch.equal(post.mode(), post.mean) and torch.equal(post.mean, post.parameters[:, :zc])
    dec = m.decode(post.mean)
    e_dec = rel_l2(dec, case["dec"])
    print(f"{name}: moments rel-L2 {e_mom:.2e}, decode(mean) rel-L2 {e_dec:.2e}")
    assert post.parameters.shape == case["moments"].shape and e_mom < TOL
    assert dec.shape == case["dec"].shape and e_dec < TOL
    rec, post2 = m(x, sample_posterior=False)
    assert torch.equal(rec, dec) and torch.equal(post2.parameters, post.parameters)
    with pytest.raises(NotImplementedError):
        m(x, sample_posterior=True)
    with pytest.raises(NotImplementedError):
        m(x)


@pytest.mark.parametrize("name", ["vq-f8-n256", "vq-f16"])
def test_vq_vs_reference(cuda_dev, name):
    g = golden("first_stage.pt")
    case = g["cases"][name]
    cfg = arch.FIRST_STAGES[name]
    m = _golden_model(name, cuda_dev)
    x = _input(case).to(cuda_dev)
    h = m.encode_to_prequant(x)
    e_h = rel_l2(h, case["h"])
    assert h.shape == case["h"].shape and e_h < TOL

    # the quantizer on the reference's own latent makes the reference's decisions
    _, none, (_, _, idx_ref_h) = m.quantize(case["h"].to(cuda_dev))
    assert none is None and torch.equal(idx_ref_h.cpu(), case["indices"])

    quant, loss, (p0, p1, idx) = m.encode(x)
    assert p0 is None and p1 is None and idx.dtype == torch.int64 and idx.shape == case["indices"].shape
    ref_idx = case["indices"].to(cuda_dev)
    same = idx == ref_idx
    share = float(same.double().mean())
    # a decision may differ only where the reference's two nearest codes are closer than the latent's error can move
    # them: d(j) - d(i) changes by 2 (z_engine - z_ref) . (e_i - e_j), plus the fp32 rounding of the distances
    book = m.W["codebook"]
    e_dim = cfg["embed_dim"]
    z = h.permute(0, 2, 3, 1).reshape(-1, e_dim).double()
    z_ref = case["h"].to(cuda_dev).permute(0, 2, 3, 1).reshape(-1, e_dim).double()
    gap = (case["d_top2"][:, 1] - case["d_top2"][:, 0]).to(cuda_dev).double()
    moved = 2 * (z - z_ref).norm(dim=1) * (book[idx] - book[ref_idx]).double().norm(dim=1)
    slack = 1e-5 * (z_ref.pow(2).sum(1) + book.double().pow(2).sum(1).max())
    bad = ~same & (gap > moved + slack)
    print(f"{name}: latent rel-L2 {e_h:.2e}; indices equal {share:.4f} ({int((~same).sum())} of {same.numel()} differ, "
          f"all within the latent's error: {not bool(bad.any())})")
    assert share >= 0.99 and not bool(bad.any())

    e_loss = abs(float(loss) / float(case["emb_loss"]) - 1)
    assert loss.shape == () and e_loss < 5e-3, e_loss
    dec, diff, ind = m(x, return_pred_indices=True)
    assert torch.equal(diff, loss) and torch.equal(ind, idx) and torch.equal(dec, m.decode(quant))
    # forward's dec of every image whose decisions all agree with the reference's (a flipped near-tie selects another
    # code, which changes that image by far more than rounding), and the decoder on the reference's own decisions
    k = g["image_stride"]
    nb = dec.shape[0]
    agree = same.view(nb, -1).all(dim=1).tolist()
    e_dec = [rel_l2(dec[i, :, ::k, ::k], case["dec"][i]) for i in range(nb) if agree[i]]
    e_ref_codes = rel_l2(m.decode_code(ref_idx.view(nb, *h.shape[2:]))[..., ::k, ::k], case["dec"])
    print(f"{name}: emb_loss rel {e_loss:.2e}; dec rel-L2 {max(e_dec, default=0):.2e} over the {len(e_dec)} of {nb} "
          f"images with equal decisions; decode of the reference's codes {e_ref_codes:.2e}")
    assert len(e_dec) >= nb // 2 and max(e_dec) < TOL and e_ref_codes < TOL

    # decode_code: the codebook rows of the indices, decoded
    b, _, hh, ww = h.shape
    code = idx.view(b, hh, ww)
    rows = book[idx].view(b, hh, ww, e_dim).permute(0, 3, 1, 2).contiguous()
    assert torch.equal(m.get_codebook_entry(idx, (b, hh, ww, e_dim)), rows)
    from_code = m.decode_code(code)
    assert torch.equal(from_code, m.decode(rows))
    assert rel_l2(from_code, dec) < 1e-4       # quant is the straight-through z + (e - z): e to within rounding
    with pytest.raises(IndexError):
        m.decode_code(torch.full_like(code, cfg["n_embed"]))


# ------------------------------------------------------------------------------------------------ small members
@pytest.mark.parametrize("cfg_name", ["TINY_KL_F4", "TINY_KL_F32", "TINY_VQ_F16"])
def test_small_members_vs_oracle(cuda_dev, cfg_name):
    """Level attention 128 / 256 wide on the per-image path, a 4x4 bottom level, 128 -> 128 quant_conv, codes of 8."""
    cfg = getattr(arch, cfg_name)
    sd = arch.random_state_dict(_shapes(cfg), 5)
    m = _model(cfg, 5, cuda_dev)
    x = torch.randn(2, 3, 128, 128, generator=torch.Generator().manual_seed(6)).clamp(-1, 1)
    if "n_embed" in cfg:
        h_ref = F8.vq_encode(sd, x)
        h = m.encode_to_prequant(x.to(cuda_dev))
        dec = m.decode(m.get_codebook_entry(m.quantize(h_ref.to(cuda_dev))[2][2],
                                            (2, h.shape[2], h.shape[3], cfg["embed_dim"])))
        errs = rel_l2(h, h_ref), rel_l2(dec, F8.vq_decode(sd, h_ref))
    else:
        mom_ref = RO.kl_encode_moments(sd, x)
        post = m.encode(x.to(cuda_dev))
        errs = rel_l2(post.parameters, mom_ref), rel_l2(m.decode(post.mean), RO.kl_decode(sd, post.mean.cpu()))
    print(f"{cfg_name}: encode rel-L2 {errs[0]:.2e}, decode rel-L2 {errs[1]:.2e}")
    assert max(errs) < TOL


# ------------------------------------------------------------------------------------------------ VQModel vs interface
@pytest.mark.parametrize("name", ["vq-f4", "vq-f8"])
def test_vq_model_equals_interface(cuda_dev, name):
    cfg = arch.FIRST_STAGES[name]
    _models.clear()
    a = _model(cfg, 9, cuda_dev, sdb200.VQModel)
    b = _model(cfg, 9, cuda_dev, sdb200.VQModelInterface)
    x = torch.randn(1, 3, 128, 128, generator=torch.Generator().manual_seed(10)).clamp(-1, 1).to(cuda_dev)
    h = b.encode(x)
    assert torch.equal(a.encode_to_prequant(x), h)
    quant, _, (_, _, idx) = a.encode(x)
    q2, _, (_, _, idx2) = b.quantize(h)
    assert torch.equal(quant, q2) and torch.equal(idx, idx2)
    assert torch.equal(a.decode(quant), b.decode(h))
    assert torch.equal(a.decode(h), b.decode(h, force_not_quantize=True))


# ------------------------------------------------------------------------------------------------ 1x1 latent heads
@pytest.mark.parametrize("cin,cout,alpha", [(33, 33, 1.0), (64, 64, 1.0), (128, 128, 1.0), (33, 128, 1.0),
                                            (128, 64, 1.0), (64, 64, 1 / 0.18215), (128, 128, -0.5),
                                            (128, 128, 1 / 0.18215)])
def test_pointwise_small_wide_vs_fp64(cuda_dev, cin, cout, alpha):
    """quant_conv / post_quant_conv up to 128 channels: elementwise within the sweep's bound, repeat launches equal."""
    g = torch.Generator(device=cuda_dev).manual_seed(cin * 1000 + cout)
    x = 2.0 * torch.randn(2, 9, 13, cin, generator=g, device=cuda_dev)
    w = torch.randn(cout, cin, generator=g, device=cuda_dev) * cin ** -0.5
    b = torch.randn(cout, generator=g, device=cuda_dev)
    out = ops.pointwise_small(x, w, b, alpha=alpha)
    ref = (alpha * x.double()) @ w.double().t() + b.double()
    absref = (abs(alpha) * x.double().abs()) @ w.double().abs().t() + b.double().abs()
    assert bool(torch.isfinite(out).all())
    assert float(((out.double() - ref).abs() / (LS_REL * absref)).max()) <= 1.0
    assert torch.equal(ops.pointwise_small(x, w, b, alpha=alpha), out)
    no_bias = ops.pointwise_small(x, w, alpha=alpha)
    assert float(((no_bias.double() - (ref - b.double())).abs() / (LS_REL * absref)).max()) <= 1.0


def test_pointwise_small_rejects_past_128(cuda_dev):
    x = torch.zeros(4, 129, device=cuda_dev)
    with pytest.raises(RuntimeError, match="sdb_pointwise_small"):
        ops.pointwise_small(x, torch.zeros(8, 129, device=cuda_dev))
    with pytest.raises(RuntimeError, match="sdb_pointwise_small"):
        ops.pointwise_small(x[:, :8].contiguous(), torch.zeros(129, 8, device=cuda_dev))


# ------------------------------------------------------------------------------------------------ the script
@pytest.mark.parametrize("name", sorted(arch.FIRST_STAGES))
def test_autoencode_script_random_init(cuda_dev, tmp_path, name):
    from PIL import Image
    _models.clear()
    S = script("autoencode")
    cfg_path = tmp_path / "config.yaml"
    cfg_path.write_text(yaml.safe_dump(golden("first_stage.pt")["yamls"][name]))
    out = tmp_path / "out"
    written = S.main(["--config", str(cfg_path), "--random_init", "--n_samples", "2", "--H", "256", "--W", "256",
                      "--outdir", str(out), "--save_latents"])
    assert len(written) == 2
    imgs = [np.array(Image.open(p)) for p in written]
    assert all(i.shape == (256, 256, 3) and i.dtype == np.uint8 for i in imgs) and imgs[0].std() > 0
    lat = torch.load(out / "latents.pt", weights_only=True)["synthetic"]
    cfg = arch.FIRST_STAGES[name]
    f = 2 ** (len(cfg["ddconfig"]["ch_mult"]) - 1)
    if "n_embed" in cfg:
        assert lat["h"].shape == (2, cfg["embed_dim"], 256 // f, 256 // f)
        assert lat["indices"].shape == (2 * (256 // f) ** 2,)
        assert int(lat["indices"].min()) >= 0 and int(lat["indices"].max()) < cfg["n_embed"]
    else:
        assert lat["mean"].shape == (2, cfg["embed_dim"], 256 // f, 256 // f)
        assert bool(torch.isfinite(lat["mean"]).all())
