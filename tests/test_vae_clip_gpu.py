"""AutoencoderKL decode/encode and CLIP text encoder on the H100 against the reference's outputs (golden fixtures)."""
import pytest
import torch

from helpers import CFGS, golden, rel_l2, weights

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
TOL = 2e-3  # fp16 operands / fp32 accumulate over ~30 conv layers; measured values are printed


@pytest.mark.parametrize("idx", range(2))
def test_vae_decode_encode_vs_reference(cuda_dev, idx):
    import sdb200
    case = golden("vae.pt")[idx]
    vae = sdb200.AutoencoderKL(**CFGS["vae"][case["cfg"]]).load_weights(weights("vae", case["cfg"], case["seed"]), cuda_dev)
    dec = vae.decode(case["z"].to(cuda_dev))
    e_dec = rel_l2(dec, case["dec"])
    post = vae.encode(case["img"].to(cuda_dev))
    e_mean = rel_l2(post.mean, case["mean"])
    e_lv = rel_l2(post.logvar, case["logvar"])
    print(f"vae {case['cfg']}: decode {e_dec:.2e} mean {e_mean:.2e} logvar {e_lv:.2e}")
    assert dec.shape == case["dec"].shape
    assert e_dec < TOL and e_mean < TOL and e_lv < TOL
    # posterior sample with given noise == (mean + exp(0.5 logvar) eps) * scale
    noise = torch.randn(case["mean"].shape, generator=torch.Generator().manual_seed(1))
    z = post.sample(noise=noise.to(cuda_dev), scale=0.18215)
    ref = 0.18215 * (case["mean"] + torch.exp(0.5 * case["logvar"]) * noise)
    assert rel_l2(z, ref) < TOL


@pytest.mark.parametrize("idx", range(2))
def test_clip_vs_transformers(cuda_dev, idx):
    import sdb200
    case = golden("clip.pt")[idx]
    cfg = CFGS["clip"][case["cfg"]]
    enc = sdb200.FrozenCLIPEmbedder(config=cfg).load_weights(weights("clip", case["cfg"], case["seed"]), cuda_dev)
    z = enc.encode_ids(case["ids"].to(cuda_dev))
    err = rel_l2(z, case["z"])
    print(f"clip {case['cfg']}: {err:.2e}")
    assert z.shape == case["z"].shape and err < TOL
    with pytest.raises(RuntimeError):
        enc.encode(["a photo of a cat"])  # no tokenizer vocabulary offline: must fail loudly, not fall back
