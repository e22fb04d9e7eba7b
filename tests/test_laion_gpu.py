"""The LAION-400M text-to-image LDM on the H100: the BERT text encoder (exact-GELU GEMM epilogue) and the UNet with a
1280-wide context against the unmodified reference (tests/golden/laion.pt), the CUDA-graph path against eager, a tiny
guided PLMS run from token ids to the decoded image, scripts/txt2img.py --laion400m end to end, the exact-GELU epilogue
and every GEMM plan at the encoder's and the UNet's GEMM problems against fp64."""
import os
import subprocess
import sys

import pytest
import torch

import helpers  # noqa: F401
import test_gemm_plans_gpu as GP
from helpers import golden, rel_l2
from sdb200 import arch, ops
from sdb200.lib import ACT_GELU
from workloads import GEMM_MODEL_WORKLOADS

pytestmark = pytest.mark.gpu
BCFG = {"tiny": arch.TINY_BERT, "full": arch.LAION_BERT}
UCFG = {"tiny": arch.TINY_LAION_UNET, "full": arch.LAION_UNET}


def _ctx(case, cfg):
    return torch.randn((case["x"].shape[0], 77, cfg["context_dim"]), generator=torch.Generator().manual_seed(case["ctx_seed"]))


def _bert(tag, dev, seed):
    import sdb200
    sd = arch.random_state_dict(arch.bert_param_shapes(BCFG[tag]), seed)
    return sdb200.BERTEmbedder(**BCFG[tag], use_tokenizer=False).load_weights(sd, dev)


@pytest.mark.parametrize("idx", range(2))
def test_bert_matches_reference(cuda_dev, idx):
    g = golden("laion.pt")
    case = g["bert"][idx]
    emb = _bert(case["cfg"], cuda_dev, g["bert_seed"])
    z = emb.encode(case["ids"])
    assert z.shape == (2, 77, BCFG[case["cfg"]]["n_embed"]) and z.dtype == torch.float32 and z.is_cuda
    errs = [rel_l2(z[i], case["z"][i].float()) for i in range(2)]
    print(f"\nBERT {case['cfg']}: rel-L2 prompt row {errs[0]:.2e}, empty-prompt row {errs[1]:.2e}")
    assert max(errs) < 2e-3
    assert torch.equal(emb(case["ids"].to(cuda_dev)), z)            # ids on the device, through forward
    short = emb.encode(case["ids"][:, :20])                          # n < 77: positions 0 .. n-1
    assert short.shape == (2, 20, z.shape[-1]) and rel_l2(short[0], z[0, :20]) > 1e-3
    with pytest.raises(IndexError):
        emb.encode(torch.full((1, 77), BCFG[case["cfg"]]["vocab_size"]))


@pytest.mark.parametrize("idx", range(4))
def test_unet_eps_matches_reference(cuda_dev, idx):
    import sdb200
    g = golden("laion.pt")
    case = g["unet"][idx]
    cfg = UCFG[case["cfg"]]
    net = sdb200.UNetModel(**cfg).load_weights(arch.random_state_dict(arch.unet_param_shapes(cfg), g["unet_seed"]), cuda_dev)
    x, t, c = case["x"].to(cuda_dev), case["t"].to(cuda_dev), _ctx(case, cfg).to(cuda_dev)
    eps = net(x, t, context=c)
    err = rel_l2(eps, case["eps"])
    print(f"\nUNet {case['cfg']} {tuple(x.shape)} context (77, {cfg['context_dim']}): eps rel-L2 {err:.2e}")
    assert err < 1e-3
    if case["cfg"] == "full" and idx == 2:
        net.use_cuda_graph = True
        first = net(x, t.float(), context=c).clone()
        replay = net(x, t.float(), context=c)
        net.use_cuda_graph = False
        eager = net(x, t.float(), context=c)
        print(f"graph replay rel-L2 {rel_l2(replay, case['eps']):.2e}")
        assert torch.equal(first, replay) and torch.equal(replay, eager)


def test_tiny_guided_plms_from_ids_to_image(cuda_dev):
    import sdb200
    from sdb200 import pipeline
    g = golden("laion.pt")
    d = g["plms"]
    model = pipeline.build_laion_model(arch.TINY_LAION_UNET, arch.TINY_VAE, arch.TINY_BERT)
    model = pipeline.load_random_weights(model, cuda_dev, seeds=(g["unet_seed"], g["vae_seed"], g["bert_seed"])).eval()
    assert isinstance(model.cond_stage_model, sdb200.BERTEmbedder)
    pipe = pipeline.Txt2Img(model, sampler="plms", steps=10, scale=7.5, height=32, width=32, f=2)
    ids, un, x_T = d["ids"].to(cuda_dev), d["uc_ids"].to(cuda_dev), d["x_T"].to(cuda_dev)
    s = pipe(ids, un, x_T=x_T, return_latent=True)
    x_dec = model.decode_first_stage(s)
    ref_dec = model.decode_first_stage(d["sample"].to(cuda_dev))
    errs = dict(latent=rel_l2(s, d["sample"]), decode_of_reference_latent=rel_l2(ref_dec, d["x_dec"]),
                image=rel_l2(x_dec, d["x_dec"]))
    print("\ntiny guided PLMS-10: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert errs["latent"] < 2e-2 and errs["decode_of_reference_latent"] < 2e-3 and errs["image"] < 2e-2
    img = pipe(ids, un, x_T=x_T)
    assert img.shape == (2, 32, 32, 3) and img.dtype == torch.uint8


def test_txt2img_laion400m_random_init(cuda_dev, tmp_path):
    """scripts/txt2img.py --laion400m --random_init end to end (full-size model, 256², 5 PLMS steps, stand-in ids)."""
    script = os.path.join(helpers.ROOT, "scripts", "txt2img.py")
    r = subprocess.run([sys.executable, script, "--laion400m", "--random_init", "--plms", "--ddim_steps", "5",
                        "--H", "256", "--W", "256", "--n_samples", "2", "--n_iter", "1", "--skip_save"],
                       cwd=tmp_path, capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, HF_HUB_OFFLINE="1"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "Falling back to LAION 400M model..." in r.stdout and "seeded token ids" in r.stdout
    assert (tmp_path / "outputs" / "txt2img-samples-laion400m" / "samples").is_dir()
    assert "2 images in" in r.stdout


@pytest.mark.parametrize("act", [-1, 5, 99])
def test_sdb_gemm_rejects_unknown_activation(cuda_dev, act):
    a = torch.randn(128, 64, device=cuda_dev).half()
    b = torch.randn(64, 64, device=cuda_dev).half()
    with pytest.raises(RuntimeError, match="unknown activation"):
        ops.gemm(a, b, act=act, want_f32=True)


@pytest.mark.parametrize("f16", [False, True])
def test_gelu_epilogue_against_fp64(cuda_dev, f16):
    """ACT_GELU is exact nn.GELU: 0.5 v (1 + erf(v / sqrt 2)) of v = A B^T + bias."""
    g = torch.Generator(device=cuda_dev).manual_seed(5)
    a = torch.randn(154, 1280, generator=g, device=cuda_dev).half()
    b = (torch.randn(5120, 1280, generator=g, device=cuda_dev) * 1280 ** -0.5 * 3).half()
    bias = torch.randn(5120, generator=g, device=cuda_dev) * 0.5
    h, f = ops.gemm(a, b, bias=bias, act=ACT_GELU, want_f16=f16, want_f32=not f16)
    v = a.double() @ b.double().t() + bias.double()
    ref = 0.5 * v * (1.0 + torch.erf(v * 0.5 ** 0.5))
    out = (h if f16 else f).double()
    err = float((out - ref).abs().max())
    print(f"\nGELU epilogue ({'fp16' if f16 else 'fp32'} out): max |err| {err:.2e}, rel-L2 {rel_l2(out, ref):.2e}")
    assert float(v.abs().max()) > 4.0 and float((v < -1).float().mean()) > 0.05    # both tails are exercised
    assert rel_l2(out, ref) < (5e-4 if f16 else 1e-5)


# ------------------------------------------------------------------------------------------------ GEMM plan sweep
@pytest.mark.timeout(900)
def test_every_plan_of_every_laion_gemm_problem(cuda_dev):
    """BERT on the cond + uncond ids of a batch of 3, then the UNet at batches 2 and 6."""
    problems = GP.catalogue(GEMM_MODEL_WORKLOADS["laion"], cuda_dev)
    gelu = [p for p in problems if p["act"] == ACT_GELU]
    print(f"\nLAION BERT (6 x 77 tokens) + UNet (2 and 6, 4, 64²), context (77, 1280): {len(problems)} distinct GEMM "
          f"problems, {len(gelu)} with ACT_GELU")
    assert gelu and any(p["chans"] == (1280,) and p["n"] == 1280 * 4 for p in gelu)
    GP.run_sweep(problems, cuda_dev, "laion")
    torch.cuda.empty_cache()


GELU_SYNTHETIC = {
    "gelu_f16": GP._synthetic(geo=(400,), chans=(1280,), n=5120, act=ACT_GELU, f16=True, f32=False),
    "gelu_f32_res": GP._synthetic(geo=(300,), chans=(640,), n=640, act=ACT_GELU, res=True),
    "gelu_f16_single": GP._synthetic(geo=(154,), chans=(128,), n=512, act=ACT_GELU, f16=True, f32=False, splits=0),
    "gelu_f32_split": GP._synthetic(geo=(256,), chans=(2560,), n=320, act=ACT_GELU, splits=4),
    "gelu_f16_split_scalar": GP._synthetic(geo=(200,), chans=(1280,), n=6, act=ACT_GELU, f16=True, splits=3),
    "gelu_conv": GP._synthetic(geo=(2, 8, 8), taps=9, chans=(320,), n=320, act=ACT_GELU, f16=True),
}


@pytest.mark.timeout(600)
def test_every_plan_of_synthetic_gelu_problems(cuda_dev):
    GP.run_sweep(list(GELU_SYNTHETIC.values()), cuda_dev, "gelu synthetic")
