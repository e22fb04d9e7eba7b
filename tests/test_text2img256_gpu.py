"""The text-conditional LDM-VQ-4 (models/ldm/text2img256) on the H100: the BERT-640 x 32 text encoder and the UNet with
heads of 32 channels on a 640-wide context against the unmodified reference (tests/golden/text2img256.pt), graph replay
against eager, tiny guided DDIM (eta 0 and 1), PLMS and DPM-Solver trajectories from a text2img256-layout checkpoint
and the unchanged YAML through scripts/txt2img.py's loader, the script end to end, every GEMM plan of the model's GEMM
problems and every attention launch of its UNet against fp64."""
import os
import subprocess
import sys

import pytest
import torch
import yaml

import helpers  # noqa: F401
import test_attention_sweep_gpu as AS
import test_gemm_plans_gpu as GP
from helpers import golden, rel_l2, script
from sweeps import record
from test_text2img256_cpu import tiny_node, tiny_state_dict
from workloads import _run_unet, text2img256
from sdb200 import arch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
TOL = 1e-3


def _gen(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------------ full size
def test_full_bert_matches_reference(cuda_dev):
    import sdb200
    g = golden("text2img256.pt")
    d = g["bert"]
    emb = sdb200.BERTEmbedder(**arch.TEXT2IMG256_BERT, use_tokenizer=False).load_weights(
        arch.random_state_dict(arch.bert_param_shapes(arch.TEXT2IMG256_BERT), g["bert_seed"]), cuda_dev)
    z = emb.encode(d["ids"])
    assert z.shape == (2, 77, 640) and z.dtype == torch.float32
    errs = [rel_l2(z[i], d["z"][i].float()) for i in range(2)]
    print(f"\nBERT-640 x 32: rel-L2 prompt row {errs[0]:.2e}, empty-prompt row {errs[1]:.2e}")
    assert max(errs) < TOL


@pytest.mark.parametrize("idx", range(2))
def test_full_unet_eps_matches_reference(cuda_dev, idx):
    """A guidance batch [uncond; cond] of one x_t: both halves within 1e-3 of the reference; graph replay equals eager."""
    import sdb200
    g = golden("text2img256.pt")
    case = g["unet"][idx]
    net = sdb200.UNetModel(**arch.TEXT2IMG256_UNET).load_weights(
        arch.random_state_dict(arch.unet_param_shapes(arch.TEXT2IMG256_UNET), g["unet_seed"]), cuda_dev)
    x = _gen((1, 3, 64, 64), case["x_seed"]).repeat(2, 1, 1, 1).to(cuda_dev)
    t, c = case["t"].to(cuda_dev), _gen((2, 77, 640), case["ctx_seed"]).to(cuda_dev)
    eps = net(x, t, context=c)
    errs = [rel_l2(eps[i], case["eps"][i]) for i in range(2)]
    print(f"\nUNet text2img256 (2, 3, 64, 64) t={int(case['t'][0])}: eps rel-L2 uncond {errs[0]:.2e}, cond {errs[1]:.2e}")
    assert max(errs) < TOL
    if idx == 0:
        net.use_cuda_graph = True
        first = net(x, t.float(), context=c).clone()
        replay = net(x, t.float(), context=c)
        net.use_cuda_graph = False
        eager = net(x, t.float(), context=c)
        assert torch.equal(first, replay) and torch.equal(replay, eager)


# ------------------------------------------------------------------------------------------------ tiny trajectories
def _tiny_model(tmp_path, dev, fmt):
    """The tiny model from the YAML's node and a text2img256-layout checkpoint, through txt2img's loader."""
    from sdb200 import checkpoint
    g = golden("text2img256.pt")
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": tiny_node(g)}))
    sd = tiny_state_dict(g, ema_seed=31)
    ck = tmp_path / f"model.{fmt}"
    if fmt == "ckpt":
        torch.save({"state_dict": sd}, ck)
    else:
        checkpoint.write_safetensors(str(ck), sd)
    return script("txt2img").load_model_from_config(str(cfg), str(ck), dev), cfg, ck


def _codes(m, z):
    """The fp64 nearest code of every pixel of latent z and its distance lead over the runner-up. Moving a pixel's
    latent by a vector of norm r moves each of its distances by at most r, so a lead above 2 r keeps the code."""
    e = m.first_stage_model._host_sd["quantize.embedding.weight"].double()
    zz = z.detach().double().cpu().permute(0, 2, 3, 1).reshape(-1, e.shape[1])
    d = torch.cdist(zz, e)
    top = d.topk(2, dim=1, largest=False)
    return top.indices[:, 0], top.values[:, 1] - top.values[:, 0]


@pytest.mark.parametrize("fmt", ["ckpt", "safetensors"])
@pytest.mark.parametrize("name", ["ddim_eta0", "ddim_eta1", "plms", "dpm_solver"])
def test_tiny_guided_trajectory_matches_reference(cuda_dev, tmp_path, monkeypatch, name, fmt):
    """Txt2Img on the ids of a prompt and of the empty prompt, the reference's x_T (and its eta 1 noise draws), scale
    5.0, 10 steps; then decode_first_stage, which re-quantizes the latent. The decoded image of the reference latent is
    compared in full; for the engine's own latent, the quantizer's codes are compared wherever the reference latent's
    nearest code leads the runner-up by more than the engine's latent error at that pixel can close (closer codes may
    swap, and the decoder then shows a different codebook row there; the tiny model's 512 codes of width 3 lie close).
    At least a quarter of the pixels must be decided that clearly."""
    from sdb200 import pipeline
    g = golden("text2img256.pt")
    d = g["tiny"]
    r = d[name]
    m, _, _ = _tiny_model(tmp_path, cuda_dev, fmt)
    assert torch.equal(m.alphas_cumprod.cpu(), g["alphas_cumprod"]) and m.scale_factor == 1.0
    eta = float(name[-1]) if name.startswith("ddim") else 0.0
    pipe = pipeline.Txt2Img(m, sampler=name.split("_eta")[0], steps=g["steps"], scale=g["scale"], height=64, width=64,
                            eta=eta, f=4, channels=3)
    draws = [_gen(tuple(d["x_T"].shape), d["noise_seed"] + i).to(cuda_dev) for i in range(r["n_noise"])] if eta else []
    if eta:
        monkeypatch.setattr(torch, "randn_like", lambda t, *a, **k: draws.pop(0).to(t.device))
    s = pipe(d["ids"].to(cuda_dev), d["uc_ids"].to(cuda_dev), x_T=d["x_T"].to(cuda_dev), return_latent=True)
    monkeypatch.undo()
    assert not draws
    ref_dec = m.decode_first_stage(r["sample"].to(cuda_dev))
    x_dec = m.decode_first_stage(s)
    mine, _ = _codes(m, s)
    want, gap = _codes(m, r["sample"])
    moved = (s.double().cpu() - r["sample"].double()).permute(0, 2, 3, 1).reshape(-1, s.shape[1]).norm(dim=1)
    clear = gap > 2 * moved
    errs = dict(latent=rel_l2(s, r["sample"]), decode_of_reference_latent=rel_l2(ref_dec, r["x_dec"]),
                image=rel_l2(x_dec, r["x_dec"]))
    print(f"\ntiny guided {name} ({fmt}): " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()) +
          f"; codes equal on {int((mine == want)[clear].sum())} of {int(clear.sum())} clear pixels "
          f"({int(clear.numel())} in all)")
    assert errs["latent"] < 2e-2 and errs["decode_of_reference_latent"] < 2e-3
    assert float(clear.float().mean()) > 0.25 and torch.equal(mine[clear], want[clear])
    img = pipe(d["ids"].to(cuda_dev), d["uc_ids"].to(cuda_dev), x_T=d["x_T"].to(cuda_dev))
    assert img.shape == (2, 64, 64, 3) and img.dtype == torch.uint8


def test_ema_scope_runs_the_checkpoint_ema_weights(cuda_dev, tmp_path):
    """Inside ema_scope() the UNet evaluates the model_ema.* set (equal to a UNet loaded with those weights), outside it
    the raw weights."""
    import sdb200
    m, _, _ = _tiny_model(tmp_path, cuda_dev, "safetensors")
    u = m.model.diffusion_model
    ema = sdb200.UNetModel(**arch.TINY_TEXT2IMG256_UNET).load_weights(
        arch.random_state_dict(arch.unet_param_shapes(arch.TINY_TEXT2IMG256_UNET), 31), cuda_dev)
    x, t, c = _gen((2, 3, 16, 16), 5).to(cuda_dev), torch.tensor([501., 501.], device=cuda_dev), \
        _gen((2, 77, 128), 6).to(cuda_dev)
    raw = u(x, t, context=c).clone()
    with m.ema_scope():
        inside = u(x, t, context=c).clone()
    assert torch.equal(inside, ema(x, t, context=c)) and not torch.equal(inside, raw)
    assert torch.equal(u(x, t, context=c), raw)


# ------------------------------------------------------------------------------------------------ scripts/txt2img.py
def test_txt2img_script_tiny_checkpoint_with_bert_vocab(cuda_dev, tmp_path):
    """The unchanged YAML's node (tiny stages) and a .ckpt through main(): --bert_vocab tokenises the prompt for the
    BERTEmbedder cond stage (no --laion400m); DPM-Solver; PNGs of 64² (--C 3 --f 4)."""
    _, cfg, ck = _tiny_model(tmp_path, cuda_dev, "ckpt")
    vocab = tmp_path / "vocab"
    vocab.mkdir()
    letters = [chr(c) for c in range(ord("a"), ord("z") + 1)]
    (vocab / "vocab.txt").write_text("\n".join(["[PAD]", "[unused0]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"] + letters +
                                               ["##" + c for c in letters] + ["virus", "monster"]) + "\n")
    out = tmp_path / "out"
    mod = script("txt2img")
    mod.main(["--config", str(cfg), "--ckpt", str(ck), "--H", "64", "--W", "64", "--C", "3", "--f", "4", "--scale", "5.0",
              "--dpm_solver", "--ddim_steps", "4", "--n_samples", "2", "--n_iter", "1", "--outdir", str(out),
              "--bert_vocab", str(vocab), "--prompt", "a virus monster", "--no_watermark"])
    from PIL import Image
    pngs = sorted((out / "samples").glob("*.png"))
    assert len(pngs) == 2 and all(Image.open(p).size == (64, 64) for p in pngs)
    enc = mod.sdb200.BERTEmbedder(**arch.TINY_BERT, vocab_dir=str(vocab))
    assert enc._tokenize(["a virus monster"])[0, :5].tolist() == [3, 6, 58, 59, 4]


def test_txt2img_script_full_size_random_init(cuda_dev, tmp_path):
    """The unchanged YAML with --random_init at 256², stand-in BERT ids, PLMS; wrong --C / --f are rejected with the
    values to pass."""
    g = golden("text2img256.pt")
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": g["yaml_node"]}))
    script = os.path.join(helpers.ROOT, "scripts", "txt2img.py")
    env = dict(os.environ, HF_HUB_OFFLINE="1")
    run = lambda *extra: subprocess.run(
        [sys.executable, script, "--config", str(cfg), "--random_init", "--H", "256", "--W", "256", "--scale", "5.0",
         "--plms", "--ddim_steps", "5", "--n_samples", "2", "--n_iter", "1", "--outdir", str(tmp_path / "out"), *extra],
        cwd=tmp_path, capture_output=True, text=True, timeout=900, env=env)
    r = run("--C", "3", "--f", "4")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "seeded token ids" in r.stdout and "2 images in" in r.stdout
    from PIL import Image
    pngs = sorted((tmp_path / "out" / "samples").glob("*.png"))
    assert len(pngs) == 2 and all(Image.open(p).size == (256, 256) for p in pngs)
    bad = run()                              # the SD-v1 defaults --C 4 --f 8
    assert bad.returncode != 0 and "pass --C 3 --f 4" in bad.stderr, bad.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ kernel sweeps
def test_every_plan_of_every_text2img256_gemm_problem(cuda_dev):
    """workloads.text2img256: BERT-640 on the cond + uncond ids of a batch of 3 (6 x 77 tokens: the K / V projections
    of K = 640 and the 8 x 64 attention's 512-wide inner dimension), the UNet at the guidance batches 2 and 8, and the
    VQ-f4 decode of a 64² latent. Its norm and elementwise launches are swept in test_first_stage_sweep_gpu.py."""
    problems = GP.catalogue(text2img256, cuda_dev)
    print(f"\ntext2img256 BERT (6 x 77 tokens) + UNet (2 and 8, 3, 64²), context (77, 640) + VQ-f4 decode (64²): "
          f"{len(problems)} distinct GEMM problems")
    assert any(p["chans"] == (640,) for p in problems)
    GP.run_sweep(problems, cuda_dev, "text2img256")
    torch.cuda.empty_cache()


def test_every_attention_launch_of_the_text2img256_unet(cuda_dev):
    """Self-attention of 12 / 18 / 30 heads of d = 32 at 32² / 16² / 8² tokens and cross-attention on the 77-token
    context, each launch elementwise against fp64."""
    wl = lambda dev: _run_unet(arch.TEXT2IMG256_UNET, [(2, 3, 64, 64)], dev, ctx=(77, 640))
    calls, problems = record(wl, cuda_dev, {"attention": AS._attn_sig})
    got = {(p["heads"], p["d"], p["nq"], p["nkv"]) for p in problems}
    print(f"\ntext2img256 UNet: {calls} attention calls, {len(problems)} distinct problems: {sorted(got)}")
    for heads, n in ((12, 1024), (18, 256), (30, 64)):
        assert (heads, 32, n, n) in got and (heads, 32, n, 77) in got
    AS.run_sweep(problems, "text2img256")
    torch.cuda.empty_cache()
