"""The layout-to-image LDM (models/ldm/layout2img-openimages256) on the H100: the BERT-512 x 16 encoder on 92 layout ids
and the UNet with spatial transformers of depth 3 against the unmodified reference (tests/golden/layout2img.pt), graph
replay against eager across a change of context, tiny unguided DDIM (eta 0 and 1) inside ema_scope() from a
layout2img-layout checkpoint and the unchanged YAML through scripts/layout2img.py's loader, the script end to end, and
the GEMM plan, norm, attention and elementwise sweeps and the pre-wait weight audit on its layout2img workload."""
import os
import subprocess
import sys
import time
from collections import defaultdict

import pytest
import torch
import yaml

import helpers  # noqa: F401
import test_attention_sweep_gpu as AS
import test_elementwise_sweep_gpu as ES
import test_gemm_plans_gpu as GP
import test_norm_sweep_gpu as NS
from helpers import golden, rel_l2, script
from sweeps import record
from test_layout2img_cpu import tiny_node, tiny_state_dict
from test_pdl_order_gpu import audit_workload
from workloads import _bert, _run_unet, _vq
from sdb200 import arch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
TOL = 1e-3
# The UNet eps bound. Every depth-1 UNet meets 1e-3; this one has three transformer blocks per spatial transformer, each
# adding its fp16 operand rounding (LayerNorm outputs, q / k / v, softmax probabilities, attention and GEGLU outputs) to
# the fp32 token stream. Restating those roundings in the oracle at t = 981 gives 3.2e-4 / 2.6e-4 / 2.3e-4 from blocks
# 0 / 1 / 2 alone and 4.9e-4 from all three: the error is spread evenly over the blocks, no single block stands out.
# The engine measures 1.10e-3 to 1.15e-3 at t = 981 and 9.2e-4 to 9.7e-4 at t = 1 (H100 80GB HBM3).
UNET_TOL = 1.5e-3
WIDTHS = ((256, 8, 1024), (384, 12, 256), (512, 16, 64))      # spatial transformer width, heads of d = 32, tokens


def layout2img(dev):
    """The sweep workload: BERT-512 x 16 on 2 x 92 layout ids (vocabulary 8192), the UNet with spatial transformers of
    depth 3 at batches 2 and 8 on a 92 x 512 context, and one VQ-f4 decode of a 64² latent, built from the
    tests/workloads.py helpers (its tables stay as they are)."""
    g = torch.Generator(device=dev).manual_seed(2)
    ids = torch.randint(0, 8192, (2, 92), generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    return (_bert(arch.LAYOUT2IMG_BERT, dev, ids),
            _run_unet(arch.LAYOUT2IMG_UNET, [(2, 3, 64, 64), (8, 3, 64, 64)], dev, ctx=(92, 512)),
            _vq(arch.VQ_F4, dev).decode(torch.randn(1, 3, 64, 64, generator=g, device=dev)))


def _gen(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------------ full size
def test_full_bert_matches_reference(cuda_dev):
    import sdb200
    g = golden("layout2img.pt")
    d = g["bert"]
    emb = sdb200.BERTEmbedder(**arch.LAYOUT2IMG_BERT, use_tokenizer=False).load_weights(
        arch.random_state_dict(arch.bert_param_shapes(arch.LAYOUT2IMG_BERT), g["bert_seed"]), cuda_dev)
    z = emb.encode(d["ids"])
    assert z.shape == (2, 92, 512) and z.dtype == torch.float32
    errs = [rel_l2(z[i], d["z"][i].float()) for i in range(2)]
    print(f"\nBERT-512 x 16 on 92 ids: rel-L2 {errs[0]:.2e}, {errs[1]:.2e}")
    assert max(errs) < TOL


def _full_unet(dev):
    import sdb200
    g = golden("layout2img.pt")
    return sdb200.UNetModel(**arch.LAYOUT2IMG_UNET).load_weights(
        arch.random_state_dict(arch.unet_param_shapes(arch.LAYOUT2IMG_UNET), g["unet_seed"]), dev)


@pytest.mark.parametrize("idx", range(2))
def test_full_unet_eps_matches_reference(cuda_dev, idx):
    """Two samples with different 92 x 512 contexts: both rows within UNET_TOL of the reference."""
    g = golden("layout2img.pt")
    case = g["unet"][idx]
    net = _full_unet(cuda_dev)
    x = _gen((2, 3, 64, 64), case["x_seed"]).to(cuda_dev)
    t, c = case["t"].to(cuda_dev), _gen((2, 92, 512), case["ctx_seed"]).to(cuda_dev)
    eps = net(x, t, context=c)
    errs = [rel_l2(eps[i], case["eps"][i]) for i in range(2)]
    print(f"\nUNet layout2img (2, 3, 64, 64) t={int(case['t'][0])}: eps rel-L2 {errs[0]:.2e}, {errs[1]:.2e}")
    assert max(errs) < UNET_TOL


def test_graph_replay_equals_eager_across_contexts(cuda_dev):
    """One captured graph per shape reads the per-block K / V^T buffers: after the context changes, replay still equals
    eager on the new context, bit for bit."""
    g = golden("layout2img.pt")
    net = _full_unet(cuda_dev)
    x = _gen((2, 3, 64, 64), 900).to(cuda_dev)
    t = torch.tensor([981., 981.], device=cuda_dev)
    c1, c2 = (_gen((2, 92, 512), s).to(cuda_dev) for s in (950, 951))
    net.use_cuda_graph = True
    first = net(x, t, context=c1).clone()
    replay = net(x, t, context=c1).clone()
    other = net(x, t, context=c2).clone()
    assert len(net._graphs) == 1 and len(net._kv_static[(2, 92)]) == 16 * 3
    net.use_cuda_graph = False
    assert torch.equal(first, replay) and torch.equal(replay, net(x, t, context=c1))
    assert torch.equal(other, net(x, t, context=c2)) and not torch.equal(other, first)
    assert g["unet"][0]["x_seed"] == 900 and g["unet"][0]["ctx_seed"] == 950
    assert rel_l2(first, g["unet"][0]["eps"]) < UNET_TOL


# ------------------------------------------------------------------------------------------------ tiny trajectories
def _tiny_model(tmp_path, dev, fmt):
    """The tiny model from the YAML's node and a layout2img-layout checkpoint with model_ema.*, through the script's
    loader."""
    from sdb200 import checkpoint
    g = golden("layout2img.pt")
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": tiny_node(g)}))
    sd = tiny_state_dict(g)
    ck = tmp_path / f"model.{fmt}"
    if fmt == "ckpt":
        torch.save({"state_dict": sd}, ck)
    else:
        checkpoint.write_safetensors(str(ck), sd)
    return script("layout2img").load_model(str(cfg), str(ck), dev), cfg, ck


def _codes(m, z):
    """The fp64 nearest code of every pixel of latent z and its distance lead over the runner-up. Moving a pixel's
    latent by a vector of norm r moves each of its distances by at most r, so a lead above 2 r keeps the code."""
    e = m.first_stage_model._host_sd["quantize.embedding.weight"].double()
    zz = z.detach().double().cpu().permute(0, 2, 3, 1).reshape(-1, e.shape[1])
    d = torch.cdist(zz, e)
    top = d.topk(2, dim=1, largest=False)
    return top.indices[:, 0], top.values[:, 1] - top.values[:, 0]


@pytest.mark.parametrize("fmt", ["ckpt", "safetensors"])
@pytest.mark.parametrize("eta", [0, 1])
def test_tiny_unguided_ddim_matches_reference(cuda_dev, tmp_path, monkeypatch, eta, fmt):
    """The script's sampling (log_images: unguided DDIM inside ema_scope(), 10 steps) on the reference's ids, x_T and
    eta 1 noise draws; then decode_first_stage, which re-quantizes the latent. The decoded image of the reference latent
    is compared in full; for the engine's own latent, the quantizer's codes are compared wherever the reference latent's
    nearest code leads the runner-up by more than the engine's latent error at that pixel can close. At least a quarter
    of the pixels must be decided that clearly."""
    g = golden("layout2img.pt")
    d = g["tiny"]
    r = d[f"ddim_eta{eta}"]
    mod = script("layout2img")
    m, _, _ = _tiny_model(tmp_path, cuda_dev, fmt)
    assert torch.equal(m.alphas_cumprod.cpu(), g["alphas_cumprod"]) and m.scale_factor == 1.0
    m.model.diffusion_model.use_cuda_graph = True
    draws = [_gen(tuple(d["x_T"].shape), d["noise_seed"] + i).to(cuda_dev) for i in range(r["n_noise"])] if eta else []
    if eta:
        monkeypatch.setattr(torch, "randn_like", lambda t, *a, **k: draws.pop(0).to(t.device))
    ids = mod.check_layout_ids(m.cond_stage_model, d["ids"])
    s = mod.sample_latents(m, ids, g["steps"], float(eta), x_T=d["x_T"].to(cuda_dev))
    monkeypatch.undo()
    assert not draws and m.model.diffusion_model._active == "raw"
    ref_dec = m.decode_first_stage(r["sample"].to(cuda_dev))
    mine, _ = _codes(m, s)
    want, gap = _codes(m, r["sample"])
    moved = (s.double().cpu() - r["sample"].double()).permute(0, 2, 3, 1).reshape(-1, s.shape[1]).norm(dim=1)
    clear = gap > 2 * moved
    errs = dict(latent=rel_l2(s, r["sample"]), decode_of_reference_latent=rel_l2(ref_dec, r["x_dec"]),
                image=rel_l2(m.decode_first_stage(s), r["x_dec"]))
    print(f"\ntiny unguided DDIM eta {eta} ({fmt}): " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()) +
          f"; codes equal on {int((mine == want)[clear].sum())} of {int(clear.sum())} clear pixels "
          f"({int(clear.numel())} in all)")
    assert errs["latent"] < 2e-2 and errs["decode_of_reference_latent"] < 2e-3
    assert float(clear.float().mean()) > 0.25 and torch.equal(mine[clear], want[clear])
    img = mod.decode(m, s)
    assert img.shape == (2, 3, 64, 64) and float(img.min()) >= 0 and float(img.max()) <= 1


def test_ema_scope_runs_the_checkpoint_ema_weights(cuda_dev, tmp_path):
    """Inside ema_scope() the depth-3 UNet evaluates the model_ema.* set (equal to a UNet loaded with those weights),
    outside it the raw weights."""
    import sdb200
    g = golden("layout2img.pt")
    m, _, _ = _tiny_model(tmp_path, cuda_dev, "safetensors")
    u = m.model.diffusion_model
    ema = sdb200.UNetModel(**arch.TINY_LAYOUT2IMG_UNET).load_weights(
        arch.random_state_dict(arch.unet_param_shapes(arch.TINY_LAYOUT2IMG_UNET), g["ema_seed"]), cuda_dev)
    x, t, c = _gen((2, 3, 16, 16), 5).to(cuda_dev), torch.tensor([501., 501.], device=cuda_dev), \
        _gen((2, 92, 128), 6).to(cuda_dev)
    raw = u(x, t, context=c).clone()
    with m.ema_scope():
        inside = u(x, t, context=c).clone()
    assert torch.equal(inside, ema(x, t, context=c)) and not torch.equal(inside, raw)
    assert torch.equal(u(x, t, context=c), raw)


# ------------------------------------------------------------------------------------------------ scripts/layout2img.py
def test_layout2img_script_full_size_random_init(cuda_dev, tmp_path):
    """The built-in model node (the reference's default config path is absent) with --random_init at 256²: seeded
    stand-in ids, 5 DDIM steps, four PNGs of 256²; a token file of the wrong length is rejected."""
    script = os.path.join(helpers.ROOT, "scripts", "layout2img.py")
    run = lambda *extra: subprocess.run(
        [sys.executable, script, "--random_init", "--ddim_steps", "5", "--outdir", str(tmp_path / "out"), *extra],
        cwd=tmp_path, capture_output=True, text=True, timeout=900)
    r = run("--n_samples", "4")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "seeded token ids" in r.stdout and "4 images in" in r.stdout
    from PIL import Image
    pngs = sorted((tmp_path / "out" / "samples").glob("*.png"))
    assert len(pngs) == 4 and all(Image.open(p).size == (256, 256) for p in pngs)
    torch.save(torch.zeros(2, 77, dtype=torch.long), tmp_path / "short.pt")
    bad = run("--tokens", str(tmp_path / "short.pt"))
    assert bad.returncode != 0 and "exactly 92" in bad.stderr, bad.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ kernel sweeps
def test_every_plan_of_every_layout2img_gemm_problem(cuda_dev):
    """BERT-512 on 2 x 92 ids, the UNet at batches 2 and 8 and a VQ-f4 decode: every GEMM problem with every tile plan.
    The depth-3 problems are the feed-forward output of the blocks before the last, which writes fp32 with the residual
    (the last block's writes fp16 hi / lo for proj_out)."""
    problems = GP.catalogue(layout2img, cuda_dev)
    print(f"\nlayout2img BERT (2 x 92) + UNet (2 and 8, 3, 64²), context (92, 512) + VQ-f4 decode (64²): "
          f"{len(problems)} distinct GEMM problems")
    for ch, _, n in WIDTHS:
        for nb in (2, 8):
            ff2 = [p for p in problems if p["taps"] == 1 and p["chans"] == (4 * ch,) and p["n"] == ch
                   and p["geo"] == (nb * n,) and p["res"]]
            assert any(p["f32"] and not p["f16"] for p in ff2), (ch, nb)       # blocks 0 and 1
            assert any(p["lo"] and not p["f32"] for p in ff2), (ch, nb)        # block 2
        assert any(p["chans"] == (512,) and p["n"] == ch and p["geo"] == (2 * 92,) for p in problems)   # K / V
    assert any(p["chans"] == (512,) and p["geo"] == (2 * 92,) and p["n"] == 2048 for p in problems)     # BERT FF
    GP.run_sweep(problems, cuda_dev, "layout2img")
    torch.cuda.empty_cache()


def test_every_attention_launch_of_the_layout2img_workload(cuda_dev):
    """Self-attention of 8 / 12 / 16 heads of d = 32 at 32² / 16² / 8² tokens, the 92-key cross-attention at all three
    head counts, and BERT's 92-token self-attention at d = 64, each launch elementwise against fp64."""
    calls, problems = record(layout2img, cuda_dev, {"attention": AS._attn_sig})
    got = {(p["heads"], p["d"], p["nq"], p["nkv"]) for p in problems}
    print(f"\nlayout2img: {calls} attention calls, {len(problems)} distinct problems: {sorted(got)}")
    for _, heads, n in WIDTHS:
        assert (heads, 32, n, n) in got and (heads, 32, n, 92) in got
    assert (8, 64, 92, 92) in got
    AS.run_sweep(problems, "layout2img")
    torch.cuda.empty_cache()


def test_every_norm_launch_of_the_layout2img_workload(cuda_dev):
    """GroupNorm and the transformer blocks' LayerNorms at 256 / 384 / 512 channels (three blocks' worth per spatial
    transformer), BERT's LayerNorm at 512."""
    calls, problems = record(layout2img, cuda_dev, NS.SIGS)
    kinds = defaultdict(int)
    for p in problems:
        kinds[p["kind"]] += 1
    print(f"\nlayout2img: {calls} calls, {len(problems)} distinct problems ({dict(kinds)})")
    ln = {(p["rows"], p["c"]) for p in problems if p["kind"] == "ln"}
    for ch, _, n in WIDTHS:
        assert (2 * n, ch) in ln and (8 * n, ch) in ln, ch
    assert (2 * 92, 512) in ln
    NS.run_sweep(problems, "layout2img")
    torch.cuda.empty_cache()


def test_every_elementwise_launch_of_the_layout2img_workload(cuda_dev):
    """Layouts, casts, embeddings and the quantizer; the context's V^T for the 92-key cross-attention, padded to 96."""
    calls, problems = record(layout2img, cuda_dev, ES.SIGS)
    ops_ = defaultdict(int)
    for p in problems:
        ops_[p["op"]] += 1
    print(f"\nlayout2img: {calls} calls, {len(problems)} distinct problems ({dict(ops_)})")
    tr = {(p["B"], p["rows"], p["cols"], p["ldo"]) for p in problems if p["op"] == "transpose_f16"}
    for ch, _, _ in WIDTHS:
        assert (2, 92, ch, 96) in tr and (8, 92, ch, 96) in tr, tr
    assert any(p["op"] == "vq_quantize" and p["n_e"] == 8192 for p in problems)
    ES.run_sweep(problems, "layout2img")
    torch.cuda.empty_cache()


def test_layout2img_pre_wait_operands_are_packed_weights(cuda_dev):
    """The weight audit of test_pdl_order_gpu.py on the layout2img workload."""
    t0 = time.time()
    bad, n = audit_workload("layout2img", layout2img, cuda_dev)
    print(f"\nlayout2img: {n} gemm / groupnorm / layernorm calls audited, {len(bad)} violations, {time.time() - t0:.1f} s")
    assert not bad, "pre-wait operands outside packed weights (workload, op, slot, shape):\n" + \
        "\n".join(map(str, sorted(set(bad))))
