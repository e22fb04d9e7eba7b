"""The retrieval-augmented diffusion model (configs/retrieval-augmented-diffusion/768x768.yaml, scripts/knn2img.py) on the
H100: the projected CLIP text embedding against transformers, the exact k-NN search kernel against fp64, the UNet and
the KL-f16 first stage against the unmodified reference (tests/golden/rdm.pt), graph replay and the C handle against
eager, guided trajectories on EMA weights, every GEMM tile plan of the model's GEMM problems, and the script."""
import json
import os

import numpy as np
import pytest
import torch

import helpers  # noqa: F401
import rdm_oracle as RO
from helpers import golden, rel_l2, script
from sdb200 import arch, ops, pipeline
from workloads import GEMM_MODEL_WORKLOADS

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
UCFG = {"tiny": arch.TINY_RDM_UNET, "rdm": arch.RDM_UNET}
VCFG = {"tiny": arch.TINY_KL_F16, "kl_f16": arch.KL_F16}
TOL = 1e-3
_models = {}


def _gen(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def _unit_rows(shape, seed):
    x = _gen(shape, seed)
    return x / torch.linalg.norm(x, dim=-1, keepdim=True)


def _sub(x, g):
    """The pixels the golden stores of a decoded image: every g["image_stride"]-th in both directions."""
    k = g["image_stride"]
    return x[..., ::k, ::k]


def _esub(eps, g):
    """The latent pixels the golden stores of a UNet output: every g["eps_stride"]-th in both directions."""
    k = g["eps_stride"]
    return eps[..., ::k, ::k]


def _unet(tag, dev):
    import sdb200
    if tag not in _models:
        _models[tag] = sdb200.UNetModel(**UCFG[tag]).load_weights(
            arch.random_state_dict(arch.unet_param_shapes(UCFG[tag]), golden("rdm.pt")["unet_seed"]), dev)
    return _models[tag]


def _kl(tag, dev):
    import sdb200
    key = "kl_" + tag
    if key not in _models:
        _models[key] = sdb200.AutoencoderKL(**VCFG[tag]).load_weights(
            arch.random_state_dict(arch.vae_param_shapes(VCFG[tag]), golden("rdm.pt")["vae_seed"]), dev)
    return _models[key]


# ------------------------------------------------------------------------------------------------ CLIP text embedding
@pytest.mark.parametrize("tag", ["tiny", "vit_l14"])
def test_clip_text_embedding_vs_transformers(cuda_dev, tag):
    """encode() = transformers CLIPTextModelWithProjection's text_embeds at the EOT (largest) id, L2-normalised."""
    import sdb200
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    cfg = arch.TINY_CLIP_TEXT_PROJ if tag == "tiny" else arch.CLIP_TEXT_PROJ
    sd = arch.random_state_dict(arch.clip_text_proj_param_shapes(cfg), 13)
    hf_cfg = CLIPTextConfig(vocab_size=cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                            intermediate_size=cfg["intermediate_size"], num_hidden_layers=cfg["num_hidden_layers"],
                            num_attention_heads=cfg["num_attention_heads"],
                            max_position_embeddings=cfg["max_position_embeddings"], projection_dim=cfg["projection_dim"],
                            layer_norm_eps=cfg["layer_norm_eps"], hidden_act="quick_gelu", eos_token_id=2)
    ref = CLIPTextModelWithProjection(hf_cfg).eval()
    ref.load_state_dict(sd, strict=False)
    V = cfg["vocab_size"]
    g = torch.Generator().manual_seed(5)
    ids = torch.zeros((3, 77), dtype=torch.long)
    for b, n in enumerate((5, 40, 75)):          # BOS + n tokens + EOT, zero padding (clip.tokenize)
        ids[b, 0] = V - 2
        ids[b, 1:1 + n] = torch.randint(1, V - 2, (n,), generator=g)
        ids[b, 1 + n] = V - 1
    with torch.no_grad():
        z_ref = ref(input_ids=ids).text_embeds.double()
    z_ref = z_ref / z_ref.norm(dim=-1, keepdim=True)
    enc = sdb200.FrozenCLIPTextEmbedder(config=cfg).load_weights(sd, cuda_dev)
    z = enc.encode(ids)
    assert tuple(z.shape) == (3, 1, cfg["projection_dim"])
    err = rel_l2(z[:, 0], z_ref)
    print(f"CLIP text embedding {tag}: rel-L2 {err:.2e} vs transformers")
    assert err < 2e-3
    assert torch.allclose(z.double().norm(dim=-1).cpu(), torch.ones(3, 1, dtype=torch.float64), atol=1e-5)
    assert rel_l2(z[:, 0], RO.clip_text_embed(sd, ids, cfg["num_attention_heads"])) < 2e-3


# ------------------------------------------------------------------------------------------------ k-NN search
def _db(n, dim, seed, dev):
    x = _unit_rows((n, dim), seed)
    return x, x.half().to(dev)


def _check_topk(db32, q32, scores, rows, k):
    """Indices equal the fp64 top-k of the unrounded vectors except where fp64 scores lie within the margin fp16
    rounding of both unit vectors (2 * 2^-11) and fp32 accumulation (dim * 2^-24) allow; returned scores equal the fp64
    dot products of the fp16-rounded vectors to fp32 accumulation; order is score descending, then row ascending."""
    dim = db32.shape[1]
    margin = 2 * 2.0 ** -11 + dim * 2.0 ** -24
    exact = q32.double() @ db32.double().t()
    rounded = q32.half().double() @ db32.half().double().t()
    rows, scores = rows.cpu(), scores.cpu().double()
    for b in range(q32.shape[0]):
        kth = exact[b].topk(k).values[-1]
        must = set(torch.nonzero(exact[b] > kth + 2 * margin).flatten().tolist())
        got = rows[b].tolist()
        assert len(set(got)) == k and must <= set(got), (b, sorted(must - set(got)))
        assert bool((exact[b, rows[b]] >= kth - 2 * margin).all())
        assert torch.allclose(scores[b], rounded[b, rows[b]], atol=dim * 2.0 ** -24 * 4, rtol=0)
        for i in range(k - 1):
            assert scores[b, i] > scores[b, i + 1] or (scores[b, i] == scores[b, i + 1] and got[i] < got[i + 1])


@pytest.mark.parametrize("k", [1, 10, 64])
@pytest.mark.parametrize("B", [1, 3, 64])
def test_knn_topk_vs_fp64(cuda_dev, B, k):
    n, dim = 64 * 157 + 37, 768        # not a multiple of the 64-row tile; more tiles than SMs
    db32, db = _db(n, dim, 1, cuda_dev)
    q32 = _unit_rows((B, dim), 2 + B)
    scores, rows = ops.knn_topk(db, q32.half().to(cuda_dev), k)
    s2, r2 = ops.knn_topk(db, q32.half().to(cuda_dev), k)
    torch.cuda.synchronize()
    assert torch.equal(scores, s2) and torch.equal(rows, r2), "two runs differ"
    _check_topk(db32, q32, scores, rows, k)


def test_knn_topk_small_database_and_dims(cuda_dev):
    """Fewer rows than one tile per SM (N = 70, one partial tile), dim 64 and 512."""
    for n, dim, k in ((70, 64, 64), (70, 512, 5), (1000, 512, 33)):
        db32, db = _db(n, dim, 7, cuda_dev)
        q32 = _unit_rows((5, dim), 8)
        scores, rows = ops.knn_topk(db, q32.half().to(cuda_dev), k)
        _check_topk(db32, q32, scores, rows, k)


def test_knn_exact_ties_go_to_the_lower_row(cuda_dev):
    """Copies of one row spread over the database (several CTAs) tie exactly: they come back in ascending row order."""
    n, dim = 64 * 300 + 5, 768
    db32, _ = _db(n, dim, 3, cuda_dev)
    copies = [19000, 5, 700, 64 * 150 + 1, 64 * 299 + 3, 12345]
    q = _unit_rows((2, dim), 4)
    db32[copies] = q[0]
    db32[9999] = q[1]
    db32[77] = q[1]
    db = db32.half().to(cuda_dev)
    scores, rows = ops.knn_topk(db, q.half().to(cuda_dev), 8)
    assert rows[0, :len(copies)].tolist() == sorted(copies)
    assert len(set(scores[0, :len(copies)].tolist())) == 1
    assert rows[1, :2].tolist() == [77, 9999] and scores[1, 0] == scores[1, 1]


def test_knn_rejects_bad_arguments(cuda_dev):
    db = torch.zeros((100, 768), dtype=torch.float16, device=cuda_dev)
    for q, k in ((torch.zeros((65, 768), dtype=torch.float16, device=cuda_dev), 4),
                 (torch.zeros((2, 768), dtype=torch.float16, device=cuda_dev), 65),
                 (torch.zeros((2, 768), dtype=torch.float16, device=cuda_dev), 101)):
        with pytest.raises(RuntimeError, match="sdb_knn_topk"):
            ops.knn_topk(db, q, k)
    with pytest.raises(RuntimeError, match="dim"):
        ops.knn_topk(torch.zeros((100, 96), dtype=torch.float16, device=cuda_dev),
                     torch.zeros((2, 96), dtype=torch.float16, device=cuda_dev), 4)


def _write_db(path, n, dim, seed, n_files=2):
    os.makedirs(path, exist_ok=True)
    rng = np.random.default_rng(seed)
    emb = (rng.standard_normal((n, dim)) * rng.uniform(0.5, 2.0, (n, 1))).astype(np.float32)
    cuts = np.linspace(0, n, n_files + 1).astype(int)
    for i in range(n_files):
        sl = slice(cuts[i], cuts[i + 1])
        np.savez(os.path.join(path, f"part{i:02d}.npz"), embedding=emb[sl], img_id=np.arange(n)[sl],
                 patch_coords=np.stack([np.arange(n)[sl]] * 4, 1))
    return emb


def test_searcher_matches_reference_formula(cuda_dev, tmp_path):
    """Searcher.search: the reference's dict, nn_embeddings bit-equal to the reference formula on the same indices,
    and batches larger than one launch (70 queries) split on the host."""
    from sdb200.retrieval import Searcher, normalize_rows
    emb = _write_db(str(tmp_path / "db"), 5000, 768, 0)
    s = Searcher("test", device=cuda_dev, path=str(tmp_path / "db"))
    assert len(s) == 5000
    x = _unit_rows((70, 1, 768), 9) * 3.0
    out = s.search(x, 10)
    assert set(out) == {"nn_embeddings", "img_ids", "patch_coords", "queries", "exec_time", "nns", "q_embeddings"}
    nns = out["nns"]
    assert nns.shape == (70, 10) and out["nn_embeddings"].shape == (70, 10, 768)
    ref = emb[nns] / np.linalg.norm(emb[nns], axis=-1)[..., np.newaxis]
    assert np.array_equal(out["nn_embeddings"], ref) and np.array_equal(out["img_ids"], nns)
    q = out["q_embeddings"]
    assert np.array_equal(q, x[:, 0].numpy() / np.linalg.norm(x[:, 0].numpy(), axis=1)[:, np.newaxis])
    exact = torch.from_numpy(q).double() @ torch.from_numpy(normalize_rows(emb)).double().t()
    margin = 2 * 2.0 ** -11 + 768 * 2.0 ** -24
    for b in range(70):
        kth = exact[b].topk(10).values[-1]
        must = set(torch.nonzero(exact[b] > kth + 2 * margin).flatten().tolist())
        assert must <= set(nns[b].tolist())


# ------------------------------------------------------------------------------------------------ UNet
def _case_inputs(case, dev):
    x = _gen(case["shape"], case["seed"])
    c = _unit_rows((case["shape"][0], case["n_ctx"], UCFG[case["cfg"]]["context_dim"]), case["seed"] + 1)
    return x.to(dev), case["t"].to(dev), c.to(dev)


@pytest.mark.parametrize("idx", range(4))
def test_unet_vs_reference(cuda_dev, idx):
    """Tiny with a 3-token context; RDM at (2,16,48,48) with 11 tokens (text + 10 neighbours) and 1 token (text only:
    the one-token fold), and (1,16,24,48)."""
    g = golden("rdm.pt")
    case = g["unet"][idx]
    net = _unet(case["cfg"], cuda_dev)
    x, t, c = _case_inputs(case, cuda_dev)
    eps = net(x, t, context=c)
    err = rel_l2(_esub(eps, g), case["eps"])
    print(f"unet {case['cfg']} {tuple(case['shape'])} ctx {case['n_ctx']}: rel-L2 {err:.3e}")
    assert tuple(eps.shape) == tuple(case["shape"]) and err < TOL


@pytest.mark.parametrize("n_ctx", [1, 3])
def test_tiny_unet_all_zero_context_vs_oracle(cuda_dev, n_ctx):
    """The unconditional half of knn2img's guidance: uc = zeros_like(c)."""
    sd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_RDM_UNET), 11)
    x, t = _gen((2, 16, 16, 24), 3), torch.tensor([900, 20])
    c = torch.zeros(2, n_ctx, 64)
    eps = _unet("tiny", cuda_dev)(x.to(cuda_dev), t.to(cuda_dev), context=c.to(cuda_dev))
    err = rel_l2(eps, RO.unet_forward(sd, x, t, c))
    print(f"tiny zero context {n_ctx}: rel-L2 {err:.2e}")
    assert err < TOL


def test_rdm_graph_and_c_handle_equal_eager(cuda_dev):
    """Graph replay (with autotuning) and the C handle equal the eager forward bit for bit, for the 11-token and the
    one-token context."""
    g = golden("rdm.pt")
    net = _unet("rdm", cuda_dev)
    for case in (g["unet"][1], g["unet"][2]):
        x, t, c = _case_inputs(case, cuda_dev)
        t = t.float()
        net.use_cuda_graph = True
        first = net(x, t, context=c).clone()
        replay = net(x, t, context=c)
        net.use_cuda_graph = False
        eager = net(x, t, context=c)
        h = net.c_handle(tuple(x.shape), c)
        try:
            out = h.forward(x, t)
            torch.cuda.synchronize()
            assert torch.equal(first, replay) and torch.equal(replay, eager) and torch.equal(out, eager)
            assert rel_l2(_esub(replay, g), case["eps"]) < TOL
        finally:
            h.close()


# ------------------------------------------------------------------------------------------------ first stage
@pytest.mark.parametrize("idx", range(3))
def test_kl_f16_decode_vs_reference(cuda_dev, idx):
    """Tiny (level attention 128 wide on the per-image path, 512 wide in the flash kernel) and 48x48 -> 768²."""
    g = golden("rdm.pt")
    case = g["decode"][idx]
    x = _kl(case["cfg"], cuda_dev).decode(_gen(case["shape"], case["seed"]).to(cuda_dev))
    err = rel_l2(_sub(x, g), case["x"])
    print(f"decode {case['cfg']} {tuple(case['shape'])}: rel-L2 {err:.2e}")
    assert tuple(x.shape) == tuple(case["x_shape"]) and err < 2e-3


def test_kl_f16_encode_vs_reference(cuda_dev):
    case = golden("rdm.pt")["encode"][0]
    post = _kl(case["cfg"], cuda_dev).encode(_gen(case["shape"], case["seed"]).clamp(-1, 1).to(cuda_dev))
    err = rel_l2(post.parameters, case["moments"])
    print(f"encode {case['cfg']} {tuple(case['shape'])}: rel-L2 {err:.2e}")
    assert post.parameters.shape == case["moments"].shape and err < 2e-3
    with pytest.raises(NotImplementedError):
        post.sample()


# ------------------------------------------------------------------------------------------------ sampling
def _tiny_model(dev):
    from sdb200.util import instantiate_from_config, remap_config
    g = golden("rdm.pt")
    m = instantiate_from_config(remap_config(script("knn2img").rdm_config(arch.TINY_RDM_UNET, arch.TINY_KL_F16)))
    m = pipeline.load_random_weights(m, dev, seeds=(g["unet_seed"], g["vae_seed"]))
    m.model.diffusion_model.set_weight_set("ema", arch.random_state_dict(arch.unet_param_shapes(arch.TINY_RDM_UNET),
                                                                         g["ema_seed"]))
    return m.eval()


@pytest.mark.parametrize("name", ["ddim_eta0", "ddim_eta1", "plms"])
@pytest.mark.parametrize("graph", [False, True])
def test_tiny_guided_trajectories_match_reference(cuda_dev, monkeypatch, name, graph):
    """c = [text | 2 neighbours], uc = 0, scale 5, inside ema_scope(); the reference's noise draws replayed at eta 1."""
    from sdb200.samplers import DDIMSampler, PLMSSampler
    g = golden("rdm.pt")
    d = g["sampling"]
    r = d[name]
    m = _tiny_model(cuda_dev)
    assert torch.equal(m.alphas_cumprod.cpu(), g["alphas_cumprod"])
    m.model.diffusion_model.use_cuda_graph = graph
    x_T = _gen((2, 16, 16, 16), d["x_T_seed"]).to(cuda_dev)
    c = _unit_rows((2, 3, 64), d["c_seed"]).to(cuda_dev)
    # the reference draws noise at eta 0 too (multiplied by sigma 0); the engine draws only at eta > 0
    stochastic = name == "ddim_eta1"
    draws = [_gen((2, 16, 16, 16), d["noise_seed"] + i) for i in range(r["n_noise"] if stochastic else 0)]
    if stochastic:
        monkeypatch.setattr(torch, "randn_like", lambda t, *a, **k: draws.pop(0).to(t.device))
    kw = dict(batch_size=2, shape=[16, 16, 16], conditioning=c, verbose=False, x_T=x_T,
              unconditional_guidance_scale=g["guidance"], unconditional_conditioning=torch.zeros_like(c))
    with m.ema_scope():
        if name == "plms":
            s, _ = PLMSSampler(m).sample(10, eta=0.0, **kw)
        else:
            s, _ = DDIMSampler(m).sample(10, eta=float(name[-1]), **kw)
    monkeypatch.undo()
    m.model.diffusion_model.use_cuda_graph = False
    assert not draws
    e_s = rel_l2(s, r["sample"])
    e_d = rel_l2(_sub(m.decode_first_stage(r["sample"].to(cuda_dev)), g), r["x_dec"])
    print(f"tiny guided {name} graph {graph}: latent rel-L2 {e_s:.2e}; decode {e_d:.2e}")
    # guidance at scale 5 multiplies the eps difference by 5 at every step: the guided samplers' 2e-3 (and below the
    # 2e-2 of the LAION and non-square guided runs)
    assert e_s < 2e-3 and e_d < 2e-3


def _tiny_vocab(path):
    """A CLIP-format vocabulary covering every byte (ids < 1000 for the tiny CLIP): no merges."""
    from sdb200.tokenizer import bytes_to_unicode
    chars = list(bytes_to_unicode().values())
    vocab = {c: i for i, c in enumerate(chars)}
    vocab.update({c + "</w>": 256 + i for i, c in enumerate(chars)})
    vocab.update({"<|startoftext|>": 998, "<|endoftext|>": 999})
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "vocab.json"), "w") as f:
        json.dump(vocab, f)
    with open(os.path.join(path, "merges.txt"), "w") as f:
        f.write("#version: 0.2\n")
    return path


@pytest.mark.parametrize("neighbors", [False, True])
def test_knn2img_script_tiny(cuda_dev, tmp_path, monkeypatch, neighbors):
    mod = script("knn2img")
    monkeypatch.chdir(tmp_path)
    _write_db(str(tmp_path / "data" / "rdm" / "retrieval_databases" / "artbench-surrealism"), 3000, 64, 1)
    vocab = _tiny_vocab(str(tmp_path / "vocab"))
    args = ["--random_init", "--tiny", "--clip_vocab", vocab, "--outdir", str(tmp_path / "out"), "--H", "256", "--W",
            "256", "--ddim_steps", "4", "--n_samples", "2", "--seed", "0"] + (["--use_neighbors", "--knn", "4"] if
                                                                             neighbors else [])
    paths = mod.main(args)
    from PIL import Image
    assert len(paths) == 3 and Image.open(paths[0]).size == (256, 256)
    assert Image.open(paths[-1]).size == (2 * 258 + 2, 258 + 2)


# ------------------------------------------------------------------------------------------------ GEMM plans
def test_every_plan_of_every_rdm_gemm_problem(cuda_dev):
    """The RDM UNet at (6, 16, 48, 48) with an 11-token context (knn2img's guided batch of 3) and the KL-f16 decoder at
    a 24x24 latent (the decoder's widths at a smaller image)."""
    from test_gemm_plans_gpu import catalogue, run_sweep
    problems = catalogue(GEMM_MODEL_WORKLOADS["rdm"], cuda_dev)
    print(f"\nRDM UNet (6, 16, 48²) and KL-f16 decoder (1, 16, 24²): {len(problems)} distinct GEMM problems")
    assert problems
    run_sweep(problems, cuda_dev, "rdm")
    torch.cuda.empty_cache()
