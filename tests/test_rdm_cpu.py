"""The retrieval-augmented diffusion model (configs/retrieval-augmented-diffusion/768x768.yaml, scripts/knn2img.py) on
the host: the oracle (oracle/rdm_oracle.py) against the unmodified reference's outputs (tests/golden/rdm.pt), the
architecture tables against the reference's key list of the whole model, the YAML node, the schedule, the retrieval
database's loading and normalisation, the Searcher's host logic, CLIP tokenization and the script's arguments."""
import json
import os

import numpy as np
import pytest
import torch

import helpers  # noqa: F401  (sys.path for the oracle)
import rdm_oracle as RO
from helpers import golden, rel_l2, script
from sdb200 import arch

UCFG = {"tiny": arch.TINY_RDM_UNET, "rdm": arch.RDM_UNET}
VCFG = {"tiny": arch.TINY_KL_F16, "kl_f16": arch.KL_F16}


def _gen(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def _unit_rows(shape, seed):
    x = _gen(shape, seed)
    return x / torch.linalg.norm(x, dim=-1, keepdim=True)


def _sub(x, g):
    k = g["image_stride"]
    return x[..., ::k, ::k]


@pytest.mark.parametrize("idx", range(4))
def test_oracle_unet_matches_reference(idx):
    g = golden("rdm.pt")
    case = g["unet"][idx]
    sd = arch.random_state_dict(arch.unet_param_shapes(UCFG[case["cfg"]]), g["unet_seed"])
    c = _unit_rows((case["shape"][0], case["n_ctx"], UCFG[case["cfg"]]["context_dim"]), case["seed"] + 1)
    k = g["eps_stride"]
    eps = RO.unet_forward(sd, _gen(case["shape"], case["seed"]), case["t"], c)
    assert rel_l2(eps[..., ::k, ::k], case["eps"]) < 1e-5


def test_oracle_first_stage_matches_reference():
    g = golden("rdm.pt")
    sds = {tag: arch.random_state_dict(arch.vae_param_shapes(cfg), g["vae_seed"]) for tag, cfg in VCFG.items()}
    for case in g["decode"]:
        x = RO.kl_decode(sds[case["cfg"]], _gen(case["shape"], case["seed"]))
        assert tuple(x.shape) == tuple(case["x_shape"]) and rel_l2(_sub(x, g), case["x"]) < 1e-5
    for case in g["encode"]:
        x = _gen(case["shape"], case["seed"]).clamp(-1, 1)
        assert rel_l2(RO.kl_encode_moments(sds[case["cfg"]], x), case["moments"]) < 1e-5
    assert ("kl_f16", (1, 16, 48, 48), (1, 3, 768, 768)) in {(c["cfg"], tuple(c["shape"]), tuple(c["x_shape"]))
                                                             for c in g["decode"]}


@pytest.mark.parametrize("name", ["ddim_eta0", "ddim_eta1", "plms"])
def test_oracle_guided_trajectories_match_reference(name):
    g = golden("rdm.pt")
    d = g["sampling"]
    r = d[name]
    esd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_RDM_UNET), g["ema_seed"])
    x_T = _gen((2, 16, 16, 16), d["x_T_seed"])
    c = _unit_rows((2, 3, 64), d["c_seed"])
    fn = lambda x, t, ctx: RO.unet_forward(esd, x, t, ctx)
    if name == "plms":
        s = RO.plms_sample(fn, x_T, c, torch.zeros_like(c), g["guidance"], g["alphas_cumprod"], 10)
    else:
        eta = float(name[-1])
        noises = torch.stack([_gen(x_T.shape, d["noise_seed"] + i) for i in range(r["n_noise"])])
        s = RO.ddim_sample(fn, x_T, c, torch.zeros_like(c), g["guidance"], g["alphas_cumprod"], 10, eta,
                           noises if eta else torch.zeros_like(noises))
    assert rel_l2(s, r["sample"]) < 1e-5
    vsd = arch.random_state_dict(arch.vae_param_shapes(arch.TINY_KL_F16), g["vae_seed"])
    assert rel_l2(_sub(RO.decode_first_stage(vsd, r["sample"], g["scale_factor"]), g), r["x_dec"]) < 1e-5


def test_arch_tables_match_reference_keys():
    """Every parameter of the reference's RDM LatentDiffusion by key and shape, with its EMA copies (use_ema defaults to
    True), the KL-f16 first stage in registration order, and the per-level heads of 32."""
    g = golden("rdm.pt")
    ref = [(k, tuple(s)) for k, s in g["rdm_keys"]]
    ushapes = arch.unet_param_shapes(arch.RDM_UNET)
    vshapes = arch.vae_param_shapes(arch.KL_F16)
    mine = [("model.diffusion_model." + k, tuple(s)) for k, s in ushapes.items()]
    mine += [("first_stage_model." + k, tuple(s)) for k, s in vshapes.items()]
    mine += [("model_ema.diffusion_model" + k.replace(".", ""), tuple(s)) for k, s in ushapes.items()]
    stages = ("model.", "first_stage_model.", "model_ema.diffusion_model")
    assert sorted(e for e in ref if e[0].startswith(stages)) == sorted(mine)
    assert {k for k, _ in ref if k.startswith("model_ema.") and not k.startswith(stages)} == \
        {"model_ema.decay", "model_ema.num_updates"}
    assert not [k for k, _ in ref if k.startswith("cond_stage_model.")]       # the Identity cond stage
    assert [e for e in ref if e[0].startswith("first_stage_model.")] == \
        [("first_stage_model." + k, tuple(s)) for k, s in vshapes.items()]
    assert not [k for k in vshapes if ".attn." in k and not k.startswith(("encoder.down.4.", "decoder.up.4."))]
    assert ("first_stage_model.post_quant_conv.weight", (16, 16, 1, 1)) in ref
    plan = arch.unet_plan(arch.RDM_UNET)
    layers = [l for grp in plan["input"] + [plan["middle"]] + plan["output"] for l in grp]
    sts = [(a["ch"], a["heads"], a["dhead"]) for k, _, a in layers if k == "st"]
    assert sorted(set(sts)) == [(448, 14, 32), (896, 28, 32), (1344, 42, 32), (1792, 56, 32)]


def test_reference_yaml_node_resolves():
    """The YAML's model node instantiates through TARGET_MAP with the arch tables' parameters (cond stage Identity),
    and the script's built-in node is the same."""
    import sdb200
    from sdb200.util import TARGET_MAP, instantiate_from_config, remap_config
    node = golden("rdm.pt")["yaml_node"]
    p = node["params"]
    assert p["unet_config"]["params"] == arch.RDM_UNET
    assert p["first_stage_config"]["params"]["ddconfig"] == arch.KL_F16["ddconfig"]
    assert p["first_stage_config"]["params"]["embed_dim"] == 16
    for t in [node["target"], p["unet_config"]["target"], p["first_stage_config"]["target"]]:
        assert t in TARGET_MAP
    m = instantiate_from_config(remap_config(node))
    assert isinstance(m.model.diffusion_model, sdb200.UNetModel) and m.model.diffusion_model.conditional
    assert isinstance(m.first_stage_model, sdb200.AutoencoderKL)
    assert m.first_stage_model.shapes == arch.vae_param_shapes(arch.KL_F16)
    assert isinstance(m.cond_stage_model, torch.nn.Identity)
    assert m.use_ema and m.scale_factor == pytest.approx(0.22765929) and m.model.conditioning_key == "crossattn"
    assert script("knn2img").rdm_config() == node
    assert "ldm.modules.encoders.modules.FrozenCLIPTextEmbedder" in TARGET_MAP


def test_schedule_linear_end():
    """linear_start 0.0015, linear_end 0.015: the engine's schedule equals the reference's buffers."""
    from sdb200.util import instantiate_from_config, remap_config
    m = instantiate_from_config(remap_config(script("knn2img").rdm_config(arch.TINY_RDM_UNET, arch.TINY_KL_F16)))
    assert m.linear_end == 0.015 and torch.equal(m.alphas_cumprod, golden("rdm.pt")["alphas_cumprod"])


def _write_db(path, sizes, dim, seed):
    os.makedirs(path, exist_ok=True)
    rng = np.random.default_rng(seed)
    parts = []
    for i, n in enumerate(sizes):
        emb = (rng.standard_normal((n, dim)) * rng.uniform(0.5, 2.0, (n, 1))).astype(np.float32)
        ids = rng.integers(0, 10 ** 6, n)
        pc = rng.integers(0, 256, (n, 4))
        np.savez(os.path.join(path, f"{9 - i}.npz"), embedding=emb, img_id=ids, patch_coords=pc)   # names sort backwards
        parts.append((emb, ids, pc))
    return parts[::-1]


def test_database_loading_and_normalisation(tmp_path):
    """Files concatenate in sorted name order; the normalisation is the reference's numpy formula bit for bit, in
    the chunks the upload uses as well as at once."""
    from sdb200 import retrieval
    parts = _write_db(str(tmp_path / "db"), [300, 17, 1000], 64, 0)
    db = retrieval.load_database(str(tmp_path / "db"))
    for j, key in enumerate(retrieval.KEYS):
        assert np.array_equal(db[key], np.concatenate([p[j] for p in parts]))
    emb = db["embedding"]
    ref = emb / np.linalg.norm(emb, axis=1)[:, np.newaxis]
    assert np.array_equal(retrieval.normalize_rows(emb), ref)
    assert np.array_equal(np.concatenate([retrieval.normalize_rows(emb[i:i + 100]) for i in range(0, len(emb), 100)]), ref)
    one = _write_db(str(tmp_path / "one"), [50], 64, 1)
    assert np.array_equal(retrieval.load_database(str(tmp_path / "one"))["embedding"], one[0][0])
    with pytest.raises(ValueError, match="No npz-files"):
        retrieval.load_database(str(tmp_path / "none"))
    assert retrieval.database_path("openimages") == os.path.join(".", "data", "rdm", "retrieval_databases", "openimages")
    with pytest.raises(AssertionError):
        retrieval.Searcher("not-a-database")


def test_searcher_host_logic_equals_fp64_brute_force(tmp_path):
    """search(x, k) with the device search replaced by an fp64 brute force: the reference's dict, nn_embeddings by the
    reference's formula on the returned rows."""
    from sdb200 import retrieval
    _write_db(str(tmp_path / "db"), [400, 600], 32, 2)
    s = object.__new__(retrieval.Searcher)
    s.database = retrieval.load_database(str(tmp_path / "db"))
    full = s.database["embedding"].astype(np.float64)
    full = full / np.linalg.norm(full, axis=1)[:, None]
    s.search_rows = lambda q, k: (np.argsort(-(q.astype(np.float64) @ full.T), axis=1, kind="stable")[:, :k], None)
    x = torch.from_numpy(np.random.default_rng(3).standard_normal((5, 1, 32)).astype(np.float32))
    out = s.search(x, 7)
    emb = s.database["embedding"]
    nns = out["nns"]
    scores = (out["q_embeddings"].astype(np.float64) @ full.T)
    assert np.array_equal(nns, np.argsort(-scores, axis=1, kind="stable")[:, :7])
    assert np.array_equal(out["nn_embeddings"], emb[nns] / np.linalg.norm(emb[nns], axis=-1)[..., np.newaxis])
    assert np.array_equal(out["img_ids"], s.database["img_id"][nns])
    assert np.array_equal(out["patch_coords"], s.database["patch_coords"][nns])
    assert np.array_equal(out["queries"], x[:, 0].numpy())


def _tiny_vocab(path):
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


def test_tokenize_eot_position_and_padding(tmp_path):
    """clip.tokenize: BOS + tokens + EOT, zeros after; the EOT (the largest id) is where the embedding is pooled; a
    prompt longer than 77 tokens is an error, not truncated."""
    import sdb200
    enc = sdb200.FrozenCLIPTextEmbedder(version=_tiny_vocab(str(tmp_path / "v")), config=arch.TINY_CLIP_TEXT_PROJ)
    ids = enc.tokenize(["ab", "a b c d"])
    assert ids.shape == (2, 77) and ids.dtype == torch.long
    for row in ids:
        eot = int(row.argmax())
        assert row[0] == 998 and row[eot] == 999 and not row[eot + 1:].any() and (row[1:eot] < 998).all()
    assert int(ids[0].argmax()) == 3          # "ab" is two byte tokens without merges
    enc.tokenize(["x" * 75])
    with pytest.raises(RuntimeError, match="too long"):
        enc.tokenize(["x" * 76])
    with pytest.raises(RuntimeError, match="vocabulary"):
        sdb200.FrozenCLIPTextEmbedder(config=arch.TINY_CLIP_TEXT_PROJ).tokenize(["a"])


def test_clip_text_embedder_reads_clipmodel_layout():
    """`text_model.*` + `text_projection.weight` are adopted at the top level; the vision tower's keys are ignored."""
    import sdb200
    enc = sdb200.FrozenCLIPTextEmbedder(config=arch.TINY_CLIP_TEXT_PROJ)
    sd = dict(arch.random_state_dict(enc.shapes, 13))
    sd.update({"vision_model.embeddings.class_embedding": torch.zeros(8), "visual_projection.weight": torch.zeros(4, 8),
               "logit_scale": torch.tensor(1.0), "text_model.embeddings.position_ids": torch.arange(77)[None]})
    r = enc.load_state_dict(sd, strict=False)
    assert r.missing_keys == [] and r.unexpected_keys == []
    assert torch.equal(enc._host_sd["text_projection.weight"], sd["text_projection.weight"])
    assert enc.shapes["text_projection.weight"] == (64, 128)
    assert arch.clip_text_proj_param_shapes(arch.CLIP_TEXT_PROJ)["text_projection.weight"] == (768, 768)


def test_kl_first_stage_level_attention_arguments():
    """KL first stages with attention inside the levels are accepted when every attn_resolutions entry is a level's
    resolution (KL-f16's [16], KL-f32's [16, 8]); an entry no level reaches is rejected."""
    import sdb200
    kl = sdb200.AutoencoderKL(**arch.KL_F16, lossconfig={"target": "torch.nn.Identity"})
    assert kl.embed_dim == 16 and sum(".attn." in k for k in kl.shapes) == (2 + 3) * 10
    f32 = dict(double_z=True, z_channels=64, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 1, 2, 2, 4, 4],
               num_res_blocks=2, attn_resolutions=[16, 8], dropout=0.0)
    assert sum(".attn." in k for k in sdb200.AutoencoderKL(ddconfig=f32, embed_dim=64).shapes) == 2 * (2 + 3) * 10
    with pytest.raises(AssertionError, match="no level"):     # the SD-v1 f8 stage has no 16x16 level
        sdb200.AutoencoderKL(ddconfig={**arch.SD_V1_VAE["ddconfig"], "attn_resolutions": [16]}, embed_dim=4)


def test_script_arguments():
    """The reference's defaults, and the argument checks that run before anything is built."""
    mod = script("knn2img")
    opt = mod.get_parser().parse_args([])
    assert (opt.H, opt.W, opt.ddim_steps, opt.scale, opt.n_samples, opt.knn, opt.database, opt.ddim_eta) == \
        (768, 768, 50, 5.0, 3, 10, "artbench-surrealism", 0.0)
    assert not opt.plms and not opt.use_neighbors and opt.ckpt == "models/rdm/rdm768x768/model.ckpt"
    with pytest.raises(NotImplementedError):
        mod.main(["--clip_type", "RN50"])
    with pytest.raises(ValueError, match="multiples of 16"):
        mod.main(["--H", "760", "--random_init"])
    with pytest.raises(ValueError, match="PLMS"):
        mod.main(["--plms", "--ddim_eta", "1", "--random_init"])
    with pytest.raises(ValueError, match="--tiny"):
        mod.main(["--tiny"])
    with pytest.raises(SystemExit):
        mod.get_parser().parse_args(["--database", "not-a-database"])
    # the shapes the script builds at the tiny size: latent [16, H/16, W/16], context 1 + knn tokens of the CLIP width
    from sdb200.util import instantiate_from_config, remap_config
    m = instantiate_from_config(remap_config(mod.rdm_config(arch.TINY_RDM_UNET, arch.TINY_KL_F16)))
    assert m.model.diffusion_model.in_channels == 16 and m.channels == 16
    assert m.model.diffusion_model.cfg["context_dim"] == arch.TINY_CLIP_TEXT_PROJ["projection_dim"]
    assert m.first_stage_model.cfg["ddconfig"]["z_channels"] == 16 and len(m.first_stage_model.cfg["ddconfig"]["ch_mult"]) == 5
