"""The LAION-400M text-to-image LDM (txt2img --laion400m) on the host: the WordPiece tokenizer against the installed
transformers BERT fast tokenizer on a synthetic vocabulary, the BERT oracle (oracle/bert_oracle.py) against the
unmodified reference's outputs (tests/golden/laion.pt), the architecture tables against the reference's key list of the
whole model, config plumbing, checkpoint ingest, host-side input checks and the script's host logic."""
import collections

import pytest
import torch
import yaml

import helpers  # noqa: F401  (sys.path for the oracle)
import bert_oracle as BO
import ldm_oracle as O
from helpers import golden, rel_l2, script
from sdb200 import arch

CORPUS = ("a photograph of an astronaut riding a horse on mars , highly detailed digital painting . the quick brown "
          "fox jumps over the lazy dog ' s back ; it ' s 42 degrees and they ' re happy ! stable diffusion latent text "
          "to image model trending on artstation 4k 8k uhd cafe naive tokyo tower")
PROMPTS = [
    "a photograph of an astronaut riding a horse",
    "A  Painting\tof a   VIRUS monster playing guitar!!!",
    "it's the dog's 42nd birthday, they're happy; we'll see (maybe) ...",
    "café naïve — trending on ArtStation, 8K UHD ✨ 🚀",                                   # accents, symbols, emoji
    "",
    "   ",
    "under_score and-hyphen and 3.14159 and $100 #tag @user ?!?!... ((()))",            # punctuation runs
    "x" * 40 + " " + "horse " * 120,                                                     # > 77 tokens: truncated
    "y" * 101 + " " + "z" * 100 + " ok",                                                 # 101 chars: [UNK]; 100: kept
    "東京タワー at night 夜景, 서울 skyline, москва зимой",                                   # CJK split per ideograph
    "tab\there\x0bvertical\x0cform\x85next line　wide nbsp",
    "zero​width﻿bom\x00nul\x07bell�replacement",                          # dropped characters
    "é vs é, Å, ẛ̣, ÀÉÎÕÜ ñ ç Ø ß ĳ",                           # accent stripping (NFD)
    "ΟΔΟΣ Σ ﬁ ligature ＦＵＬＬ　ｗｉｄｔｈ",                                              # per-character lowercasing
    "a [CLS] horse [SEP][PAD] [MASK] [UNK] [cls] x[SEP]y",                                # literal special tokens
    "〈quoted〉 «guillemets» „low“ ¿qué? ¡sí! ‰ † ‡ • ‧ ·",                                # Unicode punctuation
]


def _vocab():
    """A synthetic uncased vocabulary: BERT's special tokens, single characters with and without `##`, the corpus words
    and some of their suffixes, so words decompose into several pieces."""
    v = ["[PAD]"] + [f"[unused{i}]" for i in range(3)] + ["[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    chars = sorted(set("abcdefghijklmnopqrstuvwxyz0123456789!\"#$%&'()*+,-./:;<=>?@[\\]^_`{|}~") |
                   set("東京夜景タワー서울москвазимойß¿¡—…"))
    v += chars + ["##" + c for c in chars]
    for w in sorted(collections.Counter(CORPUS.split())):
        if w not in v:
            v.append(w)
        for i in range(2, len(w) - 1, 2):
            if "##" + w[i:] not in v:
                v.append("##" + w[i:])
    return v + ["photo", "##graph", "astro", "##naut", "ride", "##ing", "paint"]


@pytest.fixture(scope="module")
def bert_vocab_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("bert_vocab")
    (d / "vocab.txt").write_text("\n".join(_vocab()) + "\n", encoding="utf-8")
    return d


def test_wordpiece_matches_transformers_bert_tokenizer(bert_vocab_dir, monkeypatch):
    monkeypatch.setenv("HF_HUB_OFFLINE", "1")
    transformers = pytest.importorskip("transformers")
    from sdb200.tokenizer import BertWordPieceTokenizer
    hf = transformers.BertTokenizerFast.from_pretrained(str(bert_vocab_dir), local_files_only=True)
    mine = BertWordPieceTokenizer.from_dir(str(bert_vocab_dir))
    assert len(mine) == len(_vocab()) and (mine.cls_id, mine.sep_id, mine.pad_id, mine.unk_id) == (5, 6, 0, 4)
    want = hf(PROMPTS, truncation=True, max_length=77, return_length=True, return_overflowing_tokens=False,
              padding="max_length", return_tensors="pt")["input_ids"]
    got = torch.tensor(mine(PROMPTS))
    assert got.shape == (len(PROMPTS), 77)
    for i, p in enumerate(PROMPTS):
        assert torch.equal(got[i], want[i]), (p, got[i].tolist()[:24], want[i].tolist()[:24])
    assert got[4].tolist() == [5, 6] + [0] * 75                      # the empty prompt: [CLS] [SEP] [PAD]...
    assert int((got[7] != 0).sum()) == 77 and got[7, -1] == 6         # truncated to [CLS] + 75 + [SEP]
    assert got[8, 1].item() == 4 and got[8, 2].item() != 4            # the 101-character word is [UNK]; 100 is not


def test_bert_embedder_tokenizes_from_vocab_dir_and_raises_without_one(bert_vocab_dir, monkeypatch):
    import sdb200
    from sdb200.tokenizer import BertWordPieceTokenizer
    emb = sdb200.BERTEmbedder(**arch.TINY_BERT, vocab_dir=str(bert_vocab_dir))
    ids = emb._tokenize(["a horse", ""])
    assert ids.shape == (2, 77) and ids.dtype == torch.int64
    assert ids.tolist() == BertWordPieceTokenizer.from_dir(str(bert_vocab_dir))(["a horse", ""])
    monkeypatch.setattr(sdb200.bert, "_cached_vocab", lambda: None)
    bare = sdb200.BERTEmbedder(**arch.TINY_BERT)
    with pytest.raises(RuntimeError, match="vocabulary"):
        bare.encode("a horse")
    with pytest.raises(RuntimeError, match="vocabulary"):
        bare(["a horse"])
    with pytest.raises(TypeError):
        emb._tokenize(["a horse", 3])


def test_bert_embedder_rejects_bad_ids():
    """sdb_embed_tokens clamps ids, so the host check must raise before anything reaches it."""
    import sdb200
    emb = sdb200.BERTEmbedder(**arch.TINY_BERT, use_tokenizer=False)
    ok = torch.zeros(2, 77, dtype=torch.long)
    assert torch.equal(emb.check_ids(ok), ok)
    for bad in (torch.full((1, 77), 1000), torch.full((1, 77), -1), torch.tensor([[101, 102, 30521]])):
        with pytest.raises(IndexError):
            emb.check_ids(bad)
    for bad in (torch.zeros(77, dtype=torch.long), torch.zeros(2, 77), torch.zeros(1, 77, dtype=torch.bool),
                torch.zeros(1, 1, 77, dtype=torch.long)):
        with pytest.raises(TypeError):
            emb.check_ids(bad)
    for bad in (torch.zeros(1, 78, dtype=torch.long), torch.zeros(0, 77, dtype=torch.long),
                torch.zeros(2, 0, dtype=torch.long)):
        with pytest.raises(ValueError):
            emb.check_ids(bad)
    with pytest.raises(AssertionError, match="weights not loaded"):
        emb.encode_ids(ok)


@pytest.mark.parametrize("idx", range(2))
def test_oracle_bert_matches_reference(idx):
    g = golden("laion.pt")
    case = g["bert"][idx]
    cfg = {"tiny": arch.TINY_BERT, "full": arch.LAION_BERT}[case["cfg"]]
    sd = arch.random_state_dict(arch.bert_param_shapes(cfg), g["bert_seed"])
    z = BO.bert_embed(sd, case["ids"])
    assert case["ids"][-1].tolist() == [101, 102] + [0] * 75
    assert rel_l2(z, case["z"]) < (5e-4 if case["cfg"] == "full" else 1e-5)     # the full-size output is stored as fp16


@pytest.mark.parametrize("idx", [0, 1])
def test_oracle_tiny_unet_matches_reference(idx):
    g = golden("laion.pt")
    case = g["unet"][idx]
    assert case["cfg"] == "tiny"
    sd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_LAION_UNET), g["unet_seed"])
    ctx = torch.randn((case["x"].shape[0], 77, 128), generator=torch.Generator().manual_seed(case["ctx_seed"]))
    assert rel_l2(O.unet_forward(sd, case["x"], case["t"], ctx, num_heads=2), case["eps"]) < 1e-5


def test_oracle_guided_plms_matches_reference():
    g = golden("laion.pt")
    d = g["plms"]
    usd = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_LAION_UNET), g["unet_seed"])
    bsd = arch.random_state_dict(arch.bert_param_shapes(arch.TINY_BERT), g["bert_seed"])
    fn = lambda x, t, ctx: O.unet_forward(usd, x, t, ctx, num_heads=2)
    s = O.plms_sample(fn, d["x_T"], BO.bert_embed(bsd, d["ids"]), BO.bert_embed(bsd, d["uc_ids"]), 7.5, S=10)
    assert rel_l2(s, d["sample"]) < 1e-4


def test_arch_tables_match_reference_keys():
    """Every parameter of the reference's LAION LatentDiffusion, by key and shape, to_logits included; the rest of its
    state_dict is the schedule buffers."""
    ref = [(k, tuple(s)) for k, s in golden("laion.pt")["laion_keys"]]
    mine = [("model.diffusion_model." + k, tuple(s)) for k, s in arch.unet_param_shapes(arch.LAION_UNET).items()]
    mine += [("first_stage_model." + k, tuple(s)) for k, s in arch.vae_param_shapes(arch.SD_V1_VAE).items()]
    bert = [("cond_stage_model." + k, tuple(s)) for k, s in arch.bert_param_shapes(arch.LAION_BERT).items()]
    stages = ("model.", "first_stage_model.", "cond_stage_model.")
    assert sorted(e for e in ref if e[0].startswith(stages)) == sorted(mine + bert)
    assert [e for e in ref if e[0].startswith("cond_stage_model.")] == bert          # same order as the reference
    assert ("cond_stage_model.transformer.to_logits.weight", (30522, 1280)) in ref
    assert ("model.diffusion_model.input_blocks.1.1.transformer_blocks.0.attn2.to_k.weight", (320, 1280)) in ref
    assert all("." not in k for k, _ in ref if not k.startswith(stages))
    assert len(bert) == 2 + 64 * 2 + 32 * 5 + 32 * 4 + 4


def test_random_init_layer_norms_are_gains():
    sd = arch.random_state_dict(arch.bert_param_shapes(arch.TINY_BERT), 13)
    g = sd["transformer.attn_layers.layers.1.0.weight"]
    assert 0.7 < float(g.min()) and float(g.max()) < 1.3
    assert float(sd["transformer.attn_layers.layers.1.1.net.0.0.weight"].std()) < 0.2


def test_target_map_and_builtin_config():
    import sdb200
    from sdb200 import pipeline
    from sdb200.util import TARGET_MAP, get_obj_from_str, instantiate_from_config, remap_config
    assert get_obj_from_str(TARGET_MAP["ldm.modules.encoders.modules.BERTEmbedder"]) is sdb200.BERTEmbedder
    node = pipeline.laion_model_config()
    p = node["params"]
    assert p["unet_config"]["params"]["context_dim"] == 1280 and p["cond_stage_config"]["params"]["n_layer"] == 32
    assert (p["linear_start"], p["linear_end"], p["scale_factor"], p["use_ema"]) == (0.00085, 0.012, 0.18215, False)
    m = instantiate_from_config(remap_config(pipeline.laion_model_config(arch.TINY_LAION_UNET, arch.TINY_VAE,
                                                                         arch.TINY_BERT)))
    assert isinstance(m.cond_stage_model, sdb200.BERTEmbedder) and m.cond_stage_model.use_tknz_fn
    b =pipeline.build_laion_model(arch.TINY_LAION_UNET, arch.TINY_VAE, arch.TINY_BERT)
    assert isinstance(b.cond_stage_model, sdb200.BERTEmbedder) and b.scale_factor == 0.18215


@pytest.mark.parametrize("fmt", ["ckpt", "safetensors"])
def test_load_tiny_laion_checkpoint(tmp_path, fmt):
    """A reference-style txt2img-1p4B-eval config (tiny members, use_ema False) and a checkpoint with the reference's
    keys, to_logits included, load through load_model_from_config with nothing missing or unexpected."""
    import sdb200
    from sdb200 import checkpoint, pipeline
    node = pipeline.laion_model_config(arch.TINY_LAION_UNET, arch.TINY_VAE, arch.TINY_BERT)
    assert node["params"]["use_ema"] is False
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.safe_dump({"model": {"base_learning_rate": 5.0e-05, **node}}))
    sd = {"model.diffusion_model." + k: t for k, t in
          arch.random_state_dict(arch.unet_param_shapes(arch.TINY_LAION_UNET), 11).items()}
    sd.update({"first_stage_model." + k: t for k, t in arch.random_state_dict(arch.vae_param_shapes(arch.TINY_VAE), 12).items()})
    bsd = arch.random_state_dict(arch.bert_param_shapes(arch.TINY_BERT), 13)
    sd.update({"cond_stage_model." + k: t for k, t in bsd.items()})
    if fmt == "ckpt":
        ck = tmp_path / "model.ckpt"
        torch.save({"state_dict": sd, "global_step": 7}, ck)
    else:
        ck = tmp_path / "model.safetensors"
        checkpoint.write_safetensors(str(ck), sd)
    model = checkpoint.load_model_from_config(str(cfg), str(ck), device=None)
    info = model.load_info
    schedule = ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod")
    assert [k for k in info["missing"] if k not in schedule] == [] and info["unexpected"] == []
    enc = model.cond_stage_model
    assert isinstance(enc, sdb200.BERTEmbedder) and model.cond_stage_key == "caption"
    assert "transformer.to_logits.weight" not in enc._host_sd
    assert torch.equal(enc._host_sd["transformer.token_emb.weight"], bsd["transformer.token_emb.weight"])
    # a missing encoder tensor is an error, an extra unknown one is reported as unexpected
    del sd["cond_stage_model.transformer.norm.bias"]
    sd["cond_stage_model.transformer.extra"] = torch.zeros(1)
    ck2 = tmp_path / "broken.safetensors"
    checkpoint.write_safetensors(str(ck2), sd)
    with pytest.raises(RuntimeError, match="lacks"):
        checkpoint.load_model_from_config(str(cfg), str(ck2), device=None)


def test_txt2img_laion400m_host_logic(tmp_path, monkeypatch):
    """--laion400m switches config / checkpoint / output directory as the reference does; the built-in LAION config is
    used when the YAML is absent; the stand-in and unconditional ids are bert-base-uncased's."""
    mod = script("txt2img")
    import argparse
    opt = argparse.Namespace(laion400m=True, config=mod.DEFAULT_CONFIG, ckpt="x.ckpt", outdir="outputs/txt2img-samples")
    mod.apply_laion400m(opt)
    assert (opt.config, opt.ckpt, opt.outdir) == ("configs/latent-diffusion/txt2img-1p4B-eval.yaml",
                                                  "models/ldm/text2img-large/model.ckpt",
                                                  "outputs/txt2img-samples-laion400m")
    sd_opt = argparse.Namespace(laion400m=False, config=mod.DEFAULT_CONFIG, ckpt="x.ckpt", outdir="o")
    assert vars(mod.apply_laion400m(sd_opt)) == dict(laion400m=False, config=mod.DEFAULT_CONFIG, ckpt="x.ckpt", outdir="o")
    ids = mod.synthetic_bert_ids(3, 1234, "cpu")
    assert ids.shape == (3, 77) and (ids[:, 0] == 101).all() and (ids[:, 20] == 102).all() and (ids[:, 21:] == 0).all()
    assert ((ids[:, 1:20] >= 999) & (ids[:, 1:20] < 30522)).all() and torch.equal(ids, mod.synthetic_bert_ids(3, 1234, "cpu"))
    un = mod.bert_uncond_ids(3, "cpu")
    assert un.tolist() == [[101, 102] + [0] * 75] * 3
    # the SD-v1 stand-ins are unchanged
    sdv = mod.synthetic_ids(2, 1234, "cpu")
    assert (sdv[:, 0] == 49406).all() and (sdv[:, 20:] == 49407).all()
    # built-in config fallback: the LAION YAML path is absent, so the LAION model config is used with the checkpoint
    monkeypatch.chdir(tmp_path)
    seen = {}
    monkeypatch.setattr(mod.sdb200.checkpoint, "load_model_from_config",
                        lambda cfg, ckpt, **kw: seen.update(cfg=cfg, ckpt=ckpt) or "model")
    (tmp_path / "m.ckpt").write_bytes(b"")
    assert mod.load_model_from_config(mod.LAION_CONFIG, "m.ckpt", "cpu") == "model"
    assert seen["cfg"]["model"]["params"]["cond_stage_config"]["target"] == "ldm.modules.encoders.modules.BERTEmbedder"
    mod.load_model_from_config(mod.DEFAULT_CONFIG, "m.ckpt", "cpu")
    assert seen["cfg"]["model"]["params"]["cond_stage_config"]["target"] == "ldm.modules.encoders.modules.FrozenCLIPEmbedder"
    with pytest.raises(FileNotFoundError):
        mod.load_model_from_config("configs/other.yaml", "m.ckpt", "cpu")
    with pytest.raises(FileNotFoundError):
        mod.load_model_from_config(mod.LAION_CONFIG, "missing.ckpt", "cpu")
