"""The LDM inpainting model on the host: the oracle (oracle/inpaint_oracle.py) against the unmodified reference's
make_batch / interpolate / composite outputs (tests/golden/inpaint.pt), the architecture tables against the reference's
state-dict keys, and config / checkpoint ingest (DummyLoss, __is_first_stage__, both key prefixes)."""

import numpy as np
import pytest
import torch

import helpers  # noqa: F401  (sys.path for the oracle)
import inpaint_oracle as P
from helpers import golden, script
from sdb200 import arch


def _x_dec(case):
    h, w = case["image"].shape[:2]
    return torch.randn((1, 3, h, w), generator=torch.Generator().manual_seed(case["x_dec_seed"])) * 0.6


@pytest.mark.parametrize("idx", range(4))
def test_oracle_matches_reference_make_batch_interpolate_composite(idx):
    case = golden("inpaint.pt")["prepare"][idx]
    b = P.make_batch(case["image"].numpy(), case["mask"].numpy())
    assert torch.equal(b["masked_image"], case["masked_image"]) and torch.equal(b["mask"], case["batch_mask"])
    for size, cc in case["cc"]:
        assert torch.equal(P.mask_channel(b["mask"], size), cc)
    assert np.array_equal(P.composite(b, _x_dec(case)), case["composite"].numpy())


def test_rgb_mask_is_converted_to_luma_on_the_host():
    from PIL import Image
    case = [c for c in golden("inpaint.pt")["prepare"] if c["tag"] == "rgb_mask"][0]
    assert case["mask_raw"].dim() == 3
    assert np.array_equal(np.array(Image.fromarray(case["mask_raw"].numpy()).convert("L")), case["mask"].numpy())


def test_threshold_case_covers_127_and_128():
    case = [c for c in golden("inpaint.pt")["prepare"] if c["tag"] == "threshold"][0]
    m, bm = case["mask"], case["batch_mask"][0, 0]
    assert bool((m == 127).any()) and bool((m == 128).any())
    assert bool((bm[m == 127] == -1).all()) and bool((bm[m == 128] == 1).all())


def test_arch_tables_match_reference_keys():
    keys = [(k, tuple(s)) for k, s in golden("inpaint.pt")["ld_keys"]]
    sub = lambda pre: [(k[len(pre):], s) for k, s in keys if k.startswith(pre)]
    unet = [(k, tuple(s)) for k, s in arch.unet_param_shapes(arch.INPAINTING_BIG_UNET).items()]
    vq = [(k, tuple(s)) for k, s in arch.vq_param_shapes(arch.VQ_F4_NOATTN).items()]
    assert sub("model.diffusion_model.") == unet
    assert sub("first_stage_model.") == vq and sub("cond_stage_model.") == vq
    assert not [k for k, _ in vq if ".mid.attn_1." in k]
    plan = arch.unet_plan(arch.INPAINTING_BIG_UNET)
    layers = [l for grp in plan["input"] + [plan["middle"]] + plan["output"] for l in grp]
    assert sorted({(a["ch"], a["heads"], a["dhead"]) for k, _, a in layers if k == "attn"}) == \
        [(512, 8, 64), (768, 8, 96), (1024, 8, 128)]
    assert {a["updown"] for k, _, a in layers if k == "res"} == {None, "down", "up"}
    assert not any(a["ss"] for k, _, a in layers if k == "res")


def test_config_instantiates_with_first_stage_as_cond_stage():
    import sdb200
    from sdb200.util import instantiate_from_config, remap_config
    node = script("inpaint").inpaint_config(arch.TINY_INPAINT_UNET, arch.TINY_VQ_NOATTN)
    assert node["params"]["first_stage_config"]["params"]["lossconfig"]["target"].endswith("DummyLoss")
    model = instantiate_from_config(remap_config(node))
    assert isinstance(model, sdb200.LatentDiffusion)
    assert isinstance(model.first_stage_model, sdb200.VQModelInterface)
    assert model.cond_stage_model is model.first_stage_model
    assert model.model.conditioning_key == "concat" and model.model.diffusion_model.in_channels == 7


def test_checkpoint_with_both_prefixes_loads_without_missing_keys():
    from sdb200.util import instantiate_from_config, remap_config
    node = script("inpaint").inpaint_config(arch.TINY_INPAINT_UNET, arch.TINY_VQ_NOATTN)
    model = instantiate_from_config(remap_config(node))
    u = arch.random_state_dict(arch.unet_param_shapes(arch.TINY_INPAINT_UNET), 11)
    v = arch.random_state_dict(arch.vq_param_shapes(arch.TINY_VQ_NOATTN), 12)
    sd = {"model.diffusion_model." + k: t for k, t in u.items()}
    for pre in ("first_stage_model.", "cond_stage_model."):     # the reference saves the shared module twice
        sd.update({pre + k: t for k, t in v.items()})
    sd.update({k: t for k, t in model.state_dict().items() if "." not in k})         # the schedule buffers
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert missing == [] and unexpected == []
    assert torch.equal(model.first_stage_model._host_sd["quantize.embedding.weight"], v["quantize.embedding.weight"])


def test_unsupported_options_raise():
    import sdb200
    from sdb200.diffusion import DiffusionWrapper
    ucfg = {"target": "ldm.modules.diffusionmodules.openaimodel.UNetModel", "params": dict(arch.TINY_INPAINT_UNET)}
    for key in ("hybrid", "adm"):
        with pytest.raises(NotImplementedError):
            DiffusionWrapper(ucfg, key)
    lin = {**arch.TINY_VQ, "ddconfig": {**arch.TINY_VQ["ddconfig"], "attn_type": "linear"}}
    with pytest.raises(NotImplementedError):
        sdb200.VQModelInterface(**lin)
    with pytest.raises(NotImplementedError):
        arch.vae_param_shapes({**arch.TINY_VAE, "ddconfig": {**arch.TINY_VAE["ddconfig"], "attn_type": "linear"}})
    # configs without attn_type keep their mid-block attention
    assert "encoder.mid.attn_1.q.weight" in arch.vq_param_shapes(arch.VQ_F4)
    assert "decoder.mid.attn_1.q.weight" in arch.vae_param_shapes(arch.SD_V1_VAE)
