"""The denoising objective on the H100: sdb_q_sample_t and sdb_diffusion_loss elementwise against fp64 and the
reference, LatentDiffusion.p_losses / get_input / validation_step on the five tiny members of tests/golden/losses.pt
(oracle/make_golden_losses.py), and scripts/eval_loss.py end to end."""
import json
import math
import os
import sys

import pytest
import torch

from helpers import ROOT, golden, rel_l2
from sdb200 import arch, ops
from sdb200.util import instantiate_from_config, remap_config

pytestmark = pytest.mark.gpu

G = golden("losses.pt")
U = 2.0 ** -24                        # fp32 unit roundoff
KEYS = ("val/loss_simple", "val/loss_vlb", "val/loss")


def _fs_shapes(node):
    p = node["params"]["first_stage_config"]["params"]
    cfg = {k: p[k] for k in ("embed_dim", "n_embed", "ddconfig") if k in p}
    return arch.vq_param_shapes(cfg) if "n_embed" in cfg else arch.vae_param_shapes(cfg)


def build(name, dev, ema_seed=None, **override):
    """The engine's model of a golden member with the generator's weights (UNet seed 11, first stage 12, cond stage 13
    at the stored shapes); ema_seed also loads an EMA set of that seed and turns use_ema on."""
    m = G["members"][name]
    node = {**m["node"], "params": {**m["node"]["params"], **override}}
    if ema_seed is not None:
        node["params"]["use_ema"] = True
    ld = instantiate_from_config(remap_config(node))
    unet_cfg = node["params"]["unet_config"]["params"]
    usd = arch.random_state_dict(arch.unet_param_shapes(unet_cfg), G["unet_seed"])
    sd = {"model.diffusion_model." + k: v for k, v in usd.items()}
    sd.update({"first_stage_model." + k: v for k, v in arch.random_state_dict(_fs_shapes(node), G["fs_seed"]).items()})
    csd = arch.random_state_dict(m["cond_shapes"], G["cond_seed"]) if m["cond_shapes"] else {}
    sd.update({"cond_stage_model." + k: v for k, v in csd.items()})
    if ema_seed is not None:
        esd = arch.random_state_dict(arch.unet_param_shapes(unet_cfg), ema_seed)
        sd.update({"model_ema." + ("diffusion_model." + k).replace(".", ""): v for k, v in esd.items()})
    if node["params"].get("scale_by_std"):
        sd["scale_factor"] = torch.tensor(m["scale_factor"])
    res = ld.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys, res.unexpected_keys
    return ld.to(dev).eval()


def batch_of(name):
    """The member's batch dict as get_input reads it: the stored uint8 images as u / 127.5 - 1, the uint8 label map
    one-hot over the semantic cond stage's channels, class labels as they are."""
    out = {}
    for k, v in G["members"][name]["batch"].items():
        if k == "segmentation":
            out[k] = torch.nn.functional.one_hot(v.long(), arch.TINY_SEMANTIC_COND["in_channels"]).float()
        elif v.dtype == torch.uint8:
            out[k] = v.float() / 127.5 - 1.0
        else:
            out[k] = v
    return out


# ------------------------------------------------------------------------------------------------ sdb_q_sample_t
@pytest.mark.parametrize("name", sorted(G["members"]))
def test_q_sample_t_bit_exact_vs_reference(cuda_dev, name):
    m = G["members"][name]
    ld = build(name, cuda_dev)
    out = ops.q_sample_t(m["x_start"].to(cuda_dev), m["noise"].to(cuda_dev), m["t"].to(cuda_dev),
                         ld.sqrt_alphas_cumprod, ld.sqrt_one_minus_alphas_cumprod)
    assert torch.equal(out.cpu(), m["x_noisy"])


@pytest.mark.parametrize("t", [0, 1, 500, 999])
def test_q_sample_t_uniform_equals_axpby2(cuda_dev, t):
    ld = build("sd", cuda_dev)
    g = torch.Generator().manual_seed(t)
    x = torch.randn(3, 4, 13, 7, generator=g).to(cuda_dev)
    n = torch.randn(3, 4, 13, 7, generator=g).to(cuda_dev)
    ts = torch.full((3,), t, dtype=torch.long, device=cuda_dev)
    new = ops.q_sample_t(x, n, ts, ld.sqrt_alphas_cumprod, ld.sqrt_one_minus_alphas_cumprod)
    old = ld.q_sample(x, ts, n)             # the samplers' route: one timestep, sdb_axpby2
    assert torch.equal(new, old)
    assert torch.equal(ld._q_sample_per_sample(x, ts, n), old)


def test_q_sample_t_rejects_out_of_range_t(cuda_dev):
    ld = build("sd", cuda_dev)
    x = torch.zeros(2, 4, 8, 8, device=cuda_dev)
    tables = (ld.sqrt_alphas_cumprod, ld.sqrt_one_minus_alphas_cumprod)
    torch.cuda.synchronize()
    before = ops.launch_count()
    for bad in ([0, 1000], [-1, 3]):
        t = torch.tensor(bad, device=cuda_dev)
        with pytest.raises(IndexError):
            ops.q_sample_t(x, x, t, *tables)
        with pytest.raises(IndexError):
            ops.diffusion_loss(x, x, "l2", t, ld.logvar, ld.lvlb_weights)
        with pytest.raises(IndexError):
            ld.p_losses(x, torch.zeros(2, 77, 64, device=cuda_dev), t)
    with pytest.raises(IndexError):
        ld._q_sample_per_sample(x, torch.tensor([1000, 1000], device=cuda_dev), x)
    assert ops.launch_count() == before


# ------------------------------------------------------------------------------------------------ sdb_diffusion_loss
def loss_ref(pred, target, kind, t, logvar, lvlb):
    """fp64 restatement: per-sample mean of |d| or d^2 with d = target - pred exact, then the two weightings."""
    d = target.double() - pred.double()
    e = d.abs() if kind == "l1" else d * d
    simple = e.flatten(1).mean(1)
    lv = logvar.double()[t]
    return torch.stack([simple, simple / lv.exp() + lv, lvlb.double()[t] * simple]), e.flatten(1).mean(1)


def check_loss(out, pred, target, kind, t, logvar, lvlb):
    """Per value: the fp32 difference and square cost (1 + u)^2 per term, the fp64 sum nothing visible, and each fp32
    result one more rounding, so |k - r| <= 4u r (+ the logvar / exp terms, each a few u of their own magnitude). A
    square below the fp32 normal range is rounded to the subnormal grid instead, an absolute error of at most
    2^-150 per term, so the mean carries up to 2^-149 more."""
    ref, mag = loss_ref(pred.cpu(), target.cpu(), kind, t.cpu(), logvar.cpu(), lvlb.cpu())
    out = out.cpu().double()
    lv = logvar.cpu().double()[t.cpu()]
    simple = 4 * U * mag + 2.0 ** -149
    bound = torch.stack([simple, 2 * simple / lv.exp() + 4 * U * lv.abs(), 2 * simple * lvlb.cpu().double()[t.cpu()]])
    err = (out - ref).abs()
    assert bool((err <= bound + 1e-300).all()), (err / bound.clamp_min(1e-300)).max()
    return float((err / bound.clamp_min(1e-300)).max())


NS = sorted({1, 7, 1023, 4097} | {G["members"][n]["x_start"][0].numel() for n in G["members"]} | {4 * 64 * 64})


@pytest.mark.parametrize("kind", ["l1", "l2"])
@pytest.mark.parametrize("n", NS)
def test_diffusion_loss_vs_fp64(cuda_dev, kind, n):
    g = torch.Generator().manual_seed(n)
    logvar = (torch.randn(1000, generator=g) * 0.5).to(cuda_dev)
    lvlb = torch.rand(1000, generator=g).to(cuda_dev)
    for nb in (1, 2, 5, 64):
        pred = torch.randn(nb, n, generator=g).to(cuda_dev)
        target = torch.randn(nb, n, generator=g).to(cuda_dev)
        t = torch.randint(0, 1000, (nb,), generator=g).to(cuda_dev)
        out = ops.diffusion_loss(pred, target, kind, t, logvar, lvlb)
        check_loss(out, pred, target, kind, t, logvar, lvlb)


@pytest.mark.parametrize("kind", ["l1", "l2"])
def test_diffusion_loss_large_and_cancelling(cuda_dev, kind):
    g = torch.Generator().manual_seed(3)
    n, nb = 5000, 6
    base = torch.randn(nb, n, generator=g) * 1e15 if kind == "l1" else torch.randn(nb, n, generator=g) * 1e17
    cases = [
        (base, base * (1 + 1e-6)),                                    # large magnitudes
        (base, base.clone()),                                         # exact cancellation: 0
        (torch.full((nb, n), 1.0), torch.full((nb, n), 1.0) + torch.randn(nb, n, generator=g) * 1e-7),
        (torch.randn(nb, n, generator=g) * 1e-20, torch.zeros(nb, n)),  # tiny
    ]
    logvar, lvlb = torch.zeros(1000, device=cuda_dev), torch.ones(1000, device=cuda_dev)
    t = torch.arange(nb, device=cuda_dev)
    for p, q in cases:
        p, q = p.float().to(cuda_dev), q.float().to(cuda_dev)
        out = ops.diffusion_loss(p, q, kind, t, logvar, lvlb)
        assert bool(torch.isfinite(out).all())
        check_loss(out, p, q, kind, t, logvar, lvlb)
    out = ops.diffusion_loss(cases[1][0].float().to(cuda_dev), cases[1][1].float().to(cuda_dev), kind, t, logvar, lvlb)
    assert bool((out == 0).all())


@pytest.mark.parametrize("kind", ["l1", "l2"])
def test_diffusion_loss_deterministic_and_batch_independent(cuda_dev, kind):
    g = torch.Generator().manual_seed(9)
    n, nb = 16384, 32
    pred = torch.randn(nb, 4, 64, 64, generator=g).to(cuda_dev)
    target = torch.randn(nb, 4, 64, 64, generator=g).to(cuda_dev)
    t = torch.randint(0, 1000, (nb,), generator=g).to(cuda_dev)
    logvar = torch.randn(1000, generator=g).to(cuda_dev)
    lvlb = torch.rand(1000, generator=g).to(cuda_dev)
    out = ops.diffusion_loss(pred, target, kind, t, logvar, lvlb)
    for _ in range(3):
        assert torch.equal(ops.diffusion_loss(pred, target, kind, t, logvar, lvlb), out)
    for b in (0, 7, nb - 1):
        alone = ops.diffusion_loss(pred[b:b + 1].contiguous(), target[b:b + 1].contiguous(), kind, t[b:b + 1].contiguous(),
                                   logvar, lvlb)
        assert torch.equal(alone[:, 0], out[:, b])
    mixed = torch.cat([pred[5:9], torch.randn(3, 4, 64, 64, generator=g).to(cuda_dev)])
    tm = torch.cat([t[5:9], t[:3]])
    other = ops.diffusion_loss(mixed, torch.cat([target[5:9], target[:3]]), kind, tm, logvar, lvlb)
    assert torch.equal(other[:, :4], out[:, 5:9])
    assert n == pred[0].numel()


# ------------------------------------------------------------------------------------------------ p_losses
@pytest.mark.parametrize("name", sorted(G["members"]))
def test_p_losses_vs_reference(cuda_dev, name):
    """The engine's loss_dict against the reference's, within the bound its own eps error implies: for l2,
    |mean(a^2) - mean(b^2)| <= (2 ||b|| ||a - b|| + ||a - b||^2) / N with a - b = delta eps and b = eps_ref - noise;
    for l1, |mean|a| - mean|b|| <= ||a - b|| / sqrt(N). vlb weighs each sample by at most max lvlb_weights[t]."""
    m = G["members"][name]
    ld = build(name, cuda_dev)
    dev = lambda v: v.to(cuda_dev) if torch.is_tensor(v) else v
    t, noise = m["t"].to(cuda_dev), m["noise"].to(cuda_dev)
    eps = ld.apply_model(m["x_noisy"].to(cuda_dev), t, dev(m["cond"])).cpu()
    loss, d = ld.p_losses(m["x_start"].to(cuda_dev), dev(m["cond"]), t, noise=noise)
    assert list(d) == list(KEYS) and torch.equal(loss, d["val/loss"])
    de = (eps.double() - m["model_output"].double())
    N = de.numel()
    if ld.loss_type == "l2":
        b = m["model_output"].double() - m["noise"].double()
        bound = (2 * b.norm() * de.norm() + de.norm() ** 2) / N
    else:
        bound = de.norm() / math.sqrt(N)
    bound = float(bound) + 8 * U * float(m["loss_dict"]["val/loss_simple"])
    wmax = float(m["lvlb_weights"][m["t"]].max())
    for k, scale in zip(KEYS, (1.0, wmax, 1.0)):
        err = abs(float(d[k]) - float(m["loss_dict"][k]))
        assert err <= scale * bound, (k, err, scale * bound)
    print(f"{name}: eps rel-L2 {rel_l2(eps, m['model_output']):.2e}, |dloss| "
          f"{abs(float(d['val/loss']) - float(m['loss_dict']['val/loss'])):.2e} <= {bound:.2e}")
    ld.train()
    _, dt = ld.p_losses(m["x_start"].to(cuda_dev), dev(m["cond"]), t, noise=noise)
    assert list(dt) == [k.replace("val/", "train/") for k in KEYS]


@pytest.mark.parametrize("name", ["lsun", "cin", "semantic", "bsr"])
def test_get_input_vs_reference(cuda_dev, name):
    m = G["members"][name]
    ld = build(name, cuda_dev)
    torch.manual_seed(G["get_input_seed"])
    z, c = ld.get_input(batch_of(name), ld.first_stage_key)
    assert rel_l2(z, m["get_input_z"]) < 5e-3, rel_l2(z, m["get_input_z"])
    if name == "lsun":
        assert c is None
        return
    key = ld.cond_stage_key
    if key != "class_label":                  # an image-like key: the batch entry in NCHW, as DDPM.get_input makes it
        assert torch.equal(c.cpu(), batch_of(name)[key].permute(0, 3, 1, 2))
    c_enc = ld.get_learned_conditioning(c) if ld.cond_stage_trainable else c
    assert rel_l2(c_enc, m["get_input_c_enc"]) < 1e-5


def test_validation_step_keys_and_ema(cuda_dev):
    ld = build("lsun", cuda_dev, ema_seed=31)
    out = ld.validation_step(batch_of("lsun"), 0)
    assert list(out) == list(KEYS) + [k + "_ema" for k in KEYS]
    assert all(math.isfinite(float(v)) for v in out.values())
    m = G["members"]["lsun"]
    args = (m["x_start"].to(cuda_dev), None, m["t"].to(cuda_dev))
    noise = m["noise"].to(cuda_dev)
    raw = ld.p_losses(*args, noise=noise)[1]
    with ld.ema_scope():
        ema = ld.p_losses(*args, noise=noise)[1]
    assert all(float(raw[k]) != float(ema[k]) for k in KEYS)
    same = build("lsun", cuda_dev)                          # no EMA set: ema_scope keeps the raw weights
    raw2 = same.p_losses(*args, noise=noise)[1]
    with same.ema_scope():
        ema2 = same.p_losses(*args, noise=noise)[1]
    assert all(torch.equal(raw2[k], ema2[k]) for k in KEYS)
    assert all(torch.equal(raw2[k], raw[k]) for k in KEYS)


def test_forward_draws_one_t_per_sample(cuda_dev):
    ld = build("cin", cuda_dev)
    torch.manual_seed(0)
    z, c = ld.get_input(batch_of("cin"), "image")
    loss, d = ld(z, c)                                        # cond_stage_trainable: c is the batch, encoded here
    assert math.isfinite(float(loss)) and list(d) == list(KEYS)
    assert float(ld.get_loss(z, z)) == 0.0


# ------------------------------------------------------------------------------------------------ eval_loss.py
def test_eval_loss_script_both_modes(cuda_dev, tmp_path):
    import yaml
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import eval_loss
    node = {**G["members"]["lsun"]["node"]}
    cfg = tmp_path / "tiny.yaml"
    cfg.write_text(yaml.safe_dump({"model": node}))
    out = tmp_path / "random_t.json"
    eval_loss.main(["--config", str(cfg), "--random_init", "--n_samples", "6", "--batch_size", "4", "--out", str(out)])
    res = json.loads(out.read_text())
    assert set(res["loss"]) == set(KEYS) | {k + "_ema" for k in KEYS}
    assert all(math.isfinite(v) for v in res["loss"].values()) and res["n_samples"] == 6
    out2 = tmp_path / "per_t.json"
    eval_loss.main(["--config", str(cfg), "--random_init", "--n_samples", "3", "--batch_size", "2",
                    "--timesteps", "0,250,999", "--out", str(out2)])
    rows = json.loads(out2.read_text())["per_t"]
    assert [r["t"] for r in rows] == [0, 250, 999]
    assert all(math.isfinite(r[k]) for r in rows for k in ("loss_simple", "loss_simple_ema", "loss_vlb", "loss_vlb_ema"))
