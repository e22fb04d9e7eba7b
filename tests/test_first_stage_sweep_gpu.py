"""The fp64 kernel sweeps over the nine first-stage autoencoders of arch.FIRST_STAGES (workloads.FIRST_STAGE_WORKLOADS:
encode, decode at a scale and, for VQ, decode_code, at 256², 256x384 batch 2 and the thin f x 8f with its 1 x 8 latent),
and the norm and elementwise sweeps over text2img256 (BERT-640, its UNet and a VQ-f4 decode). Each test reuses one sweep
file's recording signatures and run_sweep, and the PDL file's weight audit:
  - every GEMM problem with every tile plan (test_gemm_plans_gpu.py);
  - every GroupNorm / LayerNorm / softmax launch (test_norm_sweep_gpu.py);
  - every attention launch (test_attention_sweep_gpu.py);
  - every layout, 1x1 head and quantizer launch (test_elementwise_sweep_gpu.py);
  - every operand read before griddepcontrol.wait lies in packed weights (test_pdl_order_gpu.py).
Each test also asserts that its workload reached the paths it exists for, so that a change to a builder cannot drop one
quietly. text2img256's GEMM and attention sweeps are in test_text2img256_gpu.py."""
import time
from collections import defaultdict

import pytest
import torch

import helpers  # noqa: F401
import test_attention_sweep_gpu as AS
import test_elementwise_sweep_gpu as ES
import test_gemm_plans_gpu as GP
import test_norm_sweep_gpu as NS
from sweeps import record
from test_pdl_order_gpu import audit_workload
from workloads import DECODE_SCALE, FIRST_STAGE_WORKLOADS, first_stage_geometries, text2img256
from sdb200 import arch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
NAMES = list(FIRST_STAGE_WORKLOADS)
WITH_T2I = {**FIRST_STAGE_WORKLOADS, "text2img256": text2img256}


def _factor(name):
    return 2 ** (len(arch.FIRST_STAGES[name]["ddconfig"]["ch_mult"]) - 1)


def _has_attention(name):
    return arch.FIRST_STAGES[name]["ddconfig"].get("attn_type", "vanilla") != "none"


@pytest.mark.parametrize("name", NAMES)
def test_every_plan_of_every_first_stage_gemm_problem(cuda_dev, name):
    """Every geometry runs the Downsample's stride-2 conv down to a 1 x 8 output (input 2 x 16); KL-f32's decoder feeds
    its 64-channel latent to the implicit-GEMM conv in fp16."""
    problems = GP.catalogue(FIRST_STAGE_WORKLOADS[name], cuda_dev)
    one_row = [p for p in problems if p["taps"] == 9 and p["conv_stride"] == 2 and p["geo"] == (1, 2, 16)]
    assert one_row, "no stride-2 conv down to a single output row"
    if name == "kl-f32":
        assert any(p["taps"] == 9 and p["conv_stride"] == 1 and p["chans"] == (64,) for p in problems)
    print(f"\n{name}: {len(problems)} distinct GEMM problems")
    GP.run_sweep(problems, cuda_dev, name)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(WITH_T2I))
def test_every_norm_launch_of_every_first_stage(cuda_dev, name):
    """GroupNorm over 512 channels down to 8 pixels (the thin latent) in every first stage; text2img256's LayerNorm at
    BERT-640's width."""
    calls, problems = record(WITH_T2I[name], cuda_dev, NS.SIGS)
    kinds = defaultdict(int)
    for p in problems:
        kinds[p["kind"]] += 1
    print(f"\n{name}: {calls} calls, {len(problems)} distinct problems ({dict(kinds)})")
    if name == "text2img256":
        assert any(p["kind"] == "ln" and p["c"] == 640 for p in problems)
    else:
        assert any(p["kind"] == "gn" and p["h"] * p["w"] == 8 and p["c0"] + p["c1"] == 512 for p in problems)
    NS.run_sweep(problems, name)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", NAMES)
def test_every_attention_launch_of_every_first_stage(cuda_dev, name):
    """The d = 512 attention (mid block and level attention) at each geometry: 8 tokens at the thin latent; KL-f32's
    level attention also at 2 x 16 and 1 x 8. vq-f4-noattn has none."""
    calls, problems = record(FIRST_STAGE_WORKLOADS[name], cuda_dev, {"attention": AS._attn_sig})
    got = sorted({(p["B"], p["nq"], p["nkv"], p["d"]) for p in problems})
    print(f"\n{name}: {calls} attention calls, {len(problems)} distinct problems: {got}")
    if not _has_attention(name):
        assert not problems
        return
    f = _factor(name)
    for nb, h, w in first_stage_geometries(f):
        n = h // f * (w // f)
        assert (nb, n, n, 512) in got, (nb, n)                         # the mid-block attention on the latent
    assert (1, 8, 8, 512) in got
    if name == "kl-f32":
        assert (1, 32, 32, 512) in got                                # level attention at 2 x 16
    AS.run_sweep(problems, name)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(WITH_T2I))
def test_every_elementwise_launch_of_every_first_stage(cuda_dev, name):
    """Layouts, casts, im2col, upsampling, the 1x1 heads and the quantizer: kl-f32's heads at 128 -> 128 and 64 -> 64;
    vq-f16's 16384 x 8 codebook and vq-f8-n256's 256 x 4, each with and without indices and at the decode scale."""
    calls, problems = record(WITH_T2I[name], cuda_dev, ES.SIGS)
    ops_ = defaultdict(int)
    for p in problems:
        ops_[p["op"]] += 1
    print(f"\n{name}: {calls} calls, {len(problems)} distinct problems ({dict(ops_)})")
    pw = {(p["cin"], p["cout"]) for p in problems if p["op"] == "pointwise_small"}
    vq = {(p["e_dim"], p["n_e"], p["idx"], p["scale"]) for p in problems if p["op"] == "vq_quantize"}
    if name == "kl-f32":
        assert {(128, 128), (64, 64)} <= pw, pw
    cfg = arch.FIRST_STAGES.get(name, {})
    if "n_embed" in cfg:
        e, n = cfg["embed_dim"], cfg["n_embed"]
        assert {(e, n, True, 1.0), (e, n, False, DECODE_SCALE)} <= vq, vq
    if name == "vq-f16":
        assert (8, 16384) in {v[:2] for v in vq}
    if name == "vq-f8-n256":
        assert (4, 256) in {v[:2] for v in vq}
    ES.run_sweep(problems, name)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(WITH_T2I))
def test_first_stage_pre_wait_operands_are_packed_weights(cuda_dev, name):
    """The weight audit of test_pdl_order_gpu.py on the encoders too, whose level attention (VQ-f8, KL-f16, KL-f32,
    VQ-f16) makes b_dynamic GEMMs."""
    t0 = time.time()
    bad, n = audit_workload(name, WITH_T2I[name], cuda_dev)
    print(f"\n{name}: {n} gemm / groupnorm / layernorm calls audited, {len(bad)} violations, {time.time() - t0:.1f} s")
    assert not bad, "pre-wait operands outside packed weights (workload, op, slot, shape):\n" + \
        "\n".join(map(str, sorted(set(bad))))

