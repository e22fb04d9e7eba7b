"""scripts/measure.py on the host: the UNet FLOP count every bench script reports, the JSON line they print, and that
the measurement helpers live only there (no bench script defines its own or imports another bench script)."""
import ast
import json
import os

import pytest

import helpers
from sdb200 import arch

SCRIPTS = os.path.join(helpers.ROOT, "scripts")
measure = helpers.script("measure")

# (config, batch, latent h, w, context tokens) -> FLOPs, as the bench scripts count them for their workloads
UNET_FLOPS = [
    ("INPAINTING_BIG_UNET", 1, 128, 128, 0, 1345415282688),       # bench_inpaint b1
    ("INPAINTING_BIG_UNET", 4, 128, 128, 0, 5381661130752),       # bench_inpaint b4
    ("BSR_SR_UNET", 9, 128, 128, 0, 2903019356160),               # bench_superres, 9 tiles
    ("SEMANTIC_SYNTHESIS_UNET", 8, 64, 64, 0, 1660952772608),     # bench_semantic 256² b8
    ("SEMANTIC_SYNTHESIS_UNET", 1, 128, 256, 0, 1675985158144),   # bench_semantic 512x1024
    ("LSUN_CHURCHES_UNET", 10, 32, 32, 0, 417902592000),
    ("CELEBAHQ_UNET", 10, 64, 64, 0, 2023747747840),
    ("TEXT2IMG256_UNET", 8, 64, 64, 77, 1674767499264),           # bench_text2img256, 4 prompts guided
    ("TEXT2IMG256_UNET", 32, 64, 64, 77, 6699069997056),          # 16 prompts guided
    ("SD_V1_UNET", 2, 64, 64, 77, 1600531333120),
    ("LAION_UNET", 2, 64, 64, 77, 1600531333120),
    ("CIN256_V2_UNET", 12, 64, 64, 1, 2500944592896),
    ("CIN256_F8_UNET", 6, 32, 32, 1, 684189548544),
    ("RDM_UNET", 6, 48, 48, 1, 4162027290624),                    # bench_rdm text only
    ("RDM_UNET", 6, 48, 48, 11, 4164132962304),                   # bench_rdm with 10 neighbours
]


@pytest.mark.parametrize("name,nb,h,w,n_ctx,flops", UNET_FLOPS)
def test_unet_flops(name, nb, h, w, n_ctx, flops):
    assert measure.unet_flops(getattr(arch, name), nb, h, w, n_ctx) == flops


def test_unet_flops_rejects_unknown_layer_kind(monkeypatch):
    plan = arch.unet_plan(arch.TINY_UNET)
    plan["middle"] = plan["middle"] + [("mystery", "middle_block.3", dict(ch=64))]
    monkeypatch.setattr(measure.arch, "unet_plan", lambda cfg: plan)
    with pytest.raises(ValueError, match="mystery"):
        measure.unet_flops(arch.TINY_UNET, 1, 16, 16)


def test_emit_prints_and_writes_one_line(tmp_path, capsys):
    res = {"images_per_s": 2.5, "run_s": [0.4, 0.41], "gpu": "H100"}
    out = tmp_path / "sub" / "r.json"
    measure.emit(res, str(out))
    assert capsys.readouterr().out == json.dumps(res) + "\n"
    assert out.read_text() == json.dumps(res) + "\n"


def _scripts():
    for f in sorted(os.listdir(SCRIPTS)):
        if f.endswith(".py"):
            with open(os.path.join(SCRIPTS, f)) as fh:
                yield f, fh.read()


def test_measurement_helpers_live_only_in_measure():
    helper_names = {"unet_flops", "gpu_info", "card", "timed", "event_ms", "unet_ms"}
    bad = []
    for f, src in _scripts():
        tree = ast.parse(src, f)
        for node in ast.walk(tree):
            if isinstance(node, ast.Import):
                mods = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom):
                mods = [node.module or ""]
            else:
                mods = []
            if f.startswith("bench_"):
                bad += [f"{f} imports {m}" for m in mods if m.split(".")[0].startswith("bench_")]
            if f == "measure.py":
                continue
            if isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef)) and node.name in helper_names:
                bad.append(f"{f} defines {node.name}")
            if isinstance(node, ast.Constant) and isinstance(node.value, str) and "nvidia-smi" in node.value:
                bad.append(f"{f} queries nvidia-smi")
    assert not bad, bad
