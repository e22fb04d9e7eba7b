"""Where the attention time of one SD-v1 UNet evaluation goes (eager, (2, 4, 64, 64), ops.PROFILE event pairs): every
sdb_attention launch with its shape, time, algorithmic FLOPs, tensor floor (FLOPs / 989 TFLOP/s, the H100 SXM dense
fp16 data-sheet rate) and MUFU floor (B * heads * nq * nkv exponentials / (16 per clock per SM * SMs * SM clock)),
plus the QK and V^T projection GEMMs (the two GEMMs right before each self-attention launch).

usage: python scripts/attn_breakdown.py [reps]"""
import collections
import statistics
import sys

import torch

sys.path.insert(0, ".")
import sdb200
from sdb200 import arch, ops
from measure import card

dev = torch.device("cuda:0")
REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 7
gpu = card()
print("GPU:", ", ".join(gpu.values()))
clk = float(gpu["max_sm_clock"].split()[0]) * 1e6
sms = torch.cuda.get_device_properties(dev).multi_processor_count
net = sdb200.UNetModel(**arch.SD_V1_UNET).load_weights(
    arch.random_state_dict(arch.unet_param_shapes(arch.SD_V1_UNET), 11, device=dev), dev)
g = torch.Generator(device=dev).manual_seed(0)
x = torch.randn(2, 4, 64, 64, generator=g, device=dev)
ctx = torch.randn(2, 77, 768, generator=g, device=dev)
t = torch.full((2,), 981.0, device=dev)
net.use_cuda_graph = False
net(x, t, context=ctx)   # tile choices / module load
runs = []
for _ in range(REPS):
    ops.PROFILE = []
    net(x, t, context=ctx)
    torch.cuda.synchronize()
    runs.append(ops.PROFILE)
ops.PROFILE = None
n = len(runs[0])
us = [statistics.median(r[i][2].elapsed_time(r[i][3]) for r in runs) * 1e3 for i in range(n)]
recs = runs[0]
rows = collections.OrderedDict()
proj_us = 0.0
print(f"{'B':>2} {'H':>3} {'nq':>5} {'nkv':>5} {'d':>4} |     us   GFLOP  TF/s  tensor_us  mufu_us")
for i, (kind, fl, _, _, shp) in enumerate(recs):
    if kind != "attention":
        continue
    B, H, nq, nkv, d = shp
    tens = fl / 989e12 * 1e6
    mufu = B * H * nq * nkv / (16.0 * sms * clk) * 1e6
    print(f"{B:2d} {H:3d} {nq:5d} {nkv:5d} {d:4d} | {us[i]:6.1f} {fl / 1e9:7.2f} {fl / us[i] / 1e6:5.0f} {tens:10.1f} "
          f"{mufu:8.1f}")
    e = rows.setdefault(shp, [0, 0.0, 0.0, 0.0])
    e[0] += 1
    e[1] += us[i]
    e[2] += tens
    e[3] += mufu
    if nq == nkv:
        proj_us += sum(us[j] for j in range(i - 2, i) if recs[j][0] == "gemm")
print("by shape:")
for shp, e in rows.items():
    print(f"  {shp}: n={e[0]}  {e[1]:8.1f} us  tensor floor {e[2]:6.1f} us  MUFU floor {e[3]:6.1f} us")
lvl1 = sum(e[1] for shp, e in rows.items() if shp[2] == shp[3] == 4096)
print(f"level-1 self-attention (nq = nkv = 4096): {lvl1:.1f} us per evaluation")
print(f"all attention: {sum(e[1] for e in rows.values()):.1f} us; QK + V^T projection GEMMs: {proj_us:.1f} us")
