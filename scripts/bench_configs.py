"""Timings of the other BASELINE.json configurations on one H100 (not the headline bench line):
C3 txt2img DDIM-50 batch 32, C4-per-GPU txt2img PLMS-50 batch 8, C5 img2img 768x768 strength 0.75 batch 4."""
import json, sys, torch
sys.path.insert(0, ".")
import sdb200
from sdb200 import pipeline
from measure import emit, event_ms

dev = torch.device("cuda:0")
model = pipeline.build_model()
pipeline.load_random_weights(model, dev, gen_device=dev)

def ids(n, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, 49406, (n, 77), generator=g); t[:, 0] = 49406; t[:, 20:] = 49407
    u = torch.full((n, 77), 49407, dtype=torch.long); u[:, 0] = 49406
    return t.to(dev), u.to(dev)

out = {}
which = sys.argv[1:] or ["c4", "c3", "c5"]
if "c4" in which:
    B = 8
    p = pipeline.Txt2Img(model, sampler="plms", steps=50, scale=7.5)
    i, u = ids(B, 1); xT = sdb200.dist.batch_noise(0, B, (4, 64, 64)).to(dev)
    ms = event_ms(lambda: p(i, u, x_T=xT), 2, warmup=1)
    out["C4_per_gpu_txt2img_plms50_b8"] = {"ms_per_batch": ms, "images_per_s": B / ms * 1e3}
    print(out, flush=True)
if "c3" in which:
    B = 32
    p = pipeline.Txt2Img(model, sampler="ddim", steps=50, scale=7.5)
    i, u = ids(B, 2); xT = sdb200.dist.batch_noise(0, B, (4, 64, 64)).to(dev)
    ms = event_ms(lambda: p(i, u, x_T=xT), 1, warmup=1)
    out["C3_txt2img_ddim50_b32"] = {"ms_per_batch": ms, "images_per_s": B / ms * 1e3,
                                    "achieved_tflops": B * 82.84 / (ms * 1e-3)}
    print(out, flush=True)
if "c5" in which:
    B = 4
    p = pipeline.Img2Img(model, steps=50, scale=5.0, strength=0.75)
    i, u = ids(B, 3)
    init = torch.rand(B, 3, 768, 768, generator=torch.Generator().manual_seed(0)).to(dev) * 2 - 1
    ms = event_ms(lambda: p(init, i, u), 1, warmup=1)
    out["C5_img2img_768_b4"] = {"ms_per_batch": ms, "images_per_s": B / ms * 1e3, "achieved_tflops": B * 167.6 / (ms * 1e-3)}
import os
os.makedirs("gpurun_out", exist_ok=True)
meta = {"gpu": torch.cuda.get_device_name(0), "weights": "random-init SD-v1 (seeded)", "timing": "CUDA events around the public "
        "pipeline call (CLIP encode -> sampler loop -> VAE decode [-> uint8]), inputs resident in HBM, 1 warm-up call"}
for key, tag in (("C3_txt2img_ddim50_b32", "r02_c3"), ("C4_per_gpu_txt2img_plms50_b8", "r02_c4_per_gpu"), ("C5_img2img_768_b4", "r02_c5")):
    if key in out:
        json.dump({"config": key, **out[key], **meta}, open(f"gpurun_out/{tag}.json", "w"), indent=1)
emit(out)
