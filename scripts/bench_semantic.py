#!/usr/bin/env python
"""LDM semantic-synthesis speed on the H100 engine, on seeded random weights and seeded Voronoi label maps:
  (a) SS256: 256x256 maps, batch 8, DDIM-200 (log_images' defaults, eta 1), cond stage + sampling + decode_first_stage;
  (b) a 512x1024 landscape with the 512 config (the same weights and keys), batch 1, the same sampler.
Also reports, with CUDA events: one graph-replayed UNet evaluation per workload with its TFLOP from the layer shapes and
TFLOP/s; the decode; and the fused label kernel (sdb_seg_labels_rescale) against the torch path it replaces
(F.one_hot -> float -> 2 x F.interpolate -> conv2d) at 256x256 and 1024x2048. Prints one JSON line with the card name and
power limit read in the same run.

  python scripts/bench_semantic.py --repeats 2 --out outputs/semantic.json
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
from sdb200 import arch, ops  # noqa: E402
from sdb200.samplers import DDIMSampler  # noqa: E402
from measure import card, emit, event_ms, unet_flops, wall_s  # noqa: E402
import semantic_oracle as SO  # noqa: E402


def run_workload(S, m, maps, steps, repeats):
    """Wall time per run (synchronised) of cond + DDIM + decode over `repeats` runs after one short warm-up run."""
    sampler = DDIMSampler(m)
    with m.ema_scope():
        S.synthesize(m, sampler, maps, steps=2)        # warm-up: autotune, graph capture, decoder
        torch.cuda.synchronize()
        times, (x, c, s) = wall_s(lambda: S.synthesize(m, sampler, maps, steps=steps, eta=1.0, return_latents=True),
                                  repeats)
    assert bool(torch.isfinite(x).all())
    return times, c, s


def unet_eval(m, c, dev):
    u = m.model.diffusion_model
    nb, _, h, w = c.shape
    g = torch.Generator(device=dev).manual_seed(1)
    xt = torch.randn(nb, 3, h, w, generator=g, device=dev)
    t = torch.linspace(1, 981, nb, device=dev).round()
    ms = event_ms(lambda: u(xt, t, concat=c), 10, warmup=2)
    fl = unet_flops(arch.SEMANTIC_SYNTHESIS_UNET, nb, h, w)
    return ms, fl


def label_kernels(m, h, w, dev):
    """(fused ms, torch ms, equal) for one map of h x w through the full cond stage."""
    cs = m.cond_stage_model
    lab = torch.from_numpy(SO.voronoi_labels(h, w, 182, 7))[None].to(dev)
    wt, n = cs.W["weight"], cs.n_stages
    w4 = wt[:, :, None, None]
    fused = lambda: ops.seg_labels_rescale(lab, 182, n, wt)

    def torch_path():
        x = F.one_hot(lab.long(), 182).permute(0, 3, 1, 2).float()
        for _ in range(n):
            x = F.interpolate(x, scale_factor=0.5, mode="bilinear")
        return F.conv2d(x, w4)
    t_f, t_t = event_ms(fused, 20, warmup=2), event_ms(torch_path, 5, warmup=2)
    err = float((fused() - torch_path()).abs().max())
    return t_f, t_t, err


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=2)
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    import semantic_synthesis as S
    dev = torch.device("cuda")
    res = {}
    # (a) SS256: 8 maps of 256x256
    m = S.load_model(random_init=True)
    m.model.diffusion_model.use_cuda_graph = True
    maps = torch.stack([torch.from_numpy(SO.voronoi_labels(256, 256, 182, 100 + i)) for i in range(8)])
    times, c, s = run_workload(S, m, maps, a.steps, a.repeats)
    ms, fl = unet_eval(m, c, dev)
    dec = event_ms(lambda: m.decode_first_stage(s), 3, warmup=2)
    res["ss256"] = dict(workload=f"semantic_synthesis256, 8 maps of 256x256, DDIM-{a.steps} eta 1, cond + sampling + "
                                 "decode, random weights", images_per_s=8 / min(times), run_s=times,
                        unet_eval_ms_graph=ms, unet_tflop=fl / 1e12, unet_tflops=fl / (ms * 1e-3) / 1e12,
                        decode_ms=dec)
    for h, w in ((256, 256), (1024, 2048)):
        t_f, t_t, err = label_kernels(m, h, w, dev)
        res[f"cond_{h}x{w}"] = dict(fused_label_kernel_ms=t_f, torch_one_hot_interpolate_conv_ms=t_t,
                                    max_abs_diff=err)
    del m, c, s
    torch.cuda.empty_cache()
    # (b) a 512x1024 landscape with the 512 config
    m = S.load_model(random_init=True, image_size=128)
    m.model.diffusion_model.use_cuda_graph = True
    maps = torch.from_numpy(SO.voronoi_labels(512, 1024, 182, 200))[None]
    times, c, s = run_workload(S, m, maps, a.steps, a.repeats)
    ms, fl = unet_eval(m, c, dev)
    dec = event_ms(lambda: m.decode_first_stage(s), 3, warmup=2)
    res["landscape512x1024"] = dict(workload=f"semantic_synthesis512, one 512x1024 map (latent 128x256), DDIM-{a.steps} "
                                             "eta 1, cond + sampling + decode, random weights",
                                    images_per_s=1 / min(times), run_s=times, unet_eval_ms_graph=ms,
                                    unet_tflop=fl / 1e12, unet_tflops=fl / (ms * 1e-3) / 1e12, decode_ms=dec)
    res.update(card())
    emit(res, a.out)


if __name__ == "__main__":
    main()
