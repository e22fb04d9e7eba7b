#!/usr/bin/env python
"""Retrieval-augmented diffusion sampling speed on the H100 engine: the reference workload of scripts/knn2img.py (768²,
DDIM-50, eta 0, scale 5.0, batch 3, CLIP text encode, decode_first_stage included) on seeded random weights, text-only
and with --knn 10 neighbours from a seeded synthetic database (search included). Also reports one graph-replayed UNet
evaluation at the guided batch with the 11-token context (CUDA events) with its FLOPs from the layer shapes, and the
k-NN search kernel alone at N = 1 M, 4 M and 16 M rows of 768 (fp16): time and the database bytes streamed per second
against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s). Prints one JSON line with the card name and power limit read
in the same run.

  python scripts/bench_rdm.py --out outputs/rdm.json
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sdb200 import arch, ops, retrieval  # noqa: E402
from measure import card, emit, event_ms, unet_flops, wall_s  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def synthetic_searcher(n, dim, dev, seed=0):
    """A Searcher over n seeded rows, built in memory (no .npz files)."""
    g = torch.Generator().manual_seed(seed)
    s = object.__new__(retrieval.Searcher)
    emb = torch.randn((n, dim), generator=g).numpy()
    s.database = {"embedding": emb, "img_id": torch.arange(n).numpy(), "patch_coords": torch.zeros(n, 4).numpy()}
    s.device = dev
    s.db = torch.from_numpy(retrieval.normalize_rows(emb)).to(dev).half()
    return s


def time_search(n, dim, b, k, dev, reps=20):
    db = torch.empty((n, dim), device=dev, dtype=torch.float16)
    g = torch.Generator(device=dev).manual_seed(n)
    for i in range(0, n, 1 << 20):       # unit rows, 1 M at a time (no fp32 copy of the whole database)
        x = torch.randn((min(1 << 20, n - i), dim), device=dev, generator=g)
        db[i:i + x.shape[0]] = (x / x.norm(dim=1, keepdim=True)).half()
    q = torch.randn((b, dim), device=dev, generator=g)
    q = (q / q.norm(dim=1, keepdim=True)).half()
    ms = event_ms(lambda: ops.knn_topk(db, q, k), reps, warmup=3)
    del db
    torch.cuda.empty_cache()
    gbs = n * dim * 2 / (ms * 1e-3) / 1e9
    return dict(rows=n, dim=dim, queries=b, k=k, ms=round(ms, 3), gb_per_s=round(gbs, 1),
                share_of_hbm_peak=round(gbs * 1e9 / HBM_BYTES_PER_S, 3))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--db_rows", type=int, default=200000, help="rows of the synthetic database of the --knn workload")
    p.add_argument("--out", type=str, default=None)
    a = p.parse_args()
    import knn2img as K
    dev = torch.device("cuda")
    m = K.load_model(random_init=True, device=dev)
    u = m.model.diffusion_model
    u.use_cuda_graph = True
    clip = K.load_clip(random_init=True, device=dev)
    ids = torch.zeros((3, 77), dtype=torch.long)
    ids[:, 0], ids[:, 1:9], ids[:, 9] = 49406, torch.arange(400, 408), 49407
    ids = ids.to(dev)

    class Ids:   # the prompt batch as token ids: no vocabulary in the benchmark
        def encode(self, _):
            return clip.encode(ids)

    searcher = synthetic_searcher(a.db_rows, 768, dev)
    res = dict(workload=f"knn2img 768², DDIM-{a.steps} eta 0, scale 5.0, batch 3 (UNet batch 6 at 48x48x16), CLIP text "
                        f"encode, decode_first_stage, random weights", **card())
    for tag, s, k in (("text_only", None, 0), ("knn10", searcher, 10)):
        torch.manual_seed(0)
        K.sample(m, Ids(), ["p"] * 3, s, max(k, 1), ddim_steps=a.steps)   # warm-up: autotune, graph capture
        torch.cuda.synchronize()
        times, (img, c) = wall_s(lambda: K.sample(m, Ids(), ["p"] * 3, s, max(k, 1), ddim_steps=a.steps), a.repeats)
        assert img.shape == (3, 3, 768, 768) and bool(torch.isfinite(img).all()) and c.shape[1] == 1 + k
        res[f"images_per_s_{tag}"] = 3 / min(times)
        res[f"run_s_{tag}"] = times
    # one UNet evaluation at the guided batch with the 11-token context
    x = torch.randn(6, 16, 48, 48, device=dev)
    t = torch.full((6,), 501.0, device=dev)
    c = torch.randn(6, 11, 768, device=dev)
    unet_ms = event_ms(lambda: u(x, t, context=c), 30, warmup=5)
    flops = unet_flops(arch.RDM_UNET, 6, 48, 48, c.shape[1])
    res.update(unet_eval_ms_graph=unet_ms, unet_eval_gflop=flops / 1e9, unet_tflop_per_s=flops / (unet_ms * 1e-3) / 1e12)
    del m, u, clip, searcher, x, c
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    res["search_kernel"] = [time_search(n, 768, 3, 10, dev) for n in (1 << 20, 4 << 20, 16 << 20)]
    res["search_kernel"].append(time_search(16 << 20, 768, 64, 64, dev))
    emit(res, a.out)


if __name__ == "__main__":
    main()
