"""Nearest-neighbour retrieval of the retrieval-augmented diffusion model: drop-in for the `Searcher` of the reference's
scripts/knn2img.py (`search(x, k)` -> the same dict), exact search on the GPU.

The reference searches with ScaNN's `score_brute_force` searcher over the L2-normalised database embeddings by dot
product. Here the normalised rows live on the device as fp16 (half the bytes of fp32) and `ops.knn_topk`
(sdb_knn_topk) streams them once per batch of <= 64 queries: exact top-k of the fp32 dot products of the fp16 rows and
queries, ties to the lower row. The returned `nn_embeddings` are gathered from the host's fp32 rows and normalised
with the reference's numpy formula, so for the same indices the conditioning is bit-equal to the reference's.
"""
from __future__ import annotations

import glob
import os
import time

import numpy as np
import torch

from . import ops

# scripts/knn2img.py DATABASES
DATABASES = [
    "openimages",
    "artbench-art_nouveau",
    "artbench-baroque",
    "artbench-expressionism",
    "artbench-impressionism",
    "artbench-post_impressionism",
    "artbench-realism",
    "artbench-romanticism",
    "artbench-renaissance",
    "artbench-surrealism",
    "artbench-ukiyo_e",
]
KEYS = ("embedding", "img_id", "patch_coords")
UPLOAD_ROWS = 1 << 18   # rows normalised and uploaded per step (bounds the host's fp32 temporary)


def database_path(name, root="."):
    """The directory the reference reads a database from (knn2img.py Searcher.database_path)."""
    return os.path.join(root, "data", "rdm", "retrieval_databases", name)


def load_database(path):
    """The `.npz` files of a database directory, concatenated in sorted file-name order: {key: array} for `embedding`
    [N, dim], `img_id` and `patch_coords`."""
    files = sorted(glob.glob(os.path.join(path, "*.npz")))
    if not files:
        raise ValueError(f'No npz-files in specified path "{path}" is this directory existing?')
    parts = {k: [] for k in KEYS}
    for f in files:
        with np.load(f) as d:
            for k in KEYS:
                parts[k].append(d[k])
    return {k: v[0] if len(v) == 1 else np.concatenate(v, axis=0) for k, v in parts.items()}


def normalize_rows(x):
    """The reference's normalisation (knn2img.py:80-81, 143, 153): x / ||x|| per row, numpy."""
    return x / np.linalg.norm(x, axis=-1)[..., np.newaxis]


class Searcher:
    """`Searcher(database)` loads `data/rdm/retrieval_databases/<database>/*.npz` (or `path`) and uploads the normalised
    embeddings to `device` as fp16; `search(x, k)` returns the reference's dict. A database larger than the device's
    free memory is an error that states both sizes."""

    def __init__(self, database, device="cuda", path=None, root="."):
        if path is None:
            assert database in DATABASES, f"unknown database {database!r} (one of {DATABASES})"
            path = database_path(database, root)
        self.database_name = database
        self.database_path = path
        self.device = torch.device(device)
        self.database = load_database(path)
        emb = self.database["embedding"]
        n, dim = emb.shape
        need = n * dim * 2
        free, _ = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise MemoryError(f"retrieval database {path!r}: {n} x {dim} fp16 rows need {need / 2**30:.2f} GiB on the "
                              f"device, {free / 2**30:.2f} GiB free (databases larger than device memory are not "
                              "supported)")
        self.db = torch.empty((n, dim), dtype=torch.float16, device=self.device)
        for i in range(0, n, UPLOAD_ROWS):
            rows = normalize_rows(emb[i:i + UPLOAD_ROWS]).astype(np.float16)
            self.db[i:i + UPLOAD_ROWS].copy_(torch.from_numpy(rows))

    def __len__(self):
        return self.db.shape[0]

    def search_rows(self, q, k):
        """Top-k rows of normalised queries q (numpy [B, dim]) on the device: (indices int64 [B, k], scores fp32)."""
        q16 = torch.from_numpy(np.ascontiguousarray(q, dtype=np.float32)).to(self.device).half()
        idx, scores = [], []
        for i in range(0, q16.shape[0], ops.KNN_MAX_QUERIES):
            s, r = ops.knn_topk(self.db, q16[i:i + ops.KNN_MAX_QUERIES].contiguous(), k)
            idx.append(r)
            scores.append(s)
        return torch.cat(idx).cpu().numpy(), torch.cat(scores).cpu().numpy()

    def search(self, x, k):
        if isinstance(x, torch.Tensor):
            x = x.detach().cpu().numpy()
        if len(x.shape) == 3:
            x = x[:, 0]
        query_embeddings = normalize_rows(x)
        start = time.time()
        nns, _ = self.search_rows(query_embeddings, k)
        end = time.time()
        out_embeddings = self.database["embedding"][nns]
        return {"nn_embeddings": normalize_rows(out_embeddings),
                "img_ids": self.database["img_id"][nns],
                "patch_coords": self.database["patch_coords"][nns],
                "queries": x,
                "exec_time": end - start,
                "nns": nns,
                "q_embeddings": query_embeddings}

    def __call__(self, x, n):
        return self.search(x, n)
