"""Build a retrieval database for the retrieval-augmented model (scripts/knn2img.py) from a directory tree of images:

  python scripts/build_rdm_database.py --images <dir> --outdir <db dir> --clip_ckpt <clip-vit-large-patch14 weights>
  python scripts/knn2img.py --use_neighbors --database_dir <db dir> ...

Every image under --images (png, jpg, jpeg, webp, bmp, in sorted relative-path order) is embedded whole with
FrozenClipImageEmbedder('ViT-L/14'): bicubic resize of the whole image to 224² (aspect ratio not kept), CLIP's
normalisation and the vision tower with its projection, on the GPU. The output directory holds
  manifest.txt            one relative image path per line; line i is img_id i
  shard_NNNNNN.npz        `embedding` float32 [N, 768] (unnormalised, as encode_image returns it), `img_id` int64 [N],
                          `patch_coords` int32 [N, 4] = the whole-image box (0, 0, W, H)
which sdb200.retrieval.load_database (and so knn2img.py's Searcher) reads in sorted file order. Shard k holds manifest
rows [k * shard_size, (k + 1) * shard_size).

Images are decoded to RGB uint8 on a pool of host processes; each batch is packed into one of two pinned buffers and
uploaded on a copy stream while the GPU embeds the previous batch, and one launch preprocesses the whole ragged batch.
A shard is written to a temporary name and renamed when complete, so --resume (which requires the same image list)
skips complete shards and redoes the rest. Without --resume an output directory that already holds a database is an
error. --random_init uses seeded weights instead of --clip_ckpt (--tiny: the 64-wide test member that matches
knn2img.py --tiny). Patch-level databases (crops), ScaNN searchers and train_searcher.py are not built.
"""
import argparse
import multiprocessing as mp
import os
import sys
import time
from collections import deque

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import sdb200  # noqa: E402
from sdb200 import arch  # noqa: E402

EXTENSIONS = (".png", ".jpg", ".jpeg", ".webp", ".bmp")
MANIFEST = "manifest.txt"


# ------------------------------------------------------------------------------------------------ host logic
def list_images(root):
    """Relative paths ('/'-separated) of the image files under root, sorted."""
    out = []
    for d, dirs, files in os.walk(root):
        dirs.sort()
        for f in files:
            if f.lower().endswith(EXTENSIONS):
                out.append(os.path.relpath(os.path.join(d, f), root).replace(os.sep, "/"))
    return sorted(out)


def shard_name(k):
    return f"shard_{k:06d}.npz"


def shard_ranges(n, shard_size):
    """[(k, start, stop)] of the shards of n manifest rows."""
    return [(k, s, min(s + shard_size, n)) for k, s in enumerate(range(0, n, shard_size))]


def shard_complete(path, start, stop):
    """True when path is a readable shard holding exactly manifest rows [start, stop)."""
    try:
        with np.load(path) as d:
            ids = d["img_id"]
            return (d["embedding"].shape[0] == stop - start and d["patch_coords"].shape == (stop - start, 4)
                    and np.array_equal(ids, np.arange(start, stop, dtype=np.int64)))
    except Exception:  # noqa: BLE001 - missing, truncated or foreign file: not complete
        return False


def write_shard(path, embedding, img_id, patch_coords):
    """Write one shard under a temporary name (not *.npz, so load_database never sees it) and rename it."""
    tmp = path + ".partial"
    with open(tmp, "wb") as f:
        np.savez(f, embedding=np.asarray(embedding, dtype=np.float32), img_id=np.asarray(img_id, dtype=np.int64),
                 patch_coords=np.asarray(patch_coords, dtype=np.int32))
    os.replace(tmp, path)


def prepare_outdir(outdir, paths, resume):
    """Write (or, with resume, check) the manifest. Returns the manifest rows."""
    os.makedirs(outdir, exist_ok=True)
    mpath = os.path.join(outdir, MANIFEST)
    existing = os.path.exists(mpath) or any(f.endswith(".npz") for f in os.listdir(outdir))
    if existing and not resume:
        raise FileExistsError(f"{outdir} already holds a database: pass --resume to complete it, or another --outdir")
    if resume and os.path.exists(mpath):
        with open(mpath) as f:
            old = f.read().splitlines()
        if old != list(paths):
            raise ValueError(f"--resume: the images under --images differ from {mpath} ({len(old)} listed, "
                             f"{len(paths)} found)")
        return old
    with open(mpath + ".partial", "w") as f:
        f.write("".join(p + "\n" for p in paths))
    os.replace(mpath + ".partial", mpath)
    return list(paths)


def decode(path):
    """One image file -> RGB uint8 [H, W, 3] (runs in the decoding processes)."""
    from PIL import Image
    with Image.open(path) as im:
        return np.ascontiguousarray(np.asarray(im.convert("RGB"), dtype=np.uint8))


# ------------------------------------------------------------------------------------------------ GPU side
def load_embedder(clip_ckpt=None, random_init=False, tiny=False, device="cuda", unsafe_ckpt=False):
    """FrozenClipImageEmbedder('ViT-L/14') with its weights from a transformers CLIPModel checkpoint, or seeded."""
    cfg = arch.TINY_CLIP_VISION_PROJ if tiny else arch.CLIP_VISION_PROJ
    emb = sdb200.FrozenClipImageEmbedder("ViT-L/14", config=cfg)
    if clip_ckpt:
        sd, _ = sdb200.checkpoint.read_state_dict(clip_ckpt, allow_pickle=unsafe_ckpt)
        return emb.load_weights(sd, device)
    if not random_init:
        raise ValueError("pass --clip_ckpt (CLIP ViT-L/14 in the transformers CLIPModel layout), or --random_init")
    return emb.load_weights(arch.random_state_dict(emb.shapes, 16, device=torch.device(device)), device)


class Uploader:
    """Two pinned host buffers used in turn: a batch is packed into one while the copy of the other may still run;
    the copies go on their own stream and the compute stream waits on each copy's event."""

    def __init__(self, device):
        self.device = device
        self.stream = torch.cuda.Stream(device)
        self.bufs = [None, None]
        self.done = [None, None]
        self.slot = 0

    def upload(self, arrays):
        s = self.slot
        self.slot ^= 1
        if self.done[s] is not None:
            self.done[s].synchronize()            # the previous copy out of this buffer has finished
        n = sum(a.size for a in arrays)
        if self.bufs[s] is None or self.bufs[s].numel() < n:
            self.bufs[s] = torch.empty(max(n, 1 << 20), dtype=torch.uint8, pin_memory=True)
        host = self.bufs[s].numpy()
        off = 0
        for a in arrays:
            host[off:off + a.size] = a.reshape(-1)
            off += a.size
        with torch.cuda.stream(self.stream):
            dev = self.bufs[s][:n].to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.done[s] = ev
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(ev)
        dev.record_stream(cur)
        return dev


def build(images_root, outdir, embedder, pool, batch=256, shard_size=100000, resume=False, log=print):
    """Embed every image under images_root into shards in outdir, decoding on `pool` (a multiprocessing pool).
    Returns (rows embedded, shards written)."""
    paths = prepare_outdir(outdir, list_images(images_root), resume)
    if not paths:
        raise ValueError(f"no images ({', '.join(EXTENSIONS)}) under {images_root}")
    todo = [(k, s, e) for k, s, e in shard_ranges(len(paths), shard_size)
            if not (resume and shard_complete(os.path.join(outdir, shard_name(k)), s, e))]
    skipped = len(shard_ranges(len(paths), shard_size)) - len(todo)
    if skipped:
        log(f"--resume: {skipped} complete shard(s) kept")
    ends = {k: (s, e) for k, s, e in todo}
    batches = [(k, i, min(i + batch, e)) for k, s, e in todo for i in range(s, e, batch)]
    up = Uploader(embedder.W["device"])
    ahead = deque()
    n_rows, t0 = 0, time.time()
    parts = {}                       # shard -> [(first row, embeddings, (H, W) per image)]

    def submit(j):
        if j < len(batches):
            _, a, b = batches[j]
            ahead.append(pool.map_async(decode, [os.path.join(images_root, p) for p in paths[a:b]]))

    for j in range(3):               # decode up to three batches ahead of the GPU
        submit(j)
    pending = None
    for j in range(len(batches) + 1):
        cur = None
        if j < len(batches):
            arrays = ahead.popleft().get()
            submit(j + 3)
            hw = [(x.shape[0], x.shape[1]) for x in arrays]
            emb = embedder.encode_packed(up.upload(arrays), hw)
            host = torch.empty(emb.shape, dtype=torch.float32, pin_memory=True)
            host.copy_(emb, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            cur = (batches[j], host, ev, hw)
        if pending is not None:      # the previous batch's result, while the GPU works on this one
            (k, a, b), host, ev, hw = pending
            ev.synchronize()
            parts.setdefault(k, []).append((a, host.numpy().copy(), hw))
            n_rows += b - a
            s, e = ends[k]
            if b == e:
                _flush(outdir, k, s, e, parts.pop(k))
                log(f"{shard_name(k)}: rows {s}..{e - 1} ({n_rows} embedded, {n_rows / (time.time() - t0):.1f} img/s)")
        pending = cur
    return n_rows, len(todo)


def _flush(outdir, k, start, stop, chunks):
    chunks.sort(key=lambda c: c[0])
    emb = np.concatenate([c[1] for c in chunks], 0)
    hw = [x for c in chunks for x in c[2]]
    coords = np.array([(0, 0, w, h) for h, w in hw], dtype=np.int32)
    assert emb.shape[0] == stop - start
    write_shard(os.path.join(outdir, shard_name(k)), emb, np.arange(start, stop, dtype=np.int64), coords)


def get_parser():
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--images", type=str, required=True, help="directory tree of images")
    p.add_argument("--outdir", type=str, required=True, help="database directory (knn2img.py --database_dir)")
    p.add_argument("--batch", type=int, default=256, help="images per GPU batch")
    p.add_argument("--shard_size", type=int, default=100000, help="rows per .npz shard")
    p.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1), help="image decoding processes")
    p.add_argument("--resume", action="store_true", help="keep complete shards of an interrupted run, redo the rest")
    p.add_argument("--clip_ckpt", type=str, default=None,
                   help="CLIP ViT-L/14 weights in the transformers CLIPModel layout (.safetensors or .ckpt)")
    p.add_argument("--random_init", action="store_true", help="seeded random weights instead of --clip_ckpt")
    p.add_argument("--tiny", action="store_true", help="the small test configuration (with --random_init)")
    p.add_argument("--unsafe-ckpt", action="store_true", help="allow full unpickling of a .ckpt (runs code from the file)")
    return p


def main(argv=None):
    opt = get_parser().parse_args(argv)
    if opt.batch < 1 or opt.shard_size < 1 or opt.workers < 1:
        raise ValueError("--batch, --shard_size and --workers must be at least 1")
    if opt.tiny and not opt.random_init:
        raise ValueError("--tiny needs --random_init")
    if not os.path.isdir(opt.images):
        raise FileNotFoundError(f"--images {opt.images}: not a directory")
    # the decoding processes are forked before CUDA is initialised in this process
    with mp.get_context("fork").Pool(opt.workers) as pool:
        embedder = load_embedder(opt.clip_ckpt, opt.random_init, opt.tiny, "cuda", opt.unsafe_ckpt)
        t0 = time.time()
        n, shards = build(opt.images, opt.outdir, embedder, pool, opt.batch, opt.shard_size, opt.resume)
        dt = time.time() - t0
    print(f"{n} images embedded into {shards} shard(s) in {dt:.1f} s ({n / max(dt, 1e-9):.1f} img/s): {opt.outdir}")


if __name__ == "__main__":
    main()
