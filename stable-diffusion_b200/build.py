"""Build the sm_90a (H100) C-ABI library in-tree: stable-diffusion_b200/csrc/libsdb200.so.

nvcc cross-compiles without a GPU. Objects are rebuilt only when a source (or header) is newer.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
LIB = CSRC / "libsdb200.so"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]
if os.environ.get("SDB_BUILD_TRACE"):   # debug build: in-kernel phase stamps (sdb_debug_trace) and SDB_DBG switches
    FLAGS.append("-DSDB_TRACE")


def _newer(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build(verbose: bool = False, force: bool = False) -> Path:
    sources = sorted(CSRC.glob("*.cu"))
    headers = sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + sorted((CSRC.parent.parent / "include").glob("*.h"))
    objs = []
    jobs = []
    for src in sources:
        obj = src.with_suffix(".o")
        objs.append(obj)
        if force or _newer(obj, [src] + headers):
            cmd = [NVCC, *FLAGS, "-c", str(src), "-o", str(obj)]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for out in ex.map(run, jobs):
                if verbose and out:
                    print(out, file=sys.stderr)
    if force or jobs or _newer(LIB, objs):
        cmd = [NVCC, "-shared", "-o", str(LIB), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a"]
        run(cmd)
    return LIB


if __name__ == "__main__":
    p = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(p)
