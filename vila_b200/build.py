"""In-tree build of libvila_b200.so (sm_90a, H100) with nvcc.

`python -m vila_b200.build` or `__graft_entry__.build()`.  The .so and the object files are
git-ignored build products; nothing is JIT-compiled at run time.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
OBJ_DIR = ROOT / "_build"
LIB = ROOT / "libvila_b200.so"

SOURCES = [
    "host.cu",
    "api.cu",
    "gemm_wgmma.cu",
    "fmha_wgmma.cu",
    "norm.cu",
    "data_movement.cu",
    "decode.cu",
    "gemv_tma.cu",
    "kv_fp8.cu",
    "sample.cu",
    "prefix_hash.cu",
    "penalties.cu",
    "logprobs_row.cu",
    "token_bitmask.cu",
    "pdl_test.cu",
]
HEADERS = ["common.cuh", "wgmma.cuh", "kernels.h", "../../include/vila_b200.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: vila_b200 needs the CUDA 12.9 toolkit to build")


def _digest() -> str:
    h = hashlib.sha256()
    for name in SOURCES + HEADERS:
        h.update((CSRC / name).read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    stamp = OBJ_DIR / "stamp.txt"
    digest = _digest()
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB
    OBJ_DIR.mkdir(exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: str) -> Path:
        obj = OBJ_DIR / (Path(src).stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        (OBJ_DIR / (Path(src).stem + ".ptxas.log")).write_text(res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{res.stderr[-8000:]}")
        if verbose:
            print(res.stderr, file=sys.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    link = [nvcc, "-shared", "-o", str(LIB), *map(str, objs),
            "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    res = subprocess.run(link, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stderr[-4000:]}")
    stamp.write_text(digest)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
