"""In-tree build of libgigaam_b200.so (sm_90a only) with nvcc.

The library is the product: the Python classes in this package only marshal pointers into it.
`build_library()` is what `__graft_entry__.build()` calls; it cross-compiles without a GPU.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
BUILD_DIR = PKG_DIR / "build"
LIB_PATH = PKG_DIR / "libgigaam_b200.so"

SOURCES = ["gam_api.cu", "gemm.cu", "attention_sm90.cu", "attention_relpos_sm90.cu", "rowops.cu", "frontend.cu", "ctc.cu", "words.cu", "comm.cu", "rnnt.cu", "rnnt_cluster.cu", "heads.cu", "pooled_head.cu", "emo_time.cu", "head_grads.cu", "align.cu", "spot.cu", "bias.cu", "rnnt_loss.cu", "resample.cu"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libgigaam_b200.so cannot be built (no CPU fallback exists)")


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(CSRC.glob("*")) + [PKG_DIR.parent / "include" / "gigaam_b200.h"]:
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build_library(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA translation unit for sm_90a and link libgigaam_b200.so in-tree."""
    BUILD_DIR.mkdir(exist_ok=True)
    stamp = BUILD_DIR / "stamp.txt"
    digest = _digest()
    if not force and LIB_PATH.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB_PATH
    nvcc = _nvcc()

    def compile_one(src: str) -> str:
        obj = BUILD_DIR / (src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        (BUILD_DIR / (src + ".log")).write_text(res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{res.stdout}\n{res.stderr}")
        if verbose:
            print(res.stderr)
        return str(obj)

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-o", str(LIB_PATH), *objs, "-cudart", "static", "-ldl", "-gencode", "arch=compute_90a,code=sm_90a"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    stamp.write_text(digest)
    return LIB_PATH


if __name__ == "__main__":
    import sys

    print(build_library(force="--force" in sys.argv, verbose=True))
