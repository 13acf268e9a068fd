"""In-tree nvcc build of libpigeon_b200.so (sm_90a only).

The shared object is built next to the sources so that it travels with a snapshot of the repo.  `build()` is idempotent: it rebuilds only when a
source, header or flag changed (content hash), and never needs a GPU (nvcc cross-compiles).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
INCLUDE = PKG_DIR.parent / "include"
LIB_PATH = PKG_DIR / "libpigeon_b200.so"
OBJ_DIR = CSRC / "build"

SOURCES = [
    "tma_host.cu",
    "gemm_wgmma.cu",
    "gemm_pingpong.cu",
    "gemm_wide.cu",
    "gemm_wide_resid.cu",
    "attention_wgmma.cu",
    "nccl_gather.cu",
    "vit_misc.cu",
    "head.cu",
    "head_fused_wgmma.cu",
    "view_attention.cu",
    "refiner.cu",
    "train.cu",
    "preprocess.cu",
    "train_vit.cu",
    "attention_bwd_wgmma.cu",
    "vit_train_capi.cu",
    "capi.cu",
    "clip.cu",
    "clip_capi.cu",
    "clip_train.cu",
    "pretrain.cu",
    "optics.cu",
    "geo_metrics.cu",
    "jpeg.cu",
    "png.cu",
]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: pigeon_b200 needs the CUDA 12.9 toolkit to build its sm_90a kernels")
    return exe


def _flags() -> list:
    """NVCC_FLAGS plus the debugging extras of PG_NVCC_EXTRA (e.g. -DPG_DEADLOCK_REPORT)."""
    return NVCC_FLAGS + os.environ.get("PG_NVCC_EXTRA", "").split()


def _digest() -> str:
    h = hashlib.sha256()
    h.update(" ".join(_flags()).encode())
    files = sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + sorted(INCLUDE.glob("*.h"))
    for f in files:
        h.update(f.name.encode())
        h.update(f.read_bytes())
    return h.hexdigest()


def is_current() -> bool:
    """True when libpigeon_b200.so exists and was built from exactly the sources in the tree."""
    stamp = OBJ_DIR / "digest.txt"
    return LIB_PATH.exists() and stamp.exists() and stamp.read_text() == _digest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA source for sm_90a and link libpigeon_b200.so in-tree."""
    stamp = OBJ_DIR / "digest.txt"
    digest = _digest()
    if not force and LIB_PATH.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB_PATH
    nvcc = _nvcc()
    OBJ_DIR.mkdir(parents=True, exist_ok=True)

    def compile_one(src: str) -> Path:
        obj = OBJ_DIR / (Path(src).stem + ".o")
        cmd = [nvcc, *_flags(), "-I", str(INCLUDE), "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    tmp = LIB_PATH.with_suffix(".so.tmp")
    cmd = [nvcc, "-shared", "-o", str(tmp), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a",
           "-cudart", "static", "-Xlinker", "--exclude-libs,ALL", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB_PATH)
    stamp.write_text(digest)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
