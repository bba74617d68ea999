"""Builds runbookai_b200/lib/librbk_knn.so (hand-written sm_90a CUDA + the C ABI) in-tree.

nvcc cross-compiles without a GPU, so the library can be built on a machine without one and
used wherever the tree is copied.
"""
from __future__ import annotations

import os
import shutil
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "lib" / "librbk_knn.so"
SOURCES = ["rbk_capi.cu", "rbk_group.cu", "rbk_scan.cu", "rbk_scan_f16.cu", "rbk_ingest.cu", "rbk_finalize.cu", "rbk_compact.cu", "rbk_gather.cu", "rbk_mmr.cu"]
HEADERS = ["rbk_internal.h", "rbk_index_impl.h", "rbk_group_plan.h", "rbk_ptx.cuh", "rbk_epilogue.cuh", "rbk_scan_kernel.cuh", "rbk_f16.cuh", "../../include/rbk_knn.h"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false",            # fp64 re-rank must never contract a*b+c (parity contract)
    "--extended-lambda",
    "-Xcompiler", "-fPIC", "-shared", "-ldl",
]


def _nvcc() -> str:
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(cand).exists():
        raise RuntimeError("nvcc not found (set NVCC or add /usr/local/cuda/bin to PATH)")
    return cand


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = [CSRC / s for s in SOURCES] + [(CSRC / h).resolve() for h in HEADERS] + [Path(__file__)]
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    LIB.parent.mkdir(parents=True, exist_ok=True)
    cmd = [_nvcc(), *NVCC_FLAGS, *[str(CSRC / s) for s in SOURCES], "-o", str(LIB)]
    for flag in os.environ.get("RBK_EXTRA_NVCC_FLAGS", "").split():   # development probes, e.g. -DRBK_SCAN_CYCLE_STATS
        cmd.insert(1, flag)
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return LIB


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
