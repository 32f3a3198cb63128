#!/usr/bin/env python
"""Build lib/libprisma_b200.so (sm_90a, H100) from csrc/*.cu with nvcc.

    python vit-prisma_b200/build.py [--force]

Objects are compiled in parallel into build/ and linked into ONE shared library that exports
exactly the `extern "C"` entry points of include/prisma_b200.h.  nvcc cross-compiles without a
GPU, so this also runs on a machine without one.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OBJ = HERE / "build"
LIB = HERE / "lib" / "libprisma_b200.so"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
]


def _stale(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = True) -> Path:
    sources = sorted(CSRC.glob("*.cu"))
    headers = sorted(CSRC.glob("*.cuh")) + [HERE.parent / "include" / "prisma_b200.h"]
    OBJ.mkdir(exist_ok=True)
    LIB.parent.mkdir(exist_ok=True)
    stamp = OBJ / "flags.txt"            # objects built with other flags (another architecture) are stale whatever their age
    if not stamp.exists() or stamp.read_text() != " ".join(FLAGS):
        force = True

    def compile_one(src: Path):
        obj = OBJ / (src.stem + ".o")
        if force or _stale(obj, [src, *headers]):
            cmd = [NVCC, *FLAGS, "-c", str(src), "-o", str(obj)]
            if verbose:
                print("[build]", " ".join(cmd), flush=True)
            subprocess.run(cmd, check=True)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(sources))) as pool:
        objs = list(pool.map(compile_one, sources))
    if force or _stale(LIB, objs):
        cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB), *map(str, objs)]
        if verbose:
            print("[build]", " ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)
    stamp.write_text(" ".join(FLAGS))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
