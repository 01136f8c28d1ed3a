"""Builds the C-ABI CUDA library in-tree: autovfx_b200/csrc/*.cu -> autovfx_b200/lib/libgsr_b200.so.

Plain nvcc, sm_90a (H100) only, no torch headers (the library has no torch dependency; the boundary is
include/gsr_b200.h).  The .so is git-ignored but travels to the GPU box with the repo snapshot.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "lib", "obj")
SO_PATH = os.path.join(LIBDIR, "libgsr_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build libgsr_b200.so (the library must be prebuilt with "
                           "`python -m autovfx_b200.build` where the CUDA toolkit is available)")
    return exe


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime() -> float:
    files = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(INCLUDE, "gsr_b200.h")]
    return max(os.path.getmtime(f) for f in files)


def is_stale() -> bool:
    return not os.path.exists(SO_PATH) or os.path.getmtime(SO_PATH) < _deps_mtime()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return SO_PATH
    nvcc = _nvcc()
    os.makedirs(OBJDIR, exist_ok=True)
    hdr_mtime = max(os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if not f.endswith(".cu"))
    hdr_mtime = max(hdr_mtime, os.path.getmtime(os.path.join(INCLUDE, "gsr_b200.h")))

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".o")
        if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(src), hdr_mtime):
            return obj
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed for %s" % src)
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(compile_one, sources()))
    tmp = SO_PATH + ".tmp"
    subprocess.check_call([nvcc, "-shared", "-o", tmp] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    os.replace(tmp, SO_PATH)
    return SO_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
