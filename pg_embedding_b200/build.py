"""Build libpgemb_b200.so (the C-ABI shared library: CUDA kernels for sm_90a + host code) in-tree.

    python -m pg_embedding_b200.build          # or: python pg_embedding_b200/build.py

nvcc cross-compiles without a GPU.  The build products are git-ignored and stay in the package directory, so the
package is importable from the source tree.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libpgemb_b200.so")
SOURCES = ["capi.cu"]
HEADERS = ["common.cuh", "dist_exact.cuh", "search_kernel.cuh", "aux_kernels.cuh", "bind_kernel.cuh", "scan_tile_kernel.cuh", "scan_umma_kernel.cuh",
           "search_config.h",
           os.path.join("..", "..", "include", "pgemb_b200.h")]


# the GPU-owning sidecar process and the CUDA-free client library backends link against (csrc/sidecar)
SIDECAR_DIR = os.path.join(CSRC, "sidecar")
OUT_SIDECAR = os.path.join(HERE, "pgemb_sidecar")
OUT_CLIENT = os.path.join(HERE, "libpgemb_client.so")


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build(out: str = OUT) -> bool:
    if not os.path.isfile(out):
        return True
    t = os.path.getmtime(out)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.isfile(d))


def _cmd(out: str, verbose: bool) -> list:
    return [
        nvcc_path(), "-shared", "-Xcompiler", "-fPIC", "-std=c++17", "-O3", "-lineinfo",
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-fmad=false",  # exact kernels use explicit _rn intrinsics; never contract anything else either
        "-Xptxas", "-v" if verbose else "-warn-spills",
        "-I", os.path.join(HERE, "..", "include"),
        "-o", out,
    ] + [os.path.join(CSRC, f) for f in SOURCES]


def build(force: bool = False, verbose: bool = False) -> str:
    """Build the C-ABI library in-tree; returns its path."""
    jobs = []
    if force or needs_build(OUT):
        cmd = _cmd(OUT, verbose)
        jobs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)))
    build_sidecar(force)
    for cmd, pr in jobs:
        so, se = pr.communicate()
        if pr.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + so + "\n" + se)
        if verbose:
            print(so)
            print(se)
    return OUT


def build_sidecar(force: bool = False) -> tuple:
    """pgemb_sidecar (C++, dlopen()s the C-ABI library) and libpgemb_client.so (plain C): host code only, no nvcc."""
    inc = os.path.join(HERE, "..", "include")
    deps = [os.path.join(SIDECAR_DIR, f) for f in ("server.cpp", "client.c", "ipc.h")] + [os.path.join(inc, "pgemb_b200.h"), os.path.join(inc, "pgemb_client.h")]
    cmds = [
        (OUT_SIDECAR, ["g++", "-std=c++17", "-O2", "-Wall", "-o", OUT_SIDECAR, os.path.join(SIDECAR_DIR, "server.cpp"), "-ldl", "-lrt"]),
        (OUT_CLIENT, ["gcc", "-std=gnu11", "-O2", "-Wall", "-fPIC", "-shared", "-o", OUT_CLIENT, os.path.join(SIDECAR_DIR, "client.c"), "-lrt", "-lm"]),
    ]
    for out, cmd in cmds:
        if force or not os.path.isfile(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            res = subprocess.run(cmd, capture_output=True, text=True)
            if res.returncode != 0:
                raise RuntimeError("sidecar build failed:\n" + " ".join(cmd) + "\n" + res.stdout + "\n" + res.stderr)
    return OUT_SIDECAR, OUT_CLIENT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
