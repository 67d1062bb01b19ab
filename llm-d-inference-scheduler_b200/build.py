"""Builds libepp_engine.so IN-TREE with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python llm-d-inference-scheduler_b200/build.py [--force] [--verbose]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libepp_engine.so")
SOURCES = ["engine.cu", "batcher.cu", "hash_kernels.cu", "hash_fused.cu", "index_kernels.cu", "index_store.cu", "pick_kernels.cu", "match_sparse.cu", "cycle_small.cu", "shard_p2p.cu", "nohit_lru.cu", "inflight.cu", "subset_pick.cu", "admit.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false",                      # fp64 scoring must never fuse x*y+z (Go/amd64 semantics)
    "-Xcompiler", "-fPIC,-O2,-Wall,-fvisibility=hidden",
    "--shared", "-cudart", "shared",
]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [
        os.path.join(HERE, "..", "include", "epp_engine.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
        [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))] + ["-o", OUT]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building libepp_engine.so")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
