"""Build libfiery_b200.so in-tree with nvcc for sm_90a (H100; no torch, no cmake).

    python -m fiery_b200.build [--force] [--verbose]

The shared library has a plain C ABI (include/fiery_b200.h) and links only the CUDA runtime; the driver entry point
for TMA descriptors is resolved at run time through cudaGetDriverEntryPoint.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libfiery_b200.so")
STAMP_PATH = os.path.join(PKG_DIR, "csrc", ".build_stamp")
SOURCES = ["c_api.cu", "lift_plan.cu", "lift_fwd.cu", "lift_fwd_cols.cu", "lift_det.cu", "lift_bwd.cu", "bev_conv.cu", "bev_conv_bwd.cu", "depth_layer.cu", "voxels_summing.cu", "warp.cu", "temporal_entry.cu", "causal_conv.cu", "spatial_sums.cu", "batch_norm.cu", "spatial_gru.cu", "bottleneck.cu", "output_head.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo", "--use_fast_math=false",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: set NVCC or put it on PATH")


def _source_hash() -> str:
    h = hashlib.sha256()
    files = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h")))
    files = [os.path.join(CSRC, f) for f in files] + [os.path.join(os.path.dirname(PKG_DIR), "include", "fiery_b200.h")]
    for f in files:
        with open(f, "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_current() -> bool:
    if not (os.path.exists(LIB_PATH) and os.path.exists(STAMP_PATH)):
        return False
    with open(STAMP_PATH) as fh:
        return fh.read().strip() == _source_hash()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compiles every .cu under csrc/ for sm_90a into fiery_b200/libfiery_b200.so; returns its path."""
    if not force and is_current():
        return LIB_PATH
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = [nvcc, *[f for f in NVCC_FLAGS if f != "--use_fast_math=false"], "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stdout.write(out)
        if p.returncode != 0:
            failed = True
            print(f"nvcc failed on {src}", file=sys.stderr)
    if failed:
        raise RuntimeError("nvcc compilation failed")
    link = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH, *objs, "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
    subprocess.run(link, check=True)
    with open(STAMP_PATH, "w") as fh:
        fh.write(_source_hash())
    return LIB_PATH


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(force=a.force, verbose=a.verbose))
