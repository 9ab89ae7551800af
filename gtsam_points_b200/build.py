"""Builds gtsam_points_b200/lib/libb2points.so (hand-written CUDA for sm_90a) in-tree with nvcc.

`python -m gtsam_points_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a GPU.
The host compiler is pinned to /usr/bin/g++ rather than $CXX, so that the build does not depend on the caller's environment.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libb2points.so")

SOURCES = ["b2_context.cu", "b2_cloud.cu", "b2_voxelmap.cu", "b2_kdtree.cu", "b2_factors.cu", "b2_registration.cu", "b2_filter.cu", "b2_segmentation.cu", "b2_occupancy.cu", "b2_optimize.cu"]
HEADERS = ["b2_internal.hpp", "b2_device.cuh", "b2_kdtree.cuh", "b2_factor_kernel_ws.cuh", os.path.join("..", "..", "include", "b2points.h")]

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HOST_CXX = "/usr/bin/g++"
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-ccbin", HOST_CXX,
    "-Xcompiler", "-fPIC,-fvisibility=hidden",
    "-Xcudafe", "--diag_suppress=177",
]

# The pose optimizer's loop arithmetic is restated on the host bit for bit: no fused multiply-adds, on the device or the host.
EXTRA_FLAGS = {"b2_optimize.cu": ["-fmad=false", "-Xcompiler", "-ffp-contract=off"]}


def _mtime(p):
    return os.path.getmtime(p) if os.path.exists(p) else 0.0


def _compile(src, verbose):
    obj = os.path.join(OBJDIR, src.replace(".cu", ".o"))
    deps = [os.path.join(CSRC, src)] + [os.path.join(CSRC, h) for h in HEADERS]
    if _mtime(obj) > max(_mtime(d) for d in deps):
        return obj, False
    cmd = [NVCC] + NVCC_FLAGS + EXTRA_FLAGS.get(src, []) + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    return obj, True


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJDIR):
            os.remove(os.path.join(OBJDIR, f))
    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        results = list(ex.map(lambda s: _compile(s, verbose), SOURCES))
    objs = [o for o, _ in results]
    if any(changed for _, changed in results) or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-ccbin", HOST_CXX, "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
