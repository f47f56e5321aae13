"""Builds libo2345_sm90.so (sm_90a only, NVIDIA H100) in-tree with nvcc.

    python one-2-3-45_b200/build.py [--force]

The shared library lands in one-2-3-45_b200/lib/ (git-ignored), object files in one-2-3-45_b200/build/.
nvcc cross-compiles without a GPU.
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
LIB = os.path.join(LIBDIR, "libo2345_sm90.so")
SOURCES = ["api.cu", "sdf_mlp.cu", "costvol.cu", "spconv.cu", "mcubes.cu", "featnet.cu", "render.cu", "render_tc.cu", "sdf_mlp_tc.cu", "gemm_tc.cu", "unet_ops.cu", "attention.cu", "raster.cu", "metrics.cu", "simplify.cu", "texture.cu", "project.cu", "clean.cu", "ao.cu", "lbvh.cu", "remesh.cu", "scan.cu", "mesh_common.cu"]
# no --use_fast_math: parity with the fp32 reference comes first
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC"]


def nvcc():
    cand = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else "nvcc"


def _deps(src):
    # every header of csrc/: an edit of sdf_common.cuh / blend_common.cuh must rebuild the objects that include them
    headers = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cuh")]
    return [os.path.join(CSRC, src), *headers, os.path.join(HERE, "..", "include", "o2345.h")]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True):
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    objs, jobs = [], []
    for s in SOURCES:
        o = os.path.join(OBJDIR, s.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, _deps(s)):
            jobs.append([nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, s), "-o", o])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    if force or jobs or _stale(LIB, objs):
        run([nvcc(), "-shared", *ARCH, "-o", LIB, *objs, "-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
