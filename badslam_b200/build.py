"""Builds libbadba_b200.so (the product's CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m badslam_b200.build [--force]

The shared object and the objects under _obj/ are build products and are git-ignored.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libbadba_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "--expt-relaxed-constexpr"]
# (source, extra flags).  kernels.cu is built with -use_fast_math like the reference
# (applications/badslam/CMakeLists.txt:74-75); the fp64 pose solve, the exact sum's debug kernels and the host code are not.
UNITS = [
    ("kernels.cu", ["-use_fast_math", "-Xptxas", "-v"]),
    ("spatial_order.cu", ["-use_fast_math", "-Xptxas", "-v"]),
    ("intrinsics.cu", ["-use_fast_math", "-Xptxas", "-v"]),
    ("pcg.cu", ["-use_fast_math", "-Xptxas", "-v"]),
    ("lifecycle.cu", ["-use_fast_math", "-Xptxas", "-v"]),
    ("preprocess.cu", ["-use_fast_math", "-Xptxas", "-v"]),
    ("odometry.cu", ["-use_fast_math", "-Xptxas", "-v"]),
    ("pose_solve.cu", []),
    ("pose_graph.cu", ["-Xptxas", "-v"]),
    ("exact_sum.cu", ["-Xptxas", "-v"]),
    ("badba.cu", []),
    ("pose_step.cu", []),
    ("bundle_adjust.cu", []),
    ("multi_gpu.cu", []),
    ("local_group.cu", ["-Xptxas", "-v"]),   # (the all-reduce sums keep denormals: no -use_fast_math)
    ("frames.cu", []),
]
HEADERS = ["device_math.cuh", "exact_sum.cuh", "kernels.cuh", "launch.hpp", "persistent.cuh", "odometry.cuh", "preprocess_tile.cuh", "host_math.hpp", "handle.hpp", "rendezvous.hpp", os.path.join("..", "..", "include", "badba.h")]


def _newer(src, dst):
    return not os.path.exists(dst) or os.path.getmtime(src) > os.path.getmtime(dst)


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = os.environ.get("NVCC", "nvcc")
    os.makedirs(OBJ, exist_ok=True)
    hdr_time = max(os.path.getmtime(os.path.join(CSRC, h)) for h in HEADERS)
    objs = []
    procs = []
    for src, extra in UNITS:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src + ".o")
        objs.append(o)
        if force or _newer(s, o) or hdr_time > os.path.getmtime(o):
            cmd = [nvcc] + ARCH + COMMON + extra + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd), flush=True)
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            print(out)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}")
        with open(os.path.join(OBJ, src + ".log"), "w") as f:
            f.write(out)
    if force or procs or not os.path.exists(LIB):
        cmd = [nvcc] + ARCH + ["-shared", "-o", LIB] + objs + ["-cudart", "static"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
