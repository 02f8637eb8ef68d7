"""ctypes binding of oracle/preprocess_raw_oracle.c: the host stages in front of keyframe preprocessing (bad_slam.cc:649-689).

TEST INFRASTRUCTURE ONLY: imported by tests/.  The shared object is compiled on first use into oracle/_build/ (git-ignored)
with the same compiler and warnings as the oracle's Makefile.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "preprocess_raw_oracle.c")
_LIB_PATH = os.path.join(_HERE, "_build", "libpreprocess_raw_oracle.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(_SRC) > os.path.getmtime(_LIB_PATH):
            os.makedirs(os.path.dirname(_LIB_PATH), exist_ok=True)
            cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
            tmp = f"{_LIB_PATH}.{os.getpid()}"
            subprocess.check_call([cc, "-O2", "-fPIC", "-std=gnu11", "-Wall", "-Wextra", "-ffp-contract=off", "-shared", "-o",
                                   tmp, _SRC, "-lm"])
            os.replace(tmp, _LIB_PATH)   # atomic: a concurrent test process never loads a half-written object
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_downscale_rgb_to_half_size.restype = C.c_int
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def median_filter_and_densify(raw_depth, iterations=1):
    """MedianFilterAndDensifyDepthMap applied `iterations` times (BadSlamConfig::median_filter_and_densify_iterations)."""
    cur = np.ascontiguousarray(raw_depth, np.uint16)
    h, w = cur.shape
    for _ in range(iterations):
        out = np.zeros_like(cur)
        lib().orc_median_filter_and_densify(C.c_int(w), C.c_int(h), _p(cur, C.c_uint16), _p(out, C.c_uint16))
        cur = out
    return cur


def downscale_depth(raw_depth, out_w, out_h):
    """Image::DownscaleUsingMedianWhileExcluding(0, out_w, out_h): the raw depth at pyramid_level_for_depth."""
    raw = np.ascontiguousarray(raw_depth, np.uint16)
    out = np.zeros((out_h, out_w), np.uint16)
    lib().orc_downscale_using_median_excluding_zero(C.c_int(raw.shape[1]), C.c_int(raw.shape[0]), _p(raw, C.c_uint16),
                                                    C.c_int(out_w), C.c_int(out_h), _p(out, C.c_uint16))
    return out


def downscale_color(rgb, levels):
    """ImagePyramid level `levels` of a uchar3 image: DownscaleToHalfSize applied `levels` times (even sizes at every level)."""
    cur = np.ascontiguousarray(rgb, np.uint8)
    for _ in range(levels):
        h, w = cur.shape[:2]
        out = np.zeros((h // 2, w // 2, 3), np.uint8)
        if lib().orc_downscale_rgb_to_half_size(C.c_int(w), C.c_int(h), _p(cur, C.c_uint8), _p(out, C.c_uint8)) != 0:
            raise ValueError(f"DownscaleToHalfSize needs even sizes, got {w}x{h}")
        cur = out
    return cur


def scaled_size(size, level):
    """Camera::Scaled(2^-level) of an image size (camera.h:1696-1704): int(size / 2^level + 0.5)."""
    return int(size / float(1 << level) + 0.5)


def raw_frame_stage0(raw_depth, rgb, depth_size, median_filter_and_densify_iterations=0, pyramid_level_for_depth=0,
                     pyramid_level_for_color=0):
    """The images BadSlam::PreprocessFrame uploads (bad_slam.cc:649-689) from a frame as the sensor delivers it: the input of
    cpu_oracle.Oracle.preprocess_frame / bba_preprocess_frame.  depth_size = (w, h) of the depth camera."""
    depth = np.ascontiguousarray(raw_depth, np.uint16)
    if median_filter_and_densify_iterations > 0:
        assert pyramid_level_for_depth == 0, "Simultaneous downscaling and median filtering of depth maps is not implemented."
        depth = median_filter_and_densify(depth, median_filter_and_densify_iterations)
    if pyramid_level_for_depth > 0:
        depth = downscale_depth(depth, *depth_size)
    if rgb is not None and pyramid_level_for_color > 0:
        rgb = downscale_color(rgb, pyramid_level_for_color)
    return depth, rgb
