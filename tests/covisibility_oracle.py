"""numpy restatement of the keyframe co-visibility measurement (bba_measure_keyframe_covisibility, DESIGN.md §3.19).  Not in the
reference, whose only keyframe-to-keyframe relation is the frustum-intersection list (bba_get_covisibility); this oracle is pinned by
its own properties (tests/test_oracle_covisibility.py) and checks the CUDA kernels (tests/test_gpu_covisibility.py).

A surfel is associated with keyframe k when stage 3 of the association test (surfel_deform_oracle.associate, the voter test of the
surfel deformation) passes at k's current pose.  A = [surfels, keyframes] of that test, C = A^T A in int64.  The kernels use fast
maths, so a pair within rounding of a threshold may be decided the other way there: near[a][b] counts the surfels whose margin to
a deciding test is <= NEAR for keyframe a or for keyframe b, the most any entry C[a][b] can move by such flips.
"""
from __future__ import annotations

import numpy as np

import surfel_deform_oracle as D

NEAR = 1e-4


def association(cam, depth, normals, surfels, n, frame_T_global):
    """(A [n, K] bool, margin [n, K]) of surfels[:, :n] against keyframes at frame_T_global [K, 7] (the inverses of their
    current global_T_frame).  Deleted surfels (x = NaN) are associated with no keyframe and have an infinite margin."""
    p = np.asarray(surfels, np.float32)[0:3, :n]
    live = ~np.isnan(p[0])
    nrm = D.unpack_normal(np.asarray(surfels, np.float32)[3, :n])
    K = len(frame_T_global)
    A = np.zeros((n, K), bool)
    margin = np.full((n, K), np.inf)
    for k in range(K):
        a, m = D.associate(cam, D.quat_to_matrix_f32(frame_T_global[k]), depth[k], normals[k], p, nrm)
        A[:, k] = a & live
        margin[:, k] = np.where(live, m, np.inf)
    return A, margin


def covisibility(cam, depth, normals, surfels, n, frame_T_global):
    """(C [K, K] int64, near [K, K] int64, A, margin); see the module docstring."""
    A, margin = association(cam, depth, normals, surfels, n, frame_T_global)
    Ai = A.astype(np.int64)
    C = Ai.T @ Ai
    N = (margin <= NEAR).astype(np.int64)
    per = N.sum(axis=0)
    near = per[:, None] + per[None, :] - N.T @ N   # surfels near for a or for b
    return C, near, A, margin
