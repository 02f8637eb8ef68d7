"""numpy restatement of keyframe exposure estimation (bba_estimate_keyframe_exposures, DESIGN.md §3.21).  Not in the reference,
which assumes a fixed exposure; this oracle is pinned by its own properties (tests/test_oracle_exposure.py) and checks the CUDA
kernels (tests/test_gpu_keyframe_exposure.py).

Observations: a (surfel, keyframe) pair associated by the co-visibility test (covisibility_oracle.association) whose colour pixel
lies in the colour image and whose raw luma v (the .w byte of the keyframe's RGBA image at the floor of the colour coordinates) is
in [min_luma, max_luma]; its value is y = LOG_Q16[v] = round(2^16 ln v).  Model y_sa = x_a + z_s with z_s eliminated pairwise:
L x = r with L = diag(rowsum(C) - diag C) - offdiag(C), C = M^T M over the inlier table M, r_a = sum_s M_sa (n_s y_sa - Y_s).
The gauge keyframe has x = 0; keyframes outside its component of C > 0 get NaN.  Round 1 takes every observation; round k keeps an
observation iff |n_s (y_sa - xq_a) - sum_b (y_sb - xq_b)| <= n_s tau_q over the inliers of round k - 1, xq = rint(x of round k - 1).
"""
from __future__ import annotations

import numpy as np

import covisibility_oracle as CO
import surfel_deform_oracle as D

f32 = np.float32
LOG_Q16 = np.zeros(256, np.int64)
LOG_Q16[1:] = np.rint(65536.0 * np.log(np.arange(1, 256, dtype=np.float64))).astype(np.int64)


def depth_to_color(depth_K, color_K):
    """(d2c_fx, d2c_cx, d2c_fy, d2c_cy) as MakeCamera computes them in float32."""
    fx, fy, cx, cy = (f32(v) for v in depth_K)
    cfx, cfy, ccx, ccy = (f32(v) for v in color_K)
    return (f32(cfx / fx), f32(f32(f32(-cfx) * cx) / fx) + ccx, f32(cfy / fy), f32(f32(f32(-cfy) * cy) / fy) + ccy)


def _fma(a, b, c):
    """float32 a * b + c rounded once (the product is exact in float64)."""
    return (np.float64(a) * b.astype(np.float64) + np.float64(c)).astype(f32)


NEAR_PIXEL = 1e-3


def observations(cam, depth_K, color_K, depth, normals, color, surfels, n, frame_T_global, min_luma=8, max_luma=247):
    """(valid [n, K] bool, y [n, K] int64 (0 where not valid), near [n, K] bool) of surfels[:, :n] against keyframes with images
    depth / normals / color [K][h][w(4)] at frame_T_global [K, 7].  The kernels project with fast maths, so a pair may be decided
    the other way there when it is near: its association margin is <= covisibility_oracle.NEAR or its colour coordinates lie
    within NEAR_PIXEL of a texel edge."""
    A, margin = CO.association(cam, depth, normals, surfels, n, frame_T_global)
    p = np.asarray(surfels, f32)[0:3, :n]
    d2c_fx, d2c_cx, d2c_fy, d2c_cy = depth_to_color(depth_K, color_K)
    K = len(frame_T_global)
    valid = np.zeros((n, K), bool)
    y = np.zeros((n, K), np.int64)
    near = margin <= CO.NEAR
    with np.errstate(all="ignore"):
        for k in range(K):
            T = D.quat_to_matrix_f32(frame_T_global[k])
            lz = T[8] * p[0] + T[9] * p[1] + T[10] * p[2] + T[11]
            lx = T[0] * p[0] + T[1] * p[1] + T[2] * p[2] + T[3]
            ly = T[4] * p[0] + T[5] * p[1] + T[6] * p[2] + T[7]
            inv_z = f32(1) / lz
            pxf = cam.fx * (lx * inv_z) + cam.cx
            pyf = cam.fy * (ly * inv_z) + cam.cy
            ccx = _fma(d2c_fx, pxf, d2c_cx)
            ccy = _fma(d2c_fy, pyf, d2c_cy)
            ch, cw = color[k].shape[:2]
            frac = lambda v: np.abs(v - np.round(v))
            near[:, k] |= A[:, k] & ((frac(ccx) <= NEAR_PIXEL) | (frac(ccy) <= NEAR_PIXEL))
            ok = A[:, k] & (ccx >= 0) & (ccy >= 0)
            ix = np.where(ok, ccx, 0).astype(np.int64)
            iy = np.where(ok, ccy, 0).astype(np.int64)
            ok &= (ix < cw) & (iy < ch)
            v = np.asarray(color[k])[np.where(ok, iy, 0), np.where(ok, ix, 0), 3].astype(np.int64)
            ok &= (v >= min_luma) & (v <= max_luma)
            valid[:, k] = ok
            y[:, k] = np.where(ok, LOG_Q16[v], 0)
    return valid, y, near


def system(member, y):
    """(C [K, K] int64, r [K] int64) of the inlier table member [n, K]."""
    M = member.astype(np.int64)
    C = M.T @ M
    ns = M.sum(axis=1)
    Y = (M * y).sum(axis=1)
    r = (M * (ns[:, None] * y - Y[:, None])).sum(axis=0)
    return C, r


def component(C, gauge):
    """[K] bool: the keyframes connected to gauge by C > 0."""
    K = len(C)
    adj = (C > 0) & ~np.eye(K, dtype=bool)
    reached = np.zeros(K, bool)
    reached[gauge] = True
    frontier = [gauge]
    while frontier:
        nxt = np.flatnonzero(adj[frontier].any(axis=0) & ~reached)
        reached[nxt] = True
        frontier = list(nxt)
    return reached


def solve(C, r, gauge):
    """(x [K] float64 in Q16 units, NaN outside the gauge's component; reached [K])."""
    K = len(C)
    reached = component(C, gauge)
    Cf = C.astype(np.float64)
    L = np.diag(Cf.sum(axis=1) - np.diag(Cf)) - (Cf - np.diag(np.diag(Cf)))
    U = reached.copy()
    U[gauge] = False
    x = np.full(K, np.nan)
    x[reached] = 0.0
    if U.any():
        x[U] = np.linalg.solve(L[np.ix_(U, U)], r[U].astype(np.float64))
    return x, reached


def estimate(valid, y, gauge, inlier_threshold=0.1, outer_iterations=2):
    """The estimate of an observation table: dict of gains [K] (float64, NaN outside the component), log (x / 2^16), observations,
    inliers, C, r and member [n, K] of the last round, rounds (per round: C, r, member, x)."""
    tau = int(round(65536.0 * inlier_threshold))
    y = np.where(valid, y, 0).astype(np.int64)
    member = valid.copy()
    rounds = []
    x = None
    for k in range(1, outer_iterations + 1):
        if k >= 2:
            xq = np.where(np.isnan(x), 0, np.rint(np.nan_to_num(x))).astype(np.int64)
            M = member.astype(np.int64)
            tn = M.sum(axis=1)
            ts = (M * (y - xq[None, :])).sum(axis=1)
            d = tn[:, None] * (y - xq[None, :]) - ts[:, None]
            member = valid & (np.abs(d) <= tn[:, None] * tau)
        C, r = system(member, y)
        x, reached = solve(C, r, gauge)
        rounds.append(dict(C=C, r=r, member=member.copy(), x=x.copy()))
    log = x / 65536.0
    return dict(gains=np.exp(log), log=log, observations=valid.sum(axis=0), inliers=np.where(reached, np.diag(rounds[-1]["C"]), 0),
                C=rounds[-1]["C"], r=rounds[-1]["r"], member=member, rounds=rounds)


def scale_colors(color, gains):
    """color [K][h][w][4] u8 with each keyframe's rgb scaled: clip(rint(rgb * g)), the luma recomputed by compute_brightness."""
    from badslam_b200.scene import compute_brightness
    out = np.array(color, copy=True)
    for k, g in enumerate(gains):
        rgb = np.clip(np.rint(np.asarray(color[k])[..., :3].astype(np.float64) * g), 0, 255).astype(np.uint8)
        out[k] = compute_brightness(rgb)
    return out


def compensated_luma(v, g):
    """min(255, rint(v / g)) in float32, as the luma extraction writes it."""
    return np.minimum(f32(255), np.rint(np.asarray(v, f32) / f32(g))).astype(np.uint8)
