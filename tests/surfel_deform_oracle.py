"""numpy restatement of the surfel deformation (bba_deform_surfels, DESIGN.md §3.13).  Not in the reference: it has no such
operation (its loop closure moves keyframes and frames only), so this oracle is pinned by its own properties
(tests/test_oracle_surfel_deformation.py) and checks the CUDA kernel (tests/test_gpu_surfel_deformation.py).

The association test is the geometry passes' (ProjectIntoImage + LoadPixel + Associate, device_math.cuh; oracle/badba_oracle.c
orc_pair_residuals bit 0), evaluated in fp32 for all surfels against one keyframe at a time.  The kernels are built with fast
maths and fused multiply-adds, so a pair that lies within rounding of a threshold may be decided the other way there: every
surfel gets its smallest relative margin to the tests that decide its voting set, so that tests can tell such flips from errors.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
K_DEPTH_TUKEY = f32(10.0)
K_DEPTH_UNCERTAINTY = f32(0.1)
K_COS_NORMAL = f32(0.76604)


def quat_to_matrix_f32(pose):
    """host_math.hpp QuatToMatrix + ToMatrix3x4 of a pose [7] (qx qy qz qw tx ty tz), fp32: the keyframe record's T."""
    q = np.asarray(pose[:4], f32)
    tx, ty, tz = f32(2) * q[0], f32(2) * q[1], f32(2) * q[2]
    twx, twy, twz = tx * q[3], ty * q[3], tz * q[3]
    txx, txy, txz = tx * q[0], ty * q[0], tz * q[0]
    tyy, tyz, tzz = ty * q[1], tz * q[1], tz * q[2]
    one = f32(1)
    R = [one - (tyy + tzz), txy - twz, txz + twy, txy + twz, one - (txx + tzz), tyz - twx, txz - twy, tyz + twx, one - (txx + tyy)]
    t = np.asarray(pose[4:], f32)
    return np.array([R[0], R[1], R[2], t[0], R[3], R[4], R[5], t[1], R[6], R[7], R[8], t[2]], f32)


def _rot64(q):
    q = np.asarray(q, np.float64)
    x, y, z, w = q / np.sqrt(np.sum(q * q))
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def keyframe_change(global_T_frame, original, inverse_of_current):
    """(D [12] fp32, centre [3] fp32, unmoved) of one keyframe: D = global_T_frame * original in fp64, rounded."""
    unmoved = np.asarray(inverse_of_current, f32).tobytes() == np.asarray(original, f32).tobytes()
    if unmoved:
        D = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], f32)
    else:
        Rc, Ro = _rot64(global_T_frame[:4]), _rot64(original[:4])
        to = np.asarray(original[4:], np.float32).astype(np.float64)
        R = Rc @ Ro
        t = Rc @ to + np.asarray(global_T_frame[4:], np.float32).astype(np.float64)
        D = np.concatenate([R, t[:, None]], axis=1).reshape(12).astype(f32)
    Ro = _rot64(original[:4])
    centre = (-(Ro.T @ np.asarray(original[4:], np.float32).astype(np.float64))).astype(f32)
    return D, centre, unmoved


def unpack_normal(bits):
    v = np.asarray(bits, np.float32).view(np.uint32)

    def s10(u):
        s = ((u & 0x3ff).astype(np.int32) << 22) >> 22
        return s.astype(f32) * f32(1.0 / 511)
    n = np.stack([s10(v), s10(v >> 10), s10(v >> 20)])
    return n * (f32(1) / np.sqrt(np.sum(n * n, axis=0, dtype=f32)))


def pack_normal(n):
    def s10(x):
        r = np.trunc(x * f32(511) + np.where(x > 0, f32(0.5), f32(-0.5))).astype(np.int32)
        return (r & 0x3ff).astype(np.uint32)
    return (s10(n[0]) | (s10(n[1]) << 10) | (s10(n[2]) << 20)).astype(np.uint32).view(np.float32)


def _transform(T, p):
    return np.stack([T[4 * r] * p[0] + T[4 * r + 1] * p[1] + T[4 * r + 2] * p[2] + T[4 * r + 3] for r in range(3)])


def _rotate(T, n):
    return np.stack([T[4 * r] * n[0] + T[4 * r + 1] * n[1] + T[4 * r + 2] * n[2] for r in range(3)])


class Camera:
    """The kernels' CameraParams (badba.cu MakeCamera) of a scene or of a handle's current cameras."""

    def __init__(self, width, height, depth_K, cell, cfactor, depth_a, raw_to_float, baseline_fx):
        self.w, self.h = int(width), int(height)
        self.fx, self.fy, self.cx, self.cy = (f32(v) for v in depth_K)
        self.fx_inv, self.fy_inv = f32(1) / self.fx, f32(1) / self.fy
        self.cx_inv = -(self.cx - f32(0.5)) * self.fx_inv
        self.cy_inv = -(self.cy - f32(0.5)) * self.fy_inv
        self.cell = int(cell)
        self.cfactor = np.ascontiguousarray(cfactor, f32)
        self.a, self.raw_to_float, self.baseline_fx = f32(depth_a), f32(raw_to_float), f32(baseline_fx)

    @classmethod
    def of_scene(cls, sc):
        c = sc.cfg
        return cls(c.width, c.height, sc.depth_K, c.cell, sc.cfactor, sc.depth_a, c.raw_to_float_depth, c.baseline_fx)


def associate(cam, T, depth, normals, p, n):
    """Stage 3 of ProjectAssociate for every column of p / n against one keyframe at T: (associated [N] bool, margin [N])."""
    with np.errstate(all="ignore"):
        N = p.shape[1]
        lz = T[8] * p[0] + T[9] * p[1] + T[10] * p[2] + T[11]
        lx = T[0] * p[0] + T[1] * p[1] + T[2] * p[2] + T[3]
        ly = T[4] * p[0] + T[5] * p[1] + T[6] * p[2] + T[7]
        front = lz > 0
        inv_z = f32(1) / lz
        pxf = cam.fx * (lx * inv_z) + cam.cx
        pyf = cam.fy * (ly * inv_z) + cam.cy
        inimg = front & (pxf >= 0) & (pyf >= 0) & (pxf < cam.w) & (pyf < cam.h)
        px = np.where(inimg, pxf, 0).astype(np.int64)
        py = np.where(inimg, pyf, 0).astype(np.int64)
        measured = depth[py, px]
        kfn = normals[py, px]
        cf = cam.cfactor[py // cam.cell, px // cam.cell]
        invalid = (measured & 0x8000) != 0
        inv_depth = f32(1) / (cam.raw_to_float * measured.astype(f32))
        d = f32(1) / (inv_depth + cf * np.exp(-cam.a * inv_depth))
        ln = _rotate(T, n)
        nx = cam.fx_inv * px.astype(f32) + cam.cx_inv
        ny = cam.fy_inv * py.astype(f32) + cam.cy_inv
        stddev = (K_DEPTH_UNCERTAINTY * np.abs(ln[0] * nx + ln[1] * ny + ln[2]) * (d * d)) / cam.baseline_fx
        thr = K_DEPTH_TUKEY * stddev
        diff = np.abs(lz - d)
        facing = lx * ln[0] + ly * ln[1] + lz * ln[2]
        kx = (kfn & 0xff).astype(np.uint8).view(np.int8).astype(f32) * f32(1.0 / 127)
        ky = (kfn >> 8).astype(np.uint8).view(np.int8).astype(f32) * f32(1.0 / 127)
        kz = -np.sqrt(np.maximum(f32(1) - kx * kx - ky * ky, f32(0)))
        compat = ln[0] * kx + ln[1] * ky + ln[2] * kz
        assoc = inimg & ~invalid & ~(diff > thr) & ~(facing > 0) & ~(compat < K_COS_NORMAL)
        # margins of the tests that decide the pair: the pixel the surfel projects to, then the depth, facing and normal tests
        margin = np.full(N, np.inf)
        frac = lambda v: np.abs(v - np.round(v))
        margin = np.where(front, np.minimum(frac(pxf), frac(pyf)), margin)
        valid = inimg & ~invalid
        lp_norm = np.sqrt(lx * lx + ly * ly + lz * lz)
        m = np.minimum(np.minimum(np.abs(diff - thr) / thr, np.abs(facing) / lp_norm), np.abs(compat - K_COS_NORMAL) / K_COS_NORMAL)
        margin = np.where(valid, np.minimum(margin, m), margin)
        margin = np.where(np.isnan(margin), 0.0, margin)
        return assoc, margin


def deform_surfels(cam, depth, normals, surfels, n, current_poses, original, inverse_of_current):
    """The deformation of surfels[:, :n] (17-row layout; a copy is returned) by keyframes 0 .. len(original)-1.

    current_poses [count, 7] global_T_frame now; original [count, 7] frame_T_global before; inverse_of_current [count, 7] is
    bba_host_se3_inverse of current_poses (the unmoved test).  Returns (surfels, moved, unobserved, voters [n, count] bool,
    margin [n])."""
    count = len(original)
    out = np.array(surfels, f32, copy=True)
    p = out[0:3, :n].copy()
    live = ~np.isnan(p[0])
    nrm = unpack_normal(out[3, :n])
    sums = np.zeros((8, n), f32)
    voters = np.zeros((n, count), bool)
    margin = np.full(n, np.inf)
    changes = [keyframe_change(current_poses[k], original[k], inverse_of_current[k]) for k in range(count)]

    def vote(k, mask):
        D, _, unmoved = changes[k]
        q = _transform(D, p)
        rn = _rotate(D, nrm)
        terms = [q[0] - p[0], q[1] - p[1], q[2] - p[2], rn[0], rn[1], rn[2], np.ones(n, f32),
                 np.full(n, f32(0) if unmoved else f32(1))]
        for r in range(8):
            sums[r] = np.where(mask, sums[r] + terms[r], sums[r])

    for k in range(count):
        a, m = associate(cam, quat_to_matrix_f32(original[k]), depth[k], normals[k], p, nrm)
        a &= live
        voters[:, k] = a
        margin = np.minimum(margin, np.where(live, m, np.inf))
        vote(k, a)
    unobserved = live & (sums[6] == 0)
    if count and unobserved.any():
        centres = np.stack([c[1] for c in changes])
        d2 = np.stack([np.sum(((p - centres[k][:, None]) ** 2).astype(f32), axis=0, dtype=f32) for k in range(count)])
        best = np.argmin(d2, axis=0)   # first minimum: the smaller id on a tie
        if count > 1:
            part = np.sort(d2, axis=0)
            gap = (part[1] - part[0]) / np.maximum(part[0], 1e-30)
            margin = np.where(unobserved, np.minimum(margin, gap), margin)
        for k in range(count):
            vote(k, unobserved & (best == k))
    moved = live & (sums[7] != 0)
    with np.errstate(all="ignore"):
        newp = p + sums[0:3] / sums[6]
        ns = sums[3:6]
        length = np.sqrt(ns[0] * ns[0] + ns[1] * ns[1] + ns[2] * ns[2])
        packed = pack_normal(ns / length)
    out[0:3, :n] = np.where(moved, newp, out[0:3, :n])
    out[3, :n] = np.where(moved & (length > 0), packed, out[3, :n])
    return out, int(moved.sum()), int(unobserved.sum()), voters, margin
