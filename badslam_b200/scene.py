"""Seeded synthetic RGB-D scenes in the reference's on-device encodings.

The generator follows the scene of the reference's own BA tests
(applications/badslam/src/badslam/test/test_intrinsics_optimization_photometric_residual.cc:50-94
RenderPlanes, :182-211 planes + keyframe poses) and emits every buffer in the exact
format the BA kernels consume:

* depth   u16, raw units, 65535 = unknown, bit 15 = invalid        (kernels.cuh:38-41)
* normals u16 = two s8                                              (util.cuh:120-146)
* radius  u16 = IEEE half of r^2                                    (cuda_depth_processing.cu:331-358)
* colour  uchar4, .w = luma                                         (cuda_image_processing.cu:165-176)
* surfels 17-row SoA, normal packed 3 x s10                         (kernels.cuh:69-93, util_nvcc_only.cuh:67-95)

Keyframe preprocessing (normals from depth, radii, isolated-pixel removal, min/max depth)
restates cuda_depth_processing.cu:134-279,284-358,389-420 in numpy; surfel initialisation
restates kernel_create_surfels.cu:96-161 with a deterministic "first valid pixel of the
cell in raster order" winner instead of the reference's atomicCAS race (:68).

Everything is numpy on the host: the arrays are the single source of truth that the
CUDA path, the CPU oracle and the reference's own kernels all consume.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

KF_ACTIVE, KF_COVIS_ACTIVE, KF_INACTIVE = 0, 1, 2
SURFEL_ROWS = 17
UNKNOWN_DEPTH = 65535


@dataclass
class SceneConfig:
    width: int = 640
    height: int = 480
    num_keyframes: int = 20
    num_surfels: int = 200_000
    cell: int = 4                      # sparse_surfel_cell_size (bad_slam_config.h:136)
    seed: int = 2
    raw_to_float_depth: float = 1.0 / 1000.0
    baseline_fx: float = 40.0
    plane_count: int = 20
    pose_spread_t: float = 3.0         # test_intrinsics_optimization_photometric_residual.cc:202-211
    pose_spread_r: float = 0.7
    pose_noise_t: float = 0.002        # perturbation BA has to undo (SURVEY 8d)
    pose_noise_r: float = 0.001
    surfel_depth_noise: float = 0.0    # metres, along the viewing ray
    depth_a: float = 0.0
    cfactor: float = 0.0
    name: str = "custom"


def config_by_name(name: str) -> SceneConfig:
    """The BASELINE.json configs (SURVEY.md 8d table)."""
    if name == "cfg1":
        return SceneConfig(80, 60, 2, 4000, cell=1, seed=1, name="cfg1")
    if name == "cfg2":
        return SceneConfig(640, 480, 20, 200_000, cell=4, seed=2, name="cfg2")
    if name == "cfg3":
        return SceneConfig(640, 480, 200, 3_000_000, cell=4, seed=3, name="cfg3")
    if name == "cfg4":
        return SceneConfig(640, 480, 500, 4_000_000, cell=4, seed=4, depth_a=0.03, cfactor=0.005,
                           pose_spread_t=1.5, name="cfg4")
    if name == "cfg5":
        return SceneConfig(1280, 720, 400, 8_000_000, cell=4, seed=5, name="cfg5")
    if name == "cfg3_rank8":
        # what ONE rank of an 8-GPU cfg3 job sees in the geometry step: every keyframe, an eighth of the surfels (development
        # workload for tuning the geometry kernels at small shards on a single GPU, tools/ab_fast.py --workload cfg3_rank8)
        return SceneConfig(640, 480, 200, 375_000, cell=4, seed=3, name="cfg3_rank8")
    if name == "tiny":
        return SceneConfig(160, 120, 4, 6000, cell=2, seed=7, name="tiny")
    if name == "small":
        return SceneConfig(320, 240, 6, 30_000, cell=2, seed=8, name="small")
    raise KeyError(name)


# ----------------------------------------------------------------------------------------------
# SE3 helpers (float64 maths, float32 storage).  Pose layout = Sophus::SE3f::data():
# [qx, qy, qz, qw, tx, ty, tz].


def quat_to_R(q):
    x, y, z, w = [float(v) for v in q]
    return np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
        [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
        [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], dtype=np.float64)


def R_to_quat(R):
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        w = 0.25 * s
        x = (R[2, 1] - R[1, 2]) / s
        y = (R[0, 2] - R[2, 0]) / s
        z = (R[1, 0] - R[0, 1]) / s
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = np.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2]) * 2
        w = (R[2, 1] - R[1, 2]) / s
        x = 0.25 * s
        y = (R[0, 1] + R[1, 0]) / s
        z = (R[0, 2] + R[2, 0]) / s
    elif R[1, 1] > R[2, 2]:
        s = np.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2]) * 2
        w = (R[0, 2] - R[2, 0]) / s
        x = (R[0, 1] + R[1, 0]) / s
        y = 0.25 * s
        z = (R[1, 2] + R[2, 1]) / s
    else:
        s = np.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1]) * 2
        w = (R[1, 0] - R[0, 1]) / s
        x = (R[0, 2] + R[2, 0]) / s
        y = (R[1, 2] + R[2, 1]) / s
        z = 0.25 * s
    q = np.array([x, y, z, w])
    return q / np.linalg.norm(q)


def se3_exp(a):
    a = np.asarray(a, dtype=np.float64)
    ups, om = a[:3], a[3:]
    th = np.linalg.norm(om)
    O = np.array([[0, -om[2], om[1]], [om[2], 0, -om[0]], [-om[1], om[0], 0]])
    if th < 1e-10:
        R = np.eye(3) + O
        V = np.eye(3) + 0.5 * O
    else:
        R = np.eye(3) + np.sin(th) / th * O + (1 - np.cos(th)) / th ** 2 * (O @ O)
        V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * O + (th - np.sin(th)) / th ** 3 * (O @ O)
    return np.concatenate([R_to_quat(R), V @ ups]).astype(np.float32)


def se3_mul(A, B):
    RA, RB = quat_to_R(A[:4]), quat_to_R(B[:4])
    t = RA @ np.asarray(B[4:], dtype=np.float64) + np.asarray(A[4:], dtype=np.float64)
    return np.concatenate([R_to_quat(RA @ RB), t]).astype(np.float32)


def se3_inverse(A):
    R = quat_to_R(A[:4]).T
    return np.concatenate([R_to_quat(R), -R @ np.asarray(A[4:], dtype=np.float64)]).astype(np.float32)


def se3_matrix(A):
    M = np.eye(4)
    M[:3, :3] = quat_to_R(A[:4])
    M[:3, 3] = A[4:]
    return M


def pose_error(A, B):
    """(translation error in m, rotation error in rad) between two poses.

    The angle comes from the vector part of the normalised relative quaternion (2*atan2(|v|, |w|)),
    which stays accurate at the 1e-7 rad level; arccos of a rotation-matrix trace does not."""
    A = np.asarray(A, np.float64)
    B = np.asarray(B, np.float64)
    qa = A[:4] / np.linalg.norm(A[:4])
    qb = B[:4] / np.linalg.norm(B[:4])
    ax, ay, az, aw = -qa[0], -qa[1], -qa[2], qa[3]
    bx, by, bz, bw = qb
    w = aw * bw - ax * bx - ay * by - az * bz
    v = np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                  aw * bz + az * bw + ax * by - ay * bx])
    ang = 2.0 * np.arctan2(np.linalg.norm(v), abs(w))
    # translation of A^-1 * B
    Ra = quat_to_R(qa)
    dt = Ra.T @ (B[4:] - A[4:])
    return float(np.linalg.norm(dt)), float(ang)


# ----------------------------------------------------------------------------------------------
# Encodings


def small_float_to_s8(v):
    """util.cuh:120-123 SmallFloatToEightBitSigned (C cast truncates toward zero)."""
    v = np.asarray(v, dtype=np.float32)
    return np.trunc(v * np.float32(127) + np.where(v > 0, np.float32(0.5), np.float32(-0.5))).astype(np.int8)


def image_space_normal_to_u16(x, y):
    return (small_float_to_s8(x).view(np.uint8).astype(np.uint16)
            | (small_float_to_s8(y).view(np.uint8).astype(np.uint16) << 8))


def u16_to_image_space_normal(v):
    v = np.asarray(v, dtype=np.uint16)
    x = (v & 0xFF).astype(np.uint8).view(np.int8).astype(np.float32) * np.float32(1.0 / 127)
    y = (v >> 8).astype(np.uint8).view(np.int8).astype(np.float32) * np.float32(1.0 / 127)
    z = np.float32(1) - x * x - y * y
    z = -np.sqrt(np.maximum(z, np.float32(0)))
    return np.stack([x, y, z], axis=-1)


def small_float_to_s10(v):
    """util_nvcc_only.cuh:67-69."""
    v = np.asarray(v, dtype=np.float32)
    i = np.trunc(v * np.float32(511) + np.where(v > 0, np.float32(0.5), np.float32(-0.5))).astype(np.int16)
    return i.view(np.uint16).astype(np.uint32) & np.uint32(0x3FF)


def pack_surfel_normal(n):
    n = np.asarray(n, dtype=np.float32)
    return (small_float_to_s10(n[..., 0]) | (small_float_to_s10(n[..., 1]) << 10)
            | (small_float_to_s10(n[..., 2]) << 20)).astype(np.uint32)


def unpack_surfel_normal(p):
    p = np.asarray(p, dtype=np.uint32)

    def s10(u):
        u = (u & 0x3FF).astype(np.int32)
        u = np.where(u & 0x200, u - 1024, u)
        return u.astype(np.float32) * np.float32(1.0 / 511)

    n = np.stack([s10(p), s10(p >> 10), s10(p >> 20)], axis=-1)
    return n / np.linalg.norm(n, axis=-1, keepdims=True).astype(np.float32)


def raw_to_calibrated_depth(a, cfactor, raw_to_float, raw):
    """util.cuh:62-69."""
    inv = np.float32(1.0) / (np.float32(raw_to_float) * raw.astype(np.float32))
    return np.float32(1.0) / (inv + np.float32(cfactor) * np.exp(-np.float32(a) * inv, dtype=np.float32))


def tex_luma(luma_u8, x, y, weight_mode=3):
    """tex2D(..).w of a clamp / linear-filter / normalized-float u8 texture (keyframe.cc:67-73).
    weight_mode 3 (default) reproduces the hardware texture unit bit-exactly, 1 rounds the two fractions to 1/256 and
    interpolates in float, 0 uses exact float weights."""
    h, w = luma_u8.shape
    xb = np.asarray(x, dtype=np.float32) - np.float32(0.5)
    yb = np.asarray(y, dtype=np.float32) - np.float32(0.5)
    fi, fj = np.floor(xb), np.floor(yb)
    al, be = xb - fi, yb - fj
    if weight_mode == 3:
        # The filter of the hardware texture unit as measured (tools/tex_probe*.cu, bit-exact): 1.8 fixed-point fractions,
        # w11 = round(a*b/256), w10 = a - w11, w01 = b - w11, w00 = 256 - rest, unorm16 texels, one final rounding.
        a = np.floor(al * 256 + np.float32(0.5)).astype(np.int64)
        b = np.floor(be * 256 + np.float32(0.5)).astype(np.int64)
        i, j = fi.astype(np.int64), fj.astype(np.int64)
        T16 = luma_u8.astype(np.int64) * 257

        def t16(ii, jj):
            return T16[np.clip(jj, 0, h - 1), np.clip(ii, 0, w - 1)]

        w11 = (a * b + 128) >> 8
        w10, w01 = a - w11, b - w11
        w00 = 256 - w11 - w10 - w01
        s = w00 * t16(i, j) + w10 * t16(i + 1, j) + w01 * t16(i, j + 1) + w11 * t16(i + 1, j + 1)
        return (((s + 128) >> 8).astype(np.float32) / np.float32(65535.0)).astype(np.float32)
    if weight_mode == 1:
        al = np.floor(al * 256 + np.float32(0.5)) / np.float32(256)
        be = np.floor(be * 256 + np.float32(0.5)) / np.float32(256)
    i, j = fi.astype(np.int64), fj.astype(np.int64)
    T = luma_u8.astype(np.float32) * np.float32(1.0 / 255.0)

    def tx(ii, jj):
        return T[np.clip(jj, 0, h - 1), np.clip(ii, 0, w - 1)]

    return ((1 - al) * (1 - be) * tx(i, j) + al * (1 - be) * tx(i + 1, j)
            + (1 - al) * be * tx(i, j + 1) + al * be * tx(i + 1, j + 1)).astype(np.float32)


# ----------------------------------------------------------------------------------------------


@dataclass
class Scene:
    cfg: SceneConfig
    depth_K: np.ndarray            # fx fy cx cy, pixel-corner convention
    color_K: np.ndarray
    depth: np.ndarray              # [K,h,w] u16
    normals: np.ndarray            # [K,h,w] u16
    radius: np.ndarray             # [K,h,w] u16
    color: np.ndarray              # [K,h,w,4] u8
    poses_true: np.ndarray         # [K,7] global_T_frame
    poses_init: np.ndarray         # [K,7] perturbed start
    min_depth: np.ndarray
    max_depth: np.ndarray
    surfels: np.ndarray            # [17, pitch] f32
    num_surfels: int
    cfactor: np.ndarray            # [cf_h, cf_w] f32 (the model's current estimate, zeros)
    depth_a: float = 0.0
    planes: np.ndarray = field(default=None)

    @property
    def pitch(self):
        return self.surfels.shape[1]


def _render_keyframe(cfg, K4, pose, planes):
    """RenderPlanes (test_intrinsics_optimization_photometric_residual.cc:50-94), vectorised."""
    w, h = cfg.width, cfg.height
    fx, fy, cx, cy = [np.float32(v) for v in K4]
    xs = (np.arange(w, dtype=np.float32) + np.float32(0.5) - cx) / fx   # UnprojectFromPixelCenterConv
    ys = (np.arange(h, dtype=np.float32) + np.float32(0.5) - cy) / fy
    dirs = np.stack([np.broadcast_to(xs[None, :], (h, w)), np.broadcast_to(ys[:, None], (h, w)),
                     np.ones((h, w), np.float32)], axis=-1)
    R = quat_to_R(pose[:4]).astype(np.float32)
    t = pose[4:].astype(np.float32)
    gd = dirs @ R.T                                                   # global ray directions
    n = planes[:, :3].astype(np.float32)
    off = planes[:, 3].astype(np.float32)
    denom = gd @ n.T                                                  # [h,w,P]
    num = -(n @ t + off)                                              # [P]
    with np.errstate(divide="ignore", invalid="ignore"):
        lam = num[None, None, :] / denom
    lam = np.where((lam > 0) & np.isfinite(lam), lam, np.float32(np.inf))
    z = lam.min(axis=-1)
    valid = np.isfinite(z)
    raw = np.full((h, w), UNKNOWN_DEPTH, np.uint16)
    zq = np.minimum(np.float32(65535.0), z[valid] / np.float32(cfg.raw_to_float_depth) + np.float32(0.5))
    raw[valid] = zq.astype(np.uint32).astype(np.uint16)
    # optional depth deformation of the *measurement*: measured = f^-1(true)  (cfg4). Keep simple: apply the
    # forward model's inverse by fixed-point iteration in inverse depth.
    if cfg.depth_a != 0.0 or cfg.cfactor != 0.0:
        inv_true = np.float32(1.0) / np.maximum(z[valid], np.float32(1e-6))
        inv_raw = inv_true.copy()
        for _ in range(30):
            inv_raw = inv_true - np.float32(cfg.cfactor) * np.exp(-np.float32(cfg.depth_a) * inv_raw)
        zr = np.float32(1.0) / inv_raw
        raw[valid] = np.minimum(np.float32(65535.0), zr / np.float32(cfg.raw_to_float_depth)
                                + np.float32(0.5)).astype(np.uint32).astype(np.uint16)
    gp = t[None, None, :] + gd * np.where(valid, z, 0)[..., None]
    kF = np.float32(200.0)

    def chan(a, b):
        return (np.float32(255 / 2.0) * (1 + np.sin(np.float32(0.15) * kF * a
                                                    + np.float32(0.5) * np.sin(np.float32(0.25) * kF * b))))

    rgb = np.zeros((h, w, 3), np.uint8)
    rgb[..., 0] = np.where(valid, chan(gp[..., 0], gp[..., 1]), 0).astype(np.uint8)
    rgb[..., 1] = np.where(valid, chan(gp[..., 1], gp[..., 2]), 0).astype(np.uint8)
    rgb[..., 2] = np.where(valid, chan(gp[..., 2], gp[..., 0]), 0).astype(np.uint8)
    return raw, rgb


def compute_brightness(rgb):
    """cuda_image_processing.cu:165-176."""
    r, g, b = [rgb[..., i].astype(np.float32) for i in range(3)]
    lum = (np.float32(0.299) * r + np.float32(0.587) * g + np.float32(0.114) * b + np.float32(0.5)).astype(np.uint8)
    return np.concatenate([rgb, lum[..., None]], axis=-1)


def preprocess_depth(cfg, K4, raw_in, cfactor_grid, depth_a):
    """Keyframe ctor (keyframe.cc:96-144): ComputeNormalsCUDA -> ComputePointRadiiAndRemoveIsolatedPixelsCUDA
    -> ComputeMinMaxDepthCUDA.  Returns depth, normals, radius (all u16), min_depth, max_depth."""
    h, w = raw_in.shape
    fx, fy, cx, cy = [np.float32(v) for v in K4]
    fx_inv, fy_inv = np.float32(1) / fx, np.float32(1) / fy
    cx_inv, cy_inv = -(cx - np.float32(0.5)) * fx_inv, -(cy - np.float32(0.5)) * fy_inv
    cell = cfg.cell
    yy, xx = np.mgrid[0:h, 0:w]
    cf = cfactor_grid[yy // cell, xx // cell]
    invalid = (raw_in & 0x8000) != 0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        d = raw_to_calibrated_depth(depth_a, cf, cfg.raw_to_float_depth, raw_in)
    pts = np.stack([d * (fx_inv * xx.astype(np.float32) + cx_inv), d * (fy_inv * yy.astype(np.float32) + cy_inv), d], -1)

    # --- ComputeNormalsCUDAKernel (cuda_depth_processing.cu:134-250)
    depth1 = np.full((h, w), UNKNOWN_DEPTH, np.uint16)
    normals = np.full((h, w), int(image_space_normal_to_u16(np.float32(0), np.float32(0))), np.uint16)
    inner = np.zeros((h, w), bool)
    inner[1:-1, 1:-1] = True
    ok = inner & ~invalid
    ok[1:-1, 1:-1] &= ~invalid[1:-1, 2:] & ~invalid[1:-1, :-2] & ~invalid[2:, 1:-1] & ~invalid[:-2, 1:-1]
    c = pts[1:-1, 1:-1]
    left, right = pts[1:-1, :-2], pts[1:-1, 2:]
    top, bottom = pts[:-2, 1:-1], pts[2:, 1:-1]

    def sq(a):   # (a * a).sum(-1) over the 3 components, in the same order, without the generic reduction machinery
        return a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1] + a[..., 2] * a[..., 2]

    with np.errstate(divide="ignore", invalid="ignore"):
        ld, rd = sq(left - c), sq(right - c)
        ratio = ld / rd
        l2r = np.where(((ratio < 4) & (ratio > 0.25))[..., None], right - left,
                       np.where((ld < rd)[..., None], c - left, right - c))
        bd, td = sq(bottom - c), sq(top - c)
        ratio2 = bd / td
        b2t = np.where(((ratio2 < 4) & (ratio2 > 0.25))[..., None], top - bottom,
                       np.where((bd < td)[..., None], c - bottom, top - c))
        nrm = np.stack([l2r[..., 1] * b2t[..., 2] - b2t[..., 1] * l2r[..., 2],
                        b2t[..., 0] * l2r[..., 2] - l2r[..., 0] * b2t[..., 2],
                        l2r[..., 0] * b2t[..., 1] - b2t[..., 0] * l2r[..., 1]], -1).astype(np.float32)
        length = np.sqrt(sq(nrm))
        good = length > 1e-6
        inv_len = (np.float32(-1.0) if fy_inv < 0 else np.float32(1.0)) / np.where(good, length, 1)
        nx = np.where(good, nrm[..., 0] * inv_len, 0).astype(np.float32)
        ny = np.where(good, nrm[..., 1] * inv_len, 0).astype(np.float32)
    nu16 = image_space_normal_to_u16(np.nan_to_num(nx), np.nan_to_num(ny))
    oki = ok[1:-1, 1:-1]
    normals[1:-1, 1:-1] = np.where(oki, nu16, normals[1:-1, 1:-1])
    depth1[1:-1, 1:-1] = np.where(oki, raw_in[1:-1, 1:-1], UNKNOWN_DEPTH)

    # --- ComputePointRadiiAndRemoveIsolatedPixelsCUDAKernel (:284-358), operates on depth1 with metric depth
    inv1 = (depth1 & 0x8000) != 0
    dm = np.float32(cfg.raw_to_float_depth) * depth1.astype(np.float32)
    p1 = np.stack([dm * (fx_inv * xx.astype(np.float32) + cx_inv), dm * (fy_inv * yy.astype(np.float32) + cy_inv), dm], -1)
    radius = np.zeros((h, w), np.uint16)
    depth2 = np.full((h, w), UNKNOWN_DEPTH, np.uint16)
    cnt = np.zeros((h, w), np.int32)
    mind = np.full((h, w), np.inf, np.float32)
    for dy, dx in ((0, 1), (0, -1), (1, 0), (-1, 0)):
        sh = np.roll(p1, (-dy, -dx), axis=(0, 1))
        shinv = np.roll(inv1, (-dy, -dx), axis=(0, 1))
        edge = np.zeros((h, w), bool)   # rolled-in borders are invalid neighbours
        if dy == 1: edge[-1, :] = True
        if dy == -1: edge[0, :] = True
        if dx == 1: edge[:, -1] = True
        if dx == -1: edge[:, 0] = True
        nb_ok = ~shinv & ~edge
        dist = sq(sh - p1).astype(np.float32)
        cnt += nb_ok
        mind = np.where(nb_ok & (dist < mind), dist, mind)
    valid = ~inv1 & (cnt >= 4)
    with np.errstate(over="ignore"):
        radius = np.where(valid, mind, 0).astype(np.float16).view(np.uint16)
    radius = np.where(inv1, 0, radius).astype(np.uint16)
    depth2 = np.where(valid, depth1, UNKNOWN_DEPTH).astype(np.uint16)

    # --- ComputeMinMaxDepthCUDA runs on depth1 (keyframe.cc:136-143 passes the normals-stage buffer)
    v1 = ~inv1
    if v1.any():
        mn = float(np.float32(cfg.raw_to_float_depth) * np.float32(depth1[v1].min()))
        mx = float(np.float32(cfg.raw_to_float_depth) * np.float32(depth1[v1].max()))
    else:
        mn, mx = float("inf"), 0.0
    return depth2, normals, radius, mn, mx


def _create_surfels_for_keyframe(cfg, depth_K, color_K, pose, depth, normals, radius, color, cfactor_grid, depth_a,
                                 quota, rng):
    """CreateNewSurfel (kernel_create_surfels.cu:96-161) for one winner pixel per sparse cell."""
    h, w = depth.shape
    cell = cfg.cell
    ok = (depth & 0x8000) == 0
    ok[0, :] = ok[-1, :] = False
    ok[:, 0] = ok[:, -1] = False
    ys, xs = np.nonzero(ok)                       # raster order
    cell_id = (ys // cell) * ((w - 1) // cell + 1) + (xs // cell)
    _, first = np.unique(cell_id, return_index=True)
    first.sort()
    if quota < len(first):
        sel = np.sort(rng.choice(len(first), size=quota, replace=False))
        first = first[sel]
    ys, xs = ys[first], xs[first]
    fx, fy, cx, cy = [np.float32(v) for v in depth_K]
    fx_inv, fy_inv = np.float32(1) / fx, np.float32(1) / fy
    cx_inv, cy_inv = -(cx - np.float32(0.5)) * fx_inv, -(cy - np.float32(0.5)) * fy_inv
    d = raw_to_calibrated_depth(depth_a, cfactor_grid[ys // cell, xs // cell], cfg.raw_to_float_depth, depth[ys, xs])
    if cfg.surfel_depth_noise > 0:
        d = d + rng.normal(0, cfg.surfel_depth_noise, d.shape).astype(np.float32)
    local = np.stack([d * (fx_inv * xs.astype(np.float32) + cx_inv), d * (fy_inv * ys.astype(np.float32) + cy_inv), d], -1)
    R = quat_to_R(pose[:4]).astype(np.float32)
    t = pose[4:].astype(np.float32)
    gp = local @ R.T + t
    ln = u16_to_image_space_normal(normals[ys, xs])
    gn = (ln @ R.T).astype(np.float32)
    r2 = radius[ys, xs].view(np.float16).astype(np.float32)
    # descriptors: ComputeRawDescriptorResidual with zero descriptors (cost_function.cuh:140-156)
    cfx, cfy, ccx, ccy = [np.float32(v) for v in color_K]
    d2c_fx, d2c_cx = cfx / fx, -cfx * cx / fx + ccx
    d2c_fy, d2c_cy = cfy / fy, -cfy * cy / fy + ccy
    cpx = d2c_fx * (xs.astype(np.float32) + np.float32(0.5)) + d2c_cx
    cpy = d2c_fy * (ys.astype(np.float32) + np.float32(0.5)) + d2c_cy
    Rinv = R.T
    tinv = -(Rinv @ t)

    def proj(p):
        lp = p @ Rinv.T + tinv
        return cfx * (lp[:, 0] / lp[:, 2]) + ccx, cfy * (lp[:, 1] / lp[:, 2]) + ccy

    # the surfel stores the PACKED normal; the reference computes tangents from the unpacked global normal it
    # just wrote only later -- at creation it uses the float normal (kernel_create_surfels.cu:131-139).
    axis = np.where((np.abs(gn[:, 0]) > 0.9)[:, None], np.array([0, 1, 0], np.float32), np.array([1, 0, 0], np.float32))
    t1 = np.stack([gn[:, 1] * axis[:, 2] - axis[:, 1] * gn[:, 2], axis[:, 0] * gn[:, 2] - gn[:, 0] * axis[:, 2],
                   gn[:, 0] * axis[:, 1] - axis[:, 0] * gn[:, 1]], -1).astype(np.float32)
    t1 = t1 * (np.float32(2.0) * np.sqrt(r2 / np.maximum(np.float32(1e-12), (t1 * t1).sum(-1))))[:, None]
    t2 = np.stack([gn[:, 1] * t1[:, 2] - t1[:, 1] * gn[:, 2], t1[:, 0] * gn[:, 2] - gn[:, 0] * t1[:, 2],
                   gn[:, 0] * t1[:, 1] - t1[:, 0] * gn[:, 1]], -1).astype(np.float32)
    t2 = t2 * (np.float32(2.0) * np.sqrt(r2 / np.maximum(np.float32(1e-12), (t2 * t2).sum(-1))))[:, None]
    luma = color[..., 3]
    t1x, t1y = proj(gp + t1)
    t2x, t2y = proj(gp + t2)
    inten = tex_luma(luma, cpx, cpy)
    d1 = np.float32(180.0) * (tex_luma(luma, t1x, t1y) - inten)
    d2 = np.float32(180.0) * (tex_luma(luma, t2x, t2y) - inten)
    n = len(xs)
    rows = np.zeros((8, n), np.float32)
    rows[0:3] = gp.T
    rows[3] = pack_surfel_normal(gn).view(np.float32)
    rows[4] = r2
    rgb = color[np.clip(cpy.astype(np.int64), 0, h - 1), np.clip(cpx.astype(np.int64), 0, w - 1), :3].astype(np.uint32)
    rows[5] = (rgb[:, 0] | (rgb[:, 1] << 8) | (rgb[:, 2] << 16)).astype(np.uint32).view(np.float32)
    rows[6] = d1
    rows[7] = d2
    return rows


def make_scene(cfg: SceneConfig, verbose: bool = False) -> Scene:
    """The seeded scene of a configuration.  BADBA_SCENE_CACHE=<dir> keeps a pickle per configuration there, so that several
    processes of one GPU session (tests, tools, both bench arms) generate a large scene once (cfg5: minutes of host time)."""
    import os
    cache = os.environ.get("BADBA_SCENE_CACHE")
    if not cache:
        return _make_scene(cfg, verbose)
    import pickle
    os.makedirs(cache, exist_ok=True)
    path = scene_cache_path(cfg, cache)
    if os.path.exists(path):
        with open(path, "rb") as f:
            return pickle.load(f)
    sc = _make_scene(cfg, verbose)
    tmp = f"{path}.{os.getpid()}.tmp"
    with open(tmp, "wb") as f:
        pickle.dump(sc, f, protocol=4)
    os.replace(tmp, path)
    return sc


def scene_cache_path(cfg: SceneConfig, cache_dir: str) -> str:
    import hashlib
    import os
    return os.path.join(cache_dir, f"{cfg.name}_{hashlib.sha1(repr(cfg).encode()).hexdigest()[:12]}.pkl")


def _make_scene(cfg: SceneConfig, verbose: bool = False) -> Scene:
    rng = np.random.Generator(np.random.PCG64(cfg.seed))
    w, h, K = cfg.width, cfg.height, cfg.num_keyframes
    depth_K = np.array([0.5 * h, 0.5 * h, 0.5 * w - 0.5, 0.5 * h - 0.5], np.float32)
    color_K = depth_K.copy()
    # planes: normal = normalise((u1, u2, -1)), offset 2.5  (test_..._photometric_residual.cc:182-190)
    pn = np.concatenate([rng.uniform(-1, 1, (cfg.plane_count, 2)), -np.ones((cfg.plane_count, 1))], axis=1)
    pn /= np.linalg.norm(pn, axis=1, keepdims=True)
    planes = np.concatenate([pn, np.full((cfg.plane_count, 1), 2.5)], axis=1).astype(np.float32)
    T0 = se3_exp([0.01, 0.02, 0.03, 0.004, 0.005, 0.006])
    cf_w, cf_h = (w - 1) // cfg.cell + 1, (h - 1) // cfg.cell + 1
    cfactor_grid = np.zeros((cf_h, cf_w), np.float32)

    depth = np.empty((K, h, w), np.uint16)
    normals = np.empty((K, h, w), np.uint16)
    radius = np.empty((K, h, w), np.uint16)
    color = np.empty((K, h, w, 4), np.uint8)
    poses_true = np.empty((K, 7), np.float32)
    poses_init = np.empty((K, 7), np.float32)
    mind = np.empty(K, np.float32)
    maxd = np.empty(K, np.float32)
    quota = -(-cfg.num_surfels // K)
    surfel_blocks = []
    for k in range(K):
        xi = np.concatenate([cfg.pose_spread_t * rng.uniform(-0.5, 0.5, 3), cfg.pose_spread_r * rng.uniform(-1, 1, 3)])
        pose = se3_mul(T0, se3_exp(xi))
        poses_true[k] = pose
        noise = np.concatenate([rng.normal(0, cfg.pose_noise_t, 3), rng.normal(0, cfg.pose_noise_r, 3)])
        poses_init[k] = se3_mul(pose, se3_exp(noise))
        raw, rgb = _render_keyframe(cfg, depth_K, pose, planes)
        color[k] = compute_brightness(rgb)
        depth[k], normals[k], radius[k], mind[k], maxd[k] = preprocess_depth(cfg, depth_K, raw, cfactor_grid, 0.0)
        surfel_blocks.append(_create_surfels_for_keyframe(cfg, depth_K, color_K, pose, depth[k], normals[k], radius[k],
                                                          color[k], cfactor_grid, 0.0, quota, rng))
        if verbose and (k % 10 == 0):
            print(f"[scene] keyframe {k}/{K}", flush=True)
    rows = np.concatenate(surfel_blocks, axis=1)[:, :cfg.num_surfels]
    n = rows.shape[1]
    pitch = ((n + 127) // 128) * 128          # cudaMallocPitch-style 512-byte row alignment
    surfels = np.zeros((SURFEL_ROWS, max(pitch, 128)), np.float32)
    surfels[:8, :n] = rows
    return Scene(cfg, depth_K, color_K, depth, normals, radius, color, poses_true, poses_init, mind, maxd,
                 surfels, n, cfactor_grid, 0.0, planes)


def render_frame(scene, global_T_frame):
    """A preprocessed RGB-D frame of the scene's planes seen from an arbitrary pose, in the keyframe format
    (depth, normals, radius u16 [h, w]; colour uchar4 [h, w, 4] with .w = luma): the input of frame tracking / odometry."""
    cfg = scene.cfg
    pose = np.asarray(global_T_frame, np.float32)
    raw, rgb = _render_keyframe(cfg, scene.depth_K, pose, scene.planes)
    color = compute_brightness(rgb)
    depth, normals, radius, _, _ = preprocess_depth(cfg, scene.depth_K, raw, scene.cfactor, scene.depth_a)
    return depth, normals, radius, color


def displace_surfels(scene, seed=3):
    """A copy of `scene` with three groups of surfels displaced, to exercise the end-of-BA maintenance
    (PerformBASchemeEndTasks): moved out of every view (unobserved), pulled towards keyframe 0's camera (in front of the
    measured surface: free-space violations) and pushed away from it (behind the surface: occluded)."""
    import copy
    sc = copy.copy(scene)
    sc.surfels = scene.surfels.copy()
    n = sc.num_surfels
    idx = np.random.default_rng(seed).permutation(n)
    k1, k2 = max(n // 150, 8), max(n // 100, 12)
    away, front, behind = idx[:k1], idx[k1:k1 + k2], idx[k1 + k2:k1 + 2 * k2]
    sc.surfels[0:3, away] += np.float32(1000.0)
    c0 = np.asarray(scene.poses_true[0][4:7], np.float32)
    for sel, f in ((front, np.float32(0.7)), (behind, np.float32(1.3))):
        p = sc.surfels[0:3, sel]
        sc.surfels[0:3, sel] = c0[:, None] + f * (p - c0[:, None])
    return sc, away, front, behind


def raw_frame(scene, k, noise_raw=3.0, hole_fraction=0.01, far_fraction=0.01, seed=11):
    """The sensor's view of keyframe k before preprocessing: raw u16 depth (0 = no measurement; Gaussian noise of `noise_raw`
    raw units, a fraction of pixels dropped, a fraction pushed beyond any sensible max_depth) and the uchar3 colour image --
    the inputs of BadSlam::PreprocessFrame (bad_slam.cc:640-765)."""
    cfg = scene.cfg
    raw, rgb = _render_keyframe(cfg, scene.depth_K, np.asarray(scene.poses_true[k]), scene.planes)
    rng = np.random.default_rng(seed + 1000 * k)
    valid = raw != UNKNOWN_DEPTH
    out = raw.astype(np.float64)
    out += rng.normal(0.0, noise_raw, raw.shape)
    out = np.clip(np.rint(out), 1, 32000).astype(np.uint16)
    out[~valid] = 0
    out[rng.random(raw.shape) < hole_fraction] = 0
    far = (rng.random(raw.shape) < far_fraction) & valid
    out[far] = np.uint16(30000)
    return out, rgb


def blank_scene(width, height, cell=4, seed=9, depth_a=0.02, cfactor_scale=1e-3):
    """A camera model without content (one empty keyframe, no surfels, a random depth-deformation grid): what the
    preprocessing tests need to build a DirectBA / oracle / reference context for an arbitrary image size."""
    cfg = SceneConfig(width, height, 1, 0, cell=cell, seed=seed, name=f"blank{width}x{height}")
    rng = np.random.default_rng(seed)
    depth_K = np.array([0.5 * height + 7, 0.5 * height + 7, 0.5 * width - 0.5, 0.5 * height - 0.5], np.float32)
    z16 = np.full((1, height, width), UNKNOWN_DEPTH, np.uint16)
    cf = (cfactor_scale * rng.random(((height - 1) // cell + 1, (width - 1) // cell + 1))).astype(np.float32)
    ident = np.array([[0, 0, 0, 1, 0, 0, 0]], np.float32)
    return Scene(cfg, depth_K, depth_K.copy(), z16, np.zeros_like(z16), np.zeros_like(z16),
                 np.zeros((1, height, width, 4), np.uint8), ident, ident.copy(), np.ones(1, np.float32), np.ones(1, np.float32),
                 np.zeros((17, 128), np.float32), 0, cf, depth_a, None)


def random_raw_frame(width, height, seed=0, hole_fraction=0.05):
    """Raw depth of a slanted surface around 1.5 - 2 m with 2 raw units of noise and holes, and random colours.  (White-noise
    depth would make the bilateral filter return its centre sample, rcp(rcp(c)) truncated: c or c - 1 depending on the last
    bit of the arithmetic -- a coin flip no two implementations share.)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:height, 0:width]
    raw = (1500.3 + 0.83 * xx + 0.47 * yy + rng.normal(0, 2.0, (height, width))).astype(np.uint16)
    raw[rng.random((height, width)) < hole_fraction] = 0
    rgb = rng.integers(0, 256, (height, width, 3), dtype=np.uint8)
    return raw, rgb
