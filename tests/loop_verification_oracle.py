"""numpy restatement of the loop-closure verification (bba_verify_loop_closures, DESIGN §3.16; loop_detector.cc:436-668).

* poses are float[7] = (qx, qy, qz, qw, tx, ty, tz) global_T_frame / a_T_b as on the library side; the arithmetic here is fp64
  on rotation matrices, so nothing but the statement of the rules is shared with the library;
* `neighbours` is the rule of loop_detector.cc:455-496 on contiguous keyframe ids;
* `initial_estimates` and `refined` compose the tracked pairs' poses (:498-548);
* `agreement` is the pair test of :575-599 and `average_pose` is AveragePose (util.cc:110-128) through scipy's SVD;
* `necessity` is the pixel test of :630-666 over every valid pixel of a depth image (the library's stand-in for the keypoints).
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

ACCEPTED, NO_NEIGHBOUR, ROTATION_DISAGREES, TRANSLATION_DISAGREES, CORRECTION_TOO_SMALL = range(5)
MAX_ANGLE = np.pi / 180.0 * 10.0
MAX_TRANSLATION = 0.02
MAX_PIXELS = 1.0
INVALID_DEPTH_BIT = 0x8000


def quat_to_R(q):
    x, y, z, w = np.asarray(q, np.float64) / np.linalg.norm(np.asarray(q, np.float64))
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def R_to_quat(R):
    R = np.asarray(R, np.float64)
    w = np.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    x = np.sqrt(max(0.0, 1.0 + R[0, 0] - R[1, 1] - R[2, 2])) / 2
    y = np.sqrt(max(0.0, 1.0 - R[0, 0] + R[1, 1] - R[2, 2])) / 2
    z = np.sqrt(max(0.0, 1.0 - R[0, 0] - R[1, 1] + R[2, 2])) / 2
    x = np.copysign(x, R[2, 1] - R[1, 2])
    y = np.copysign(y, R[0, 2] - R[2, 0])
    z = np.copysign(z, R[1, 0] - R[0, 1])
    q = np.array([x, y, z, w])
    return q / np.linalg.norm(q)


def to_T(p):
    p = np.asarray(p, np.float64)
    T = np.eye(4)
    T[:3, :3] = quat_to_R(p[:4])
    T[:3, 3] = p[4:7]
    return T


def from_T(T):
    return np.concatenate([R_to_quat(T[:3, :3]), T[:3, 3]])


def same_pose(a, b):
    """(translation distance, rotation angle) between two float[7] poses."""
    A, B = to_T(a), to_T(b)
    D = np.linalg.inv(A) @ B
    return float(np.linalg.norm(A[:3, 3] - B[:3, 3])), float(np.arccos(np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1)))


def neighbours(matched, K):
    """(matched, next, previous or the second next) with K keyframes, or None (NO_NEIGHBOUR)."""
    nxt = matched + 1
    if nxt >= K:
        return None
    prev = matched - 1 if matched > 0 else nxt + 1
    if prev >= K:
        return None
    return matched, nxt, prev


def matched_T_this(global_T_frame, ids):
    """matched.frame_T_global * old_i.global_T_frame for the three ids (identity for the matched keyframe)."""
    M = np.linalg.inv(to_T(global_T_frame[ids[0]]))
    return [np.eye(4) if i == 0 else M @ to_T(global_T_frame[k]) for i, k in enumerate(ids)]


def initial_estimates(old_T_cur_initial, global_T_frame, ids):
    """base_T_tracked_initial_estimate = old_T_cur_initial^-1 * matched_T_this of each tracked pair (fp64 4x4)."""
    inv = np.linalg.inv(to_T(old_T_cur_initial))
    return [inv @ m for m in matched_T_this(global_T_frame, ids)]


def refined(cur_T_tracked, global_T_frame, ids):
    """cur_T_old_refined[i] = (matched_T_this * cur_T_tracked^-1)^-1 (fp64 4x4)."""
    return [np.linalg.inv(m @ np.linalg.inv(to_T(c))) for m, c in zip(matched_T_this(global_T_frame, ids), cur_T_tracked)]


def agreement(poses, max_angle=MAX_ANGLE, max_translation=MAX_TRANSLATION):
    """(status, largest angle, largest translation distance) of three poses [3][7] in the reference's pair order."""
    T = [to_T(p) for p in poses]
    status, angle, trans = ACCEPTED, 0.0, 0.0
    for i in range(2):
        for k in range(i + 1, 3):
            rot = float(np.arccos(np.clip(T[i][:3, 2] @ T[k][:3, 2], -1.0, 1.0)))
            tr = float(np.linalg.norm(T[i][:3, 3] - T[k][:3, 3]))
            if status == ACCEPTED and rot > max_angle:
                status = ROTATION_DISAGREES
            if status == ACCEPTED and tr > max_translation:
                status = TRANSLATION_DISAGREES
            angle, trans = max(angle, rot), max(trans, tr)
    return status, angle, trans


def average_pose(poses):
    """AveragePose: U V^T of the SVD of the summed rotation matrices, the mean translation (float[7], fp64)."""
    T = [to_T(p) for p in poses]
    M = sum(t[:3, :3] for t in T)
    U, _, Vt = scipy.linalg.svd(M)
    R = U @ Vt
    out = np.eye(4)
    out[:3, :3] = R
    out[:3, 3] = sum(t[:3, 3] for t in T) / len(T)
    return from_T(out)


def necessity(depth_u16, depth_K, color_K, color_size, raw_to_float, a, cfactor, cell, cur_T_old, matched_global_T_frame,
              current_global_T_frame):
    """(average pixel distance or NaN, pixel count) of the necessity test over every valid pixel of the current keyframe's depth:
    the calibrated depth at each pixel centre, moved by (cur_T_old * matched.frame_T_global) * current.global_T_frame, both
    points projected by the colour camera (pixel-corner convention, no border)."""
    depth = np.asarray(depth_u16).astype(np.int64)
    h, w = depth.shape
    ys, xs = np.mgrid[0:h, 0:w]
    valid = (depth & INVALID_DEPTH_BIT) == 0
    raw = depth[valid].astype(np.float64)
    cf = np.asarray(cfactor, np.float64)[ys[valid] // cell, xs[valid] // cell]
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / (raw_to_float * raw)
        d = 1.0 / (inv + cf * np.exp(-a * inv))
    fx, fy, cx, cy = depth_K
    P = np.stack([d * (xs[valid] + 0.5 - cx) / fx, d * (ys[valid] + 0.5 - cy) / fy, d])
    M = to_T(cur_T_old) @ np.linalg.inv(to_T(matched_global_T_frame)) @ to_T(current_global_T_frame)
    Q = M[:3, :3] @ P + M[:3, 3:4]
    cfx, cfy, ccx, ccy = color_K
    cw, ch = color_size

    def project(X):
        with np.errstate(divide="ignore", invalid="ignore"):
            u = cfx * (X[0] / X[2]) + ccx
            v = cfy * (X[1] / X[2]) + ccy
        return u, v, (X[2] > 0) & (u >= 0) & (v >= 0) & (u < cw) & (v < ch)
    ue, ve, vis_e = project(Q)
    uc, vc, vis_c = project(P)
    both = vis_e & vis_c
    n = int(both.sum())
    if n == 0:
        return float("nan"), 0
    return float(np.hypot(ue[both] - uc[both], ve[both] - vc[both]).mean()), n


def verdict(average, count, max_pixels=MAX_PIXELS):
    return CORRECTION_TOO_SMALL if count >= 5 and average <= max_pixels else ACCEPTED
