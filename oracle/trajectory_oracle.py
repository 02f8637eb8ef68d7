"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the trajectory deformation BadSlam runs around every bundle adjustment call.

What it follows (applications/badslam/src/badslam/trajectory_deformation.cc):
  RememberKeyframePoses                          :33-42    frame_T_global of every keyframe before the BA call
  ExtrapolateAndInterpolateKeyframePoseChanges   :45-130   for every frame in [start, end] that is not a keyframe:
      before the first / after the last keyframe   new = kf.global_T_frame * (original_kf_T_global * frame.global_T_frame)
      between keyframes prev and next              correction_x = frame.frame_T_global * kf_x.global_T_frame * original_x * frame.global_T_frame
                                                   factor = (frame - prev) / (next - prev)
                                                   t = (1 - factor) t_prev + factor t_next;  q = slerp(q_prev, factor, q_next), normalised
                                                   new = frame.global_T_frame * (q, t)
  A frame's frame_T_global is the inverse of its global_T_frame (libvis ImageFrame::SetGlobalTFrame).

SE3 products and inverses are the oracle's C restatement of Sophus (orc_se3_mul / orc_se3_inverse, oracle/badba_oracle.c).  The
quaternion interpolation is Eigen's QuaternionBase::slerp, written here from its definition in fp32:
  d = <q0, q1>;  if |d| >= 1 - eps(float):  s0 = 1 - t,  s1 = t
                 else:  theta = acos(|d|),  s0 = sin((1 - t) theta) / sin(theta),  s1 = sin(t theta) / sin(theta)
  s1 = -s1 if d < 0  (the short arc);  result = s0 q0 + s1 q1
followed by Sophus' SO3::normalize (q / |q|) behind setQuaternion.  Each fp32 operation is rounded on its own (numpy float32
scalars); the 4-term sums (dot product, squared norm) add as Eigen's SSE reduction does, (x + z) + (y + w); acos and sin are the
C library's acosf / sinf, which is what std::acos / std::sin resolve to for float.

Pinning: PARITY UNPINNED against the reference binary -- the function needs a DirectBA and an RGBDVideo of the application, and
Eigen (the slerp) is not part of the reference tree.  It is anchored on what the deformation must do by construction
(tests/test_oracle_trajectory.py): keyframes are not touched, an unchanged keyframe set changes nothing, a rigid motion of all
keyframes moves every frame with them, the interpolation tends to the one-sided extrapolation at either end, and the slerp takes
the short arc.  Only tests/ may import this module.
"""
from __future__ import annotations

import ctypes
import ctypes.util

import numpy as np

from . import cpu_oracle as O

f32 = np.float32
EPS_F = f32(np.finfo(np.float32).eps)   # NumTraits<float>::epsilon()

_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.acosf.restype = _libm.sinf.restype = ctypes.c_float
_libm.acosf.argtypes = _libm.sinf.argtypes = [ctypes.c_float]


def acosf(x):
    return f32(_libm.acosf(float(x)))


def sinf(x):
    return f32(_libm.sinf(float(x)))


def dot4(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return (a[0] * b[0] + a[2] * b[2]) + (a[1] * b[1] + a[3] * b[3])


def slerp(q0, t, q1):
    """Eigen::QuaternionBase<float>::slerp(t, q1) of q0 ({x, y, z, w}), fp32."""
    q0, q1, t = np.asarray(q0, f32), np.asarray(q1, f32), f32(t)
    one = f32(1) - EPS_F
    d = dot4(q0, q1)
    abs_d = abs(d)
    if abs_d >= one:
        scale0, scale1 = f32(1) - t, t
    else:
        theta = acosf(abs_d)
        sin_theta = sinf(theta)
        scale0 = sinf((f32(1) - t) * theta) / sin_theta
        scale1 = sinf(t * theta) / sin_theta
    if d < 0:
        scale1 = -scale1
    return np.array([scale0 * q0[i] + scale1 * q1[i] for i in range(4)], f32)


def normalized(q):
    """Sophus SO3::normalize: q / |q|, |q| = sqrt of the squared norm."""
    q = np.asarray(q, f32)
    length = f32(np.sqrt(dot4(q, q)))
    return np.array([q[i] / length for i in range(4)], f32)


def interpolate_correction(from_prev, from_next, factor):
    """The SE3f built at trajectory_deformation.cc:114-121: translation linear, rotation slerp + setQuaternion."""
    factor = f32(factor)
    a, b = np.asarray(from_prev, f32), np.asarray(from_next, f32)
    t = [(f32(1) - factor) * a[4 + i] + factor * b[4 + i] for i in range(3)]
    q = normalized(slerp(a[:4], factor, b[:4]))
    return np.concatenate([q, np.array(t, f32)]).astype(f32)


def correction(original_kf_T_global, kf_global_T_frame, global_T_other):
    """other_old_T_other_new (trajectory_deformation.cc:89-110) seen from one keyframe."""
    new_global_T_other = O.se3_mul(kf_global_T_frame, O.se3_mul(original_kf_T_global, global_T_other))
    return O.se3_mul(O.se3_inverse(global_T_other), new_global_T_other)


def extrapolate(original_kf_T_global, kf_global_T_frame, global_T_other):
    """trajectory_deformation.cc:79-86."""
    return O.se3_mul(kf_global_T_frame, O.se3_mul(original_kf_T_global, global_T_other))


def deform_trajectory(keyframe_frame_index, original_keyframe_T_global, keyframe_global_T_frame, start_frame, end_frame,
                      frame_global_T_frame):
    """ExtrapolateAndInterpolateKeyframePoseChanges on arrays; returns a new [N, 7] array (end_frame <= N - 1)."""
    idx = [int(v) for v in keyframe_frame_index]
    orig = np.asarray(original_keyframe_T_global, f32).reshape(-1, 7)
    cur = np.asarray(keyframe_global_T_frame, f32).reshape(-1, 7)
    out = np.array(frame_global_T_frame, f32, copy=True)
    K = len(idx)
    for frame in range(start_frame, end_frame + 1):
        # the keyframe at or before the frame (or the first one) and the one after it
        prev = max([k for k in range(K) if idx[k] <= frame], default=0)
        nxt = next((k for k in range(K) if idx[k] > frame), None)
        if idx[prev] == frame:
            continue
        g = out[frame].copy()
        if nxt is None or idx[prev] > frame:
            out[frame] = extrapolate(orig[prev], cur[prev], g)
        else:
            factor = f32(frame - idx[prev]) / f32(idx[nxt] - idx[prev])
            c = interpolate_correction(correction(orig[prev], cur[prev], g), correction(orig[nxt], cur[nxt], g), factor)
            out[frame] = O.se3_mul(g, c)
    return out
