"""numpy fp64 restatement of the attitude priors (DESIGN §3.17), on top of tests/pose_graph_oracle.py and robust_pose_oracle.py.

* an attitude prior (k, d_ref, d_meas, L, loss) costs rho(s) / 2 with s = L theta^2, theta the angle between p = R_k^-1 d_ref and
  d_meas (both unit);
* its terms for the update T exp(delta) (`blocks`): b = L theta n in the rotation rows, n = (p x m) / |p x m| (0 where p x m = 0),
  H = L (I - p p^T) in the rotation block, zero translation rows;
* the held rule (`held_keyframes`): pose_graph_oracle's, except that in a component with neither the gauge nor a pose prior but
  with attitude priors the lowest id is held only in translation and, when the component's reference directions are parallel, in
  rotation about them (held = 2, axis = that direction or None);
* `gauss_newton` is IRLS Gauss-Newton over the free directions: a partially held keyframe's update is B y with B an orthonormal
  basis of the rotations perpendicular to R^-1 axis (or of every rotation) at the current pose.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import pose_graph_oracle as P
import robust_pose_oracle as RP


class Attitude:
    def __init__(self, k, d_ref, d_meas, L, loss=(0, 0.0)):
        self.a, self.b = int(k), -2
        self.d_ref = np.asarray(d_ref, np.float64) / np.linalg.norm(d_ref)
        self.d_meas = np.asarray(d_meas, np.float64) / np.linalg.norm(d_meas)
        self.L = float(L)
        self.loss = loss


def angle(term, T):
    p = T[0].T @ term.d_ref
    m = term.d_meas
    return np.arctan2(np.linalg.norm(np.cross(p, m)), p @ m)


def s_of(term, T):
    return term.L * angle(term, T) ** 2


def blocks(term, T):
    """(H [6, 6], b [6], cost) of the closed form."""
    p = T[0].T @ term.d_ref
    x = np.cross(p, term.d_meas)
    sn = np.linalg.norm(x)
    th = np.arctan2(sn, p @ term.d_meas)
    H, b = np.zeros((6, 6)), np.zeros(6)
    H[3:, 3:] = term.L * (np.eye(3) - np.outer(p, p))
    b[3:] = term.L * (th / sn if sn > 0 else 1.0) * x
    return H, b, 0.5 * term.L * th * th


def tilt(R, d):
    """The direction d of the map frame in the camera frames of R [..., 3, 3]."""
    return np.swapaxes(R, -1, -2) @ d


def yaw_about(R_new, R_old, d):
    """The twist angle about d (map frame) of R_new R_old^T."""
    q = P.quat_from_matrix(R_new @ R_old.T)
    return 2.0 * np.arctan2(q[:3] @ d, q[3])


def total_cost(terms, losses, atts, poses):
    c = RP.total_cost(terms, losses, poses) if terms else 0.0
    return c + sum(0.5 * RP.rho_weight(a.loss, s_of(a, P.pose(poses, a.a)))[0] for a in atts)


def held_keyframes(K, terms, atts, gauge):
    """(held [K] in {0, 1, 2}, axes {k: unit map-frame axis or None} of the keyframes with held = 2)."""
    parent = list(range(K))

    def find(k):
        while parent[k] != k:
            parent[k] = parent[parent[k]]
            k = parent[k]
        return k
    touched = np.zeros(K, bool)
    for t in terms:
        touched[t.a] = True
        if t.b >= 0:
            touched[t.b] = True
            ra, rb = find(t.a), find(t.b)
            if ra != rb:
                parent[max(ra, rb)] = min(ra, rb)
    for a in atts:
        touched[a.a] = True
    anchored = set(find(t.a) for t in terms if t.b < 0)
    if gauge >= 0:
        anchored.add(find(gauge))
    dirs = {}
    for a in sorted(atts, key=lambda a: a.a):
        dirs.setdefault(find(a.a), []).append(a.d_ref)
    held = np.zeros(K, np.int32)
    axes = {}
    seen = set()
    for k in range(K):
        r = find(k)
        first = r not in seen
        seen.add(r)
        lowest_free = first and r not in anchored
        if k == gauge or not touched[k] or (lowest_free and r not in dirs):
            held[k] = 1
        elif lowest_free:
            held[k] = 2
            d0 = dirs[r][0]
            axes[k] = d0 if all(np.linalg.norm(np.cross(d, d0)) <= 1e-6 for d in dirs[r]) else None
    return held, axes


def _basis(R, axis):
    """[6, m]: the free directions of a partially held keyframe's update."""
    if axis is None:
        B = np.zeros((6, 3))
        B[3:, :] = np.eye(3)
        return B
    u = R.T @ axis
    e = np.eye(3)[np.argmin(np.abs(u))]
    v1 = np.cross(u, e)
    v1 /= np.linalg.norm(v1)
    v2 = np.cross(u, v1)
    B = np.zeros((6, 2))
    B[3:, 0], B[3:, 1] = v1, v2
    return B


def normal_equations(terms, losses, atts, poses, held, axes):
    """IRLS H and b over the free directions, and the [6K, n] map from them to the keyframes' updates."""
    K = len(poses[0])
    Hf, bf, _ = RP.normal_equations(terms, losses, poses, np.zeros(K, bool)) if terms else (sp.csr_matrix((6 * K, 6 * K)), np.zeros(6 * K), None)
    Hd = Hf.toarray()
    b = bf.copy()
    for a in atts:
        T = P.pose(poses, a.a)
        H, g, c = blocks(a, T)
        w = RP.rho_weight(a.loss, 2.0 * c)[1]
        i = 6 * a.a
        Hd[i:i + 6, i:i + 6] += w * H
        b[i:i + 6] += w * g
    cols = []
    for k in range(K):
        if held[k] == 1:
            continue
        B = np.eye(6) if held[k] == 0 else _basis(poses[0][k], axes[k])
        E = np.zeros((6 * K, B.shape[1]))
        E[6 * k:6 * k + 6] = B
        cols.append(E)
    S = np.concatenate(cols, 1) if cols else np.zeros((6 * K, 0))
    return S.T @ Hd @ S, S.T @ b, S


def gauss_newton(terms, losses, atts, poses, gauge=0, max_iterations=50, step_tol=1e-12):
    """(poses, held, axes, robust cost, iterations) of IRLS Gauss-Newton, fp64."""
    R, t = np.array(poses[0], np.float64), np.array(poses[1], np.float64)
    K = len(R)
    held, axes = held_keyframes(K, terms, atts, gauge)
    cost = total_cost(terms, losses, atts, (R, t))
    its = 0
    for its in range(1, max_iterations + 1):
        H, b, S = normal_equations(terms, losses, atts, (R, t), held, axes)
        if H.shape[0] == 0:
            break
        delta = S @ spl.spsolve(sp.csc_matrix(H), -b)
        Rn, tn = P.mul((R, t), P.se3_exp(delta.reshape(K, 6)))
        new_cost = total_cost(terms, losses, atts, (Rn, tn))
        if new_cost > cost:
            break
        R, t, cost = Rn, tn, new_cost
        if np.max(np.abs(delta)) <= step_tol:
            break
    return (R, t), held, axes, cost, its


def tilted(truth, roll_pitch_per_kf, seed=0):
    """The truth with a tilt drift that grows along the keyframes: keyframe k turned by k * roll_pitch_per_kf about random
    horizontal axes (z is up), each keyframe's position kept."""
    rng = np.random.default_rng(seed)
    R, t = np.array(truth[0]), np.array(truth[1])
    K = len(R)
    acc = np.eye(3)
    out = np.empty_like(R)
    for k in range(K):
        if k:
            phi = rng.uniform(0, 2 * np.pi)
            acc = P.so3_exp(roll_pitch_per_kf * np.array([np.cos(phi), np.sin(phi), 0.0])) @ acc
        out[k] = acc @ R[k]
    return out, t
