"""numpy fp64 restatement of the robust losses on the pose terms (DESIGN §3.15), on top of tests/pose_graph_oracle.py.

* a loss is (type, scale) with bba_loss_type's numbers: 0 trivial, 1 Huber, 2 Cauchy; scale = delta in units of sqrt(s);
* a term with s = r^T L r costs rho(s) / 2, with Ceres' rho (scipy's least_squares with f_scale = delta uses the same);
* `gauss_newton` is IRLS Gauss-Newton: every term's H and b are scaled by w = rho'(s) at the current poses, the step is accepted
  when the robust cost does not rise, and the held rule is pose_graph_oracle's.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import pose_graph_oracle as P

TRIVIAL, HUBER, CAUCHY = 0, 1, 2


def rho_weight(loss, s):
    """(rho(s), rho'(s)) of loss = (type, scale), closed forms in fp64."""
    kind, scale = loss
    d2 = float(scale) ** 2
    if kind == HUBER and s > d2:
        return 2.0 * scale * np.sqrt(s) - d2, scale / np.sqrt(s)
    if kind == CAUCHY:
        return d2 * np.log1p(s / d2), 1.0 / (1.0 + s / d2)
    return s, 1.0


def term_s(term, poses):
    r = P.residual(term, P.pose(poses, term.a), None if term.b < 0 else P.pose(poses, term.b))
    return float(r @ term.L @ r)


def total_cost(terms, losses, poses):
    """sum rho(s) / 2 over the terms."""
    return sum(0.5 * rho_weight(l, term_s(t, poses))[0] for t, l in zip(terms, losses))


def weights(terms, losses, poses):
    return np.array([rho_weight(l, term_s(t, poses))[1] for t, l in zip(terms, losses)])


def normal_equations(terms, losses, poses, held):
    """pose_graph_oracle.normal_equations with every term's H and b scaled by its weight at `poses`."""
    K = len(poses[0])
    rows, cols, vals = [], [], []
    b = np.zeros(6 * K)
    for t, loss in zip(terms, losses):
        if t.b < 0:
            H, g, c = P.term_blocks(t, P.pose(poses, t.a))
            idx = np.arange(6 * t.a, 6 * t.a + 6)
        else:
            H, g, c = P.term_blocks(t, P.pose(poses, t.a), P.pose(poses, t.b))
            idx = np.r_[6 * t.a:6 * t.a + 6, 6 * t.b:6 * t.b + 6]
        w = rho_weight(loss, 2.0 * c)[1]
        ii, jj = np.meshgrid(idx, idx, indexing="ij")
        rows.append(ii.ravel())
        cols.append(jj.ravel())
        vals.append((w * H).ravel())
        b[idx] += w * g
    H = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * K, 6 * K))
    free = np.repeat(~held, 6)
    return H[free][:, free], b[free], np.nonzero(free)[0]


def gauss_newton(terms, losses, poses, gauge=0, max_iterations=50, step_tol=1e-12):
    """IRLS Gauss-Newton over the free keyframes, fp64: (poses, held, robust cost, iterations).  With every loss trivial it takes
    the steps of pose_graph_oracle.gauss_newton."""
    R, t = np.array(poses[0], np.float64), np.array(poses[1], np.float64)
    K = len(R)
    held = P.held_keyframes(K, terms, gauge)
    cost = total_cost(terms, losses, (R, t))
    its = 0
    for its in range(1, max_iterations + 1):
        H, b, idx = normal_equations(terms, losses, (R, t), held)
        if H.shape[0] == 0:
            break
        delta = np.zeros(6 * K)
        delta[idx] = spl.spsolve(H.tocsc(), -b)
        Rn, tn = P.mul((R, t), P.se3_exp(delta.reshape(K, 6)))
        new_cost = total_cost(terms, losses, (Rn, tn))
        if new_cost > cost:
            break
        R, t, cost = Rn, tn, new_cost
        if np.max(np.abs(delta)) <= step_tol:
            break
    return (R, t), held, cost, its


def cost_gradient(terms, losses, poses, held, h=1e-6):
    """Central-difference gradient of the robust total cost in the free keyframes' tangent updates T <- T exp(delta) [6 free]."""
    K = len(poses[0])
    free = np.nonzero(~held)[0]
    g = np.zeros(6 * len(free))
    for i in range(len(g)):
        d = np.zeros((K, 6))
        d[free[i // 6], i % 6] = h
        up = total_cost(terms, losses, P.mul(poses, P.se3_exp(d)))
        down = total_cost(terms, losses, P.mul(poses, P.se3_exp(-d)))
        g[i] = (up - down) / (2 * h)
    return g
