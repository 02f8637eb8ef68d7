"""numpy fp64 restatement of the keyframe pose graph (bba_optimize_pose_graph, DESIGN §3.14).

The reference solves its pose graph with g2o on the host; the C oracle has no such solver, so this module states the same cost
independently:
* a pose is (R [3, 3], t [3]) in fp64; poses on the library side are global_T_frame float[7] = (qx, qy, qz, qw, tx, ty, tz);
* a term is (a, b, Z, L): b = -1 is a prior on a with r = log(Z^-1 T_a), otherwise r = log(Z^-1 T_a^-1 T_b); the tangent order is
  (translation, rotation) and an update is T <- T exp(delta);
* the Jacobians are central differences of these residuals in the update's own parameters, so no closed-form Jacobian is shared
  with the library;
* `gauss_newton` runs Gauss-Newton with sparse direct solves, `held_keyframes` the held rule, `pcg_iterations` preconditioned CG
  with the block-tridiagonal part of H (the library's preconditioner) or its block diagonal.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl


# ---- SE(3) in fp64 ---------------------------------------------------------------------------------------------------------
def hat(w):
    w = np.asarray(w, np.float64)
    O = np.zeros(w.shape[:-1] + (3, 3))
    O[..., 0, 1], O[..., 0, 2] = -w[..., 2], w[..., 1]
    O[..., 1, 0], O[..., 1, 2] = w[..., 2], -w[..., 0]
    O[..., 2, 0], O[..., 2, 1] = -w[..., 1], w[..., 0]
    return O


def so3_exp(w):
    w = np.asarray(w, np.float64)
    th = np.linalg.norm(w, axis=-1)[..., None, None]
    W = hat(w)
    small = th < 1e-8
    ths = np.where(small, 1.0, th)
    a = np.where(small, 1.0 - th ** 2 / 6.0, np.sin(ths) / ths)
    b = np.where(small, 0.5 - th ** 2 / 24.0, (1.0 - np.cos(ths)) / ths ** 2)
    return np.eye(3) + a * W + b * (W @ W)


def quat_from_matrix(R):
    """Unit quaternions (x, y, z, w), w >= 0, of rotation matrices [..., 3, 3] (Shepperd's method, stable at any angle): each
    matrix takes the branch of the largest of (trace, R00, R11, R22), the first one on a tie."""
    R = np.asarray(R, np.float64)
    M = R.reshape(-1, 3, 3)
    tr = M[:, 0, 0] + M[:, 1, 1] + M[:, 2, 2]
    k = np.argmax(np.stack([tr, M[:, 0, 0], M[:, 1, 1], M[:, 2, 2]], -1), -1)
    q = np.zeros((len(M), 4))
    sel = k == 0
    s = 2.0 * np.sqrt(1.0 + tr[sel])
    Ms = M[sel]
    q[sel] = np.stack([(Ms[:, 2, 1] - Ms[:, 1, 2]) / s, (Ms[:, 0, 2] - Ms[:, 2, 0]) / s, (Ms[:, 1, 0] - Ms[:, 0, 1]) / s, s / 4], -1)
    for b in (1, 2, 3):   # the largest diagonal entry m = b - 1, then j and l in cyclic order
        m, j, l = b - 1, b % 3, (b + 1) % 3
        sel = k == b
        Ms = M[sel]
        s = 2.0 * np.sqrt(1.0 + Ms[:, m, m] - Ms[:, j, j] - Ms[:, l, l])
        q[sel, m] = s / 4
        q[sel, j] = (Ms[:, j, m] + Ms[:, m, j]) / s
        q[sel, l] = (Ms[:, l, m] + Ms[:, m, l]) / s
        q[sel, 3] = (Ms[:, l, j] - Ms[:, j, l]) / s
    q *= np.where(q[:, 3:] < 0, -1.0, 1.0)
    return q.reshape(R.shape[:-2] + (4,))


def so3_log(R):
    q = quat_from_matrix(R)
    n = np.linalg.norm(q[..., :3], axis=-1)
    th = 2.0 * np.arctan2(n, q[..., 3])
    f = np.where(n > 1e-12, th / np.where(n > 1e-12, n, 1.0), 2.0)
    return f[..., None] * q[..., :3]


def _V(w):
    th = np.linalg.norm(w, axis=-1)[..., None, None]
    W = hat(w)
    small = th < 1e-6
    ths = np.where(small, 1.0, th)
    a = np.where(small, 0.5 - th ** 2 / 24.0, (1.0 - np.cos(ths)) / ths ** 2)
    b = np.where(small, 1.0 / 6.0 - th ** 2 / 120.0, (ths - np.sin(ths)) / ths ** 3)
    return np.eye(3) + a * W + b * (W @ W)


def se3_exp(x):
    """x = (rho, phi) [..., 6] -> (R, t)."""
    x = np.asarray(x, np.float64)
    return so3_exp(x[..., 3:]), (_V(x[..., 3:]) @ x[..., :3, None])[..., 0]


def se3_log(R, t):
    w = so3_log(R)
    rho = np.linalg.solve(_V(w), np.asarray(t, np.float64)[..., None])[..., 0]
    return np.concatenate([rho, w], -1)


def mul(A, B):
    return A[0] @ B[0], (A[0] @ B[1][..., None])[..., 0] + A[1]


def inv(A):
    Rt = np.swapaxes(A[0], -1, -2)
    return Rt, -(Rt @ A[1][..., None])[..., 0]


def from_array(p):
    """float[..., 7] (qx qy qz qw tx ty tz) -> (R, t) in fp64 with the quaternion normalised."""
    p = np.asarray(p, np.float64)
    q = p[..., :4] / np.linalg.norm(p[..., :4], axis=-1, keepdims=True)
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                  2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                  2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1).reshape(p.shape[:-1] + (3, 3))
    return R, p[..., 4:].copy()


def to_array(A):
    """(R, t) -> float64[..., 7] with qw >= 0."""
    return np.concatenate([quat_from_matrix(A[0]), np.asarray(A[1], np.float64)], -1)


# ---- the cost ----------------------------------------------------------------------------------------------------------------
def upper_to_matrix(u):
    u = np.asarray(u, np.float64)
    M = np.zeros((6, 6))
    M[np.triu_indices(6)] = u
    return M + np.triu(M, 1).T


class Term:
    def __init__(self, a, b, Z, L):
        self.a, self.b = int(a), int(b)
        self.Z = (np.asarray(Z[0], np.float64), np.asarray(Z[1], np.float64)) if isinstance(Z, tuple) else from_array(Z)
        L = np.asarray(L, np.float64)
        self.L = upper_to_matrix(L) if L.shape == (21,) else L


def residual(term, Ta, Tb=None, da=None, db=None):
    """r of a term at T_a exp(da), T_b exp(db)."""
    if da is not None:
        Ta = mul(Ta, se3_exp(da))
    if term.b < 0:
        return se3_log(*mul(inv(term.Z), Ta))
    if db is not None:
        Tb = mul(Tb, se3_exp(db))
    return se3_log(*mul(inv(term.Z), mul(inv(Ta), Tb)))


def _residuals(Zi, Ta, Tb=None):
    """residual over a batch: Zi = Z^-1, Ta, Tb (R [..., 3, 3], t [..., 3]) broadcast against each other; Tb None for priors."""
    return se3_log(*mul(Zi, Ta if Tb is None else mul(inv(Ta), Tb)))


def _batch_blocks(Zi, Ta, Tb=None, h=1e-6):
    """(r [N, 6], J [N, 6, n]) of N terms of one kind (n = 6 for priors, 12 for constraints): r at (Ta, Tb), J by central
    differences in every column of (da[, db]) at once, the columns of term_jacobian."""
    n = 6 if Tb is None else 12
    steps = np.concatenate([h * np.eye(n), -h * np.eye(n)])   # [2n, n]: +h e_i, then -h e_i
    Zb = (Zi[0][:, None], Zi[1][:, None])
    Xa = se3_exp(steps[:, :6])
    Ta_p = mul((Ta[0][:, None], Ta[1][:, None]), Xa)
    if Tb is None:
        rp = _residuals(Zb, Ta_p)
    else:
        Tb_p = mul((Tb[0][:, None], Tb[1][:, None]), se3_exp(steps[:, 6:]))
        rp = _residuals(Zb, Ta_p, Tb_p)
    J = np.swapaxes(rp[:, :n] - rp[:, n:], -1, -2) / (2 * h)
    return _residuals(Zi, Ta, Tb), J


def _stack(terms):
    """(a [N], b [N], Z^-1 (R [N, 3, 3], t [N, 3])) of a list of terms."""
    a = np.array([t.a for t in terms], np.int64)
    b = np.array([t.b for t in terms], np.int64)
    Zi = inv((np.array([t.Z[0] for t in terms]).reshape(-1, 3, 3), np.array([t.Z[1] for t in terms]).reshape(-1, 3)))
    return a, b, Zi


def _linearise(terms, poses, jacobians=True):
    """Every term's residual r [6] and, with `jacobians`, its term_jacobian J, in term order.  The terms of one kind are
    evaluated together, each with term_blocks' own arithmetic, so the values are the per-term ones bit for bit."""
    rs, Js = [None] * len(terms), [None] * len(terms)
    if not terms:
        return rs, Js
    a, b, Zi = _stack(terms)
    for sel in (np.nonzero(b < 0)[0], np.nonzero(b >= 0)[0]):
        if len(sel) == 0:
            continue
        Z = (Zi[0][sel], Zi[1][sel])
        Ta = (poses[0][a[sel]], poses[1][a[sel]])
        Tb = None if b[sel[0]] < 0 else (poses[0][b[sel]], poses[1][b[sel]])
        r, J = _batch_blocks(Z, Ta, Tb) if jacobians else (_residuals(Z, Ta, Tb), [None] * len(sel))
        for i, n in enumerate(sel):
            rs[n], Js[n] = r[i], J[i]
    return rs, Js


def term_jacobian(term, Ta, Tb=None, h=1e-6):
    """[6, 6] (prior) or [6, 12] (constraint): central differences of the residual in (da[, db])."""
    one = lambda T: None if T is None else (np.asarray(T[0], np.float64)[None], np.asarray(T[1], np.float64)[None])
    return _batch_blocks(_stack([term])[2], one(Ta), None if term.b < 0 else one(Tb), h)[1][0]


def term_blocks(term, Ta, Tb=None):
    """(H = J^T L J, b = J^T L r, cost = r^T L r / 2) in fp64."""
    r = residual(term, Ta, Tb)
    J = term_jacobian(term, Ta, Tb)
    return J.T @ term.L @ J, J.T @ term.L @ r, 0.5 * r @ term.L @ r


def total_cost(terms, poses):
    c = 0.0
    for t, r in zip(terms, _linearise(terms, poses, jacobians=False)[0]):
        c += 0.5 * r @ t.L @ r
    return c


def pose(poses, k):
    return poses[0][k], poses[1][k]


def odometry_chain(poses, L):
    """The chain edges (k, k + 1) at the given poses: Z = T_k^-1 T_{k+1}."""
    K = len(poses[0])
    return [Term(k, k + 1, mul(inv(pose(poses, k)), pose(poses, k + 1)), L) for k in range(K - 1)]


def held_keyframes(K, terms, gauge):
    """The held rule: the gauge, every keyframe no term touches, and the lowest id of every connected component of the binary
    terms that holds neither the gauge nor a prior."""
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
    anchored = set(find(t.a) for t in terms if t.b < 0)
    if gauge >= 0:
        anchored.add(find(gauge))
    held = np.zeros(K, bool)
    seen = set()
    for k in range(K):
        r = find(k)
        first = r not in seen
        seen.add(r)
        held[k] = k == gauge or not touched[k] or (first and r not in anchored)
    return held


def normal_equations(terms, poses, held):
    """Sparse H [6K, 6K] and b [6K] with held rows / columns removed (their indices: free)."""
    K = len(poses[0])
    rows, cols, vals = [], [], []
    b = np.zeros(6 * K)
    for t, r, J in zip(terms, *_linearise(terms, poses)):   # term_blocks' H and b of every term, summed in term order
        if t.b < 0:
            idx = np.arange(6 * t.a, 6 * t.a + 6)
        else:
            idx = np.r_[6 * t.a:6 * t.a + 6, 6 * t.b:6 * t.b + 6]
        ii, jj = np.meshgrid(idx, idx, indexing="ij")
        rows.append(ii.ravel())
        cols.append(jj.ravel())
        vals.append((J.T @ t.L @ J).ravel())
        b[idx] += J.T @ t.L @ r
    H = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * K, 6 * K))
    free = np.repeat(~held, 6)
    return H[free][:, free], b[free], np.nonzero(free)[0]


def gauss_newton(terms, poses, gauge=0, max_iterations=50, step_tol=1e-12):
    """The optimum of the cost over the free keyframes, fp64: (poses, held, cost, iterations)."""
    R, t = np.array(poses[0], np.float64), np.array(poses[1], np.float64)
    K = len(R)
    held = held_keyframes(K, terms, gauge)
    cost = total_cost(terms, (R, t))
    its = 0
    for its in range(1, max_iterations + 1):
        H, b, idx = normal_equations(terms, (R, t), held)
        if H.shape[0] == 0:
            break
        delta = np.zeros(6 * K)
        delta[idx] = spl.spsolve(H.tocsc(), -b)
        d = delta.reshape(K, 6)
        Rn, tn = mul((R, t), se3_exp(d))
        new_cost = total_cost(terms, (Rn, tn))
        if new_cost > cost:
            break
        R, t, cost = Rn, tn, new_cost
        if np.max(np.abs(delta)) <= step_tol:
            break
    return (R, t), held, cost, its


def least_squares_whitened(terms, poses, held):
    """The whitened residuals L^(1/2) r of every term as a function of the free keyframes' updates, for scipy's optimiser."""
    K = len(poses[0])
    free = np.nonzero(~held)[0]
    roots = []
    for t in terms:
        w, V = np.linalg.eigh(t.L)
        roots.append((V * np.sqrt(np.maximum(w, 0.0))) @ V.T)

    def unpack(x):
        R, tt = np.array(poses[0]), np.array(poses[1])
        d = np.zeros((K, 6))
        d[free] = x.reshape(-1, 6)
        return mul((R, tt), se3_exp(d))

    def fun(x):
        P = unpack(x)
        return np.concatenate([S @ residual(t, pose(P, t.a), None if t.b < 0 else pose(P, t.b)) for t, S in zip(terms, roots)])
    return fun, unpack, 6 * len(free)


# ---- the preconditioned linear solve -----------------------------------------------------------------------------------------
def block_tridiagonal(H):
    """The blocks (i, j) with |i - j| <= 1 of H (6x6 blocks)."""
    C = H.tocoo()
    m = np.abs(C.row // 6 - C.col // 6) <= 1
    return sp.csc_matrix((C.data[m], (C.row[m], C.col[m])), shape=H.shape)


def block_diagonal(H):
    C = H.tocoo()
    m = C.row // 6 == C.col // 6
    return sp.csc_matrix((C.data[m], (C.row[m], C.col[m])), shape=H.shape)


def pcg_iterations(H, b, M, tol=1e-10, max_iterations=None):
    """Iterations of preconditioned CG on H x = -b from x = 0 to ||r|| <= tol ||b||, M applied by a sparse LU."""
    lu = spl.splu(M.tocsc())
    n = H.shape[0]
    max_iterations = max_iterations or 6 * n
    x = np.zeros(n)
    r = -b.copy()
    nb = np.linalg.norm(b)
    if nb == 0.0:
        return 0, x
    z = lu.solve(r)
    p = z.copy()
    rz = r @ z
    for it in range(1, max_iterations + 1):
        q = H @ p
        alpha = rz / (p @ q)
        x += alpha * p
        r -= alpha * q
        if np.linalg.norm(r) <= tol * nb:
            return it, x
        z = lu.solve(r)
        rz_next = r @ z
        p = z + rz_next / rz * p
        rz = rz_next
    return max_iterations, x


# ---- synthetic graphs ----------------------------------------------------------------------------------------------------------
def circle(K, radius=5.0):
    """Keyframes on a horizontal circle, each turned to face along it: (R, t) [K]."""
    th = 2 * np.pi * np.arange(K) / K
    w = np.zeros((K, 3))
    w[:, 2] = th
    t = np.stack([radius * np.cos(th), radius * np.sin(th), np.zeros(K)], -1)
    return so3_exp(w), t


def drift(truth, sigma_t, sigma_r, seed=0):
    """The truth's relative motions, each perturbed by exp(noise) and chained from keyframe 0: a drift that grows along it."""
    rng = np.random.default_rng(seed)
    K = len(truth[0])
    R, t = [truth[0][0]], [truth[1][0]]
    for k in range(K - 1):
        rel = mul(inv(pose(truth, k)), pose(truth, k + 1))
        noise = se3_exp(np.r_[rng.normal(0, sigma_t, 3), rng.normal(0, sigma_r, 3)])
        n = mul((R[-1], t[-1]), mul(rel, noise))
        R.append(n[0])
        t.append(n[1])
    return np.array(R), np.array(t)


def random_loops(K, L, seed=0):
    """L distinct pairs (a, b) with b - a > 1."""
    rng = np.random.default_rng(seed)
    out = set()
    while len(out) < L:
        a, b = sorted(rng.choice(K, 2, replace=False).tolist())
        if b - a > 1:
            out.add((a, b))
    return sorted(out)
