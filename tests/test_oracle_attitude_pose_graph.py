"""The numpy oracle of the attitude priors (tests/attitude_prior_oracle.py) on the CPU: its terms are the gradient of the cost, its
Gauss-Newton optimum is scipy's least_squares optimum of the same cost, the partially held keyframe keeps its translation and yaw,
and the optimum does not depend on which keyframe is held, up to a global yaw about d_ref and a translation."""
import numpy as np
import pytest
from scipy.optimize import least_squares

import attitude_prior_oracle as A
import pose_graph_oracle as O

UP = np.array([0.0, 0.0, 1.0])


def case(K=24, per_kf=0.01, seed=2, L_att=1e4, L_chain=1e3):
    truth = O.circle(K)
    start = A.tilted(truth, per_kf, seed=seed)
    Lc = L_chain * np.eye(6)
    terms = O.odometry_chain(start, Lc)
    terms.append(O.Term(3, K - 4, O.mul(O.inv(O.pose(truth, 3)), O.pose(truth, K - 4)), Lc))
    atts = [A.Attitude(k, UP, A.tilt(truth[0][k], UP), L_att) for k in range(K)]
    return truth, start, terms, atts


def relative_and_tilts(poses):
    """What a global yaw about UP and a translation leave unchanged: every T_0^-1 T_k, and the tilts R_k^-1 UP."""
    rel = O.mul(O.inv((poses[0][0], poses[1][0])), poses)
    return rel[0], rel[1], A.tilt(poses[0], UP)


def rotation_vector(a, T):
    """theta n, the smooth residual whose squared norm is theta^2 (the scalar theta has a kink at 0)."""
    p = T[0].T @ a.d_ref
    x = np.cross(p, a.d_meas)
    sn = np.linalg.norm(x)
    return (np.arctan2(sn, p @ a.d_meas) / sn if sn > 0 else 1.0) * x


def test_blocks_are_the_gradient():
    truth, start, terms, atts = case(K=6, per_kf=0.2)
    for a in atts:
        T = O.pose(start, a.a)
        H, b, c = A.blocks(a, T)
        g = np.zeros(6)
        for i in range(6):
            e = np.zeros(6)
            e[i] = 1e-6
            g[i] = (0.5 * A.s_of(a, O.mul(T, O.se3_exp(e))) - 0.5 * A.s_of(a, O.mul(T, O.se3_exp(-e)))) / 2e-6
        assert np.allclose(b, g, rtol=1e-6, atol=1e-9 * a.L) and c == pytest.approx(0.5 * A.s_of(a, T))


def test_held_rule():
    K = 6
    terms = [O.Term(0, 1, O.from_array([0, 0, 0, 1, 1, 0, 0]), np.eye(6)), O.Term(3, 4, O.from_array([0, 0, 0, 1, 1, 0, 0]), np.eye(6))]
    atts = [A.Attitude(1, UP, UP, 1.0), A.Attitude(4, UP, UP, 1.0), A.Attitude(3, [1, 0, 0], [1, 0, 0], 1.0), A.Attitude(5, UP, UP, 1.0)]
    held, axes = A.held_keyframes(K, terms, atts, gauge=-1)
    # {0, 1}: parallel directions -> 0 held in translation and yaw; {3, 4}: not parallel -> 3 in translation only; 2 untouched;
    # 5 alone with its attitude prior -> held in translation and yaw
    assert held.tolist() == [2, 0, 1, 2, 0, 2]
    assert np.allclose(axes[0], UP) and axes[3] is None and np.allclose(axes[5], UP)
    held, _ = A.held_keyframes(K, terms, atts, gauge=1)
    assert held.tolist() == [0, 1, 1, 2, 0, 2]
    # a pose prior anchors its component: nothing held there
    held, _ = A.held_keyframes(K, terms + [O.Term(4, -1, O.from_array([0, 0, 0, 1, 0, 0, 0]), np.eye(6))], atts, gauge=-1)
    assert held.tolist() == [2, 0, 1, 0, 0, 2]


@pytest.mark.parametrize("gauge", [-1, 0])
def test_matches_scipy_least_squares(gauge):
    truth, start, terms, atts = case(K=12, per_kf=0.02)
    K = len(start[0])
    got, held, axes, cost, its = A.gauss_newton(terms, [(0, 0.0)] * len(terms), atts, start, gauge=gauge)
    assert held[0] == (1 if gauge == 0 else 2)
    # scipy over the same free directions, parametrised at the start poses
    B = [None if held[k] == 1 else (np.eye(6) if held[k] == 0 else A._basis(start[0][k], axes.get(k))) for k in range(K)]
    sizes = [0 if b is None else b.shape[1] for b in B]
    roots = [np.linalg.cholesky(t.L).T for t in terms]

    def unpack(x):
        d = np.zeros((K, 6))
        i = 0
        for k in range(K):
            if sizes[k]:
                d[k] = B[k] @ x[i:i + sizes[k]]
                i += sizes[k]
        return O.mul(start, O.se3_exp(d))

    def fun(x):
        P = unpack(x)
        r = [S @ O.residual(t, O.pose(P, t.a), None if t.b < 0 else O.pose(P, t.b)) for t, S in zip(terms, roots)]
        r += [np.sqrt(a.L) * rotation_vector(a, O.pose(P, a.a)) for a in atts]
        return np.concatenate(r)
    sol = least_squares(fun, np.zeros(sum(sizes)), xtol=1e-12, ftol=1e-14, gtol=1e-12, max_nfev=100)
    want = unpack(sol.x)
    assert cost == pytest.approx(0.5 * np.sum(sol.fun ** 2), rel=1e-9)
    for x, y in zip(relative_and_tilts(got), relative_and_tilts(want)):
        assert np.max(np.abs(x - y)) < 1e-7
    # the held keyframe keeps its translation and its yaw
    assert np.max(np.abs(got[1][0] - start[1][0])) == 0.0
    assert abs(A.yaw_about(got[0][0], start[0][0], UP)) < 1e-6
    # and the tilt drift is gone
    before, after = [np.mean(np.arccos(np.clip(np.sum(A.tilt(P[0], UP) * A.tilt(truth[0], UP), 1), -1, 1))) for P in (start, got)]
    assert after < 0.3 * before, (before, after)


def test_optimum_does_not_depend_on_the_held_keyframe():
    truth, start, terms, atts = case(K=20)
    a = A.gauss_newton(terms, [(0, 0.0)] * len(terms), atts, start, gauge=-1)[0]
    # the same graph with its keyframes renumbered so that keyframe 7 is the lowest id
    K = len(start[0])
    perm = np.r_[7:K, 0:7]
    inv = np.argsort(perm)
    t2 = [O.Term(inv[t.a], inv[t.b], t.Z, t.L) for t in terms]
    a2 = [A.Attitude(inv[x.a], x.d_ref, x.d_meas, x.L) for x in atts]
    b = A.gauss_newton(t2, [(0, 0.0)] * len(t2), a2, (start[0][perm], start[1][perm]), gauge=-1)[0]
    b = (b[0][inv], b[1][inv])
    for x, y in zip(relative_and_tilts(a), relative_and_tilts(b)):
        assert np.max(np.abs(x - y)) < 1e-7
