"""CPU-only: the attitude prior's terms (bba_host_attitude_prior_terms, host_math.hpp AttitudePriorTerms, DESIGN §3.17) against
numpy central differences of 1/2 L theta^2(T exp(delta)), their values at theta = 0 and pi, the zero translation rows and the
yaw null direction, their robust weights, and the layout of bba_attitude_prior in the ctypes table."""
import ctypes as C

import numpy as np
import pytest

import pose_graph_oracle as P

TRIVIAL, HUBER, CAUCHY = 0, 1, 2


def _lib():
    from badslam_b200 import _lib
    return _lib.load()


def terms(d_ref, d_meas, L, pose):
    H, b, cost = np.zeros(21), np.zeros(6), C.c_double()
    f3 = lambda v: np.ascontiguousarray(v, np.float32)
    dr, dm, p = f3(d_ref), f3(d_meas), np.ascontiguousarray(pose, np.float32)
    _lib().bba_host_attitude_prior_terms(dr.ctypes.data, dm.ctypes.data, float(L), p.ctypes.data, H.ctypes.data, b.ctypes.data,
                                         C.byref(cost))
    return P.upper_to_matrix(H), b, cost.value


def half_cost(d_ref, d_meas, L, T):
    p = T[0].T @ (d_ref / np.linalg.norm(d_ref))
    m = d_meas / np.linalg.norm(d_meas)
    th = np.arctan2(np.linalg.norm(np.cross(p, m)), p @ m)
    return 0.5 * L * th * th


def setup(theta, seed):
    """A pose (as fp32 numbers, and its fp64 (R, t)), d_ref and a d_meas at angle theta from R^-1 d_ref."""
    rng = np.random.default_rng(seed)
    pose = np.float32(np.r_[P.to_array(P.se3_exp(rng.normal(0, 0.7, 6)))])
    T = P.from_array(pose)
    d_ref = np.float32(rng.normal(size=3))
    d_ref /= np.linalg.norm(d_ref)
    d_ref = np.float32(d_ref)
    p = T[0].T @ (np.float64(d_ref) / np.linalg.norm(np.float64(d_ref)))
    axis = np.cross(p, rng.normal(size=3))
    axis /= np.linalg.norm(axis)
    m = P.so3_exp(theta * axis) @ p
    return pose, T, d_ref, m


@pytest.mark.parametrize("theta", [1e-4, 0.3, 2.0, np.pi - 1e-3])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gradient_and_cost_match_central_differences(theta, seed):
    pose, T, d_ref, m = setup(theta, seed)
    d_meas = np.float32(m)
    L = 37.0
    H, b, cost = terms(d_ref, d_meas, L, pose)
    dm = np.float64(d_meas)
    want = half_cost(np.float64(d_ref), dm, L, T)
    assert cost == pytest.approx(want, rel=1e-9, abs=1e-18)
    h = 1e-6
    g = np.zeros(6)
    for i in range(6):
        e = np.zeros(6)
        e[i] = h
        g[i] = (half_cost(np.float64(d_ref), dm, L, P.mul(T, P.se3_exp(e))) - half_cost(np.float64(d_ref), dm, L, P.mul(T, P.se3_exp(-e)))) / (2 * h)
    scale = np.linalg.norm(g)
    assert np.max(np.abs(b - g)) <= 1e-6 * max(scale, 1e-300) + 1e-12 * L, (b, g)
    # H: the Gauss-Newton matrix at theta = 0, L (I - p p^T) in the rotation block
    p = T[0].T @ (np.float64(d_ref) / np.linalg.norm(np.float64(d_ref)))
    want_H = np.zeros((6, 6))
    want_H[3:, 3:] = L * (np.eye(3) - np.outer(p, p))
    assert np.max(np.abs(H - want_H)) <= 1e-12 * L


def test_hessian_near_zero_matches_central_differences():
    """At theta -> 0 the Gauss-Newton matrix is the cost's Hessian."""
    pose, T, d_ref, m = setup(1e-6, 7)
    d_meas = np.float32(m)
    L = 5.0
    H, _, _ = terms(d_ref, d_meas, L, pose)
    f = lambda d: half_cost(np.float64(d_ref), np.float64(d_meas), L, P.mul(T, P.se3_exp(d)))
    h = 1e-3
    Hn = np.zeros((6, 6))
    for i in range(6):
        for j in range(6):
            ei, ej = np.zeros(6), np.zeros(6)
            ei[i], ej[j] = h, h
            Hn[i, j] = (f(ei + ej) - f(ei - ej) - f(-ei + ej) + f(-ei - ej)) / (4 * h * h)
    assert np.max(np.abs(H - Hn)) <= 1e-5 * L


def test_finite_at_zero_and_pi():
    pose = np.float32([0, 0, 0, 1, 0.5, -1, 2])
    d = np.float32([0.0, 0.6, 0.8])
    for m, theta in ((d, 0.0), (-d, np.pi)):
        H, b, cost = terms(d, m, 2.0, pose)
        assert np.all(np.isfinite(H)) and np.all(np.isfinite(b)) and np.isfinite(cost)
        assert np.array_equal(b, np.zeros(6))   # exactly at 0 and at pi the gradient is zero
        assert cost == pytest.approx(0.5 * 2.0 * theta * theta, rel=1e-12, abs=0)
        assert np.linalg.matrix_rank(H[3:, 3:], tol=1e-9) == 2


@pytest.mark.parametrize("seed", [3, 4, 5])
def test_translation_rows_zero_and_b_orthogonal_to_yaw_axis(seed):
    pose, T, d_ref, m = setup(0.8, seed)
    H, b, _ = terms(d_ref, np.float32(m), 3.0, pose)
    assert np.array_equal(H[:3], np.zeros((3, 6))) and np.array_equal(b[:3], np.zeros(3))
    yaw = T[0].T @ np.float64(d_ref)   # R^-1 d_ref
    assert abs(b[3:] @ yaw) <= 1e-12 * np.linalg.norm(b)
    assert np.max(np.abs(H[3:, 3:] @ yaw)) <= 1e-6 * 3.0   # (fp32 d_ref vs its fp64 normalisation)


@pytest.mark.parametrize("kind,scale", [(HUBER, 0.5), (HUBER, 50.0), (CAUCHY, 0.2), (CAUCHY, 3.0)])
def test_robust_weights(kind, scale):
    """s = L theta^2 goes through the loss as a prior's s: rho / 2 and w = rho'(s) of bba_host_robust_loss."""
    import robust_pose_oracle as RP
    pose, T, d_ref, m = setup(0.4, 11)
    L = 20.0
    _, _, cost = terms(d_ref, np.float32(m), L, pose)
    s = 2.0 * cost
    assert s == pytest.approx(L * 0.4 ** 2, rel=1e-5)
    rho, w = C.c_double(), C.c_double()
    _lib().bba_host_robust_loss(kind, scale, s, C.byref(rho), C.byref(w))
    want_rho, want_w = RP.rho_weight((kind, float(np.float32(scale))), s)
    assert rho.value == pytest.approx(want_rho, rel=1e-12) and w.value == pytest.approx(want_w, rel=1e-12)
    assert (w.value < 1.0) == (kind == CAUCHY or s > scale * scale)


def test_attitude_prior_struct_layout():
    from badslam_b200 import _lib as L
    assert C.sizeof(L.AttitudePrior) == 4 * 7 + C.sizeof(L.RobustLoss) == 36
    assert L.AttitudePrior.reference_direction.offset == 0 and L.AttitudePrior.measured_direction.offset == 12
    assert L.AttitudePrior.information.offset == 24 and L.AttitudePrior.loss.offset == 28
    for name in ("bba_set_keyframe_attitude_priors", "bba_clear_keyframe_attitude_priors", "bba_get_keyframe_attitude_prior",
                 "bba_evaluate_keyframe_attitude_priors", "bba_host_attitude_prior_terms"):
        assert name in L.SYMBOLS


def test_null_pointers_write_nothing():
    H = np.full(21, 7.0)
    d = np.float32([0, 0, 1])
    _lib().bba_host_attitude_prior_terms(d.ctypes.data, d.ctypes.data, 1.0, None, H.ctypes.data, None, None)
    assert np.all(H == 7.0)
