"""CPU-only: the product's HOST arithmetic (badslam_b200/csrc/host_math.hpp, including the frustum code, exported through the
device-free bba_host_* entry points of include/badba.h) against the oracle's independent C versions, numpy and closed forms."""
import ctypes as C

import numpy as np
import pytest

from badslam_b200 import _lib
from badslam_b200 import scene as S
from oracle import cpu_oracle as O


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def f32(a):
    return np.ascontiguousarray(a, np.float32)


def call_pose(fn, *args, n_out=7):
    out = np.zeros(n_out, np.float32)
    fn(*[f32(a).ctypes.data for a in args], out.ctypes.data)
    return out


def same_rotation(qa, qb, tol):
    return min(np.abs(qa - qb).max(), np.abs(qa + qb).max()) < tol      # q and -q are the same rotation


def test_se3_exp_log_compose_inverse_match_the_oracle(lib):
    """Sophus se3.hpp:293-313 (exp), :435-468 (log), :203-207 (product), :127-130 (inverse)."""
    rng = np.random.default_rng(0)
    tangents = np.concatenate([rng.normal(0, 1.0, (200, 6)), rng.normal(0, 1e-4, (50, 6)), np.zeros((1, 6)),
                               [[0.1, -0.2, 0.3, 3.1, 0, 0]], [[1, 2, 3, 0, 0, 1e-9]]]).astype(np.float32)
    for a in tangents:
        T = call_pose(lib.bba_host_se3_exp, a)
        T_o = O.se3_exp(a)
        assert same_rotation(T[:4], T_o[:4], 2e-6) and np.abs(T[4:] - T_o[4:]).max() < 1e-5 * max(1.0, np.abs(T_o[4:]).max())
        assert abs(np.linalg.norm(T[:4]) - 1) < 1e-6
        back = call_pose(lib.bba_host_se3_log, T, n_out=6)
        if np.linalg.norm(a[3:]) < 3.0:      # log is unique below pi
            assert np.abs(back - a).max() < 2e-4 * max(1.0, np.abs(a).max()), (a, back)
        assert np.abs(back - O.se3_log(T)).max() < 2e-5 * max(1.0, np.abs(a).max())
    for _ in range(100):
        A = call_pose(lib.bba_host_se3_exp, rng.normal(0, 1, 6))
        B = call_pose(lib.bba_host_se3_exp, rng.normal(0, 1, 6))
        AB, AB_o = call_pose(lib.bba_host_se3_compose, A, B), O.se3_mul(A, B)
        assert same_rotation(AB[:4], AB_o[:4], 2e-6) and np.abs(AB[4:] - AB_o[4:]).max() < 1e-5
        inv, inv_o = call_pose(lib.bba_host_se3_inverse, A), O.se3_inverse(A)
        assert same_rotation(inv[:4], inv_o[:4], 2e-6) and np.abs(inv[4:] - inv_o[4:]).max() < 1e-5
        ident = call_pose(lib.bba_host_se3_compose, A, inv)
        assert same_rotation(ident[:4], np.array([0, 0, 0, 1], np.float32), 2e-6) and np.abs(ident[4:]).max() < 1e-5


def test_pose_update_convergence_criterion(lib):
    """convergence_analysis.h:45-52: |(x_t, 10 x_r)|^2 < 1e-6."""
    x = lambda *v: f32(v).ctypes.data
    assert lib.bba_host_pose_update_converged(x(0, 0, 0, 0, 0, 0)) == 1
    assert lib.bba_host_pose_update_converged(x(9.9e-4, 0, 0, 0, 0, 0)) == 1
    assert lib.bba_host_pose_update_converged(x(1.01e-3, 0, 0, 0, 0, 0)) == 0
    assert lib.bba_host_pose_update_converged(x(0, 0, 0, 9.9e-5, 0, 0)) == 1      # rotations weigh ten times more
    assert lib.bba_host_pose_update_converged(x(0, 0, 0, 1.01e-4, 0, 0)) == 0
    assert lib.bba_host_pose_update_converged(x(6e-4, 6e-4, 6e-4, 0, 0, 0)) == 0


@pytest.mark.parametrize("n", [4, 5, 6])
def test_ldlt_solve_matches_numpy(lib, n):
    """The fp64 solve standing in for Eigen's ldlt() (direct_ba_alternating.cc:206, kernel_opt_intrinsics.cc:171,272)."""
    rng = np.random.default_rng(n)
    iu = np.triu_indices(n)
    for trial in range(50):
        M = rng.normal(size=(n + 3, n))
        A = M.T @ M * 10.0 ** rng.uniform(-3, 6)
        if trial % 5 == 0:
            A = A + 1e6 * np.diag(rng.random(n))          # badly scaled diagonals: pivoting matters
        b = rng.normal(size=n)
        x = np.zeros(n)
        upper = np.ascontiguousarray(A[iu])
        assert lib.bba_host_solve_ldlt(n, upper.ctypes.data, b.ctypes.data, x.ctypes.data) == 1
        want = np.linalg.solve(A, b)
        assert np.abs(x - want).max() <= 1e-9 * np.linalg.cond(A) * np.abs(want).max() + 1e-300
    # a rank-deficient system (an unobserved direction): x = 0 along it, the rest solved
    A = np.diag(np.arange(1.0, n + 1))
    A[2, 2] = 0.0
    b = np.ones(n)
    x = np.full(n, 7.0)
    assert lib.bba_host_solve_ldlt(n, np.ascontiguousarray(A[iu]).ctypes.data, b.ctypes.data, x.ctypes.data) == 1
    want = np.array([0.0 if i == 2 else 1.0 / (i + 1) for i in range(n)])
    assert np.allclose(x, want, atol=1e-15)
    assert lib.bba_host_solve_ldlt(7, np.zeros(28).ctypes.data, np.zeros(7).ctypes.data, np.zeros(7).ctypes.data) == 0


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_frustum_covisibility_matches_the_oracle(lib, name):
    """DetermineNewKeyframeCoVisibility (direct_ba.cc:231-249) through CameraFrustum::Intersects (camera_frustum.h:73-143)."""
    sc = S.make_scene(S.config_by_name(name))
    orc = O.Oracle(sc)
    K = sc.cfg.num_keyframes
    Kd = f32(sc.depth_K)
    hits = 0
    for i in range(K):
        for j in range(K):
            if i == j:
                continue
            got = lib.bba_host_frusta_intersect(Kd.ctypes.data, sc.cfg.width, sc.cfg.height, f32(sc.poses_init[i]).ctypes.data,
                                                float(sc.min_depth[i]), float(sc.max_depth[i]), f32(sc.poses_init[j]).ctypes.data,
                                                float(sc.min_depth[j]), float(sc.max_depth[j]))
            assert got == int(orc.covis[i, j]), (i, j)
            hits += got
    assert hits > 0
    # two cameras back to back, and far apart: no intersection; a camera with itself: intersection
    eye = f32([0, 0, 0, 1, 0, 0, 0])
    turned = f32([0, 1, 0, 0, 0, 0, -0.5])       # 180 degrees about y, half a metre behind
    far = f32([0, 0, 0, 1, 100, 0, 0])
    args = lambda a, b: (Kd.ctypes.data, sc.cfg.width, sc.cfg.height, a.ctypes.data, 0.5, 3.0, b.ctypes.data, 0.5, 3.0)
    assert lib.bba_host_frusta_intersect(*args(eye, eye)) == 1
    assert lib.bba_host_frusta_intersect(*args(eye, turned)) == 0
    assert lib.bba_host_frusta_intersect(*args(eye, far)) == 0
