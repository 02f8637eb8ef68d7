"""CPU-only: the host steps of the loop-closure verification (bba_verify_loop_closures, DESIGN §3.16).

* bba_host_average_pose (AveragePose, util.cc:110-128) against the oracle's scipy SVD: the identity, three equal poses, spreads
  of +-5 deg, a spread around a rotation of almost pi, one pose and two poses;
* bba_host_loop_agreement just inside and just outside each threshold, for rotation and translation, and the reference's order:
  the pairs (0, 1), (0, 2), (1, 2), the rotation of a pair before its translation; a roll about the optical axis is not seen;
* the neighbour rule of loop_detector.cc:455-496 at matched = 0, K - 2 and K - 1, and the composition of the initial and the
  refined estimates, in the oracle the GPU tests compare against;
* the ctypes layouts of the three new structs against their C layout.
"""
import ctypes as C

import numpy as np
import pytest

import loop_verification_oracle as O


def _lib():
    from badslam_b200 import _lib
    return _lib.load()


def _exp(w, t=(0.0, 0.0, 0.0)):
    """float[7] pose of rotation vector w and translation t."""
    from scipy.spatial.transform import Rotation
    q = Rotation.from_rotvec(np.asarray(w, np.float64)).as_quat()
    return np.concatenate([q, t]).astype(np.float32)


def average(poses):
    P = np.ascontiguousarray(poses, np.float32).reshape(-1, 7)
    out = np.zeros(7, np.float32)
    _lib().bba_host_average_pose(len(P), P.ctypes.data, out.ctypes.data)
    return out


def agreement(poses, max_angle=0.0, max_translation=0.0):
    P = np.ascontiguousarray(poses, np.float32).reshape(21)
    out = np.zeros(7, np.float32)
    a, t = C.c_float(), C.c_float()
    st = _lib().bba_host_loop_agreement(P.ctypes.data, max_angle, max_translation, out.ctypes.data, C.byref(a), C.byref(t))
    return st, a.value, t.value, out


def _close(a, b, t_tol=2e-6, r_tol=2e-6):
    dt, dr = O.same_pose(a, b)
    assert dt < t_tol and dr < r_tol, (a, b, dt, dr)


def test_average_of_identities_and_equal_poses():
    ident = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
    assert np.array_equal(average([ident] * 3), ident)
    p = _exp([0.3, -0.2, 0.1], [1.0, -2.0, 0.5])
    got = average([p] * 3)
    _close(got, p)
    _close(average([p]), p)


@pytest.mark.parametrize("seed", range(8))
def test_average_against_scipy(seed):
    rng = np.random.default_rng(seed)
    base = rng.normal(0, 1.0, 3)
    poses = [_exp(base + rng.uniform(-1, 1, 3) * np.radians(5), rng.normal(0, 0.5, 3)) for _ in range(3)]
    want = O.average_pose(poses)
    _close(average(poses), want)
    # two poses: the midpoint rotation
    _close(average(poses[:2]), O.average_pose(poses[:2]))


def test_average_near_pi():
    axis = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    poses = [_exp(axis * (np.pi - 0.01) + d) for d in (np.zeros(3), [0.02, 0, 0], [0, -0.02, 0.01])]
    _close(average(poses), O.average_pose(poses), r_tol=1e-5)


def test_average_writes_nothing_for_no_pose():
    out = np.full(7, 7.0, np.float32)
    _lib().bba_host_average_pose(0, np.zeros(7, np.float32).ctypes.data, out.ctypes.data)
    assert np.all(out == 7.0)


ROT_LIMIT = np.float32(np.pi / 180.0 * 10.0)


def _spread(rot2=None, trans2=None, which=2):
    """Three poses: 0 and 1 equal, `which` tilted by rot2 about the x axis (which moves the optical axis) and shifted by trans2."""
    poses = [_exp([0.1, 0.2, 0.3], [0.5, -0.4, 1.2]) for _ in range(3)]
    R0 = O.to_T(poses[0])
    T = R0.copy()
    if rot2 is not None:
        from scipy.spatial.transform import Rotation
        T[:3, :3] = R0[:3, :3] @ Rotation.from_rotvec([rot2, 0, 0]).as_matrix()
    if trans2 is not None:
        T[:3, 3] = R0[:3, 3] + np.array(trans2)
    poses[which] = O.from_T(T).astype(np.float32)
    return poses


@pytest.mark.parametrize("which", [1, 2])
def test_rotation_threshold(which):
    for factor, want in ((0.995, O.ACCEPTED), (1.005, O.ROTATION_DISAGREES)):
        poses = _spread(rot2=float(ROT_LIMIT) * factor, which=which)
        st, a, t, _ = agreement(poses)
        assert st == want, (factor, st, a)
        assert st == O.agreement(poses)[0]
        assert abs(a - O.agreement(poses)[1]) < 1e-5
    # a caller's own limit
    poses = _spread(rot2=0.05, which=which)
    assert agreement(poses, max_angle=0.051)[0] == O.ACCEPTED
    assert agreement(poses, max_angle=0.049)[0] == O.ROTATION_DISAGREES


@pytest.mark.parametrize("which", [1, 2])
def test_translation_threshold(which):
    d = np.array([0.6, -0.48, 0.64])   # unit vector
    for dist, want in ((0.0199, O.ACCEPTED), (0.0201, O.TRANSLATION_DISAGREES)):
        poses = _spread(trans2=d * dist, which=which)
        st, a, t, _ = agreement(poses)
        assert st == want, (dist, st, t)
        assert st == O.agreement(poses)[0]
        assert abs(t - dist) < 1e-5
    poses = _spread(trans2=d * 0.1, which=which)
    assert agreement(poses, max_translation=0.101)[0] == O.ACCEPTED
    assert agreement(poses, max_translation=0.099)[0] == O.TRANSLATION_DISAGREES


def test_order_of_the_tests():
    # pose 1 disagrees in translation with pose 0, pose 2 in rotation: pair (0, 1) comes first -> TRANSLATION
    poses = _spread(trans2=[0.05, 0, 0], which=1)
    from scipy.spatial.transform import Rotation
    T = O.to_T(poses[0])
    T[:3, :3] = T[:3, :3] @ Rotation.from_rotvec([0.3, 0, 0]).as_matrix()
    poses[2] = O.from_T(T).astype(np.float32)
    st, a, t, _ = agreement(poses)
    assert st == O.TRANSLATION_DISAGREES == O.agreement(poses)[0]
    assert a > 0.29 and t > 0.049   # the largest distances over all pairs
    # both in one pair: the rotation is tested first
    poses = _spread(rot2=0.3, trans2=[0.05, 0, 0], which=1)
    assert agreement(poses)[0] == O.ROTATION_DISAGREES == O.agreement(poses)[0]


def test_roll_about_the_optical_axis_is_not_seen():
    from scipy.spatial.transform import Rotation
    poses = _spread()
    T = O.to_T(poses[0])
    T[:3, :3] = T[:3, :3] @ Rotation.from_rotvec([0, 0, 0.5]).as_matrix()
    poses[2] = O.from_T(T).astype(np.float32)
    st, a, _, avg = agreement(poses)
    assert st == O.ACCEPTED and a < 1e-3
    _close(avg, O.average_pose(poses), r_tol=1e-5)


def test_agreement_average_is_average_pose():
    rng = np.random.default_rng(5)
    poses = [_exp(rng.normal(0, 0.02, 3), rng.normal(0, 0.005, 3)) for _ in range(3)]
    st, _, _, avg = agreement(poses)
    assert st == O.ACCEPTED
    assert np.array_equal(avg, average(poses))


def test_neighbour_rule():
    K = 10
    assert O.neighbours(0, K) == (0, 1, 2)        # no previous keyframe: the second next instead (:481-494)
    assert O.neighbours(4, K) == (4, 5, 3)
    assert O.neighbours(K - 2, K) == (K - 2, K - 1, K - 3)
    assert O.neighbours(K - 1, K) is None         # no next keyframe (:470-476)
    assert O.neighbours(0, 2) is None             # matched 0 with two keyframes: no second next
    assert O.neighbours(0, 3) == (0, 1, 2)


def test_estimates_compose_back_to_the_truth():
    """With the true tracking result cur_T_tracked = cur_T_old_i, the refined estimates are the true cur_T_old, and the initial
    estimates of an exact old_T_cur_initial are the true cur_T_old_i."""
    rng = np.random.default_rng(3)
    poses = np.array([_exp(rng.normal(0, 0.3, 3), rng.normal(0, 1, 3)) for _ in range(6)])
    cur, ids = 5, O.neighbours(0, 6)
    true_cur_T_old = [np.linalg.inv(O.to_T(poses[cur])) @ O.to_T(poses[k]) for k in ids]
    old_T_cur = np.linalg.inv(true_cur_T_old[0])
    init = O.initial_estimates(O.from_T(old_T_cur), poses, ids)
    for a, b in zip(init, true_cur_T_old):
        assert np.allclose(a, b, atol=1e-5)
    ref = O.refined([O.from_T(t) for t in true_cur_T_old], poses, ids)
    for r in ref:
        assert np.allclose(r, true_cur_T_old[0], atol=1e-5)


def test_necessity_of_no_move_is_zero_and_of_a_shift_is_its_disparity():
    h, w = 12, 16
    depth = np.full((h, w), 2000, np.uint16)
    depth[0, :3] |= O.INVALID_DEPTH_BIT
    K4 = (10.0, 10.0, 8.0, 6.0)
    cf = np.zeros((h, w), np.float32)
    pose = _exp([0.1, 0, 0], [0, 0, 1])
    other = _exp([0.0, 0.2, 0], [1, 0, 0])
    cur_T_old = O.from_T(np.linalg.inv(O.to_T(pose)) @ O.to_T(other))
    avg, n = O.necessity(depth, K4, K4, (w, h), 1e-3, 0.0, cf, 1, cur_T_old, other, pose)
    assert n == h * w - 3 and avg < 1e-9
    # moving the current camera 1 cm sideways shifts every point at 2 m by fx * 0.01 / 2 = 0.05 px
    shifted = O.from_T(O.to_T(pose) @ O.to_T(_exp([0, 0, 0], [0.01, 0, 0])))
    avg, n = O.necessity(depth, K4, K4, (w, h), 1e-3, 0.0, cf, 1, cur_T_old, other, shifted)
    assert abs(avg - 0.05) < 1e-6 and n > 0
    assert O.verdict(avg, n) == O.CORRECTION_TOO_SMALL and O.verdict(avg, 4) == O.ACCEPTED


def test_struct_layouts():
    from badslam_b200 import _lib as L
    assert C.sizeof(L.LoopCandidate) == 4 * (2 + 7)
    assert C.sizeof(L.LoopVerificationOptions) == C.sizeof(L.OdometryOptions) + 12 == 32
    assert C.sizeof(L.OdometryResult) == 80
    assert C.sizeof(L.LoopVerification) == 4 * (1 + 3 + 21 + 7 + 3 + 1) + 3 * 80 == 384
    assert L.LoopVerification.tracking.offset == 144
    assert L.LoopVerification.cur_T_old.offset == 4 * (1 + 3 + 21)
    assert L.LoopVerification.pixel_count.offset == 140
    assert (L.LOOP_ACCEPTED, L.LOOP_NO_NEIGHBOUR, L.LOOP_ROTATION_DISAGREES, L.LOOP_TRANSLATION_DISAGREES,
            L.LOOP_CORRECTION_TOO_SMALL) == (O.ACCEPTED, O.NO_NEIGHBOUR, O.ROTATION_DISAGREES, O.TRANSLATION_DISAGREES,
                                              O.CORRECTION_TOO_SMALL)
