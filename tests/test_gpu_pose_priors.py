"""Soft pose priors on keyframes (bba_set_keyframe_pose_priors): the 1/2 r^T L r term, r = log(prior^-1 global_T_frame), in the
alternating scheme's pose solve, in bba_estimate_frame_pose and in the PCG scheme's products.

* setting and clearing priors leaves the alternating BA (intrinsics, surfel updates) bit-identical to a handle that never had one;
* the pose solve with priors follows numpy's Gauss-Newton loop over bba_accumulate_pose_coeffs + bba_host_pose_prior_terms;
* a very large L pins a keyframe to its prior; a keyframe that sees no surfel reaches its prior; fixed keyframes (inactive, the
  PCG gauge) ignore theirs;
* the PCG products with and without priors differ by the per-keyframe terms, and a PCG BA with priors ends closer to them;
* the deterministic mode stays reproducible; two and three ranks of a local group keep identical replicas and match one rank;
* bad arguments change nothing."""
import numpy as np
import pytest

import test_gpu_multi_ranks_one_device as R
from gpu_checks import POSE_R, POSE_T

pytestmark = pytest.mark.gpu

SCENES = ["tiny", "small", "many"]
_CACHE = {}


def _scene(name):
    if name not in _CACHE:
        from badslam_b200.scene import config_by_name, make_scene
        _CACHE[name] = make_scene(config_by_name(name))
    return _CACHE[name]


def _make(sc, deterministic=False, **kw):
    from badslam_b200.direct_ba import DirectBA
    ba = DirectBA.from_scene(sc, device="cuda:0", **kw)
    if deterministic:
        ba.SetDeterministic(True)
    return ba


def _info(sigma_t, sigma_r):
    return np.diag([sigma_t ** -2] * 3 + [sigma_r ** -2] * 3).astype(np.float32)


def _upper(M):
    return np.array([M[i, j] for i in range(6) for j in range(i, 6)], np.float32)


def _lib():
    from badslam_b200 import _lib
    return _lib.load()


def _host_terms(prior, pose, info21):
    import ctypes as C
    H, b, cost = np.zeros(21), np.zeros(6), C.c_double()
    p, q, L = (np.ascontiguousarray(x, np.float32) for x in (prior, pose, info21))
    _lib().bba_host_pose_prior_terms(p.ctypes.data, q.ctypes.data, L.ctypes.data, H.ctypes.data, b.ctypes.data, C.byref(cost))
    return H, b, cost.value


def _prior_ids(K):
    return np.arange(0, K, 2, dtype=np.int32)   # every other keyframe


def _all_state(ba):
    return R._state(ba)


def _same_state(a, b):
    for k in ("poses", "act", "surfels", "active", "intr", "cf"):
        assert R._same(a[k], b[k]), k


# ---- 1. set + clear = never set --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("scene", SCENES)
def test_cleared_priors_change_no_bit(scene):
    sc = _scene(scene)
    K = sc.cfg.num_keyframes
    outs = []
    for with_priors in (False, True):
        ba = _make(sc, deterministic=True)
        if with_priors:
            ids = _prior_ids(K)
            ba.SetKeyframePosePriors(ids, sc.poses_true[ids], _info(0.01, 0.01))
            ba.ClearKeyframePosePriors(ids[:1])
            ba.ClearKeyframePosePriors()
            assert all(ba.KeyframePosePrior(k) is None for k in range(K))
        r = ba.BundleAdjustment(None, True, True, True, True, True, 2, 2)
        outs.append((_all_state(ba), R._result(r), r.kernel_launches))
    _same_state(outs[0][0], outs[1][0])
    assert np.array_equal(outs[0][1], outs[1][1]) and outs[0][2] == outs[1][2]


# ---- 2. the pose solve against numpy ---------------------------------------------------------------------------------------

def _numpy_pose_step(ba, k, init, prior, info21, max_iterations=30):
    """EstimateFramePose's Gauss-Newton loop: data H, b from bba_accumulate_pose_coeffs (fp32), plus the prior's fp64 terms,
    the fp64 LDLT, pose <- pose exp(-x) and the convergence test, through the library's host building blocks."""
    lib = _lib()
    pose = np.array(init, np.float32)
    for it in range(max_iterations):
        c = ba.AccumulatePoseEstimationCoeffs(k, pose)
        H = np.array(c.H, np.float32).astype(np.float64)
        b = np.array(c.b, np.float32).astype(np.float64)
        Hp, bp, _ = _host_terms(prior, pose, info21)
        H, b = H + Hp, b + bp
        x = np.zeros(6)
        assert lib.bba_host_solve_ldlt(6, H.ctypes.data, b.ctypes.data, x.ctypes.data) == 1
        xf = x.astype(np.float32)
        neg = np.ascontiguousarray(-xf)
        step, out = np.zeros(7, np.float32), np.zeros(7, np.float32)
        lib.bba_host_se3_exp(neg.ctypes.data, step.ctypes.data)
        lib.bba_host_se3_compose(pose.ctypes.data, step.ctypes.data, out.ctypes.data)
        pose = out
        if lib.bba_host_pose_update_converged(xf.ctypes.data):
            return pose, it + 1
    return pose, max_iterations


@pytest.mark.parametrize("scene", SCENES)
def test_pose_solve_matches_numpy(scene):
    """Deterministic mode: the coefficients numpy reads are the bits the pose solve sums, so the loops agree to rounding of the
    trigonometry (host vs device) at most."""
    sc = _scene(scene)
    K = sc.cfg.num_keyframes
    ba = _make(sc, deterministic=True)
    ids = _prior_ids(K)[:4]
    # priors a little off the true poses, so that data and prior pull apart
    rng = np.random.default_rng(5)
    priors = sc.poses_true[ids].copy()
    priors[:, 4:] += rng.normal(scale=0.01, size=(len(ids), 3)).astype(np.float32)
    info = _info(1e-3, 1e-3)
    ba.SetKeyframePosePriors(ids, priors, info)
    for i, k in enumerate(ids):
        got, its, _ = ba.EstimateFramePose(None, sc.poses_init[k], int(k))
        want, want_its = _numpy_pose_step(ba, int(k), sc.poses_init[k], priors[i], _upper(info))
        assert its == want_its, (k, its, want_its)
        assert np.abs(got.astype(np.float64) - want).max() < 1e-6, (k, got, want)
        # and the prior moved the result: without it the loop ends elsewhere
        free, _ = _numpy_pose_step(ba, int(k), sc.poses_init[k], priors[i], np.zeros(21, np.float32))
        assert np.abs(free.astype(np.float64) - want).max() > 1e-5, k


# ---- 3. / 4. / 5. strong priors, a keyframe without data, fixed keyframes -------------------------------------------------

@pytest.mark.parametrize("scene", SCENES)
def test_very_large_information_pins_the_keyframe(scene):
    from badslam_b200.scene import pose_error
    sc = _scene(scene)
    K = sc.cfg.num_keyframes
    ba = _make(sc)
    ids = _prior_ids(K)
    ba.SetKeyframePosePriors(ids, sc.poses_true[ids], _info(1e-7, 1e-7))
    ba.BundleAdjustment(None, False, False, False, True, True, 1, 1)
    poses, _ = ba.GetKeyframeStates()
    for k in ids:
        assert max(pose_error(poses[k], sc.poses_true[k])) < 1e-6, k


def test_keyframe_without_data_reaches_its_prior():
    from badslam_b200.scene import pose_error
    sc = _scene("small")
    ba = _make(sc)
    far = sc.poses_true[1].copy()
    far[4] += 100.0
    assert ba.AccumulatePoseEstimationCoeffs(1, far).n_assoc == 0
    ba.SetKeyframePosePriors([1], sc.poses_true[1:2], _info(0.05, 0.05))
    est, its, conv = ba.EstimateFramePose(None, far, 1)
    assert conv and its <= 10, its
    assert max(pose_error(est, sc.poses_true[1])) < 1e-2


def test_fixed_keyframes_ignore_their_priors():
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    away = sc.poses_init.copy()
    away[:, 4] += 0.5
    # alternating: keyframe 0, moved out of every other keyframe's view, is outside the active window and co-visible with none of
    # it, so it is inactive and not in the pose step; inside the window, with no data, it would land on its prior
    poses = sc.poses_init.copy()
    poses[0, 4] += 100.0
    prior0 = poses[0:1].copy()
    prior0[0, 4] += 0.5
    for window_start, moves in ((1, False), (0, True)):
        ba = _make(sc, poses=poses)
        ba.SetKeyframePosePriors([0], prior0, _info(1e-3, 1e-3))
        before = ba.GetKeyframeStates()[0]
        ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, active_keyframe_window_start=window_start)
        after = ba.GetKeyframeStates()[0]
        if moves:
            assert abs(float(after[0, 4]) - float(prior0[0, 4])) < 1e-4
        else:
            assert np.array_equal(after[0], before[0])
    # PCG: the gauge keyframe
    ba = _make(sc)
    ba.SetKeyframePosePriors(np.arange(K), away, _info(1e-3, 1e-3))
    before = ba.GetKeyframeStates()[0]
    ba.BundleAdjustment(None, False, False, False, True, True, 2, 2, use_pcg=True, pcg_gauge_keyframe=1)
    after = ba.GetKeyframeStates()[0]
    assert np.array_equal(after[1], before[1])
    assert not np.array_equal(after[0], before[0])


# ---- 6. PCG ----------------------------------------------------------------------------------------------------------------

def _matrix(H21):
    Hm = np.zeros((6, 6))
    Hm[np.triu_indices(6)] = H21
    return Hm + np.triu(Hm, 1).T


def test_pcg_products_differ_by_the_prior_terms():
    """bba_pcg_debug's first step without priors, with a prior on keyframe K-1 only and with one on keyframe 2 only.  Keyframe
    K-1 is moved out of the map: it has no data, so its rows of J^T W J are zero and its prior changes nothing else -- r and M
    differ by -J^T L r and diag(J^T L J) on its block, g by J^T L J p there, alpha_d by p^T J^T L J p plus the lambda term of
    the block's new p, and every other entry only by the order of the fp32 atomics.  Keyframe 2 keeps its data: r and M differ
    by the terms on its block and by nothing elsewhere."""
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    poses = sc.poses_init.copy()
    poses[K - 1, 4] += 100.0
    info = _upper(_info(0.01, 0.02))
    probes = {}
    for k in (None, K - 1, 2):
        ba = _make(sc, poses=poses)
        if k is not None:
            ba.SetKeyframePosePriors([k], sc.poses_true[k:k + 1], info)
        probes[k] = ba.PCGProbe(0, False, True, True, gauge_keyframe=0)
    a = probes[None]
    n = len(a["r"])

    def close(x, y, what):
        np.testing.assert_allclose(x, y, rtol=1e-4, atol=1e-4 * max(1e-30, np.abs(y).max()), err_msg=what)

    for k in (K - 1, 2):
        b = probes[k]
        u = 6 * (k - 1)   # pose unknowns skip the gauge keyframe 0
        s = slice(u, u + 6)
        Hp, bp, _ = _host_terms(sc.poses_true[k], poses[k], info)
        Hm = _matrix(Hp)
        rest = np.ones(n, bool)
        rest[s] = False
        tol = 1e-5 * max(np.abs(bp).max(), np.abs(a["r"][s]).max())
        assert np.abs((b["r"][s] - a["r"][s]) + bp).max() <= tol, k
        tol = 1e-5 * max(np.abs(Hm).max(), np.abs(a["M"][s]).max())
        assert np.abs((b["M"][s] - a["M"][s]) - np.diag(Hm)).max() <= tol, k
        close(b["r"][rest], a["r"][rest], "r elsewhere")
        close(b["M"][rest], a["M"][rest], "M elsewhere")
        if k == K - 1:
            assert np.all(a["M"][s] == 0) and np.all(a["p"][s] == 0)
            pb = b["p"][s].astype(np.float64)
            want_g = Hm @ pb
            assert np.abs(b["g"][s] - want_g).max() <= 1e-5 * np.abs(want_g).max()
            close(b["p"][rest], a["p"][rest], "p elsewhere")
            close(b["g"][rest], a["g"][rest], "g elsewhere")
            share = float(pb @ want_g) + K * 1e-8 * float(pb @ pb)
            assert abs((b["alpha_d"] - a["alpha_d"]) - share) <= 1e-5 * (abs(a["alpha_d"]) + share), (b["alpha_d"], a["alpha_d"], share)


def test_pcg_ba_with_priors_converges_towards_them():
    from badslam_b200.scene import pose_error
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    rng = np.random.default_rng(2)
    priors = sc.poses_true.copy()
    priors[:, 4:] += rng.normal(scale=0.02, size=(K, 3)).astype(np.float32)
    errs = []
    for with_priors in (False, True):
        ba = _make(sc)
        if with_priors:
            ba.SetKeyframePosePriors(np.arange(K), priors, _info(1e-4, 1e-4))
        ba.BundleAdjustment(None, False, False, False, True, True, 4, 4, use_pcg=True, pcg_gauge_keyframe=0)
        poses = ba.GetKeyframeStates()[0]
        assert np.all(np.isfinite(poses))
        errs.append(np.mean([pose_error(poses[k], priors[k])[0] for k in range(1, K)]))
    assert errs[1] < 0.5 * errs[0], errs


# ---- 7. deterministic mode -------------------------------------------------------------------------------------------------

def test_deterministic_with_priors():
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    outs = []
    for _ in range(2):
        ba = _make(sc, deterministic=True)
        ba.SetKeyframePosePriors(_prior_ids(K), sc.poses_true[_prior_ids(K)], _info(0.01, 0.01))
        r = ba.BundleAdjustment(None, True, True, True, True, True, 2, 2)
        outs.append((_all_state(ba), R._result(r), np.float64(r.cost)))
    _same_state(outs[0][0], outs[1][0])
    assert np.array_equal(outs[0][1], outs[1][1]) and R._same(outs[0][2], outs[1][2])


# ---- 8. several ranks ------------------------------------------------------------------------------------------------------

def _priors_for(sc):
    K = sc.cfg.num_keyframes
    rng = np.random.default_rng(11)
    ids = _prior_ids(K)
    poses = sc.poses_true[ids].copy()
    poses[:, 4:] += rng.normal(scale=0.005, size=(len(ids), 3)).astype(np.float32)
    return ids, poses, _info(0.01, 0.01)


def run_alternating_with_priors(ba):
    ids, poses, info = _priors_for(R.SCENES["small"]())
    ba.SetKeyframePosePriors(ids, poses, info)
    return R.run_pose(ba)


def run_pcg_with_priors(ba):
    ids, poses, info = _priors_for(R.SCENES["small"]())
    ba.SetKeyframePosePriors(ids, poses, info)
    return R.run_pcg(ba, False)


@pytest.mark.parametrize("world", ["2", "3"])
@pytest.mark.parametrize("mode", ["gather", "peer"])
@pytest.mark.parametrize("scheme", ["alternating", "pcg"])
def test_local_group_ranks(world, mode, scheme):
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    from badslam_b200.scene import pose_error
    fn = run_alternating_with_priors if scheme == "alternating" else run_pcg_with_priors
    handles = DirectBA.create_local_ranks(R.SCENES["small"](), int(world), ["cuda:0"] * int(world))
    with LocalGroup(handles, peer_stores=mode == "peer") as group:
        outs = group.run(lambda r, ba: fn(ba))
    keys = ("poses", "act", "surfels", "active", "intr", "cf", "res")
    for o in outs[1:]:
        for k in keys:
            assert R._same(o[k], outs[0][k]), k
    want = R.one_rank(("priors", scheme), lambda: R._one("small", fn))
    got = outs[0]
    K = len(want["poses"])
    worst = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(K))
    if scheme == "alternating":
        assert np.array_equal(got["res"][:5], want["res"][:5]) and np.array_equal(got["act"], want["act"])
        assert worst <= min(POSE_T, POSE_R), worst
    else:
        assert got["res"][0] == want["res"][0] and abs(int(got["res"][5]) - int(want["res"][5])) <= 2
        assert worst < 2e-4, worst


# ---- 9. bad arguments ------------------------------------------------------------------------------------------------------

def test_bad_arguments_change_nothing(tiny_scene):
    from badslam_b200 import _lib as L
    sc = tiny_scene
    K = sc.cfg.num_keyframes
    ba = _make(sc)
    good = _upper(_info(0.1, 0.1))
    ba.SetKeyframePosePriors([1], sc.poses_true[1:2], good)
    before = (ba.KeyframePosePrior(0), ba.KeyframePosePrior(1), ba.kernel_launch_count(), ba.GetKeyframeStates()[0])
    indefinite = _info(0.1, 0.1)
    indefinite[0, 1] = indefinite[1, 0] = 2 * indefinite[0, 0]
    negative = _info(0.1, 0.1)
    negative[5, 5] = -1.0
    nan_pose = sc.poses_true[0].copy()
    nan_pose[5] = np.nan
    nan_info = good.copy()
    nan_info[3] = np.inf
    cases = [
        ([0, K], [sc.poses_true[0], sc.poses_true[0]], [good, good]),
        ([0, -1], [sc.poses_true[0], sc.poses_true[0]], [good, good]),
        ([0, 2], [sc.poses_true[0], nan_pose], [good, good]),
        ([0, 2], [sc.poses_true[0], sc.poses_true[2]], [good, nan_info]),
        ([0, 2], [sc.poses_true[0], sc.poses_true[2]], [good, _upper(indefinite)]),
        ([0, 2], [sc.poses_true[0], sc.poses_true[2]], [good, _upper(negative)]),
        ([0, 2], [sc.poses_true[0], np.zeros(7, np.float32)], [good, good]),
    ]
    for ids, poses, infos in cases:
        with pytest.raises(L.BadBAError) as e:
            ba.SetKeyframePosePriors(ids, np.array(poses), np.array(infos))
        assert e.value.status == L.ERR_INVALID_ARGUMENT
    for ids in ([K], [-2], [0, K + 3]):
        with pytest.raises(L.BadBAError):
            ba.ClearKeyframePosePriors(ids)
    after = (ba.KeyframePosePrior(0), ba.KeyframePosePrior(1), ba.kernel_launch_count(), ba.GetKeyframeStates()[0])
    assert before[0] is None and after[0] is None
    assert all(np.array_equal(x, y) for x, y in zip(before[1], after[1]))
    assert before[2] == after[2] and np.array_equal(before[3], after[3])
    # semi-definite (a translation-only prior) is accepted
    semi = np.diag([100.0] * 3 + [0.0] * 3).astype(np.float32)
    ba.SetKeyframePosePriors([0], sc.poses_true[0:1], semi)
    assert np.array_equal(ba.KeyframePosePrior(0)[1], _upper(semi))
