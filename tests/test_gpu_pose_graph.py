"""The keyframe pose graph on the device (bba_optimize_pose_graph, DESIGN §3.14) against the numpy oracle
(tests/pose_graph_oracle.py).

* circle graphs of 200 keyframes (one loop, 50 random loops, priors without a gauge) reach the oracle's optimum and cost, with
  linear_iterations / iterations <= 12 L + 4;
* held keyframes (the gauge, an untouched keyframe, the lowest id of a component without a prior) keep their bits;
* the cost never rises; a chain-only graph stays where it is; information on translation only leaves the rotations alone;
* activations, priors, constraints and surfels are untouched, and the front end reads the new poses;
* two calls, the deterministic mode on and off, and local groups of 2 and 3 ranks give the same bits;
* on `small`, a loop closure through the pose graph, the surfel deformation and BA ends closer to the truth than BA alone;
* refused arguments change nothing.

The graphs never read images: their handles hold many keyframes that share the two 80x60 images of one tiny scene."""
import ctypes as C

import numpy as np
import pytest

import pose_graph_oracle as O
from gpu_checks import POSE_R, POSE_T

pytestmark = pytest.mark.gpu

_IMAGES = {}
_I6 = np.eye(6)


def _images():
    if "scene" not in _IMAGES:
        from badslam_b200.scene import SceneConfig, make_scene
        _IMAGES["scene"] = make_scene(SceneConfig(80, 60, 2, 2000, cell=1, seed=41, name="pose_graph"))
    return _IMAGES["scene"]


def _add_keyframes(ba, K):
    sc = _images()
    for k in range(sc.cfg.num_keyframes, K):
        j = k % sc.cfg.num_keyframes
        ba.AddKeyframeHost(sc.depth[j], sc.normals[j], sc.radius[j], sc.color[j], sc.poses_init[j], sc.min_depth[j], sc.max_depth[j])


def make_handle(K, deterministic=False):
    from badslam_b200.direct_ba import DirectBA
    ba = DirectBA.from_scene(_images(), device="cuda:0", max_keyframes=K)
    _add_keyframes(ba, K)
    if deterministic:
        ba.SetDeterministic(True)
    return ba


def _f32(A):
    return np.asarray(O.to_array(A), np.float32)


def _relative(truth, a, b):
    return _f32(O.mul(O.inv(O.pose(truth, a)), O.pose(truth, b)))


def _circle(K, seed=0):
    truth = O.circle(K)
    return truth, _f32(O.drift(truth, 0.01, 0.005, seed=seed))


def _oracle(start32, constraints, priors=(), chain=True, gauge=0):
    """The oracle's optimum over the same terms: priors [(k, pose32, L)], constraints [(a, b, Z32, L)], the chain at start32."""
    S = O.from_array(start32)
    terms = [O.Term(k, -1, P, L) for k, P, L in priors] + [O.Term(a, b, Z, L) for a, b, Z, L in constraints]
    if chain:
        terms += [O.Term(k, k + 1, _f32(O.mul(O.inv(O.pose(S, k)), O.pose(S, k + 1))), _I6) for k in range(len(start32) - 1)]
    return O.gauss_newton(terms, S, gauge=gauge)


def _poses_bits(ba):
    return ba.GetKeyframeStates()[0].view(np.uint32).copy()


def _worst(got32, want):
    from badslam_b200.scene import pose_error
    W = _f32(want)
    errs = [pose_error(got32[k], W[k]) for k in range(len(got32))]
    return max(e[0] for e in errs), max(e[1] for e in errs)


CASES = {
    "one_loop": lambda K: dict(loops=[(5, K - 3)], priors=[], gauge=0),
    "random_loops": lambda K: dict(loops=O.random_loops(K, 50, seed=7), priors=[], gauge=0),
    "priors_no_gauge": lambda K: dict(loops=[(5, K - 3)], priors=[0, 50, 100, 150], gauge=-1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_matches_the_oracle(case):
    K = 200
    spec = CASES[case](K)
    truth, start = _circle(K)
    ba = make_handle(K)
    ba.SetKeyframeStates(start)
    cons = [(a, b, _relative(truth, a, b), _I6) for a, b in spec["loops"]]
    ba.AddKeyframePoseConstraints([c[0] for c in cons], [c[1] for c in cons], [c[2] for c in cons], _I6)
    Lp = np.diag([100.0] * 3 + [400.0] * 3)
    priors = [(k, _f32(O.pose(truth, k)), Lp) for k in spec["priors"]]
    if priors:
        ba.SetKeyframePosePriors([p[0] for p in priors], [p[1] for p in priors], Lp)
    r = ba.OptimizePoseGraph(gauge_keyframe=spec["gauge"])
    want, held, cost, _ = _oracle(start, cons, priors, gauge=spec["gauge"])
    got = ba.GetKeyframeStates()[0]
    dt, dr = _worst(got, want)
    print(f"{case}: {r}, oracle cost {cost:.6g}, worst pose error {dt:.3g} m / {dr:.3g} rad")
    assert dt < POSE_T and dr < POSE_R, (dt, dr)
    assert abs(r["final_cost"] - cost) <= 1e-4 * cost, (r["final_cost"], cost)
    assert r["converged"] == 1 and r["final_cost"] <= r["initial_cost"]
    assert r["held_keyframes"] == int(held.sum()) == (0 if spec["gauge"] < 0 else 1)
    L = len(spec["loops"])
    assert r["linear_iterations"] <= (12 * L + 4) * r["iterations"], r


def test_held_keyframes_keep_their_bits():
    K = 30
    truth, start = _circle(K, seed=3)
    ba = make_handle(K)
    ba.SetKeyframeStates(start)
    # the gauge's component {3, 4, 5, 6}; {10, 11, 12} without a prior; {20, 21} with a prior on 21; everything else untouched
    pairs = [(3, 4), (4, 5), (5, 6), (10, 11), (11, 12), (20, 21)]
    ba.AddKeyframePoseConstraints([a for a, _ in pairs], [b for _, b in pairs], [_relative(truth, a, b) for a, b in pairs], _I6)
    ba.SetKeyframePosePriors([21], [_f32(O.pose(truth, 21))], _I6)
    before = _poses_bits(ba)
    r = ba.OptimizePoseGraph(add_current_state_odometry_constraints=False, gauge_keyframe=5)
    after = _poses_bits(ba)
    free = [3, 4, 6, 11, 12, 20, 21]
    assert r["held_keyframes"] == K - len(free)
    for k in range(K):
        if k in free:
            assert not np.array_equal(after[k], before[k]), k
        else:
            assert np.array_equal(after[k], before[k]), k


def test_cost_never_rises_and_chain_only_stays():
    from badslam_b200.scene import pose_error
    K = 100
    truth, start = _circle(K, seed=4)
    ba = make_handle(K)
    ba.SetKeyframeStates(start)
    r = ba.OptimizePoseGraph()
    got = ba.GetKeyframeStates()[0]
    assert r["final_cost"] <= r["initial_cost"] and r["initial_cost"] < 1e-6, r
    assert max(max(pose_error(got[k], start[k])) for k in range(K)) <= 1e-6
    for seed in range(3):   # large drifts and loops: the cost never rises
        ba.SetKeyframeStates(_f32(O.drift(truth, 0.05, 0.03, seed=10 + seed)))
        ba.RemoveKeyframePoseConstraints()
        pairs = O.random_loops(K, 5, seed=seed)
        ba.AddKeyframePoseConstraints([a for a, _ in pairs], [b for _, b in pairs], [_relative(truth, a, b) for a, b in pairs], _I6)
        r = ba.OptimizePoseGraph(max_iterations=3)
        assert r["final_cost"] <= r["initial_cost"], r


def test_translation_only_information():
    K = 2
    ba = make_handle(K)
    A = O.se3_exp(np.array([0.1, 0.2, -0.1, 0.05, -0.02, 0.1]))
    B = O.mul(A, O.se3_exp(np.array([0.3, -0.2, 0.1, 0.2, 0.1, -0.15])))
    ba.SetKeyframeStates(np.stack([_f32(A), _f32(B)]))
    Z = _f32(O.se3_exp(np.array([0.25, -0.1, 0.2, 0.0, 0.0, 0.0])))
    ba.AddKeyframePoseConstraints([0], [1], [Z], np.diag([1.0, 1.0, 1.0, 0.0, 0.0, 0.0]))
    r = ba.OptimizePoseGraph(add_current_state_odometry_constraints=False)
    got = ba.GetKeyframeStates()[0]
    assert np.all(np.isfinite(got)) and r["final_cost"] <= r["initial_cost"]
    # the rotation of keyframe 1 has no information: it keeps its value, and the translation residual closes
    assert np.abs(O.so3_log(O.from_array(got[1])[0].T @ O.from_array(_f32(B))[0])).max() < 1e-6, got[1]
    assert r["final_cost"] < 1e-10, r


def test_untouched_state_and_front_end():
    K = 60
    truth, start = _circle(K, seed=5)
    ba = make_handle(K)
    ba.SetKeyframeStates(start, np.array([k % 3 for k in range(K)], np.int32))
    ba.AddKeyframePoseConstraints([2], [K - 2], [_relative(truth, 2, K - 2)], _I6)
    ba.SetKeyframePosePriors([7], [_f32(O.pose(truth, 7))], _I6)
    _, act_before = ba.GetKeyframeStates()
    cons_before = ba.KeyframePoseConstraints()
    prior_before = ba.KeyframePosePrior(7)
    surf_before = ba.GetSurfelsHost().copy()
    ba.OptimizePoseGraph()
    poses, act = ba.GetKeyframeStates()
    assert np.array_equal(act, act_before)
    for x, y in zip(ba.KeyframePoseConstraints(), cons_before):
        assert np.array_equal(x, y)
    prior = ba.KeyframePosePrior(7)
    assert np.array_equal(prior[0], prior_before[0]) and np.array_equal(prior[1], prior_before[1])
    assert np.array_equal(ba.GetSurfelsHost().view(np.uint32), surf_before.view(np.uint32))
    # the front-end reader of one keyframe sees the published poses
    p = np.zeros(7, np.float32)
    for k in (0, 1, K // 2, K - 1):
        from badslam_b200 import _lib
        assert ba._lib.bba_get_keyframe_pose(ba._h, k, p.ctypes.data_as(C.POINTER(C.c_float))) == _lib.OK
        assert np.array_equal(p, poses[k])
    assert not np.array_equal(poses, start)


def _loop_case(ba, K, seed=6):
    truth, start = _circle(K, seed=seed)
    ba.SetKeyframeStates(start)
    pairs = [(5, K - 3)] + O.random_loops(K, 4, seed=seed)
    ba.AddKeyframePoseConstraints([a for a, _ in pairs], [b for _, b in pairs], [_relative(truth, a, b) for a, b in pairs], _I6)
    r = ba.OptimizePoseGraph()
    return ba.GetKeyframeStates()[0], r


def test_reproducible_bits():
    K = 120
    outs = []
    for det in (False, True):
        ba = make_handle(K, deterministic=det)
        outs.append(_loop_case(ba, K))
        if not det:   # a second call from the same state
            again = make_handle(K)
            outs.append(_loop_case(again, K))
    for poses, r in outs[1:]:
        assert np.array_equal(poses.view(np.uint32), outs[0][0].view(np.uint32)) and r == outs[0][1]


@pytest.mark.parametrize("world", ["2", "3"])
@pytest.mark.parametrize("mode", ["gather", "peer"])
def test_local_group_ranks(world, mode):
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    K = 40

    def run(rank, ba):
        _add_keyframes(ba, K)
        return _loop_case(ba, K)
    handles = DirectBA.create_local_ranks(_images(), int(world), ["cuda:0"] * int(world), max_keyframes=K)
    with LocalGroup(handles, peer_stores=mode == "peer") as group:
        outs = group.run(run)
    want = _loop_case(make_handle(K), K)
    for poses, r in outs:
        assert np.array_equal(poses.view(np.uint32), want[0].view(np.uint32)) and r == want[1]


def _aligned_error(poses, truth32):
    """Mean translation / rotation error of the keyframes after moving the estimate so that keyframe 0 sits at the truth."""
    from badslam_b200.scene import pose_error, se3_inverse, se3_mul
    align = se3_mul(truth32[0], se3_inverse(poses[0]))
    errs = np.array([pose_error(se3_mul(align, poses[k]), truth32[k]) for k in range(len(poses))])
    return errs.mean(0)


def test_loop_closure_end_to_end_on_small(small_scene):
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import se3_exp, se3_inverse, se3_mul
    sc = small_scene
    K = sc.cfg.num_keyframes
    # the second half drifted rigidly about keyframe K/2 - 1, with the map carried along
    D = se3_exp([0.12, -0.08, 0.06, 0.03, -0.04, 0.05])
    pivot = sc.poses_true[K // 2 - 1]
    move = se3_mul(se3_mul(pivot, D), se3_inverse(pivot))
    drifted = np.array([sc.poses_true[k] if k < K // 2 else se3_mul(move, sc.poses_true[k]) for k in range(K)], np.float32)
    errors = {}
    for with_graph in (False, True):
        ba = DirectBA.from_scene(sc, poses=sc.poses_true, device="cuda:0")
        original = ba.RememberKeyframePoses()
        ba.SetKeyframeStates(drifted)
        ba.DeformSurfelsWithKeyframePoseChanges(original)
        Z = se3_mul(se3_inverse(sc.poses_true[0]), sc.poses_true[K - 1])
        ba.AddKeyframePoseConstraints([0], [K - 1], [Z], np.diag([1e4] * 3 + [1e5] * 3))
        if with_graph:
            remembered = ba.RememberKeyframePoses()
            r = ba.OptimizePoseGraph()
            assert r["final_cost"] < r["initial_cost"]
            ba.DeformSurfelsWithKeyframePoseChanges(remembered)
        ba.BundleAdjustment(None, False, False, False, True, True, 10, 10)
        errors[with_graph] = _aligned_error(ba.GetKeyframeStates()[0], sc.poses_true)
    print(f"mean keyframe error to the truth after BA: without the pose graph {errors[False]}, with it {errors[True]}")
    assert errors[True][0] < errors[False][0] and errors[True][1] < errors[False][1], errors


def test_refused_arguments_change_nothing():
    from badslam_b200._lib import BadBAError
    K = 20
    truth, start = _circle(K, seed=8)
    ba = make_handle(K)
    ba.SetKeyframeStates(start)
    ba.AddKeyframePoseConstraints([1], [K - 2], [_relative(truth, 1, K - 2)], _I6)
    before = _poses_bits(ba)
    launches = ba.kernel_launch_count()
    bad_info = np.eye(6)
    bad_info[4, 4] = -1.0
    nan_info = np.eye(6)
    nan_info[0, 1] = nan_info[1, 0] = np.nan
    for kw in (dict(gauge_keyframe=-2), dict(gauge_keyframe=K), dict(odometry_information=nan_info),
               dict(odometry_information=bad_info)):
        with pytest.raises(BadBAError):
            ba.OptimizePoseGraph(**kw)
        assert np.array_equal(_poses_bits(ba), before) and ba.kernel_launch_count() == launches, kw
    # without the chain the information is not read
    r = ba.OptimizePoseGraph(add_current_state_odometry_constraints=False, odometry_information=bad_info)
    assert r["iterations"] >= 1
    # no term at all: every keyframe is held, and the call changes nothing
    two = make_handle(2)
    before = _poses_bits(two)
    r = two.OptimizePoseGraph(add_current_state_odometry_constraints=False, gauge_keyframe=-1)
    assert r["held_keyframes"] == 2 and r["final_cost"] == 0.0 and r["converged"] == 1 and r["linear_iterations"] == 0
    assert np.array_equal(_poses_bits(two), before)
