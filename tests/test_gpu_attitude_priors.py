"""Attitude priors on keyframes (bba_set_keyframe_attitude_priors, DESIGN §3.17): a measured direction such as gravity fixes a
keyframe's roll and pitch in the alternating pose step, bba_estimate_frame_pose, the PCG products and bba_optimize_pose_graph.

* set-then-clear gives the bits and launch counts of a handle that never had attitude priors, in every solver;
* on a 200-keyframe circle with a tilt drift the pose graph reaches the numpy oracle's optimum (tests/attitude_prior_oracle.py)
  with the gauge keyframe and without it, and the partially held keyframe keeps its translation and yaw;
* end to end on `small` a progressive roll / pitch drift is taken out by the pose graph, the surfel deformation and BA in either
  scheme, far better than without attitude priors;
* bba_estimate_frame_pose follows numpy's IRLS loop over bba_accumulate_pose_coeffs;
* a 30 degree wrong attitude prior under a Cauchy loss leaves the tilt near the outlier-free result and gets w < 0.1;
* repeated calls, the deterministic mode and local groups of 2 and 3 ranks give the pose graph's bits of one rank, and BA on
  2 and 3 ranks identical replicas close to one rank's result;
* refused calls change nothing, the launch counter included."""
import ctypes as C

import numpy as np
import pytest

import attitude_prior_oracle as A
import pose_graph_oracle as O
import test_gpu_multi_ranks_one_device as R
import test_gpu_pose_constraints as PC
import test_gpu_pose_graph as PG

pytestmark = pytest.mark.gpu

TRIVIAL, HUBER, CAUCHY = 0, 1, 2
UP = np.array([0.0, 0.0, 1.0])


def _loss(kind, scale, s):
    rho, w = C.c_double(), C.c_double()
    PC._lib().bba_host_robust_loss(kind, scale, s, C.byref(rho), C.byref(w))
    return rho.value, w.value


def _attitude_terms(d_ref, d_meas, L, pose):
    H, b, cost = np.zeros(21), np.zeros(6), C.c_double()
    dr, dm, p = PC._f32(d_ref), PC._f32(d_meas), PC._f32(pose)
    PC._lib().bba_host_attitude_prior_terms(dr.ctypes.data, dm.ctypes.data, float(L), p.ctypes.data, H.ctypes.data, b.ctypes.data,
                                             C.byref(cost))
    return H, b, cost.value


def _measured(poses32, d_ref=UP):
    """d_meas = R_k^-1 d_ref of fp32 poses."""
    return np.array([A.tilt(O.from_array(p)[0], d_ref) for p in poses32], np.float32)


def _tilt_errors(poses32, truth32, d_ref=UP):
    got, want = _measured(poses32, d_ref), _measured(truth32, d_ref)
    return np.arccos(np.clip(np.sum(np.float64(got) * want, 1), -1, 1))


def _attitude_on_all(ba, sc, L=1e3, loss="trivial", scale=1.0):
    K = sc.cfg.num_keyframes
    ba.SetKeyframeAttitudePriors(np.arange(K), UP, _measured(sc.poses_true), L, loss, scale)


# ---- 1. unchanged paths --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("scheme", ["alternating", "pcg"])
@pytest.mark.parametrize("scene", ["tiny", "small"])
def test_set_then_clear_changes_no_bit(scene, scheme):
    """The alternating scheme in the deterministic mode gives the same bits, and both schemes the same results and launch counts,
    as a handle that never had attitude priors (with priors and constraints present, as in test_gpu_robust_pose_terms)."""
    import test_gpu_robust_pose_terms as RT
    sc = PC._scene(scene)
    outs = []
    for set_clear in (False, True):
        ba = PC._make(sc, deterministic=scheme == "alternating")
        RT._priors_and_constraints(ba, sc)
        if set_clear:
            _attitude_on_all(ba, sc, loss="cauchy")
            ba.ClearKeyframeAttitudePriors()
        if scheme == "alternating":
            r = ba.BundleAdjustment(None, True, True, True, True, True, 2, 2)
        else:
            r = ba.BundleAdjustment(None, False, False, False, True, True, 2, 2, use_pcg=True, pcg_gauge_keyframe=0)
        outs.append((PC._state(ba), R._result(r), r.kernel_launches))
    assert np.array_equal(outs[0][1], outs[1][1]) and outs[0][2] == outs[1][2]
    if scheme == "alternating":
        PC._same_state(outs[0][0], outs[1][0])
    else:
        from badslam_b200.scene import pose_error
        worst = max(max(pose_error(p, q)) for p, q in zip(outs[0][0]["poses"], outs[1][0]["poses"]))
        assert worst < 1e-4, worst


def test_frame_pose_and_pose_graph_change_no_bit():
    sc = PC._scene("small")
    outs = []
    for set_clear in (False, True):
        ba = PC._make(sc, deterministic=True)
        if set_clear:
            _attitude_on_all(ba, sc)
            ba.ClearKeyframeAttitudePriors(np.arange(sc.cfg.num_keyframes))
        launches = ba.kernel_launch_count()
        est, its, conv = ba.EstimateFramePose(None, sc.poses_init[2], 2)
        ba.SetKeyframeStates(sc.poses_init)
        r = ba.OptimizePoseGraph(odometry_information=np.diag([1e2] * 6))
        outs.append((est.view(np.uint32).copy(), its, conv, PG._poses_bits(ba), r, ba.kernel_launch_count() - launches))
    for x, y in zip(outs[0], outs[1]):
        assert np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y


# ---- 2. the pose graph against the oracle --------------------------------------------------------------------------------------

def _tilted_circle(K, per_kf=0.002, seed=3):
    truth = O.circle(K)
    return truth, PG._f32(A.tilted(truth, per_kf, seed=seed))


def _graph_case(ba, K, truth, start, L_att=1e4, L_chain=1e3, loops=((5, None),), atts=None):
    """The chain at `start`, a loop edge from the truth, attitude priors from the truth on every keyframe (or `atts`)."""
    ba.SetKeyframeStates(start)
    Lc = L_chain * np.eye(6)
    cons = [(a, K - 3 if b is None else b, PG._relative(truth, a, K - 3 if b is None else b)) for a, b in loops]
    ba.AddKeyframePoseConstraints([c[0] for c in cons], [c[1] for c in cons], [c[2] for c in cons], Lc)
    d_meas = _measured(PG._f32(truth)) if atts is None else atts
    ba.SetKeyframeAttitudePriors(np.arange(K), UP, d_meas, L_att)
    S = O.from_array(start)
    terms = [O.Term(a, b, Z, Lc) for a, b, Z in cons]
    terms += [O.Term(k, k + 1, PG._f32(O.mul(O.inv(O.pose(S, k)), O.pose(S, k + 1))), Lc) for k in range(K - 1)]
    attitude = [A.Attitude(k, np.float32(UP), d_meas[k], np.float32(L_att)) for k in range(K)]
    return S, terms, attitude, Lc


@pytest.mark.parametrize("gauge", [-1, 0])
def test_pose_graph_matches_the_oracle(gauge):
    K = 200
    truth, start = _tilted_circle(K)
    ba = PG.make_handle(K)
    S, terms, atts, Lc = _graph_case(ba, K, truth, start)
    r = ba.OptimizePoseGraph(gauge_keyframe=gauge, odometry_information=Lc)
    want, held, axes, cost, _ = A.gauss_newton(terms, [(TRIVIAL, 0.0)] * len(terms), atts, S, gauge=gauge)
    got = ba.GetKeyframeStates()[0]
    dt, dr = PG._worst(got, want)
    G = O.from_array(got)
    before, after = _tilt_errors(start, PG._f32(truth)), _tilt_errors(got, PG._f32(truth))
    print(f"gauge {gauge}: {r}, oracle cost {cost:.6g}, worst pose error {dt:.3g} m / {dr:.3g} rad; mean tilt error "
          f"{before.mean():.4g} -> {after.mean():.4g} rad")
    assert dt <= 1e-5 and dr <= 1e-5, (dt, dr)
    assert abs(r["final_cost"] - cost) <= 1e-4 * cost and r["converged"] == 1
    assert after.mean() < 0.2 * before.mean()
    assert held[0] == (1 if gauge == 0 else 2) and r["held_keyframes"] == (1 if gauge == 0 else 0)
    # keyframe 0 keeps its translation and its yaw about d_ref
    assert np.max(np.abs(G[1][0] - S[1][0])) <= 1e-6
    assert abs(A.yaw_about(G[0][0], S[0][0], UP)) <= 1e-6


def test_lone_keyframe_and_nonparallel_directions():
    """A keyframe with only an attitude prior is optimised (held in translation and yaw only); with reference directions that are
    not parallel only translation is held."""
    K = 4
    truth, start = _tilted_circle(K, per_kf=0.05, seed=1)
    ba = PG.make_handle(K)
    ba.SetKeyframeStates(start)
    d_meas = _measured(PG._f32(truth))
    ba.SetKeyframeAttitudePriors([2], UP, d_meas[2:3], 1e4)
    r = ba.OptimizePoseGraph(add_current_state_odometry_constraints=False)
    got = ba.GetKeyframeStates()[0]
    assert np.array_equal(got[[0, 1, 3]].view(np.uint32), start[[0, 1, 3]].view(np.uint32))
    assert _tilt_errors(got[2:3], PG._f32(truth)[2:3])[0] < 1e-5 and r["held_keyframes"] == 3
    S = O.from_array(start)
    G = O.from_array(got)
    assert np.array_equal(got[2, 4:], start[2, 4:]) and abs(A.yaw_about(G[0][2], S[0][2], UP)) <= 1e-6
    # two directions at right angles on a chained component: rotation is free, translation held at the lowest id
    ba = PG.make_handle(K)
    ba.SetKeyframeStates(start)
    side = np.array([1.0, 0.0, 0.0])
    ba.SetKeyframeAttitudePriors([0, 1, 2, 3], [UP, side, UP, side],
                                 np.array([A.tilt(O.pose(truth, k)[0], d) for k, d in enumerate([UP, side, UP, side])], np.float32), 1e4)
    ba.OptimizePoseGraph(gauge_keyframe=-1, odometry_information=1e3 * np.eye(6))
    got = ba.GetKeyframeStates()[0]
    assert np.array_equal(got[0, 4:], start[0, 4:])
    assert np.max(np.abs(got[0, :4] - start[0, :4])) > 1e-4   # its rotation moved, yaw included


# ---- 3. end to end on `small` --------------------------------------------------------------------------------------------------

def test_tilt_drift_end_to_end_on_small(small_scene):
    """A progressive roll / pitch drift (0.02 rad per keyframe about random horizontal axes) carried over to the surfels, then the
    pose graph (gauge keyframe 0, which has no drift), the surfel deformation and ten BA iterations in either scheme, with and
    without attitude priors from the truth (sigma 0.01 rad)."""
    from badslam_b200.direct_ba import DirectBA
    sc = small_scene
    K = sc.cfg.num_keyframes
    truth = O.from_array(sc.poses_true)
    drifted = PG._f32(A.tilted(truth, 0.02, seed=5))
    errors = {}
    for arm in ("none", "attitude"):
        for scheme in ("alternating", "pcg"):
            ba = DirectBA.from_scene(sc, poses=sc.poses_true, device="cuda:0")
            original = ba.RememberKeyframePoses()
            ba.SetKeyframeStates(drifted)
            ba.DeformSurfelsWithKeyframePoseChanges(original)
            if arm == "attitude":
                _attitude_on_all(ba, sc, L=1e4)
            remembered = ba.RememberKeyframePoses()
            ba.OptimizePoseGraph(odometry_information=np.diag([1e2] * 3 + [1e3] * 3))
            ba.DeformSurfelsWithKeyframePoseChanges(remembered)
            if scheme == "alternating":
                ba.BundleAdjustment(None, False, False, False, True, True, 10, 10)
            else:
                ba.BundleAdjustment(None, False, False, False, True, True, 10, 10, use_pcg=True, pcg_gauge_keyframe=0)
            errors[arm, scheme] = float(_tilt_errors(ba.GetKeyframeStates()[0], sc.poses_true).mean())
    start = float(_tilt_errors(drifted, sc.poses_true).mean())
    print(f"mean tilt error: start {start:.4g} rad; " + ", ".join(f"{a}/{s} {v:.4g}" for (a, s), v in errors.items()))
    for scheme in ("alternating", "pcg"):
        assert errors["attitude", scheme] < 0.5 * errors["none", scheme], errors


# ---- 4. bba_estimate_frame_pose ------------------------------------------------------------------------------------------------

def test_estimate_frame_pose_follows_numpy_irls():
    sc = PC._scene("small")
    ba = PC._make(sc, deterministic=True)
    k = 2
    lib = PC._lib()
    d_meas = A.tilt(O.from_array(sc.poses_true[k])[0], UP)
    wrong = np.float32(O.so3_exp(np.r_[0.05, 0.0, 0.0]) @ d_meas)
    ba.SetKeyframeAttitudePriors([k], UP, wrong[None], 1e7, "huber", 100.0)   # s = 2.5e4: w = 0.63
    got, its, _ = ba.EstimateFramePose(None, sc.poses_init[k], k)
    rec = ba.GetKeyframeAttitudePrior(k)   # the record as the solver reads it: both directions normalised in fp32
    pose = np.array(sc.poses_init[k], np.float32)
    want_its = 30
    for it in range(30):
        c = ba.AccumulatePoseEstimationCoeffs(k, pose)
        H = np.array(c.H, np.float32).astype(np.float64)
        b = np.array(c.b, np.float32).astype(np.float64)
        Hp, bp, cost = _attitude_terms(rec["reference_direction"], rec["measured_direction"], rec["information"], pose)
        w = _loss(HUBER, 100.0, 2.0 * cost)[1]
        H, b = H + w * Hp, b + w * bp
        x = np.zeros(6)
        assert lib.bba_host_solve_ldlt(6, H.ctypes.data, b.ctypes.data, x.ctypes.data) == 1
        xf = x.astype(np.float32)
        pose = PC._compose(pose, PC._exp(-xf))
        if lib.bba_host_pose_update_converged(xf.ctypes.data):
            want_its = it + 1
            break
    assert its == want_its, (its, want_its)
    assert np.abs(got.astype(np.float64) - pose).max() < 2e-6, (got, pose)
    plain, _, _ = PC._make(sc, deterministic=True).EstimateFramePose(None, sc.poses_init[k], k)
    assert np.abs(plain.astype(np.float64) - pose).max() > 1e-6


# ---- 5. robust losses ----------------------------------------------------------------------------------------------------------

def test_cauchy_keeps_a_wrong_attitude_prior_out():
    K = 60
    truth, start = _tilted_circle(K, seed=8)
    d_meas = _measured(PG._f32(truth))
    wrong = d_meas.copy()
    wrong[30] = np.float32(O.so3_exp(np.r_[np.deg2rad(30.0), 0.0, 0.0]) @ d_meas[30])
    tilts = {}
    for arm in ("clean", "outlier"):
        ba = PG.make_handle(K)
        _graph_case(ba, K, truth, start, atts=wrong if arm == "outlier" else d_meas)
        ba.SetKeyframeAttitudePriors(np.arange(K), UP, wrong if arm == "outlier" else d_meas, 1e4, "cauchy", 1.0)
        ba.OptimizePoseGraph(gauge_keyframe=0, odometry_information=1e3 * np.eye(6))
        tilts[arm] = _tilt_errors(ba.GetKeyframeStates()[0], PG._f32(truth))
        if arm == "outlier":
            s, w = ba.EvaluateKeyframeAttitudePriors()
            got = ba.GetKeyframeStates()[0]
            for k in (0, 29, 30):
                want_s = 2.0 * _attitude_terms(UP, wrong[k], 1e4, got[k])[2]
                assert s[k] == pytest.approx(want_s, rel=1e-9, abs=1e-12) and w[k] == pytest.approx(_loss(CAUCHY, 1.0, want_s)[1], rel=1e-9)
            print(f"weights: outlier {w[30]:.3g}, others min {np.delete(w, 30).min():.3g}")
            assert w[30] < 0.1 and np.all(np.delete(w, 30) > 0.5)
    worst = float(np.max(np.abs(tilts["outlier"] - tilts["clean"])))
    print(f"largest tilt change from the outlier-free result: {worst:.3g} rad")
    assert worst < 2e-3, worst


# ---- 6. reproducibility and ranks ----------------------------------------------------------------------------------------------

def _graph_run(ba, K):
    truth, start = _tilted_circle(K, seed=4)
    _graph_case(ba, K, truth, start)
    ba.SetKeyframeAttitudePriors([3], UP, np.float32([0.1, 0.0, 1.0])[None], 1e4, "huber", 2.0)
    r = ba.OptimizePoseGraph(gauge_keyframe=-1, odometry_information=1e3 * np.eye(6))
    s, w = ba.EvaluateKeyframeAttitudePriors()
    return ba.GetKeyframeStates()[0], r, np.r_[s, w]


def test_reproducible_bits():
    K = 60
    outs = [_graph_run(PG.make_handle(K, deterministic=det), K) for det in (False, False, True)]
    for poses, r, ev in outs[1:]:
        assert np.array_equal(poses.view(np.uint32), outs[0][0].view(np.uint32)) and r == outs[0][1]
        assert np.array_equal(ev.view(np.uint64), outs[0][2].view(np.uint64))
    sc = PC._scene("small")
    states = []
    for _ in range(2):
        ba = PC._make(sc, deterministic=True)
        _attitude_on_all(ba, sc, loss="huber", scale=0.5)
        r = ba.BundleAdjustment(None, True, True, True, True, True, 2, 2)
        states.append((PC._state(ba), R._result(r)))
    PC._same_state(states[0][0], states[1][0])
    assert np.array_equal(states[0][1], states[1][1])


@pytest.mark.parametrize("world", ["2", "3"])
def test_local_group_pose_graph(world):
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    K = 40

    def run(rank, ba):
        PG._add_keyframes(ba, K)
        return _graph_run(ba, K)
    handles = DirectBA.create_local_ranks(PG._images(), int(world), ["cuda:0"] * int(world), max_keyframes=K)
    with LocalGroup(handles) as group:
        outs = group.run(run)
    want = _graph_run(PG.make_handle(K), K)
    for poses, r, ev in outs:
        assert np.array_equal(poses.view(np.uint32), want[0].view(np.uint32)) and r == want[1]
        assert np.array_equal(ev.view(np.uint64), want[2].view(np.uint64))


def _with_attitude(ba):
    _attitude_on_all(ba, R.SCENES["small"]())


def run_alternating_attitude(ba):
    _with_attitude(ba)
    return R.run_pose(ba)


def run_pcg_attitude(ba):
    _with_attitude(ba)
    return R.run_pcg(ba, False)


@pytest.mark.parametrize("world", ["2", "3"])
@pytest.mark.parametrize("scheme", ["alternating", "pcg"])
def test_local_group_bundle_adjustment(world, scheme):
    """As test_gpu_robust_pose_terms.test_local_group_bundle_adjustment, with attitude priors on every keyframe: identical replicas,
    and one rank's results up to the order in which the ranks sum the pose normal equations (the alternating poses to 5e-5: the
    attitude priors move every keyframe, so that order shows in more of them than with constraints alone)."""
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    from badslam_b200.scene import pose_error
    fn = run_alternating_attitude if scheme == "alternating" else run_pcg_attitude
    handles = DirectBA.create_local_ranks(R.SCENES["small"](), int(world), ["cuda:0"] * int(world))
    with LocalGroup(handles) as group:
        outs = group.run(lambda r, ba: fn(ba))
    for o in outs[1:]:
        for k in ("poses", "act", "surfels", "active", "intr", "cf", "res"):
            assert R._same(o[k], outs[0][k]), k
    want = R.one_rank(("attitude priors", scheme), lambda: R._one("small", fn))
    got = outs[0]
    worst = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(len(want["poses"])))
    if scheme == "alternating":
        assert np.array_equal(got["res"][:5], want["res"][:5]) and np.array_equal(got["act"], want["act"])
        assert worst <= 5e-5, worst
    else:
        assert got["res"][0] == want["res"][0] and abs(int(got["res"][5]) - int(want["res"][5])) <= 2
        assert worst < 2e-4, worst


# ---- 7. refused arguments and the front end ------------------------------------------------------------------------------------

def test_refused_arguments_change_nothing():
    from badslam_b200._lib import BadBAError
    sc = PC._scene("tiny")
    ba = PC._make(sc)
    ba.SetKeyframeAttitudePriors([1], [0, 0, 2], [[0, 3, 0]], 5.0, "huber", 0.25)
    rec = ba.GetKeyframeAttitudePrior(1)
    assert np.array_equal(rec["reference_direction"], np.float32([0, 0, 1])) and np.array_equal(rec["measured_direction"], np.float32([0, 1, 0]))
    assert rec["information"] == 5.0 and (rec["loss_type"], rec["loss_scale"]) == (HUBER, 0.25)
    assert ba.GetKeyframeAttitudePrior(0) is None
    launches = ba.kernel_launch_count()
    before = [ba.GetKeyframeAttitudePrior(k) for k in range(sc.cfg.num_keyframes)]
    nan, inf = float("nan"), float("inf")
    bad = [dict(ids=[99]), dict(ids=[-1]), dict(d_ref=[0, 0, nan]), dict(d_meas=[inf, 0, 0]), dict(d_ref=[0, 0, 1e-7]),
           dict(d_meas=[0, 0, 0]), dict(L=0.0), dict(L=-1.0), dict(L=nan), dict(L=inf), dict(loss=3), dict(loss="cauchy", scale=0.0),
           dict(loss="huber", scale=nan)]
    for kw in bad:
        args = dict(ids=[0, 2], d_ref=[0, 0, 1], d_meas=[0, 1, 0], L=1.0, loss="trivial", scale=1.0)
        args.update(kw)
        n = len(args["ids"])
        with pytest.raises(BadBAError):
            ba.SetKeyframeAttitudePriors(args["ids"], args["d_ref"], np.broadcast_to(np.float32(args["d_meas"]), (n, 3)), args["L"],
                                         args["loss"], args["scale"])
        after = [ba.GetKeyframeAttitudePrior(k) for k in range(sc.cfg.num_keyframes)]
        assert [a is None for a in after] == [b is None for b in before] and ba.kernel_launch_count() == launches, kw
    with pytest.raises(BadBAError):
        ba.ClearKeyframeAttitudePriors([1, 99])
    assert ba.GetKeyframeAttitudePrior(1) is not None
    x = np.zeros(4)
    assert PC._lib().bba_evaluate_keyframe_attitude_priors(ba._h, -1, x.ctypes.data, None, None) != 0
    assert ba.kernel_launch_count() == launches
    s, w = ba.EvaluateKeyframeAttitudePriors()
    assert np.isnan(s[0]) and np.isnan(w[0]) and np.isfinite(s[1]) and np.isfinite(w[1])
    ba.ClearKeyframeAttitudePriors([1])
    assert ba.GetKeyframeAttitudePrior(1) is None
