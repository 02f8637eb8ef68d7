"""Robust losses on the keyframe pose priors and constraints (bba_set_keyframe_pose_prior_losses /
bba_set_keyframe_pose_constraint_losses, DESIGN §3.15): IRLS in the alternating pose step, bba_estimate_frame_pose, the PCG
products and bba_optimize_pose_graph.

* all-trivial losses, and Huber with delta above every term's sqrt(s), give the results of a handle that never had losses;
* circle graphs with false loops reach the robust numpy oracle's optimum and cost (tests/robust_pose_oracle.py), and
  bba_evaluate_keyframe_pose_terms gives the false loops weights far below the true loop's, matching the host functions;
* bba_estimate_frame_pose follows numpy's IRLS loop over bba_accumulate_pose_coeffs;
* the PCG products differ from those without terms by the w-scaled terms; the damping anchors carry their constraint's w;
* on `small`, a Cauchy loss keeps a false loop closure from bending the map through the pose graph, the deformation and BA;
* repeated calls, the deterministic mode and local groups of 2 and 3 ranks give the same bits;
* refused calls change nothing, and the front-end getters return the published losses."""
import ctypes as C

import numpy as np
import pytest

import pose_graph_oracle as O
import robust_pose_oracle as RO
import test_gpu_multi_ranks_one_device as R
import test_gpu_pose_constraints as PC
import test_gpu_pose_graph as PG
from gpu_checks import POSE_R, POSE_T

pytestmark = pytest.mark.gpu

TRIVIAL, HUBER, CAUCHY = 0, 1, 2


def _loss(kind, scale, s):
    rho, w = C.c_double(), C.c_double()
    PC._lib().bba_host_robust_loss(kind, scale, s, C.byref(rho), C.byref(w))
    return rho.value, w.value


def _priors_and_constraints(ba, sc):
    """Weak priors near the truth on every other keyframe and the constraints of test_gpu_pose_constraints."""
    K = sc.cfg.num_keyframes
    rng = np.random.default_rng(4)
    ids = np.arange(1, K, 2)
    P = sc.poses_true[ids].copy()
    P[:, 4:] += rng.normal(scale=0.01, size=(len(ids), 3)).astype(np.float32)
    ba.SetKeyframePosePriors(ids, P, PC._info(0.02, 0.02))
    a, b, Z, L = PC._constraints_for(sc)
    return ids, ba.AddKeyframePoseConstraints(a, b, Z, L)


# ---- 1. unchanged paths --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("losses", ["trivial", "huber_inlier"])
@pytest.mark.parametrize("scheme", ["alternating", "pcg"])
@pytest.mark.parametrize("scene", ["tiny", "small"])
def test_trivial_and_inlier_losses_change_no_bit(scene, scheme, losses):
    """The alternating scheme in the deterministic mode gives the same bits as a handle without losses; the PCG scheme stages the
    same fp32 terms (its products sum with fp32 atomics, so its poses are compared up to their run-to-run order, as in
    test_gpu_pose_constraints)."""
    sc = PC._scene(scene)
    outs = []
    for set_losses in (False, True):
        ba = PC._make(sc, deterministic=scheme == "alternating")
        priors, cons = _priors_and_constraints(ba, sc)
        if set_losses:
            kind, scale = (TRIVIAL, 0.0) if losses == "trivial" else (HUBER, 1e6)
            ba.SetKeyframePosePriorLosses(priors, kind, scale)
            ba.SetKeyframePoseConstraintLosses(cons, kind, scale)
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


@pytest.mark.parametrize("losses", ["trivial", "huber_inlier"])
def test_frame_pose_and_pose_graph_change_no_bit(losses):
    sc = PC._scene("small")
    K = sc.cfg.num_keyframes
    outs = []
    for set_losses in (False, True):
        ba = PC._make(sc, deterministic=True)
        priors, cons = _priors_and_constraints(ba, sc)
        if set_losses:
            kind, scale = (TRIVIAL, 0.0) if losses == "trivial" else (HUBER, 1e6)
            ba.SetKeyframePosePriorLosses(priors, kind, scale)
            ba.SetKeyframePoseConstraintLosses(cons, kind, scale)
        est, its, conv = ba.EstimateFramePose(None, sc.poses_init[2], 2)
        ba.SetKeyframeStates(sc.poses_init)
        r = ba.OptimizePoseGraph(odometry_information=np.diag([1e2] * 6))
        outs.append((est.view(np.uint32).copy(), its, conv, PG._poses_bits(ba), r))
    for x, y in zip(outs[0], outs[1]):
        assert np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y


# ---- 2. the pose graph against the robust oracle -------------------------------------------------------------------------------

_WRONG = np.r_[0.3, -0.3, 0.3, 0.0, 0.0, np.deg2rad(20.0)]   # 0.52 m and 20 degrees


def _false_loop_graph(K, truth, false_pairs):
    cons = [(5, K - 3, PG._relative(truth, 5, K - 3))]
    for a, b in false_pairs:
        cons.append((a, b, PG._f32(O.mul(O.mul(O.inv(O.pose(truth, a)), O.pose(truth, b)), O.se3_exp(_WRONG)))))
    return cons


@pytest.mark.parametrize("loss", ["cauchy", "huber"])
def test_pose_graph_matches_the_robust_oracle(loss):
    K = 200
    kind = CAUCHY if loss == "cauchy" else HUBER
    truth, start = PG._circle(K)
    L = 1e4 * np.eye(6)   # sigma 1 cm / 0.01 rad on every edge, the chain included
    cons = _false_loop_graph(K, truth, [(20, 30), (80, 91), (140, 149)])
    ba = PG.make_handle(K)
    ba.SetKeyframeStates(start)
    ids = ba.AddKeyframePoseConstraints([c[0] for c in cons], [c[1] for c in cons], [c[2] for c in cons], L)
    ba.SetKeyframePoseConstraintLosses(ids, kind, 1.0)
    r = ba.OptimizePoseGraph(odometry_information=L)
    S = O.from_array(start)
    terms = [O.Term(a, b, Z, L) for a, b, Z in cons]
    terms += [O.Term(k, k + 1, PG._f32(O.mul(O.inv(O.pose(S, k)), O.pose(S, k + 1))), L) for k in range(K - 1)]
    losses = [(kind, 1.0)] * len(cons) + [(TRIVIAL, 0.0)] * (K - 1)
    want, held, cost, _ = RO.gauss_newton(terms, losses, S, gauge=0)
    got = ba.GetKeyframeStates()[0]
    dt, dr = PG._worst(got, want)
    print(f"{loss}: {r}, oracle cost {cost:.6g}, worst pose error {dt:.3g} m / {dr:.3g} rad")
    assert dt < POSE_T and dr < POSE_R, (dt, dr)
    assert abs(r["final_cost"] - cost) <= 1e-4 * cost, (r["final_cost"], cost)
    assert r["converged"] == 1 and r["final_cost"] <= r["initial_cost"]
    assert r["linear_iterations"] <= (12 * len(cons) + 4) * r["iterations"], r
    # the weights afterwards, on the device and on the host
    ev = ba.EvaluateKeyframePoseTerms()
    assert np.array_equal(ev["constraint_ids"], ids) and np.all(np.isnan(ev["prior_s"]))
    for i, (a, b, Z) in enumerate(cons):
        s = 2.0 * PC._constraint_terms(Z, got[a], got[b], PC._upper(L))[2]
        w = _loss(kind, 1.0, s)[1]
        assert ev["constraint_s"][i] == pytest.approx(s, rel=1e-9, abs=1e-12) and ev["constraint_weight"][i] == pytest.approx(w, rel=1e-9)
    w = ev["constraint_weight"]
    print(f"weights: true loop {w[0]:.4g}, false loops {w[1:]}")
    assert np.all(w[1:] < 0.1 * w[0]), w


# ---- 3. bba_estimate_frame_pose ------------------------------------------------------------------------------------------------

def _numpy_irls_pose_step(ba, k, init, terms, max_iterations=30):
    """test_gpu_pose_constraints._numpy_pose_step with each (prior, L, loss) term's H and b scaled by its weight at the current
    pose."""
    lib = PC._lib()
    pose = np.array(init, np.float32)
    for it in range(max_iterations):
        c = ba.AccumulatePoseEstimationCoeffs(k, pose)
        H = np.array(c.H, np.float32).astype(np.float64)
        b = np.array(c.b, np.float32).astype(np.float64)
        for prior, info21, (kind, scale) in terms:
            Hp, bp, cost = PC._prior_terms(prior, pose, info21)
            w = _loss(kind, scale, 2.0 * cost)[1]
            H, b = H + w * Hp, b + w * bp
        x = np.zeros(6)
        assert lib.bba_host_solve_ldlt(6, H.ctypes.data, b.ctypes.data, x.ctypes.data) == 1
        xf = x.astype(np.float32)
        pose = PC._compose(pose, PC._exp(-xf))
        if lib.bba_host_pose_update_converged(xf.ctypes.data):
            return pose, it + 1
    return pose, max_iterations


def test_estimate_frame_pose_follows_numpy_irls():
    """Keyframe 2 with a Huber prior 3 cm off and two constraints, one a Cauchy outlier (its equivalent prior 5 cm off)."""
    sc = PC._scene("small")
    ba = PC._make(sc, deterministic=True)
    k = 2
    prior = sc.poses_true[k].copy()
    prior[4:] += np.float32([0.02, -0.015, 0.015])
    Lp, L1, L2 = PC._info(3e-3, 3e-3), PC._info(2e-3, 4e-3), PC._info(4e-3, 2e-3)
    Z1 = PC._compose(PC._relative(sc.poses_init[1], sc.poses_true[k]), PC._exp([0.03, 0.0, -0.04, 0.02, 0.01, 0.0]))
    Z2 = PC._compose(PC._relative(sc.poses_true[k], sc.poses_init[3]), PC._exp([-0.002, 0.003, 0.0, 0.0, -0.002, 0.001]))
    ba.SetKeyframePosePriors([k], prior[None], Lp)
    ids = ba.AddKeyframePoseConstraints([1, k], [k, 3], np.stack([Z1, Z2]), np.stack([L1, L2]))
    ba.SetKeyframePosePriorLosses([k], "huber", 2.0)
    ba.SetKeyframePoseConstraintLosses(ids[:1], "cauchy", 1.5)
    got, its, _ = ba.EstimateFramePose(None, sc.poses_init[k], k)
    terms = [(prior, PC._upper(Lp), (HUBER, 2.0)),
             (PC._compose(sc.poses_init[1], Z1), PC._upper(L1), (CAUCHY, 1.5)),
             (PC._compose(sc.poses_init[3], PC._inverse(Z2)), PC._upper(PC._info_a(Z2, L2)), (TRIVIAL, 0.0))]
    want, want_its = _numpy_irls_pose_step(ba, k, sc.poses_init[k], terms)
    assert its == want_its, (its, want_its)
    assert np.abs(got.astype(np.float64) - want).max() < 2e-6, (got, want)
    plain, _ = _numpy_irls_pose_step(ba, k, sc.poses_init[k], [(p, L, (TRIVIAL, 0.0)) for p, L, _ in terms])
    assert np.abs(plain.astype(np.float64) - want).max() > 1e-4


# ---- 4. PCG products and damping anchors ---------------------------------------------------------------------------------------

def test_pcg_products_differ_by_the_weighted_terms():
    """test_gpu_pose_constraints.test_pcg_products_differ_by_the_constraint_terms with Cauchy / Huber losses: on the two moved-out
    keyframes r and M are exactly the constraints' terms scaled by their weights at the start poses."""
    sc = PC._scene("small")
    K = sc.cfg.num_keyframes
    poses = sc.poses_init.copy()
    poses[K - 2, 4] += 100.0
    poses[K - 1, 4] += 100.0
    Z1 = PC._compose(PC._relative(poses[K - 2], poses[K - 1]), PC._exp([0.05, 0.0, -0.04, 0.0, 0.06, 0.0]))
    Z2 = PC._compose(PC._relative(poses[0], poses[K - 1]), PC._exp([0.0, 0.02, 0.0, 0.01, 0.0, 0.0]))
    L1, L2 = PC._info(0.01, 0.02), PC._info(0.02, 0.01)
    probes = []
    for with_constraints in (False, True):
        ba = PC._make(sc, poses=poses)
        if with_constraints:
            ids = ba.AddKeyframePoseConstraints([K - 2, 0], [K - 1, K - 1], np.stack([Z1, Z2]), np.stack([L1, L2]))
            ba.SetKeyframePoseConstraintLosses(ids, ["cauchy", "huber"], [1.0, 0.5])
        probes.append(ba.PCGProbe(0, False, True, True, gauge_keyframe=0))
    a, b = probes
    n = len(a["r"])
    u = 6 * (K - 3)
    s = slice(u, u + 12)
    H1, b1, c1 = PC._constraint_terms(Z1, poses[K - 2], poses[K - 1], PC._upper(L1))
    H2, b2, c2 = PC._constraint_terms(Z2, poses[0], poses[K - 1], PC._upper(L2))
    w1, w2 = _loss(CAUCHY, 1.0, 2 * c1)[1], _loss(HUBER, 0.5, 2 * c2)[1]
    assert w1 < 0.5 and w2 < 0.5, (w1, w2)
    Hm = w1 * PC._matrix(H1, 12)
    Hm[6:, 6:] += w2 * PC._matrix(H2, 12)[6:, 6:]
    bv = w1 * b1
    bv[6:] += w2 * b2[6:]
    assert np.abs(b["r"][s] + bv).max() <= 1e-5 * np.abs(bv).max()
    assert np.abs(b["M"][s] - np.diag(Hm)).max() <= 1e-5 * np.abs(np.diag(Hm)).max()
    pb = b["p"][s].astype(np.float64)
    want_g = Hm @ pb
    assert np.abs(b["g"][s] - want_g).max() <= 1e-4 * np.abs(want_g).max()
    rest = np.ones(n, bool)
    rest[s] = False
    for k in ("r", "M", "p", "g"):
        np.testing.assert_allclose(b[k][rest], a[k][rest], rtol=1e-4, atol=1e-4 * max(1e-30, np.abs(a[k]).max()), err_msg=k)


def test_damping_anchors_carry_the_constraint_weight():
    """Two free keyframes out of the map with one Cauchy constraint: one alternating BA iteration moves each end as numpy's IRLS
    loop over its equivalent prior (weighted at the current estimate) and its anchor (information w0 H_kk, w0 the constraint's
    weight at the start poses)."""
    sc = PC._scene("small")
    K = sc.cfg.num_keyframes
    a, b = K - 2, K - 1
    poses = sc.poses_init.copy()
    poses[a, 4] += 100.0
    poses[b, 4] += 100.0
    ba = PC._make(sc, poses=poses)
    Z = PC._compose(PC._relative(poses[a], poses[b]), PC._exp([0.03, 0.0, -0.02, 0.02, 0.0, 0.01]))
    Lc = PC._upper(PC._info(0.01, 0.01))
    ids = ba.AddKeyframePoseConstraints([a], [b], Z[None], Lc)
    ba.SetKeyframePoseConstraintLosses(ids, "cauchy", 2.0)
    H, _, cost = PC._constraint_terms(Z, poses[a], poses[b], Lc)
    w0 = _loss(CAUCHY, 2.0, 2 * cost)[1]
    assert w0 < 0.2, w0
    Hm = PC._matrix(H, 12)
    ba.BundleAdjustment(None, False, False, False, True, False, 1, 1)
    got = ba.GetKeyframeStates()[0]
    loss = (CAUCHY, 2.0)
    for k, eq, info, block in ((a, PC._compose(poses[b], PC._inverse(Z)), PC._upper(PC._info_a(Z, PC._matrix(Lc, 6))), Hm[:6, :6]),
                               (b, PC._compose(poses[a], Z), Lc, Hm[6:, 6:])):
        anchor = PC._upper(block * w0)
        want, _ = _numpy_irls_pose_step(ba, k, poses[k], [(eq, info, loss), (poses[k], anchor, (TRIVIAL, 0.0))])
        full, _ = _numpy_irls_pose_step(ba, k, poses[k], [(eq, info, loss), (poses[k], PC._upper(block), (TRIVIAL, 0.0))])
        err, off = np.abs(got[k].astype(np.float64) - want).max(), np.abs(full.astype(np.float64) - want).max()
        print(f"keyframe {k}: |device - numpy| {err:.3g}, |numpy with unweighted anchor - numpy| {off:.3g}")
        assert err < 2e-5 and off > 10 * err + 1e-4, (err, off)


# ---- 5. end to end on small ----------------------------------------------------------------------------------------------------

def test_false_loop_closure_end_to_end_on_small(small_scene):
    """test_gpu_pose_graph.test_loop_closure_end_to_end_on_small's drifted second half and true loop edge, plus one false
    constraint (0.52 m and 20 degrees off), then the pose graph, the surfel deformation and BA: with a Cauchy loss on the loop
    edges the map ends near the run without the false constraint; with the trivial loss it does not."""
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import se3_exp, se3_inverse, se3_mul
    sc = small_scene
    K = sc.cfg.num_keyframes
    D = se3_exp([0.12, -0.08, 0.06, 0.03, -0.04, 0.05])
    pivot = sc.poses_true[K // 2 - 1]
    move = se3_mul(se3_mul(pivot, D), se3_inverse(pivot))
    drifted = np.array([sc.poses_true[k] if k < K // 2 else se3_mul(move, sc.poses_true[k]) for k in range(K)], np.float32)
    L = np.diag([1e4] * 3 + [1e5] * 3)
    errors = {}
    for arm in ("clean", "trivial", "cauchy"):
        ba = DirectBA.from_scene(sc, poses=sc.poses_true, device="cuda:0")
        original = ba.RememberKeyframePoses()
        ba.SetKeyframeStates(drifted)
        ba.DeformSurfelsWithKeyframePoseChanges(original)
        pairs = [(0, K - 1)] + ([] if arm == "clean" else [(1, K - 2)])
        Z = [se3_mul(se3_inverse(sc.poses_true[i]), sc.poses_true[j]) for i, j in pairs]
        if arm != "clean":
            Z[1] = se3_mul(Z[1], se3_exp(_WRONG))
        ids = ba.AddKeyframePoseConstraints([p[0] for p in pairs], [p[1] for p in pairs], np.array(Z, np.float32), L)
        if arm == "cauchy":
            ba.SetKeyframePoseConstraintLosses(ids, "cauchy", 10.0)
        remembered = ba.RememberKeyframePoses()
        r = ba.OptimizePoseGraph(odometry_information=L)   # an odometry chain as certain as the loop edges claim to be
        assert r["final_cost"] < r["initial_cost"]
        ba.DeformSurfelsWithKeyframePoseChanges(remembered)
        if arm == "cauchy":   # the caller drops what the robust pose graph rejected before BA
            w = ba.EvaluateKeyframePoseTerms()["constraint_weight"]
            print(f"weights after the pose graph: true loop {w[0]:.3g}, false loop {w[1]:.3g}")
            assert w[1] < 0.1 * w[0]
            ba.RemoveKeyframePoseConstraints(ids[w < 0.1 * w.max()])
        ba.BundleAdjustment(None, False, False, False, True, True, 10, 10)
        errors[arm] = PG._aligned_error(ba.GetKeyframeStates()[0], sc.poses_true)
    print(f"mean keyframe error to the truth after BA: without the false loop {errors['clean']}, with it under the trivial loss "
          f"{errors['trivial']}, under Cauchy {errors['cauchy']}")
    assert errors["cauchy"][0] < errors["trivial"][0] and errors["cauchy"][1] < errors["trivial"][1], errors
    assert errors["cauchy"][0] < 1.5 * errors["clean"][0] + 2e-3, errors


# ---- 6. reproducibility and ranks ----------------------------------------------------------------------------------------------

def _robust_loop_case(ba, K):
    truth, start = PG._circle(K, seed=6)
    ba.SetKeyframeStates(start)
    cons = _false_loop_graph(K, truth, [(3, 9), (20, K - 10)])
    L = 1e4 * np.eye(6)
    ids = ba.AddKeyframePoseConstraints([c[0] for c in cons], [c[1] for c in cons], [c[2] for c in cons], L)
    ba.SetKeyframePoseConstraintLosses(ids, ["huber", "cauchy", "cauchy"], [3.0, 1.0, 1.0])
    r = ba.OptimizePoseGraph(odometry_information=L)
    ev = ba.EvaluateKeyframePoseTerms()
    return ba.GetKeyframeStates()[0], r, np.r_[ev["constraint_s"], ev["constraint_weight"]]


def test_reproducible_bits():
    K = 60
    outs = [_robust_loop_case(PG.make_handle(K, deterministic=det), K) for det in (False, False, True)]
    for poses, r, ev in outs[1:]:
        assert np.array_equal(poses.view(np.uint32), outs[0][0].view(np.uint32)) and r == outs[0][1]
        assert np.array_equal(ev.view(np.uint64), outs[0][2].view(np.uint64))
    sc = PC._scene("small")
    states = []
    for _ in range(2):
        ba = PC._make(sc, deterministic=True)
        priors, cons = _priors_and_constraints(ba, sc)
        ba.SetKeyframePosePriorLosses(priors, "huber", 0.5)
        ba.SetKeyframePoseConstraintLosses(cons, "cauchy", 1.0)
        r = ba.BundleAdjustment(None, True, True, True, True, True, 2, 2)
        states.append((PC._state(ba), R._result(r)))
    PC._same_state(states[0][0], states[1][0])
    assert np.array_equal(states[0][1], states[1][1])


@pytest.mark.parametrize("world", ["2", "3"])
@pytest.mark.parametrize("mode", ["gather", "peer"])
def test_local_group_pose_graph(world, mode):
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    K = 40

    def run(rank, ba):
        PG._add_keyframes(ba, K)
        return _robust_loop_case(ba, K)
    handles = DirectBA.create_local_ranks(PG._images(), int(world), ["cuda:0"] * int(world), max_keyframes=K)
    with LocalGroup(handles, peer_stores=mode == "peer") as group:
        outs = group.run(run)
    want = _robust_loop_case(PG.make_handle(K), K)
    for poses, r, ev in outs:
        assert np.array_equal(poses.view(np.uint32), want[0].view(np.uint32)) and r == want[1]
        assert np.array_equal(ev.view(np.uint64), want[2].view(np.uint64))


def _robust(ba):
    a, b, Z, L = PC._constraints_for(R.SCENES["small"]())
    ids = ba.AddKeyframePoseConstraints(a, b, Z, L)
    ba.SetKeyframePoseConstraintLosses(ids, "cauchy", 1.0)


def run_alternating_robust(ba):
    _robust(ba)
    return R.run_pose(ba)


def run_pcg_robust(ba):
    _robust(ba)
    return R.run_pcg(ba, False)


@pytest.mark.parametrize("world", ["2", "3"])
@pytest.mark.parametrize("mode", ["gather", "peer"])
@pytest.mark.parametrize("scheme", ["alternating", "pcg"])
def test_local_group_bundle_adjustment(world, mode, scheme):
    """As test_gpu_pose_constraints.test_local_group_ranks, with Cauchy losses on the constraints: identical replicas, and one
    rank's results (bit for bit in the residual counts and activations, to POSE_T / POSE_R in the poses, as there)."""
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    from badslam_b200.scene import pose_error
    fn = run_alternating_robust if scheme == "alternating" else run_pcg_robust
    handles = DirectBA.create_local_ranks(R.SCENES["small"](), int(world), ["cuda:0"] * int(world))
    with LocalGroup(handles, peer_stores=mode == "peer") as group:
        outs = group.run(lambda r, ba: fn(ba))
    for o in outs[1:]:
        for k in ("poses", "act", "surfels", "active", "intr", "cf", "res"):
            assert R._same(o[k], outs[0][k]), k
    want = R.one_rank(("robust constraints", scheme), lambda: R._one("small", fn))
    got = outs[0]
    worst = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(len(want["poses"])))
    if scheme == "alternating":
        assert np.array_equal(got["res"][:5], want["res"][:5]) and np.array_equal(got["act"], want["act"])
        assert worst <= min(POSE_T, POSE_R), worst
    else:
        assert got["res"][0] == want["res"][0] and abs(int(got["res"][5]) - int(want["res"][5])) <= 2
        assert worst < 2e-4, worst


# ---- 7. refused arguments and the front end ------------------------------------------------------------------------------------

def test_refused_arguments_change_nothing():
    from badslam_b200._lib import BadBAError
    sc = PC._scene("tiny")
    ba = PC._make(sc)
    ba.SetKeyframePosePriors([1], sc.poses_true[1][None], np.eye(6))
    ids = ba.AddKeyframePoseConstraints([0, 1], [1, 2], np.stack([sc.poses_true[0]] * 2), np.eye(6))
    ba.SetKeyframePosePriorLosses([1], "huber", 0.25)
    ba.SetKeyframePoseConstraintLosses(ids[1:], "cauchy", 2.0)
    before = (ba.KeyframePosePriorLoss(1), [x.tolist() for x in ba.GetKeyframePoseConstraintLosses()])
    assert before == ((HUBER, 0.25), [ids.tolist(), [TRIVIAL, CAUCHY], [0.0, 2.0]])
    bad = [lambda: ba.SetKeyframePosePriorLosses([1], 3, 1.0),
           lambda: ba.SetKeyframePosePriorLosses([1], "huber", 0.0),
           lambda: ba.SetKeyframePosePriorLosses([1], "cauchy", -1.0),
           lambda: ba.SetKeyframePosePriorLosses([1], "cauchy", float("nan")),
           lambda: ba.SetKeyframePosePriorLosses([1], "huber", float("inf")),
           lambda: ba.SetKeyframePosePriorLosses([1, 0], "huber", 1.0),        # keyframe 0 has no prior
           lambda: ba.SetKeyframePosePriorLosses([1, 99], "huber", 1.0),
           lambda: ba.SetKeyframePoseConstraintLosses([ids[0], 12345], "huber", 1.0),
           lambda: ba.SetKeyframePoseConstraintLosses(ids, [1, -1], 1.0)]
    for call in bad:
        with pytest.raises(BadBAError):
            call()
        assert (ba.KeyframePosePriorLoss(1), [x.tolist() for x in ba.GetKeyframePoseConstraintLosses()]) == before
    # a trivial loss ignores its scale; a replaced prior keeps its loss, a cleared one loses it; removal drops a loss
    ba.SetKeyframePoseConstraintLosses(ids[:1], "trivial", float("nan"))
    ba.SetKeyframePosePriors([1], sc.poses_true[2][None], 2 * np.eye(6))
    assert ba.KeyframePosePriorLoss(1) == (HUBER, 0.25)
    ba.ClearKeyframePosePriors([1])
    assert ba.KeyframePosePriorLoss(1) == (TRIVIAL, 0.0)
    ba.SetKeyframePosePriors([1], sc.poses_true[2][None], 2 * np.eye(6))
    assert ba.KeyframePosePriorLoss(1) == (TRIVIAL, 0.0)
    ba.RemoveKeyframePoseConstraints(ids[1:])
    new = ba.AddKeyframePoseConstraints([0], [2], sc.poses_true[0][None], np.eye(6))
    got = ba.GetKeyframePoseConstraintLosses()
    assert got[0].tolist() == [ids[0], new[0]] and got[1].tolist() == [TRIVIAL, TRIVIAL]
    x = np.zeros(4)
    assert PC._lib().bba_evaluate_keyframe_pose_terms(ba._h, -1, x.ctypes.data, None, 0, None, None, None) != 0
    ev = ba.EvaluateKeyframePoseTerms()
    assert np.isnan(ev["prior_s"][0]) and np.isfinite(ev["prior_s"][1]) and ev["prior_weight"][1] == 1.0
