"""Soft relative pose constraints between keyframes (bba_add_keyframe_pose_constraints): the 1/2 r^T L r term,
r = log(Z^-1 global_T_a^-1 global_T_b), in the alternating scheme's pose step, in bba_estimate_frame_pose and in the PCG products.

* adding and removing constraints leaves both schemes bit-identical to a handle that never had one;
* with one end fixed (inactive, or the PCG gauge) the other end moves as under the equivalent prior;
* bba_estimate_frame_pose follows numpy's Gauss-Newton loop over bba_accumulate_pose_coeffs + the equivalent prior's terms;
* the damping anchors close a constraint between two free keyframes in one step; with weak priors, the alternating scheme's
  cost does not rise and both schemes reach numpy's optimum;
* the PCG products with and without constraints differ by the constraints' terms, an edge to the gauge included;
* constraints with the true relative poses lower the relative-pose error of the constrained pairs;
* the deterministic mode stays reproducible; two and three ranks of a local group keep identical replicas and match one rank;
* refused calls change nothing, ids stay stable, and the front-end reader returns the published set."""
import ctypes as C

import numpy as np
import pytest

import test_gpu_multi_ranks_one_device as R
from gpu_checks import POSE_R, POSE_T

pytestmark = pytest.mark.gpu

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


def _lib():
    from badslam_b200 import _lib
    return _lib.load()


def _info(sigma_t, sigma_r):
    return np.diag([sigma_t ** -2] * 3 + [sigma_r ** -2] * 3).astype(np.float64)


def _upper(M):
    return np.array([M[i, j] for i in range(6) for j in range(i, 6)], np.float32)


def _matrix(H, n):
    Hm = np.zeros((n, n))
    Hm[np.triu_indices(n)] = H
    return Hm + np.triu(Hm, 1).T


def _f32(x):
    return np.ascontiguousarray(x, np.float32)


def _prior_terms(prior, pose, info21):
    H, b, cost = np.zeros(21), np.zeros(6), C.c_double()
    p, q, L = _f32(prior), _f32(pose), _f32(info21)
    _lib().bba_host_pose_prior_terms(p.ctypes.data, q.ctypes.data, L.ctypes.data, H.ctypes.data, b.ctypes.data, C.byref(cost))
    return H, b, cost.value


def _constraint_terms(Z, A, B, info21):
    H, b, cost = np.zeros(78), np.zeros(12), C.c_double()
    z, a, bb, L = _f32(Z), _f32(A), _f32(B), _f32(info21)
    _lib().bba_host_pose_constraint_terms(z.ctypes.data, a.ctypes.data, bb.ctypes.data, L.ctypes.data, H.ctypes.data, b.ctypes.data,
                                           C.byref(cost))
    return H, b, cost.value


def _compose(A, B):
    out = np.zeros(7, np.float32)
    _lib().bba_host_se3_compose(_f32(A).ctypes.data, _f32(B).ctypes.data, out.ctypes.data)
    return out


def _inverse(A):
    out = np.zeros(7, np.float32)
    _lib().bba_host_se3_inverse(_f32(A).ctypes.data, out.ctypes.data)
    return out


def _exp(x):
    out = np.zeros(7, np.float32)
    _lib().bba_host_se3_exp(_f32(x).ctypes.data, out.ctypes.data)
    return out


def _relative(A, B):   # A^-1 B
    return _compose(_inverse(A), B)


def _adjoint_inverse(Z):   # Ad(Z^-1) in the tangent order (translation, rotation), fp64
    from scipy.spatial.transform import Rotation
    q = np.asarray(Z[:4], np.float64)
    Rz = Rotation.from_quat(q / np.linalg.norm(q)).as_matrix()
    R, t = Rz.T, -Rz.T @ np.asarray(Z[4:], np.float64)
    hat = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    Ad = np.zeros((6, 6))
    Ad[:3, :3] = Ad[3:, 3:] = R
    Ad[:3, 3:] = hat @ R
    return Ad


def _info_a(Z, L):
    Ad = _adjoint_inverse(Z)
    return Ad.T @ L @ Ad


def _state(ba):
    return R._state(ba)


def _same_state(a, b):
    for k in ("poses", "act", "surfels", "active", "intr", "cf"):
        assert R._same(a[k], b[k]), k


def _chain(sc, K, rng_seed=0):
    """A constraint between every consecutive pair, with the true relative pose, and a loop pair."""
    a = list(range(K - 1)) + [0]
    b = list(range(1, K)) + [K - 1]
    Z = np.array([_relative(sc.poses_true[i], sc.poses_true[j]) for i, j in zip(a, b)], np.float32)
    return np.array(a), np.array(b), Z


# ---- 1. add + remove = never added -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("scheme", ["alternating", "pcg"])
@pytest.mark.parametrize("scene", ["tiny", "small"])
def test_removed_constraints_change_no_bit(scene, scheme):
    """The alternating scheme in the deterministic mode gives the same bits; the PCG scheme (which the deterministic mode does
    not cover) the same results, launches and poses up to the run-to-run order of its sums."""
    sc = _scene(scene)
    K = sc.cfg.num_keyframes
    outs = []
    for with_constraints in (False, True):
        ba = _make(sc, deterministic=scheme == "alternating")
        if with_constraints:
            a, b, Z = _chain(sc, K)
            ids = ba.AddKeyframePoseConstraints(a, b, Z, _info(0.01, 0.01))
            ba.RemoveKeyframePoseConstraints(ids[:1])
            ba.RemoveKeyframePoseConstraints()
            assert len(ba.KeyframePoseConstraints()[0]) == 0
        if scheme == "alternating":
            r = ba.BundleAdjustment(None, True, True, True, True, True, 2, 2)
        else:
            r = ba.BundleAdjustment(None, False, False, False, True, True, 2, 2, use_pcg=True, pcg_gauge_keyframe=0)
        outs.append((_state(ba), R._result(r), r.kernel_launches))
    assert np.array_equal(outs[0][1], outs[1][1]) and outs[0][2] == outs[1][2]
    if scheme == "alternating":
        _same_state(outs[0][0], outs[1][0])
    else:   # the PCG products sum with fp32 atomics: equal up to their run-to-run order, with the same launches
        from badslam_b200.scene import pose_error
        worst = max(max(pose_error(p, q)) for p, q in zip(outs[0][0]["poses"], outs[1][0]["poses"]))
        assert worst < 1e-4, worst


# ---- 2. one end fixed = the equivalent prior --------------------------------------------------------------------------------

def _pose64(P):
    q = np.asarray(P[:4], np.float64)
    return q / np.linalg.norm(q), np.asarray(P[4:], np.float64)


def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def _qrot(q, v):
    from scipy.spatial.transform import Rotation
    return Rotation.from_quat(q).as_matrix() @ v


def _equivalent_prior(T_other, Z, other_is_a):
    """T_a Z (the free end is b) or T_b Z^-1 (the free end is a) in fp64, rounded to fp32 once."""
    qo, to = _pose64(T_other)
    qz, tz = _pose64(Z)
    if not other_is_a:   # Z^-1 = (conj(qz), -R(qz)^T tz)
        qz = np.array([-qz[0], -qz[1], -qz[2], qz[3]])
        tz = -_qrot(qz, tz)
    return np.concatenate([_qmul(qo, qz), to + _qrot(qo, tz)]).astype(np.float32)


@pytest.mark.parametrize("scheme", ["alternating", "pcg"])
@pytest.mark.parametrize("free_end", ["a", "b"])
def test_fixed_end_acts_as_the_equivalent_prior(free_end, scheme):
    """Keyframe 0 is held fixed: moved out of every other keyframe's view and outside the active window it is inactive
    (alternating); in the PCG scheme it is the gauge.  A constraint between it and keyframe 1 moves keyframe 1 as the prior
    T_0 Z (keyframe 1 is b, same L) or T_0 Z^-1 with L_a = Ad(Z^-1)^T L Ad(Z^-1) (keyframe 1 is a) does; the reference prior is
    composed in fp64 and rounded once, so the two forms differ by the fp32 rounding of the staged pose only.
    Alternating: keyframe 1 keeps its data, so the information weighs the term against it; the deterministic mode makes both runs
    reproducible.  PCG (fp32 atomics, not covered by the deterministic mode): keyframe 1 is moved out of the map too, so both
    forms converge onto the prior pose, several centimetres from the start, far above the run-to-run jitter of the solver.  (The
    PCG weighting of an edge to the gauge is checked term by term in test_pcg_products_differ_by_the_constraint_terms.)"""
    from badslam_b200.scene import pose_error
    sc = _scene("small")
    poses = sc.poses_init.copy()
    poses[0, 4] += 100.0
    if scheme == "pcg":
        poses[1, 4] += 100.0
        assert _make(sc, poses=poses).AccumulatePoseEstimationCoeffs(1, poses[1]).n_assoc == 0
    # the relative pose the term asks for: a few centimetres from keyframe 1's true pose (alternating) or its start (PCG)
    rel = _relative(poses[0], sc.poses_true[1] if scheme == "alternating" else poses[1])
    rel = _compose(rel, _exp([0.03, -0.02, 0.01, 0.015, 0.0, -0.01]))
    L = _info(5e-4, 5e-4)
    if free_end == "b":
        a, b, Z = 0, 1, rel                           # keyframe 1 wants to sit at T_0 Z
        prior, prior_info = _equivalent_prior(poses[0], Z, other_is_a=True), L
    else:
        a, b, Z = 1, 0, _inverse(rel)                 # keyframe 1 wants to sit at T_0 Z^-1
        prior, prior_info = _equivalent_prior(poses[0], Z, other_is_a=False), _info_a(Z, L)

    def run(form):
        ba = _make(sc, deterministic=scheme == "alternating", poses=poses)
        if form == "constraint":
            ba.AddKeyframePoseConstraints([a], [b], Z[None], L)
        elif form == "prior":
            ba.SetKeyframePosePriors([1], prior[None], prior_info)
        if scheme == "alternating":
            ba.BundleAdjustment(None, False, False, False, True, True, 3, 3, active_keyframe_window_start=1)
        else:
            ba.BundleAdjustment(None, False, False, False, True, True, 8, 8, use_pcg=True, pcg_gauge_keyframe=0)
        return ba.GetKeyframeStates()[0]

    got, want, free = run("constraint"), run("prior"), run(None)
    assert np.array_equal(got[0], poses[0]) and np.array_equal(want[0], poses[0])
    err = max(pose_error(got[1], want[1]))
    moved = max(pose_error(got[1], free[1]))   # what the term did to keyframe 1
    assert err < 1e-5, err
    assert moved > 1e-3, (moved, err)
    if scheme == "pcg":
        assert max(pose_error(got[1], prior)) < 1e-5


# ---- 3. bba_estimate_frame_pose against numpy -------------------------------------------------------------------------------

def _numpy_pose_step(ba, k, init, terms, max_iterations=30):
    """EstimateFramePose's Gauss-Newton loop: data H, b from bba_accumulate_pose_coeffs (fp32) plus each (prior, L) term's fp64
    terms in list order, the fp64 LDLT, pose <- pose exp(-x) and the convergence test."""
    lib = _lib()
    pose = np.array(init, np.float32)
    for it in range(max_iterations):
        c = ba.AccumulatePoseEstimationCoeffs(k, pose)
        H = np.array(c.H, np.float32).astype(np.float64)
        b = np.array(c.b, np.float32).astype(np.float64)
        for prior, info21 in terms:
            Hp, bp, _ = _prior_terms(prior, pose, info21)
            H, b = H + Hp, b + bp
        x = np.zeros(6)
        assert lib.bba_host_solve_ldlt(6, H.ctypes.data, b.ctypes.data, x.ctypes.data) == 1
        xf = x.astype(np.float32)
        pose = _compose(pose, _exp(-xf))
        if lib.bba_host_pose_update_converged(xf.ctypes.data):
            return pose, it + 1
    return pose, max_iterations


def test_estimate_frame_pose_matches_numpy():
    """Keyframe 2 with a prior and two constraints (it is b of one and a of the other): its list is the prior, then the two
    equivalent priors with the other ends at their keyframe poses, and no anchor (the other ends are not estimated)."""
    sc = _scene("small")
    ba = _make(sc, deterministic=True)
    rng = np.random.default_rng(5)
    k = 2
    prior = sc.poses_true[k].copy()
    prior[4:] += rng.normal(scale=0.01, size=3).astype(np.float32)
    Lp, L1, L2 = _info(3e-3, 3e-3), _info(2e-3, 4e-3), _info(4e-3, 2e-3)
    Z1 = _compose(_relative(sc.poses_init[1], sc.poses_true[k]), _exp([0.004, 0.0, -0.003, 0.002, 0.001, 0.0]))
    Z2 = _compose(_relative(sc.poses_true[k], sc.poses_init[3]), _exp([-0.002, 0.003, 0.0, 0.0, -0.002, 0.001]))
    ba.SetKeyframePosePriors([k], prior[None], Lp)
    ba.AddKeyframePoseConstraints([1, k], [k, 3], np.stack([Z1, Z2]), np.stack([L1, L2]))
    got, its, _ = ba.EstimateFramePose(None, sc.poses_init[k], k)
    terms = [(prior, _upper(Lp)),
             (_compose(sc.poses_init[1], Z1), _upper(L1)),                        # k is b: T_a Z
             (_compose(sc.poses_init[3], _inverse(Z2)), _upper(_info_a(Z2, L2)))]  # k is a: T_b Z^-1, L_a
    want, want_its = _numpy_pose_step(ba, k, sc.poses_init[k], terms)
    assert its == want_its, (its, want_its)
    assert np.abs(got.astype(np.float64) - want).max() < 2e-6, (got, want)
    free, _ = _numpy_pose_step(ba, k, sc.poses_init[k], terms[:1])
    assert np.abs(free.astype(np.float64) - want).max() > 1e-5


# ---- 4. damping ------------------------------------------------------------------------------------------------------------

def test_damping_anchor_closes_a_constraint_between_two_free_keyframes():
    """Two keyframes that see no surfels, no priors, one constraint whose Z is off from their relative pose by a known motion.
    Undamped, each end would jump onto the other's old pose every step (block Jacobi without data), and the residual would flip
    sign for ever with the same size.  With the damping anchors each end moves half way: one alternating BA iteration removes the
    residual up to its second order, and a few more leave only the fp32 rounding of poses 100 m from the origin."""
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    a, b = K - 2, K - 1
    poses = sc.poses_init.copy()
    poses[a, 4] += 100.0
    poses[b, 4] += 100.0
    ba = _make(sc, poses=poses)
    assert ba.AccumulatePoseEstimationCoeffs(a, poses[a]).n_assoc == 0
    assert ba.AccumulatePoseEstimationCoeffs(b, poses[b]).n_assoc == 0
    Z = _compose(_relative(poses[a], poses[b]), _exp([0.03, 0.0, -0.02, 0.02, 0.0, 0.01]))
    Lc = _upper(_info(0.01, 0.01))
    ba.AddKeyframePoseConstraints([a], [b], Z[None], Lc)
    costs = [_constraint_terms(Z, poses[a], poses[b], Lc)[2]]
    for _ in range(4):
        ba.BundleAdjustment(None, False, False, False, True, False, 1, 1)
        p = ba.GetKeyframeStates()[0]
        costs.append(_constraint_terms(Z, p[a], p[b], Lc)[2])
    assert costs[0] > 1.0, costs
    assert costs[1] < 1e-3 * costs[0], costs
    assert costs[4] < 1e-6 * costs[0], costs
    # both ends moved, by about the same amount: the correction is shared, not taken by one end
    from badslam_b200.scene import pose_error
    da, db = pose_error(p[a], poses[a])[0], pose_error(p[b], poses[b])[0]
    assert da > 5e-3 and db > 5e-3 and 0.5 < da / db < 2.0, (da, db)


def _joint_optimum(priors, Lp, Z, Lc, start, fixed_a=False, iterations=60):
    """numpy Gauss-Newton on the two poses (a, b) over the priors' and the constraint's host terms."""
    A, B = start[0].copy(), start[1].copy()
    for _ in range(iterations):
        H = np.zeros((12, 12))
        g = np.zeros(12)
        Hc, bc, _ = _constraint_terms(Z, A, B, _upper(Lc))
        H += _matrix(Hc, 12)
        g += bc
        for i, P in enumerate((A, B)):
            Hp, bp, _ = _prior_terms(priors[i], P, _upper(Lp))
            H[6 * i:6 * i + 6, 6 * i:6 * i + 6] += _matrix(Hp, 6)
            g[6 * i:6 * i + 6] += bp
        if fixed_a:
            x = np.concatenate([np.zeros(6), np.linalg.solve(H[6:, 6:], g[6:])])
        else:
            x = np.linalg.solve(H, g)
        A = _compose(A, _exp(-x[:6]))
        B = _compose(B, _exp(-x[6:]))
    return A, B


def _total_cost(priors, Lp, Z, Lc, A, B):
    return (_prior_terms(priors[0], A, _upper(Lp))[2] + _prior_terms(priors[1], B, _upper(Lp))[2]
            + _constraint_terms(Z, A, B, _upper(Lc))[2])


def test_weak_priors_and_a_constraint_reach_the_joint_optimum():
    """Two keyframes without data, weak priors pulling them apart and a constraint holding them together.  Their data-free pose
    blocks are positive definite through the priors, so this case converges with or without the anchors (the anchor case is
    test_damping_anchor_closes_a_constraint_between_two_free_keyframes); it checks that the alternating steps lower the full cost
    monotonically to numpy's joint optimum, and that the PCG scheme reaches numpy's optimum with the gauge on one end."""
    from badslam_b200.scene import pose_error
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    a, b = K - 2, K - 1
    poses = sc.poses_init.copy()
    poses[a, 4] += 100.0
    poses[b, 4] += 100.0
    assert _make(sc, poses=poses).AccumulatePoseEstimationCoeffs(a, poses[a]).n_assoc == 0
    # the priors pull the pair apart, the constraint holds it together
    priors = [_compose(poses[a], _exp([0.03, 0.0, 0.0, 0.0, 0.01, 0.0])), _compose(poses[b], _exp([-0.03, 0.01, 0.0, 0.0, 0.0, 0.02]))]
    Z = _relative(poses[a], poses[b])
    Lp, Lc = _info(0.02, 0.02), _info(0.01, 0.01)
    want_a, want_b = _joint_optimum(priors, Lp, Z, Lc, (poses[a], poses[b]))
    ba = _make(sc, poses=poses)
    ba.SetKeyframePosePriors([a, b], np.stack(priors), Lp)
    ba.AddKeyframePoseConstraints([a], [b], Z[None], Lc)
    costs = [_total_cost(priors, Lp, Z, Lc, poses[a], poses[b])]
    for _ in range(120):
        ba.BundleAdjustment(None, False, False, False, True, False, 1, 1)
        p = ba.GetKeyframeStates()[0]
        costs.append(_total_cost(priors, Lp, Z, Lc, p[a], p[b]))
    # (the poses are fp32 100 m from the origin: near the optimum the cost moves by their rounding only)
    rises = [c1 - c0 for c0, c1 in zip(costs, costs[1:]) if c1 > c0 + 1e-5 + 1e-6 * c0]
    assert not rises, rises
    p = ba.GetKeyframeStates()[0]
    err = max(max(pose_error(p[a], want_a)), max(pose_error(p[b], want_b)))
    assert err < 1e-4, (err, costs[-1], _total_cost(priors, Lp, Z, Lc, want_a, want_b))
    # PCG, gauge on a: b reaches numpy's optimum with a fixed
    want_a, want_b = _joint_optimum(priors, Lp, Z, Lc, (poses[a], poses[b]), fixed_a=True)
    ba = _make(sc, poses=poses)
    ba.SetKeyframePosePriors([a, b], np.stack(priors), Lp)
    ba.AddKeyframePoseConstraints([a], [b], Z[None], Lc)
    ba.BundleAdjustment(None, False, False, False, True, False, 6, 6, use_pcg=True, pcg_gauge_keyframe=a)
    p = ba.GetKeyframeStates()[0]
    assert np.array_equal(p[a], poses[a])
    assert max(pose_error(p[b], want_b)) < 1e-4


# ---- 5. PCG products --------------------------------------------------------------------------------------------------------

def test_pcg_products_differ_by_the_constraint_terms():
    """bba_pcg_debug's first step without constraints and with e1 = (K-2, K-1) and e2 = (0, K-1), keyframe 0 the gauge.  Keyframes
    K-2 and K-1 are moved out of the map, so their rows of J^T W J are zero: on their blocks r and M are exactly the constraints'
    terms, g is the constraints' H p over the two blocks (p_gauge = 0), and alpha_d grows by p^T A_e p plus the lambda term of
    the blocks' new p; everything else differs only by the order of the fp32 atomics."""
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    poses = sc.poses_init.copy()
    poses[K - 2, 4] += 100.0
    poses[K - 1, 4] += 100.0
    Z1 = _compose(_relative(poses[K - 2], poses[K - 1]), _exp([0.01, 0.0, -0.01, 0.0, 0.02, 0.0]))
    Z2 = _compose(_relative(poses[0], poses[K - 1]), _exp([0.0, 0.02, 0.0, 0.01, 0.0, 0.0]))
    L1, L2 = _info(0.01, 0.02), _info(0.02, 0.01)
    probes = []
    for with_constraints in (False, True):
        ba = _make(sc, poses=poses)
        if with_constraints:
            ba.AddKeyframePoseConstraints([K - 2, 0], [K - 1, K - 1], np.stack([Z1, Z2]), np.stack([L1, L2]))
        probes.append(ba.PCGProbe(0, False, True, True, gauge_keyframe=0))
    a, b = probes
    n = len(a["r"])
    u = 6 * (K - 3)   # block K-2 (pose unknowns skip the gauge keyframe 0), then block K-1
    s = slice(u, u + 12)
    H1, b1, _ = _constraint_terms(Z1, poses[K - 2], poses[K - 1], _upper(L1))
    H2, b2, _ = _constraint_terms(Z2, poses[0], poses[K - 1], _upper(L2))
    Hm = _matrix(H1, 12)
    Hm[6:, 6:] += _matrix(H2, 12)[6:, 6:]
    bv = b1.copy()
    bv[6:] += b2[6:]
    assert np.all(a["r"][s] == 0) and np.all(a["M"][s] == 0) and np.all(a["p"][s] == 0)
    assert np.abs(b["r"][s] + bv).max() <= 1e-5 * np.abs(bv).max()
    assert np.abs(b["M"][s] - np.diag(Hm)).max() <= 1e-5 * np.abs(np.diag(Hm)).max()
    pb = b["p"][s].astype(np.float64)
    want_g = Hm @ pb
    assert np.abs(b["g"][s] - want_g).max() <= 1e-4 * np.abs(want_g).max()
    rest = np.ones(n, bool)
    rest[s] = False

    def close(x, y, what):
        np.testing.assert_allclose(x, y, rtol=1e-4, atol=1e-4 * max(1e-30, np.abs(y).max()), err_msg=what)

    for k in ("r", "M", "p", "g"):
        close(b[k][rest], a[k][rest], k + " elsewhere")
    share = float(pb @ want_g) + K * 1e-8 * float(pb @ pb)
    assert abs((b["alpha_d"] - a["alpha_d"]) - share) <= 1e-4 * (abs(a["alpha_d"]) + share), (b["alpha_d"], a["alpha_d"], share)


# ---- 6. accuracy ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("scheme", ["alternating", "pcg"])
def test_true_relative_poses_lower_the_relative_error(scheme):
    from badslam_b200.scene import pose_error
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    a, b, Z = np.arange(K - 1), np.arange(1, K), None
    Z = np.array([_relative(sc.poses_true[i], sc.poses_true[j]) for i, j in zip(a, b)], np.float32)
    errs = []
    for with_constraints in (False, True):
        ba = _make(sc)
        if with_constraints:
            ba.AddKeyframePoseConstraints(a, b, Z, _info(5e-4, 5e-4))
        if scheme == "alternating":
            ba.BundleAdjustment(None, False, False, False, True, True, 4, 4)
        else:
            ba.BundleAdjustment(None, False, False, False, True, True, 4, 4, use_pcg=True, pcg_gauge_keyframe=0)
        p = ba.GetKeyframeStates()[0]
        assert np.all(np.isfinite(p))
        errs.append(np.mean([pose_error(_relative(p[i], p[j]), Z[e])[0] for e, (i, j) in enumerate(zip(a, b))]))
    assert errs[1] < 0.9 * errs[0], errs


# ---- 7. deterministic mode and several ranks --------------------------------------------------------------------------------

def _constraints_for(sc):
    K = sc.cfg.num_keyframes
    rng = np.random.default_rng(11)
    a, b, Z = _chain(sc, K)
    Z = np.array([_compose(z, _exp(rng.normal(scale=0.003, size=6))) for z in Z], np.float32)
    return a, b, Z, _info(0.01, 0.01)


def test_deterministic_with_constraints():
    sc = _scene("small")
    outs = []
    for _ in range(2):
        ba = _make(sc, deterministic=True)
        a, b, Z, L = _constraints_for(sc)
        ba.AddKeyframePoseConstraints(a, b, Z, L)
        r = ba.BundleAdjustment(None, True, True, True, True, True, 2, 2)
        outs.append((_state(ba), R._result(r), np.float64(r.cost)))
    _same_state(outs[0][0], outs[1][0])
    assert np.array_equal(outs[0][1], outs[1][1]) and R._same(outs[0][2], outs[1][2])


def run_alternating_with_constraints(ba):
    a, b, Z, L = _constraints_for(R.SCENES["small"]())
    ba.AddKeyframePoseConstraints(a, b, Z, L)
    return R.run_pose(ba)


def run_pcg_with_constraints(ba):
    a, b, Z, L = _constraints_for(R.SCENES["small"]())
    ba.AddKeyframePoseConstraints(a, b, Z, L)
    return R.run_pcg(ba, False)


@pytest.mark.parametrize("world", ["2", "3"])
@pytest.mark.parametrize("mode", ["gather", "peer"])
@pytest.mark.parametrize("scheme", ["alternating", "pcg"])
def test_local_group_ranks(world, mode, scheme):
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    from badslam_b200.scene import pose_error
    fn = run_alternating_with_constraints if scheme == "alternating" else run_pcg_with_constraints
    handles = DirectBA.create_local_ranks(R.SCENES["small"](), int(world), ["cuda:0"] * int(world))
    with LocalGroup(handles, peer_stores=mode == "peer") as group:
        outs = group.run(lambda r, ba: fn(ba))
    for o in outs[1:]:
        for k in ("poses", "act", "surfels", "active", "intr", "cf", "res"):
            assert R._same(o[k], outs[0][k]), k
    want = R.one_rank(("constraints", scheme), lambda: R._one("small", fn))
    got = outs[0]
    K = len(want["poses"])
    worst = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(K))
    if scheme == "alternating":
        assert np.array_equal(got["res"][:5], want["res"][:5]) and np.array_equal(got["act"], want["act"])
        assert worst <= min(POSE_T, POSE_R), worst
    else:
        assert got["res"][0] == want["res"][0] and abs(int(got["res"][5]) - int(want["res"][5])) <= 2
        assert worst < 2e-4, worst


# ---- 8. refused calls, ids, the front end -----------------------------------------------------------------------------------

def test_refused_calls_ids_and_front_end(tiny_scene):
    from badslam_b200 import _lib as L
    sc = tiny_scene
    K = sc.cfg.num_keyframes
    ba = _make(sc)
    good = _info(0.1, 0.1)
    Z = _relative(sc.poses_true[0], sc.poses_true[1])
    ids = ba.AddKeyframePoseConstraints([0, 1, 0], [1, 2, 2], np.stack([Z, Z, Z]), good)
    assert list(ids) == [0, 1, 2]
    before = (ba.KeyframePoseConstraints(), ba.kernel_launch_count(), ba.GetKeyframeStates()[0])
    indefinite = good.copy()
    indefinite[0, 1] = indefinite[1, 0] = 2 * indefinite[0, 0]
    negative = good.copy()
    negative[5, 5] = -1.0
    nan_pose = Z.copy()
    nan_pose[5] = np.nan
    inf_info = _upper(good)
    inf_info[3] = np.inf
    cases = [
        ([0, K], [1, 0], [Z, Z], [_upper(good)] * 2),
        ([0, -1], [1, 0], [Z, Z], [_upper(good)] * 2),
        ([0, 1], [1, 1], [Z, Z], [_upper(good)] * 2),
        ([0, 1], [1, 2], [Z, nan_pose], [_upper(good)] * 2),
        ([0, 1], [1, 2], [Z, Z], [_upper(good), inf_info]),
        ([0, 1], [1, 2], [Z, Z], [_upper(good), _upper(indefinite)]),
        ([0, 1], [1, 2], [Z, Z], [_upper(good), _upper(negative)]),
        ([0, 1], [1, 2], [Z, np.zeros(7, np.float32)], [_upper(good)] * 2),
    ]
    for a, b, Zs, infos in cases:
        with pytest.raises(L.BadBAError) as e:
            ba.AddKeyframePoseConstraints(a, b, np.array(Zs), np.array(infos))
        assert e.value.status == L.ERR_INVALID_ARGUMENT
    for bad in ([3], [-1], [0, 7]):
        with pytest.raises(L.BadBAError):
            ba.RemoveKeyframePoseConstraints(bad)
    after = (ba.KeyframePoseConstraints(), ba.kernel_launch_count(), ba.GetKeyframeStates()[0])
    for x, y in zip(before[0], after[0]):
        assert np.array_equal(x, y)
    assert before[1] == after[1] and np.array_equal(before[2], after[2])
    # ids are never reused, and removal keeps the others' ids and records
    ba.RemoveKeyframePoseConstraints([1])
    new = ba.AddKeyframePoseConstraints([2], [0], Z[None], good)
    assert list(new) == [3]
    got_ids, ga, gb, gZ, gL = ba.KeyframePoseConstraints()
    assert list(got_ids) == [0, 2, 3] and list(ga) == [0, 0, 2] and list(gb) == [1, 2, 0]
    assert np.array_equal(gZ[0], Z) and np.array_equal(gL[2], _upper(good))
    # the front-end reader honours its capacity
    count = C.c_int()
    out_ids = np.full(2, -7, np.int32)
    recs = (L.PoseConstraint * 2)()
    assert ba._lib.bba_get_keyframe_pose_constraints(ba._h, 1, out_ids.ctypes.data, recs, C.byref(count)) == 0
    assert count.value == 3 and out_ids[0] == 0 and out_ids[1] == -7
    # a semi-definite L (translation only) is accepted
    semi = np.diag([100.0] * 3 + [0.0] * 3)
    ba.AddKeyframePoseConstraints([1], [2], Z[None], semi)
    ba.RemoveKeyframePoseConstraints()
    assert len(ba.KeyframePoseConstraints()[0]) == 0
