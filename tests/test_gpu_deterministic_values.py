"""GPU: the VALUES of the deterministic mode (bba_set_deterministic, DESIGN.md 3.10).  tests/test_gpu_deterministic.py holds the mode
to "the same bits twice"; a kernel that is deterministically wrong passes that.  Here every instantiation the mode added is run at
a fixed state and compared with the default mode on the same handle (itself pinned three-way by test_gpu_parity.py,
test_gpu_work_groups.py and test_gpu_odometry.py on these scenes), with the CPU oracle and with the bound the code implies:

  * pose kernel (see compare_pose_records for the instantiations this holds for) and the intrinsics step's 34 global sums: both
    modes add the same fp32 warp totals, the default with fp64 atomics in
    any order (one rounding of 2^-53 of the running sum per add), the mode exactly with one rounding.  With n deposits into a slot
    the two differ by at most (n + 1) 2^-53 S, S a bound on the running sums: the slot itself on a diagonal (non-negative terms),
    sqrt(H_ii H_jj) off it, sqrt(2 H_ii cost) for b (Cauchy-Schwarz; w r^2 <= 2 rho(r) for the Huber and the Tukey weights);
  * the intrinsics step's cell rows: fp32 atomics against one rounding, (obs + 1) 2^-24 of the same kind of bound per cell;
  * odometry: per-CTA totals are fixed by the static tile partition; both modes add them in fp64, so the fp32 read-backs agree to
    an ulp.

The maxima measured against these bounds are recorded in MEASURED and printed at the end of the module (pytest -s).  Every
configuration runs a fixed one or two times, on valid scenes; the one non-finite case is IEEE arithmetic inside a sum.
"""
import copy
import math

import numpy as np
import pytest

from gpu_checks import POSE_R, POSE_T, REL, distorted_scene, rel
from test_gpu_concurrent_front_end import IDENT, assert_same
from test_gpu_work_groups import distinct_poses

pytestmark = [pytest.mark.gpu]

U53, U24 = 2.0 ** -53, 2.0 ** -24
MEASURED = {}


def held(name, value, limit, where=None):
    """Records the largest value seen under `name` and holds it to `limit`."""
    value = float(value)
    MEASURED[name] = max(MEASURED.get(name, 0.0), value)
    assert value <= limit, (name, value, limit, where)


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import _lib
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    from oracle import cpu_oracle, odometry_oracle
    yield S, DirectBA, _lib, cpu_oracle, odometry_oracle
    print("\nmeasured maxima (deterministic against default mode):")
    for k in sorted(MEASURED):
        print(f"  {k}: {MEASURED[k]:.3g}")


@pytest.fixture(scope="module")
def scenes():
    from badslam_b200.scene import config_by_name, make_scene
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = make_scene(config_by_name(name))
        return cache[name]
    return get


def in_mode(ba, on, fn):
    ba.SetDeterministic(on)
    try:
        return fn()
    finally:
        ba.SetDeterministic(False)


def positive_zero(a):
    """Every element is +0.0 (no set bit)."""
    return not np.ascontiguousarray(a).view(np.uint8).any()


# ---- A. pose kernel ------------------------------------------------------------------------------------------------------------

TRI6 = [(r, c) for r in range(6) for c in range(r, 6)]   # packed upper triangle of H, row-major
DIAG6 = [i for i, (r, c) in enumerate(TRI6) if r == c]


def compare_pose_records(det, dflt, det_costs, deposits, tag, pre, listed=None):
    """(H, b, counts, costs) of the two modes, keyframe by keyframe.  pre (the instantiations with the precomputed frames, which
    the BA pose step runs from four keyframes on): in units of (deposits + 1) 2^-53 of each slot's bound; measured on an H100 (80 GB
    HBM3, 700 W): bit-equal.  Without them the fp32 partials of the two modes' instantiations are NOT the same values, although
    nothing in the source differs but the sink and both have the same FFMA / FMUL / FADD counts: measured 1.5e-8 of
    sqrt(H_ii H_jj) on H and 4.6e-6 of sqrt(2 H_ii cost) on b, in all three tile sizes alike, with and without stats, the same in
    every run; counts and costs bit-equal.  With ONE surfel, a single pair's term, H differs by 1.6e-7: the two instantiations
    round the products of a pair differently (the residuals, and so the costs, are equal), which no deposit or summation order
    can explain.  Those instantiations are held to 1e-6 / 2e-5: a few fp32 roundings of a term."""
    H1, b1, c1, k1 = det
    H0, b0, c0, k0 = dflt
    assert np.array_equal(c1, c0), tag
    unit = (deposits + 1) * U53 * (1 + 1e-5)   # (the partials are fp32 sums: Cauchy-Schwarz holds for them to fp32 rounding)
    for k in range(len(H0)):
        if listed is not None and k not in listed:
            assert positive_zero(H1[k]) and positive_zero(b1[k]) and positive_zero(k1[k]) and not c1[k].any(), (tag, k)
            assert not H0[k].any() and not b0[k].any(), (tag, k)
            continue
        if not c0[k, 2]:
            assert positive_zero(H1[k]) and positive_zero(b1[k]) and positive_zero(k1[k]), (tag, k)
            assert not H0[k].any() and not b0[k].any(), (tag, k)
            continue
        d = H0[k][DIAG6]
        assert np.all(d > 0), (tag, k)
        scale = np.array([math.sqrt(d[r] * d[c]) for r, c in TRI6])
        dH = np.max(np.abs(H1[k] - H0[k]) / scale)
        db = np.max(np.abs(b1[k] - b0[k]) / np.sqrt(2 * d * det_costs[k].sum()))
        if pre:
            held("pose H with the frames, units of (n + 1) 2^-53 sqrt(H_ii H_jj)", dH / unit, 1.0, (tag, k))
            held("pose b with the frames, units of (n + 1) 2^-53 sqrt(2 H_ii cost)", db / unit, 1.0, (tag, k))
        else:
            held("pose H without the frames, relative to sqrt(H_ii H_jj)", dH, 1e-6, (tag, k))
            held("pose b without the frames, relative to sqrt(2 H_ii cost)", db, 2e-5, (tag, k))
        if k0[k].any():
            ok = k0[k] > 0
            held("pose costs, units of (n + 1) 2^-53 cost", np.max(np.abs(k1[k] - k0[k])[ok] / k0[k][ok]) / unit, 1.0, (tag, k))
            assert positive_zero(k1[k][~ok]), (tag, k)


def test_pose_coefficients_every_variant_and_work_list(mods, scenes):
    """All five instantiations of PoseAccumulateKernel<.., DET = true>, with and without stats, over the work lists of
    test_gpu_work_groups.py; keyframe 24 is posed 100 m in front of the map (everything behind it): listed, nothing associated."""
    S, DirectBA, L, O, _ = mods
    sc = scenes("many")
    K = sc.cfg.num_keyframes
    poses = distinct_poses(S, sc)
    poses[24] = S.se3_mul(poses[24], S.se3_exp([0, 0, 100.0, 0, 0, 0]))
    ba = DirectBA.from_scene(sc)
    deposits = -(-sc.num_surfels // 128)
    lists = {"all": np.arange(K), "permuted": np.random.default_rng(37).permutation(K), "nine": [36, 0, 8, 15, 16, 17, 31, 7, 24],
             "three": [17, 8, 0], "two": [15, 36], "one": [16]}
    variants = [L.POSE_VARIANT_256_PRE, L.POSE_VARIANT_512_PRE, L.POSE_VARIANT_256, L.POSE_VARIANT_512, L.POSE_VARIANT_1024]
    for v in variants:
        for lname, ids in lists.items():
            ids = np.asarray(ids)
            costs = None
            for with_stats in (True, False):
                call = lambda: ba.PoseCoeffsBatch(ids, poses[ids], v, with_stats)
                dflt, det = call(), in_mode(ba, True, call)
                costs = det[3] if with_stats else costs
                assert dflt[2][ids[ids != 24], 2].min() > 0 and not dflt[2][24].any(), (v, lname)
                pre = v in (L.POSE_VARIANT_256_PRE, L.POSE_VARIANT_512_PRE)
                compare_pose_records(det, dflt, costs, deposits, (int(v), lname, with_stats), pre, listed=set(ids.tolist()))


def test_pose_coefficients_ragged_surfel_counts(mods, scenes):
    """1, 255, 257, 1023 and 1025 surfels in the largest tile of each kind, mode on: against the default mode and the oracle."""
    S, DirectBA, L, O, _ = mods
    many = scenes("many")
    K = many.cfg.num_keyframes
    poses = distinct_poses(S, many)
    ids = np.arange(K)
    for n in (1, 255, 257, 1023, 1025):
        sc = copy.copy(many)
        sc.num_surfels = n
        ba, orc = DirectBA.from_scene(sc), O.Oracle(sc)
        oracle = [orc.pose_coeffs(k, poses[k]) for k in range(K)]
        for v in (L.POSE_VARIANT_1024, L.POSE_VARIANT_512_PRE):
            call = lambda: ba.PoseCoeffsBatch(ids, poses, v, True)
            dflt, det = call(), in_mode(ba, True, call)
            compare_pose_records(det, dflt, det[3], -(-n // 128), (n, int(v)), v == L.POSE_VARIANT_512_PRE)
            for k in range(K):
                st = oracle[k]
                assert tuple(det[2][k]) == (st.n_inimg, st.n_depthok, st.n_assoc, st.n_photo), (n, int(v), k)
                if st.n_assoc:   # (a few pairs per keyframe: the tolerance of test_batched_pose_coefficients_ragged_surfel_counts)
                    assert rel(det[0][k], st.H[:]) < 5e-3 and rel(det[1][k], st.b[:]) < 1.5e-2, (n, int(v), k)


def test_pose_solve_against_default_and_oracle(mods, scenes):
    """PoseSolveKernel<true>: EstimateFramePose of every keyframe of `small`, and one BA iteration (poses only) on `many`."""
    S, DirectBA, L, O, _ = mods
    sc = scenes("small")
    ba, orc = DirectBA.from_scene(sc), O.Oracle(sc)
    for k in range(sc.cfg.num_keyframes):
        call = lambda: ba.EstimateFramePose(None, sc.poses_init[k], k)
        (p0, it0, cv0), (p1, it1, cv1) = call(), in_mode(ba, True, call)
        assert (it1, cv1) == (it0, cv0) and it0 > 1, (k, it0, it1)
        dt, dr = S.pose_error(p1, p0)
        held("EstimateFramePose, m", dt, 1e-6, k)
        held("EstimateFramePose, rad", dr, 1e-6, k)
        po, io, co = orc.estimate_frame_pose(k)
        dt, dr = S.pose_error(p1, po)
        assert dt < 2 * POSE_T and dr < 2 * POSE_R, (k, dt, dr)   # (ours and the oracle are each pinned to the reference at 1e-5)
    sc = scenes("many")
    out = []
    for on in (False, True):
        ba = DirectBA.from_scene(sc)
        ba.SetDeterministic(on)
        r = ba.BundleAdjustment(None, False, False, False, True, False, 1, 1)
        out.append((r, ba.GetKeyframeStates()))
    (r0, (p0, a0)), (r1, (p1, a1)) = out
    assert (r1.iterations_done, r1.converged, r1.pose_iterations_total, r1.depth_residual_count, r1.descriptor_residual_count) == \
        (r0.iterations_done, r0.converged, r0.pose_iterations_total, r0.depth_residual_count, r0.descriptor_residual_count)
    assert np.array_equal(a0, a1) and r0.pose_iterations_total > sc.cfg.num_keyframes
    held("one BA iteration on many: cost, relative", abs(r1.cost - r0.cost) / r0.cost, 1e-12)
    for k in range(sc.cfg.num_keyframes):
        dt, dr = S.pose_error(p1[k], p0[k])
        held("one BA iteration on many, m", dt, 1e-6, k)
        held("one BA iteration on many, rad", dr, 1e-6, k)


def test_pose_edge_states(mods, scenes):
    """The empty map, one keyframe and a map no keyframe sees, mode on: what the default mode gives for the same state."""
    S, DirectBA, L, O, _ = mods
    tiny = scenes("tiny")
    empty = copy.copy(tiny)
    empty.num_surfels = 0
    one = S.make_scene(S.SceneConfig(width=tiny.cfg.width, height=tiny.cfg.height, num_keyframes=1, num_surfels=3000,
                                     cell=tiny.cfg.cell, seed=5, name="one"))
    behind = copy.copy(tiny)
    behind.surfels = tiny.surfels.copy()
    behind.surfels[2] = -5.0
    for name, sc in (("empty", empty), ("one keyframe", one), ("behind", behind)):
        res = []
        for on in (False, True):
            ba = DirectBA.from_scene(sc)
            ba.SetDeterministic(on)
            pc = ba.AccumulatePoseEstimationCoeffs(0, sc.poses_init[0])
            est = ba.EstimateFramePose(None, sc.poses_init[0], 0)
            ba.UpdateSurfelActivation()
            r = ba.BundleAdjustment(None, False, False, False, True, True, 1, 2)
            res.append(dict(counts=(pc.n_inimg, pc.n_depthok, pc.n_assoc, pc.n_photo), H=np.array(pc.H[:]), b=np.array(pc.b[:]),
                            est=est, active=ba.GetActiveHost(), ba=(r.iterations_done, r.converged, r.pose_iterations_total, r.surfels_size),
                            poses=ba.GetKeyframeStates()[0]))
        d, m = res
        assert m["counts"] == d["counts"] and m["est"][1:] == d["est"][1:] and m["ba"] == d["ba"], (name, d["ba"], m["ba"])
        assert np.array_equal(m["active"], d["active"]), name
        if d["counts"][2] == 0:
            assert positive_zero(m["H"]) and positive_zero(m["b"]) and not d["H"].any(), name
            assert np.array_equal(m["est"][0], d["est"][0]) and np.array_equal(m["poses"], d["poses"]), name
            assert d["est"][1] == 1 and d["est"][2], name   # H = 0 -> x = 0 -> converged at once
        else:
            assert rel(m["H"], d["H"]) < 1e-6 and rel(m["b"], d["b"]) < 1e-6, name   # (fp32 read-backs of fp64-noise-equal sums)
            for p, q in zip(m["poses"], d["poses"]):
                assert max(S.pose_error(p, q)) < 1e-6, name


def test_pose_sums_carry_nothing_between_calls(mods, scenes):
    """The exact sums are cleared by whoever read them: the parity hooks on the host, PoseSolveKernel<true> on the device."""
    S, DirectBA, L, O, _ = mods
    sc = scenes("small")
    K = sc.cfg.num_keyframes
    ids = np.arange(K)

    def hook(ba):
        return ba.PoseCoeffsBatch(ids, sc.poses_init, L.POSE_VARIANT_AUTO, True)

    def ba_step(ba):   # (poses only, without the end tasks: the surfels stay as they are)
        ba.SetLastBAIterationCount(ba.ba_iteration_count())
        return ba.BundleAdjustment(None, False, False, False, True, False, 1, 1, increase_ba_iteration_count=False)
    ba = DirectBA.from_scene(sc)
    ba.SetDeterministic(True)
    first = hook(ba)
    # mode on -> off -> a default call -> on again
    ba.SetDeterministic(False)
    hook(ba)
    ba.SetDeterministic(True)
    assert_same(hook(ba), first, "on, off, default call, on")
    # hook -> BA -> hook at the first hook's state
    ba_step(ba)
    moved = ba.GetKeyframeStates()[0]
    assert not np.array_equal(moved, sc.poses_init)
    ba.SetKeyframeStates(poses=sc.poses_init)
    assert_same(hook(ba), first, "hook, BA, hook")
    # the single-keyframe call right after a BA call equals the same call on a fresh handle at the same state
    ba.SetKeyframeStates(poses=sc.poses_init)
    ba_step(ba)
    pc = ba.AccumulatePoseEstimationCoeffs(2, sc.poses_init[2])
    fresh = DirectBA.from_scene(sc, poses=ba.GetKeyframeStates()[0])
    fresh.SetDeterministic(True)
    want = fresh.AccumulatePoseEstimationCoeffs(2, sc.poses_init[2])
    assert bytes(pc) == bytes(want)


def test_non_finite_deposits_set_the_flags_and_do_not_outlive_the_call(mods, scenes):
    """A surfel descriptor of +Inf gives the residual -Inf: the Huber weight 10 / |r| is 0, so H stays finite, w r = 0 * Inf = NaN
    reaches b and the Huber cost +Inf the cost of descriptor 1 (device_math.cuh AccumulateHb, HuberResidual).  The slots are
    non-finite in the same places in both modes; with the surfels restored the next call gives a clean handle's bits; and in a
    Gauss-Newton loop the NaN of the first iteration (a NaN pose projects nothing: ProjectIntoImage's comparisons fail) does not
    reach the second one, whose sums are exactly zero: the loop ends as in the default mode."""
    import torch
    S, DirectBA, L, O, _ = mods
    sc = scenes("tiny")
    ids = np.arange(sc.cfg.num_keyframes)
    ba = DirectBA.from_scene(sc)
    call = lambda: ba.PoseCoeffsBatch(ids, sc.poses_init, L.POSE_VARIANT_AUTO, True)
    clean = in_mode(ba, True, call)
    surf = ba.surfels()
    saved = surf[6, :8].clone()
    surf[6, :8] = float("inf")
    torch.cuda.synchronize()
    ba.SetSurfels(surf, sc.num_surfels)
    dflt, det = call(), in_mode(ba, True, call)
    bad = ~np.isfinite(dflt[1])
    assert bad.any() and np.isinf(dflt[3][:, 1]).any()
    for a, b in zip(det, dflt):
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b)) and \
            np.array_equal(np.isneginf(a), np.isneginf(b))
    kf = int(np.flatnonzero(bad.any(axis=1))[0])
    loop = lambda: ba.EstimateFramePose(None, sc.poses_init[kf], kf)
    (p0, it0, cv0), (p1, it1, cv1) = loop(), in_mode(ba, True, loop)
    assert (it1, cv1) == (it0, cv0) and np.array_equal(np.isnan(p1), np.isnan(p0)), (it0, cv0, it1, cv1)
    assert it0 < 30, it0
    surf[6, :8] = saved
    torch.cuda.synchronize()
    ba.SetSurfels(surf, sc.num_surfels)
    assert_same(in_mode(ba, True, call), clean, "after the non-finite call")


# ---- B. intrinsics step --------------------------------------------------------------------------------------------------------

TRI5 = [(r, c) for r in range(5) for c in range(r, 5)]
TRI4 = [(r, c) for r in range(4) for c in range(r, 4)]
DIAG5 = [i for i, (r, c) in enumerate(TRI5) if r == c]
DIAG4 = [20 + i for i, (r, c) in enumerate(TRI4) if r == c]


def seeded(ba, sc):
    """The non-zero deformation model of gpu_checks.check_intrinsics_step."""
    cf = (np.random.default_rng(5).standard_normal(sc.cfactor.shape) * 0.003).astype(np.float32)
    ba.SetA(0.02)
    ba.SetCFactorBuffer(cf)
    return cf


@pytest.fixture(scope="module")
def distorted(mods):
    S = mods[0]
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = distorted_scene(S, name)
        return cache[name]
    return get


@pytest.mark.parametrize("opt_depth,opt_color", [(True, True), (True, False), (False, True)])
@pytest.mark.parametrize("name", ["small", "many"])
def test_intrinsics_normal_equations(mods, distorted, name, opt_depth, opt_color):
    """IntrinsicsAccumulateKernel<colour, depth, DET = true> + IntrinsicsFinalizeKernel through bba_debug_intrinsics_coeffs: the 34
    global sums and the cell rows B[5], D, b2, obs before the Schur complement.  `many`: 16 + 16 + 5 keyframes."""
    S, DirectBA, L, O, _ = mods
    sc = distorted(name)
    ba = DirectBA.from_scene(sc)
    cf = seeded(ba, sc)
    call = lambda: ba.IntrinsicsCoeffs(opt_depth, opt_color)
    (s0, c0), (s1, c1) = call(), in_mode(ba, True, call)
    tag = (name, opt_depth, opt_color)
    items = -(-sc.num_surfels // 256) * -(-sc.cfg.num_keyframes // 16)
    unit = (items + 1) * U53 * (1 + 1e-5)
    # which instantiation ran: depth only leaves the colour sums zero, colour only the depth sums and every cell row
    if not opt_color:
        assert positive_zero(s1[20:]) and not s0[20:].any(), tag
    else:
        d = s0[DIAG4]
        assert np.all(d > 0) and s1[32] != 0 and s1[33] != 0, tag   # (32, 33: the pair that lane 0 alone stores)
        scale = np.array([math.sqrt(d[r] * d[c]) for r, c in TRI4])
        held("intrinsics colour H, units of (items + 1) 2^-53 sqrt(H_ii H_jj)", np.max(np.abs(s1[20:30] - s0[20:30]) / scale) / unit, 1.0, tag)
        # b: the running sums are bounded by sqrt(H_ii sum w r^2), which the step does not compute: held relative to max |b|
        held("intrinsics colour b (all four, 32 and 33 among them), relative to max |b|",
             np.max(np.abs(s1[30:] - s0[30:])) / np.max(np.abs(s0[30:])), 1e-10, tag)
    if not opt_depth:
        assert positive_zero(s1[:20]) and positive_zero(c1) and not s0[:20].any() and not c0.any(), tag
        return
    d = s0[DIAG5]
    assert np.all(d > 0), tag
    scale = np.array([math.sqrt(d[r] * d[c]) for r, c in TRI5])
    held("intrinsics A, units of (items + 1) 2^-53 sqrt(A_ii A_jj)", np.max(np.abs(s1[:15] - s0[:15]) / scale) / unit, 1.0, tag)
    held("intrinsics b1, relative to max |b1|", np.max(np.abs(s1[15:20] - s0[15:20])) / np.max(np.abs(s0[15:20])), 1e-10, tag)
    # cells
    obs = c0[7].astype(np.float64)
    assert c1[7].tobytes() == c0[7].tobytes() and obs.max() > 1, tag
    orc = O.Oracle(sc)
    orc.model.a = 0.02
    orc.cfactor[:] = cf
    orc.optimize_intrinsics(True, False)
    none = obs == 0
    MEASURED[f"cells without an observation, {name}"] = int(none.sum())
    # (the step zeroes the cfactor of an unobserved cell; the oracle's IEEE arithmetic may flip a pair that sits on a threshold)
    assert np.count_nonzero((np.asarray(orc.cfactor).reshape(-1) == 0) != none) <= 2, tag
    assert positive_zero(c1[:7, none]) and not c0[:7, none].any(), tag
    D0, D1 = c0[5].astype(np.float64), c1[5].astype(np.float64)
    assert np.all(D0[~none] > 0) and np.all(D1[~none] > 0), tag
    cell_unit = (obs[~none] + 1) * U24
    held("intrinsics D per cell, units of (obs + 1) 2^-24 D", np.max(np.abs(D1 - D0)[~none] / (cell_unit * D1[~none])), 1.0, tag)
    for r in range(5):   # |running sum of B_r in a cell| <= sqrt(sum w J_r^2 * D) <= sqrt(A_rr D)
        diff = np.abs(c1[r].astype(np.float64) - c0[r])[~none]
        held("intrinsics B per cell, units of (obs + 1) 2^-24 sqrt(A_rr D)", np.max(diff / (cell_unit * np.sqrt(d[r] * D1[~none]))), 1.0, (tag, r))
    diff = np.abs(c1[6].astype(np.float64) - c0[6])[~none]
    held("intrinsics b2 per cell, units of (obs + 1) 2^-24 max |b2|", np.max(diff / cell_unit) / np.abs(c0[6]).max(), 1.0, tag)
    # a row written to another row's place moves whole-row totals, whatever slack sparse cells leave per cell
    for r in range(7):
        t0, t1 = c0[r].astype(np.float64), c1[r].astype(np.float64)
        held("intrinsics cell row totals, relative to sum |row|", abs(t1.sum() - t0.sum()) / np.abs(t0).sum(), 1e-6, (tag, r))
        assert np.abs(t0).sum() > 0, (tag, r)


@pytest.mark.parametrize("opt_depth,opt_color", [(True, True), (True, False), (False, True)])
@pytest.mark.parametrize("name", ["small", "many"])
def test_intrinsics_two_steps(mods, distorted, name, opt_depth, opt_color):
    """bba_optimize_intrinsics called directly, twice in a row, mode on: against the default mode, the oracle and itself."""
    S, DirectBA, L, O, _ = mods
    sc = distorted(name)
    tag = (name, opt_depth, opt_color)

    def run(on):
        ba = DirectBA.from_scene(sc)
        cf = seeded(ba, sc)
        ba.SetDeterministic(on)
        for _ in range(2):
            ba.OptimizeIntrinsics(opt_depth, opt_color)
        d, c, a = ba._intrinsics()
        return dict(depth_K=d, color_K=c, a=np.float32(a), cfactor=ba.cfactor_buffer()), cf
    (dflt, cf), (det, _), (again, _) = run(False), run(True), run(True)
    assert_same(again, det, "second run")
    orc = O.Oracle(sc)
    orc.model.a = 0.02
    orc.cfactor[:] = cf
    for _ in range(2):
        orc.optimize_intrinsics(opt_depth, opt_color)
    d2, c2 = np.array(orc.model.depth_K[:], np.float32), np.array(orc.model.color_K[:], np.float32)
    # (the tolerances of gpu_checks.check_intrinsics_step)
    assert np.all(np.abs(det["depth_K"] - d2) < REL * np.abs(d2) + 1e-3) and np.all(np.abs(det["color_K"] - c2) < REL * np.abs(c2) + 1e-3), tag
    assert abs(det["a"] - orc.model.a) < 1e-4, tag
    if opt_color and not opt_depth:   # (with the depth step the second colour step sees the other mode's cfactors)
        assert np.any(det["color_K"] != np.asarray(sc.color_K, np.float32)), tag
        held("two colour-only intrinsics steps: colour K, fp32 ulp",
             np.max(np.abs(det["color_K"] - dflt["color_K"]) / np.spacing(np.abs(dflt["color_K"]))), 1.0, tag)
    elif opt_color:
        held("two intrinsics steps: colour K, relative", np.max(np.abs(det["color_K"] - dflt["color_K"]) / np.abs(dflt["color_K"])), 1e-5, tag)
    else:
        assert np.array_equal(det["color_K"], np.asarray(sc.color_K, np.float32)), tag
    if opt_depth:
        assert np.abs(det["cfactor"] - orc.cfactor).max() < 1e-3 and abs(det["a"] - 0.02) > 1e-3, tag
        assert np.array_equal(det["cfactor"] == 0, dflt["cfactor"] == 0) and (det["cfactor"] == 0).any(), tag
        held("two intrinsics steps: depth K, relative", np.max(np.abs(det["depth_K"] - dflt["depth_K"]) / np.abs(dflt["depth_K"])), 1e-5, tag)
        held("two intrinsics steps: a", abs(det["a"] - dflt["a"]), 1e-5, tag)
        held("two intrinsics steps: cfactor", np.abs(det["cfactor"] - dflt["cfactor"]).max(), 1e-5, tag)
    else:
        assert_same({k: det[k] for k in ("depth_K", "a", "cfactor")},
                    dict(depth_K=np.asarray(sc.depth_K, np.float32), a=np.float32(0.02), cfactor=cf), "untouched")


# ---- C. odometry ---------------------------------------------------------------------------------------------------------------

MOTION = [0.02, -0.01, 0.015, 0.01, -0.008, 0.012]   # (tests/test_gpu_odometry.py)
RAGGED = dict(width=148, height=102, num_keyframes=2, num_surfels=2000, cell=2, seed=21, name="ragged")
ODOMETRY = {
    "default": ("small", 4, {}, {}),
    "gradient magnitude": ("small", 4, {"use_gradmag": True}, {}),
    "without level 0": ("small", 4, {"use_pyramid_level_0": False}, {}),
    "one initial estimate": ("small", 3, {"test_different_initial_estimates": False}, {}),
    "depth only": ("small", 3, {}, {"use_descriptor_residuals": False}),
    "descriptor only": ("small", 3, {}, {"use_depth_residuals": False}),
    "ragged 148 x 102": ("ragged", 3, {}, {}),
}


def to_dev(frame):
    import torch
    d, n, _, c = frame
    return (torch.from_numpy(d.view(np.int16)).cuda(), torch.from_numpy(n.view(np.int16)).cuda(), torch.from_numpy(np.ascontiguousarray(c)).cuda())


def ulps(a, b):
    """Largest difference of two fp32 arrays in units of the larger element's spacing (0 where both are zero)."""
    a, b = np.atleast_1d(np.asarray(a, np.float32)), np.atleast_1d(np.asarray(b, np.float32))
    big = np.maximum(np.abs(a), np.abs(b))
    return float(np.max(np.abs(a.astype(np.float64) - b) / np.spacing(np.where(big > 0, big, np.float32(1)))))


def odometry_pair(S, scenes, scene_name):
    if scene_name == "ragged":
        sc = S.make_scene(S.SceneConfig(**RAGGED))
        base, motion = 1, [0.01, 0.005, -0.01, 0.004, -0.003, 0.002]
    else:
        sc, base, motion = scenes(scene_name), 0, MOTION
    return sc, base, S.render_frame(sc, S.se3_mul(sc.poses_true[base], S.se3_exp(motion)))


@pytest.mark.parametrize("case", list(ODOMETRY))
def test_odometry_values(mods, scenes, case):
    """OdomTrackKernel<GRADMAG, DET = true> in every option set test_gpu_odometry.py tracks with: the tracking and the normal
    equations on every level, at the tracked and at the initial pose, against the default mode on the same handle."""
    S, DirectBA, L, O, _ = mods
    scene_name, num_scales, kw, types = ODOMETRY[case]
    sc, base, frame = odometry_pair(S, scenes, scene_name)
    ba = DirectBA.from_scene(sc, **types)
    dev = to_dev(frame)
    init2 = S.se3_exp([0.01, 0.0, 0.0, 0.0, 0.0, 0.0])
    gm = bool(kw.get("use_gradmag", False))
    first = 0 if kw.get("use_pyramid_level_0", True) else 1

    def track():
        est, res = ba.TrackFramePairwise(None, base, *dev, IDENT, init2, num_scales=num_scales, **kw)
        out = dict(pose=est, iterations=list(res.iterations), chose_initial=list(res.chose_initial), residual_count=res.residual_count,
                   residual_sum=res.residual_sum, passes=res.passes)
        out["coeffs"] = [ba.OdometryCoeffs(s, p, init2, use_gradmag=gm) for s in range(first, num_scales) for p in (est, IDENT)]
        return out
    dflt = track()
    ba.SetDeterministic(True)
    det, again = track(), track()
    ba.SetDeterministic(False)
    assert_same(again, det, "second run in the mode")
    for k in ("iterations", "chose_initial", "residual_count", "passes"):
        assert det[k] == dflt[k], (case, k, det[k], dflt[k])
    assert sum(det["iterations"]) > num_scales - first and det["residual_count"] > 0, case
    dt, dr = S.pose_error(det["pose"], dflt["pose"])
    held("odometry pose, m", dt, 1e-6, case)
    held("odometry pose, rad", dr, 1e-6, case)
    held("odometry residual_sum, fp32 ulp", ulps(det["residual_sum"], dflt["residual_sum"]), 2.0, case)
    # the two runs end at poses that may differ in the last bits, so each mode's coefficients are taken at the DETERMINISTIC pose
    at = [ba.OdometryCoeffs(s, p, init2, use_gradmag=gm) for s in range(first, num_scales) for p in (det["pose"], IDENT)]
    for i, ((H1, b1, n1, s1, cnt1, cost1), (H0, b0, n0, s0, cnt0, cost0)) in enumerate(zip(det["coeffs"], at)):
        tag = (case, first + i // 2, "tracked" if i % 2 == 0 else "initial")
        assert n1 == n0 and n0 > 0 and np.array_equal(cnt1, cnt0), tag
        held("odometry H, fp32 ulp", ulps(H1, H0), 2.0, tag)
        held("odometry b, fp32 ulp of max |b|", np.max(np.abs(b1.astype(np.float64) - b0)) / np.spacing(np.abs(b0).max()), 2.0, tag)
        held("odometry costs and residual sum, fp32 ulp", max(ulps(cost1, cost0), ulps(s1, s0)), 2.0, tag)
    if gm:   # the gradient-magnitude instantiation ran: GradientXY has two descriptor residuals per pixel where it has one, and
        # other normal equations (3.7e-4 of max |H| measured; the depth residuals dominate H, and the modes agree to an ulp)
        xy = in_mode(ba, True, lambda: ba.OdometryCoeffs(first, det["pose"], init2, use_gradmag=False))
        assert np.all(xy[4] > det["coeffs"][0][4]) and rel(xy[0], det["coeffs"][0][0]) > 1e-5, case


def test_odometry_partials_allocated_late_and_for_another_size(mods, scenes):
    """The first call in the mode on a handle that has tracked in the default mode, then a second handle with another image size
    (another grid, another partials buffer) in the same process: each equals a handle that was in the mode from the start."""
    S, DirectBA, L, O, _ = mods
    init2 = S.se3_exp([0.01, 0.0, 0.0, 0.0, 0.0, 0.0])

    def track(ba, base, dev):
        est, res = ba.TrackFramePairwise(None, base, *dev, IDENT, init2, num_scales=3)
        return dict(pose=est, iterations=list(res.iterations), residual_count=res.residual_count, residual_sum=res.residual_sum)
    for scene_name in ("small", "ragged"):
        sc, base, frame = odometry_pair(S, scenes, scene_name)
        dev = to_dev(frame)
        late, fresh = DirectBA.from_scene(sc), DirectBA.from_scene(sc)
        track(late, base, dev)
        late.SetDeterministic(True)
        fresh.SetDeterministic(True)
        assert_same(track(late, base, dev), track(fresh, base, dev), scene_name)
