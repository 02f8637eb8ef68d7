"""Checks shared by the GPU parity modules (test_gpu_parity.py, test_gpu_fullsize.py, test_gpu_work_groups.py): one step of
the CUDA path through the C ABI against the reference's kernels (recorded outputs, oracle/ref_golden.py) and the CPU oracle
from the same state, on whichever scene the calling test builds.

Tolerances (BASELINE.json north_star): 1e-4 relative on normal-equation coefficients / residual sums, 1e-5 m / 1e-5 rad on
poses (+ the reference's own run-to-run noise where its float atomics are unordered); counts are integers and must match.
"""
import dataclasses

import numpy as np

REL = 1e-4
POSE_T, POSE_R = 1e-5, 1e-5


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / (np.max(np.abs(b)) + 1e-30))


def distorted_scene(S, name):
    """Depth-distorted raw depth (true a / cfactor != the model's zeros) and perturbed camera estimates."""
    sc = S.make_scene(dataclasses.replace(S.config_by_name(name), depth_a=0.03, cfactor=0.005))
    sc.depth_K = (np.asarray(sc.depth_K, np.float32) * np.float32([1.003, 0.998, 1.002, 0.997])).astype(np.float32)
    sc.color_K = (np.asarray(sc.color_K, np.float32) * np.float32([0.998, 1.002, 1.001, 0.999])).astype(np.float32)
    return sc


def check_intrinsics_step(O, R, DirectBA, sc, opt_depth, opt_color, a_tol=1e-5):
    """OptimizeIntrinsicsCUDA (kernel_opt_intrinsics.cc:39-281): two steps from a non-zero deformation model, ours vs the
    reference kernels (two runs: its own spread) vs the oracle."""
    ba, ref, ref2, orc = DirectBA.from_scene(sc), R.RefDirectBA(sc), R.RefDirectBA(sc), O.Oracle(sc)
    # a non-zero deformation model, so that the d/da and d/dcfactor terms (kernel_opt_intrinsics.cu:97-113) are exercised
    a_init = 0.02
    cf_init = (np.random.default_rng(5).standard_normal(sc.cfactor.shape) * 0.003).astype(np.float32)
    ba.SetA(a_init); ba.SetCFactorBuffer(cf_init)
    ref.set_depth_params(a_init, cf_init)
    ref2.set_depth_params(a_init, cf_init)
    orc.model.a = a_init; orc.cfactor[:] = cf_init
    for _ in range(2):
        ba.OptimizeIntrinsics(opt_depth, opt_color)
        ref.optimize_intrinsics(opt_depth, opt_color)
        ref2.optimize_intrinsics(opt_depth, opt_color)
        orc.optimize_intrinsics(opt_depth, opt_color)
    d0, c0, a0 = ba._intrinsics()
    d1, c1, a1 = ref.intrinsics()
    # `a` is the weakly constrained unknown of this step (hence the reference's prior, kernel_opt_intrinsics.cc:146-155): the
    # reference's own run-to-run difference (unordered fp32 atomics on the per-cell terms) sets the scale of what can be asked
    a_noise = abs(a1 - ref2.intrinsics()[2])
    d2, c2, a2 = np.array(orc.model.depth_K[:], np.float32), np.array(orc.model.color_K[:], np.float32), orc.model.a
    # the UPDATE (new - old, up to ~0.5 px here) must agree to 1e-4 relative of the parameter scale + fp32 atomics noise
    tol_d = REL * np.abs(d1) + 1e-3
    assert np.all(np.abs(d0 - d1) < tol_d), (d0, d1)
    assert np.all(np.abs(c0 - c1) < REL * np.abs(c1) + 1e-3), (c0, c1)
    assert abs(a0 - a1) < a_tol + 5 * a_noise, (a0, a1, a_noise)
    assert np.all(np.abs(d0 - d2) < tol_d) and np.all(np.abs(c0 - c2) < REL * np.abs(c2) + 1e-3) and abs(a0 - a2) < 1e-4
    cf0, cf1 = ba.cfactor_buffer(), ref.cfactor()
    if opt_depth:
        assert np.any(d0 != np.asarray(sc.depth_K, np.float32)) and np.any(cf0 != cf_init) and abs(a0 - a_init) > 1e-3
        rows = R.kept_rows(cf1)
        assert (cf0[rows] != 0).sum() == (cf1[rows] != 0).sum()
        assert np.abs(cf0 - cf1).max() < 1e-4 and np.abs(cf0 - orc.cfactor).max() < 1e-3
    else:
        assert np.array_equal(d0, np.asarray(sc.depth_K, np.float32)) and np.array_equal(cf0, cf_init) and a0 == np.float32(a_init)
    if not opt_color:
        assert np.array_equal(c0, np.asarray(sc.color_K, np.float32))


def pcg_segments(K, n, stride, total):
    """The unknowns of the PCG vectors: pose (6 per keyframe but the gauge), surfel (stride per surfel), intrinsics (the rest)."""
    segs = {"pose": (0, 6 * (K - 1)), "surfel": (6 * (K - 1), 6 * (K - 1) + stride * n)}
    if total > segs["surfel"][1]:
        segs["intr"] = (segs["surfel"][1], total)
    return segs


def check_pcg_building_blocks(O, R, DirectBA, sc, intr, use_desc, a_init, gauge_keyframe, oracle_tol=1e-3):
    """PCGInit / PCGInit2 / PCGStep1 (kernel_pcg.cu:179-1037): r, M, p0, g = J^T W J p0, alpha_n, alpha_d per segment, ours vs
    the reference's kernels vs the oracle.  Returns (ours, reference, oracle)."""
    K, n = sc.cfg.num_keyframes, sc.num_surfels
    ba = DirectBA.from_scene(sc, use_descriptor_residuals=use_desc)
    ref, orc = R.RefDirectBA(sc, True, use_desc), O.Oracle(sc, True, use_desc)
    if a_init:
        cf = (np.random.default_rng(5).standard_normal(sc.cfactor.shape) * 0.003).astype(np.float32)
        ba.SetA(a_init); ba.SetCFactorBuffer(cf)
        ref.set_depth_params(a_init, cf)
        orc.model.a = a_init; orc.cfactor[:] = cf
    kw = dict(optimize_depth_intrinsics=intr, optimize_color_intrinsics=intr, gauge_keyframe=gauge_keyframe)
    ours, theirs, cpu = ba.PCGDebug(**kw), ref.pcg_debug(**kw), orc.pcg_debug(**kw)
    assert len(ours[0]) == len(theirs[0]) == len(cpu[0]) == 6 * (K - 1) + (3 if use_desc else 1) * n + ((5 + sc.cfactor.size + 4) if intr else 0)
    for idx, what in enumerate(("r", "M", "p", "g")):
        for seg, (lo, hi) in pcg_segments(K, n, 3 if use_desc else 1, len(ours[0])).items():
            scale = np.abs(theirs[idx][lo:hi]).max()
            d = np.abs(ours[idx][lo:hi].astype(np.float64) - theirs[idx][lo:hi]).max() / scale
            assert d < 5e-5, (what, seg, d)      # vs the reference's kernels: fp32 summation order only
            if seg != "surfel":                  # oracle (software texture filter, threshold flips): aggregated entries only
                dc = np.abs(cpu[idx][lo:hi].astype(np.float64) - theirs[idx][lo:hi]).max() / scale
                assert dc < oracle_tol, (what, seg, dc)
    assert np.all(np.abs(ours[4] - theirs[4]) < 1e-5 * np.abs(theirs[4]))
    assert np.all(np.abs(cpu[4] - theirs[4]) < 1e-4 * np.abs(theirs[4]))
    assert np.all(ours[1] >= 0) and ours[4][1] > 0   # M = diag(J^T W J) >= 0, p^T A p > 0
    return ours, theirs, cpu


def check_one_ba_iteration(S, R, ba, ref, ref2, sc):
    """One outer iteration of the alternation (activation, normals, position / descriptor, pose of every keyframe) from the
    same state on both sides; ref2 = a second run of the reference = its own noise floor."""
    K = sc.cfg.num_keyframes
    # no end-of-scheme maintenance on either side (it would delete surfels first: direct_ba_alternating.cc:313-319 runs
    # PerformBASchemeEndTasks at the start of a call with increase_ba_iteration_count = false once the counter has moved)
    ba.SetLastBAIterationCount(ba.ba_iteration_count())
    ro = ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, increase_ba_iteration_count=False)
    rr = ref.bundle_adjust(True, True, 1, 1, count_residuals=2, end_tasks=False)
    ref2.bundle_adjust(True, True, 1, 1, count_residuals=False, end_tasks=False)
    # residual counts at the pose step's starting state: depth residuals and descriptor pairs separately
    assert ro.depth_residual_count == rr.n_depth_count
    assert ro.depth_residual_count + ro.descriptor_residual_count // 2 == rr.n_count
    assert abs(ro.pose_iterations_total - rr.pose_iterations_total) <= max(2, K // 50)   # (1e-6 threshold, see test_gpu_parity)
    assert abs(ro.cost - rr.cost) < 5 * REL * rr.cost
    noise = max(max(S.pose_error(ref.pose(k), ref2.pose(k))) for k in range(K))
    worst = 0.0
    for k in range(K):
        dt, dr = S.pose_error(ba.keyframes()[k].global_T_frame(), ref.pose(k))
        worst = max(worst, dt, dr)
        assert dt < POSE_T + 2 * noise and dr < POSE_R + 2 * noise, (k, dt, dr, noise)
    assert R.equal(ba.GetKeyframeStates()[1], ref.activation())
    # activation flags: identical; surfel rows after the geometry step: positions to 2e-6 m, packed normals identical,
    # descriptors to 2e-3 of their +-180 range (tests/test_gpu_parity.py::test_activation_and_geometry at small size)
    assert R.equal(ba.GetActiveHost(), ref.active())
    a, b_ = ba.GetSurfelsHost(), ref.surfels()
    d = np.abs(a[:3] - b_[:3])
    assert d.max() < 1e-5 and (d > 2e-6).mean() < 1e-5, (d.max(), (d > 2e-6).mean())   # (2e-6 on every one of the 30 k surfels of `small`)
    assert (a[3].view(np.uint32) != b_[3].view(np.uint32)).sum() == 0
    assert np.max(np.abs(a[6:8] - b_[6:8])) < 2e-3
    print(f"{sc.cfg.name}: worst pose difference to the reference {worst:.2e} (reference run-to-run {noise:.2e}), "
          f"{ro.depth_residual_count + ro.descriptor_residual_count} residuals, GN iterations {ro.pose_iterations_total} / {rr.pose_iterations_total}")


def check_pcg_inner_steps(S, R, DirectBA, sc):
    """use_pcg = true with 4 inner steps per outer iteration, 2 outer iterations, gauge keyframe 2 (direct_ba_pcg.cc:43-819): few
    enough fp32 CG steps for tight parity with the reference's kernels (+ its own run-to-run noise, a second run)."""
    K = sc.cfg.num_keyframes
    ba, ref, ref2 = DirectBA.from_scene(sc), R.RefDirectBA(sc), R.RefDirectBA(sc)
    ro = ba.BundleAdjustment(None, False, False, False, True, True, 2, 2, use_pcg=True, pcg_max_inner_iterations=4, pcg_gauge_keyframe=2)
    rr = ref.bundle_adjust_pcg(min_iterations=2, max_iterations=2, max_inner_iterations=4, gauge_keyframe=2)
    ref2.bundle_adjust_pcg(min_iterations=2, max_iterations=2, max_inner_iterations=4, gauge_keyframe=2)
    assert ro.iterations_done == rr.iterations_done == 2 and ro.pcg_inner_iterations_total == rr.inner_iterations_total == 8
    assert abs(ro.pcg_last_r_norm - rr.last_r_norm) < 1e-3 * rr.last_r_norm
    noise = max(max(S.pose_error(ref.pose(k), ref2.pose(k))) for k in range(K))
    pa = ba.GetKeyframeStates()[0]
    assert np.array_equal(pa[2], sc.poses_init[2])     # the gauge keyframe does not move
    for k in range(K):
        dt, dr = S.pose_error(pa[k], ref.pose(k))
        assert dt < 1e-5 + 3 * noise and dr < 1e-5 + 3 * noise, (k, dt, dr, noise)
    a, b_ = ba.GetSurfelsHost(), ref.surfels()
    assert np.abs(a[:3] - b_[:3]).max() < 1e-4 and np.abs(a[:3] - b_[:3]).mean() < 1e-6      # 8 fp32 CG steps
    assert (a[3].view(np.uint32) != b_[3].view(np.uint32)).mean() < 1e-4   # second normals update sees 1e-6-different positions
