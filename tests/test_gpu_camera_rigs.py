"""GPU parity on camera rigs whose colour camera is not the depth camera (badslam_b200/scene.py: rig_half, rig_same,
rig_half1).  Every other scene of the suite has one symmetric camera for depth and colour, so the depth-to-colour mapping is the
identity there, no pair ever loses its descriptor residual to the colour image bounds, the tangent points project through the
same intrinsics as the surfel, and every sparse cell is whole.

  rig_half   162 x 122 depth, fx 101 / fy 93, principal point (84.3, 57.9), cell 4 (a partial last cfactor column and row);
             81 x 61 colour of a camera with 4 % longer focal lengths and a shifted principal point (d2c_fx = 0.52): the
             configuration of pyramid_level_for_color = 1, and the odometry's half-resolution colour path.
  rig_same   151 x 110 depth and colour, fx != fy, cell 3; colour focal lengths 6 % longer, principal point a few pixels away.
  rig_half1  rig_half's cameras at cell 1 (surfel creation exact against the reference).

Each check is the one the symmetric scenes pass (test_gpu_parity.py, test_gpu_work_groups.py, test_gpu_lifecycle.py,
test_gpu_odometry.py, test_gpu_frame_poses.py, gpu_checks.py), three-way against the reference's kernels (recorded outputs,
tests/golden/ref/test_gpu_camera_rigs) and the oracles, plus assertions that the rig reaches the code it is there for.
"""
import numpy as np
import pytest

import test_gpu_frame_poses as frame_poses
import test_gpu_lifecycle as lifecycle
import test_gpu_odometry as odometry
import test_gpu_parity as parity
from gpu_checks import (check_intrinsics_step, check_one_ba_iteration, check_pcg_building_blocks, check_pcg_inner_steps,
                        distorted_scene)
from test_gpu_spatial_order import border_surfels, check_same, with_surfels
from test_gpu_work_groups import check_batch, distinct_poses, variants

pytestmark = pytest.mark.gpu

RIGS = ["rig_half", "rig_same"]


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    from oracle import cpu_oracle, ref_golden
    assert ref_golden.available(), "recording needs oracle/_ref/libbadslam_ref.so (oracle/build_ref.sh)"
    return S, DirectBA, cpu_oracle, ref_golden


@pytest.fixture(scope="module")
def lib():
    from badslam_b200 import _lib
    return _lib


_scenes = {}


def rig(S, name):
    if name not in _scenes:
        _scenes[name] = S.make_scene(S.config_by_name(name))
    return _scenes[name]


@pytest.mark.parametrize("name", RIGS)
def test_pose_coefficients_three_way(mods, lib, name):
    """The single-keyframe path (test_gpu_parity.py's bars), then every instantiation of the batched pose kernel with and without
    stats on all keyframes and on one (test_gpu_work_groups.py's bars), at poses distinct per keyframe."""
    S, DirectBA, O, R = mods
    sc = rig(S, name)
    parity.test_pose_coefficients_three_way(mods, sc)
    K = sc.cfg.num_keyframes
    poses = distinct_poses(S, sc)
    ba, ref, orc = DirectBA.from_scene(sc), R.RefDirectBA(sc), O.Oracle(sc)
    single = [ba.AccumulatePoseEstimationCoeffs(k, poses[k]) for k in range(K)]
    oracle = [orc.pose_coeffs(k, poses[k]) for k in range(K)]
    reference = [ref.pose_coeffs(k, poses[k]) for k in range(K)]
    # the rig does what it is for: associated pairs whose colour pixel lies outside the colour image keep their depth residual
    # and lose the descriptor residual (never the case with one camera: n_photo == n_assoc on every other scene)
    lost = [pc.n_assoc - pc.n_photo for pc in single]
    assert sum(1 for x in lost if x > 0) >= K // 2, lost
    print(f"{name}: {sum(lost)} of {sum(pc.n_assoc for pc in single)} associated pairs "
          f"({sum(lost) / sum(pc.n_assoc for pc in single):.2%}) outside the colour image")
    for vname, v in variants(lib).items():
        for ids in (np.arange(K), np.array([K - 1])):
            try:
                check_batch(ba, ids, poses, v, single, oracle, reference)
            except AssertionError as e:
                raise AssertionError(f"variant {vname}, {len(ids)} keyframes: {e}") from e


@pytest.mark.parametrize("name", RIGS)
@pytest.mark.parametrize("use_depth,use_desc", [(True, False), (False, True)], ids=["depth_only", "descriptor_only"])
def test_single_residual_type(mods, name, use_depth, use_desc):
    S, DirectBA, O, R = mods
    parity.test_single_residual_type(mods, rig(S, name), use_depth, use_desc)


@pytest.mark.parametrize("name", RIGS)
def test_pre_culling_is_exact_on_asymmetric_borders(mods, lib, name):
    """Surfels placed on, just inside and just beyond each border of the off-centre, fx != fy depth image: the PRE instantiations
    (chunk boxes culled against the view) count exactly what a non-PRE instantiation counts."""
    S, DirectBA, O, R = mods
    sc = rig(S, name)
    K = sc.cfg.num_keyframes
    rng = np.random.default_rng(91)
    n0 = sc.num_surfels
    chosen = (0, K // 2, K - 1)
    cols = [sc.surfels[:, :n0]]
    for k in chosen:
        extra = sc.surfels[:, rng.integers(0, n0, 6 * 300)].copy()
        extra[0:3] = border_surfels(S, sc, k, rng)
        cols.append(extra)
    cols = np.concatenate(cols, axis=1)
    pre = (lib.POSE_VARIANT_256_PRE, lib.POSE_VARIANT_512_PRE)
    base = check_same(DirectBA.from_scene(sc), np.arange(K), sc.poses_init, pre, lib.POSE_VARIANT_256, "scene")
    counts = check_same(DirectBA.from_scene(with_surfels(sc, cols, cols.shape[1])), np.arange(K), sc.poses_init, pre,
                        lib.POSE_VARIANT_256, "with border surfels")
    for k in chosen:
        added = int(counts[k][0]) - int(base[k][0])
        assert 0 < added < cols.shape[1] - n0, (k, added)


@pytest.mark.parametrize("name", RIGS)
def test_estimate_frame_pose(mods, name):
    S, DirectBA, O, R = mods
    parity.test_estimate_frame_pose(mods, rig(S, name))


@pytest.mark.parametrize("name", RIGS)
def test_batched_frame_poses(mods, lib, name):
    """bba_estimate_frame_poses_for_frames with the keyframes' buffers and frames rendered through the rig as entries (colour
    buffers of the colour camera's size and pitch, uploaded as the entries' luma textures): a batch of one is the single-frame
    call, and 37 entries in calls of 1 .. 37 agree with the single-frame calls, the keyframe form, the coefficients at the
    estimate, the oracle and -- for the keyframe entries -- the reference's EstimateFramePose (test_gpu_frame_poses.py)."""
    S, DirectBA, O, R = mods
    sc = rig(S, name)
    fmods = (S, DirectBA, lib, O)
    frame_poses._scenes[name] = sc
    frame_poses.test_batch_of_one_is_the_single_frame_call(fmods, name)
    frame_poses.check_entries_agree_with_single_calls(fmods, sc, reference=R.RefDirectBA(sc))


@pytest.mark.parametrize("name", RIGS)
def test_activation_and_geometry(mods, name):
    S, DirectBA, O, R = mods
    parity.test_activation_and_geometry(mods, rig(S, name))


@pytest.mark.parametrize("name", RIGS)
@pytest.mark.parametrize("opt_depth,opt_color", [(True, True), (True, False), (False, True)])
def test_intrinsics_step_three_way(mods, name, opt_depth, opt_color):
    S, DirectBA, O, R = mods
    sc = distorted_scene(S, name)
    # (`a` ends near 5.17 here: ours differs from the reference by 3.2e-5 = 6e-6 relative, as on `many` in test_gpu_work_groups)
    check_intrinsics_step(O, R, DirectBA, sc, opt_depth, opt_color, a_tol=5e-5)
    if opt_depth and not opt_color:
        # Which cells the step observes, from the state check_intrinsics_step starts at: it sets the cfactor of an unobserved cell
        # to 0 and of an observed one to its update (kernel_opt_intrinsics.cu:374-424).  The partial last column and row of both
        # rigs (rig_half: x 160-161, y 120-121; rig_same: x 150, y 108-109) hold only the two outermost pixel columns / rows,
        # which never have valid depth (no normal on the border, and their neighbours fail the four-neighbour test of the
        # radius / isolated-pixel step), so they are never observed; the whole cells next to them are.  A cf_w stride or a cell
        # index off by one moves observations into the partial cells or out of their neighbours.
        ba = DirectBA.from_scene(sc)
        cf_init = (np.random.default_rng(5).standard_normal(sc.cfactor.shape) * 0.003).astype(np.float32)
        ba.SetA(0.02); ba.SetCFactorBuffer(cf_init)
        ba.OptimizeIntrinsics(True, False)
        observed = ba.cfactor_buffer() != 0
        assert not observed[-1, :].any() and not observed[:, -1].any(), (observed[-1, :], observed[:, -1])
        assert observed[-2, :].mean() > 0.9 and observed[:, -2].mean() > 0.9, (observed[-2, :], observed[:, -2])


@pytest.mark.parametrize("name,distort,intr,use_desc", [("rig_half", False, False, True), ("rig_half", False, False, False),
                                                         ("rig_same", True, True, True), ("rig_half", True, True, True)])
def test_pcg_building_blocks_three_way(mods, name, distort, intr, use_desc):
    S, DirectBA, O, R = mods
    sc = distorted_scene(S, name) if distort else rig(S, name)
    check_pcg_building_blocks(O, R, DirectBA, sc, intr, use_desc, 0.02 if intr else 0.0, gauge_keyframe=1, oracle_tol=1e-2)


@pytest.mark.parametrize("name,filt", [("rig_half1", False), ("rig_half1", True), ("rig_half", True), ("rig_same", False)])
def test_create_surfels_for_keyframe_three_way(mods, name, filt):
    """Creation samples the colour row and the descriptors in the colour image (clamped to its size): exact against the oracle,
    exact against the reference at cell 1, in distribution at cells 3 and 4 (test_gpu_lifecycle.py)."""
    lifecycle.test_create_surfels_for_keyframe_three_way(mods, name, filt)


@pytest.mark.parametrize("name", RIGS)
def test_merge_surfels_three_way(mods, name):
    lifecycle.test_merge_surfels_three_way(mods, name)


@pytest.mark.parametrize("name", RIGS)
def test_end_tasks_three_way(mods, name):
    lifecycle.test_end_tasks_three_way(mods, name)


@pytest.mark.parametrize("name", RIGS)
def test_one_ba_iteration(mods, name):
    S, DirectBA, O, R = mods
    sc = rig(S, name)
    check_one_ba_iteration(S, R, DirectBA.from_scene(sc), R.RefDirectBA(sc), R.RefDirectBA(sc), sc)


@pytest.mark.parametrize("name", RIGS)
def test_pcg_bundle_adjustment_against_reference(mods, name):
    """use_pcg = true, 4 inner steps per outer iteration: the tight parity of test_gpu_parity.py's PCG test."""
    S, DirectBA, O, R = mods
    check_pcg_inner_steps(S, R, DirectBA, rig(S, name))


@pytest.fixture(scope="module")
def odo_mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    from oracle import odometry_oracle, ref_golden
    assert ref_golden.available(), "recording needs oracle/_ref/libbadslam_ref.so (oracle/build_ref.sh)"
    return S, DirectBA, odometry_oracle, ref_golden


def test_odometry_pyramids_and_single_evaluation(odo_mods):
    """Half-resolution colour: the base level 0 maps every depth pixel into the 81 x 61 colour image, and the level cameras scale
    the colour camera by 2 / 2^scale.  Pyramids level by level, one evaluation per level (counts exact, H / b 1e-4)."""
    odometry.test_pyramids_and_single_evaluation_three_way(odo_mods, "rig_half", 3)


@pytest.mark.parametrize("kw", [{}, {"use_gradmag": True}, {"use_pyramid_level_0": False},
                                {"use_pyramid_level_0": False, "use_gradmag": True}],
                         ids=["default", "gradmag", "no_level0", "no_level0_gradmag"])
def test_odometry_tracking(odo_mods, kw):
    """The whole tracking against the reference (test_gpu_odometry.py's bars); without level 0 the tracked frame's level 1 takes its
    colour from the half-resolution image one to one (CalibrateAndDownsampleImagesCUDAKernel's branch for colour at half the
    depth size)."""
    S, DirectBA, O, R = odo_mods
    sc, true_rel, frame = odometry.make_pair(S, "rig_half")
    ba, ref = DirectBA.from_scene(sc), R.RefDirectBA(sc)
    init2 = S.se3_exp([0.01, 0.0, 0.0, 0.0, 0.0, 0.0])
    est0, res0, est1, res1, noise, dt, dr = odometry.run_tracking(S, ba, ref, sc, frame, true_rel, odometry.IDENT, init2,
                                                                  num_scales=3, **kw)
    first = 0 if kw.get("use_pyramid_level_0", True) else 1
    odometry.check_levels(ba, ref, None, 3, first)
    its0, its1 = list(res0.iterations)[:3], list(res1.iterations)[:3]
    print(f"rig_half {kw}: iterations {its0} / reference {its1}; pose difference {dt:.2e} m {dr:.2e} rad, reference run-to-run "
          f"{noise:.2e}; error to the rendered motion {S.pose_error(est0, true_rel)} / {S.pose_error(est1, true_rel)}")
    assert list(res0.chose_initial)[:3] == list(res1.chose_initial)[:3]
    # closer to the rendered motion than the start on both sides.  (With level 0 the tracked frame's colour is read at depth pixel
    # coordinates from the half-resolution image, as in the reference -- pairwise_frame_tracking.cc:298 -- so the finest level's
    # descriptor residuals compare mismatched images and the gain is smaller than with one camera.)
    e_init = S.pose_error(odometry.IDENT, true_rel)[0]
    assert S.pose_error(est0, true_rel)[0] < 0.9 * e_init and S.pose_error(est1, true_rel)[0] < 0.9 * e_init
    gm = bool(kw.get("use_gradmag", False))
    _, _, _, _, counts, costs = ba.OdometryCoeffs(first, est0, est1, use_gradmag=gm)
    assert costs[0] <= costs[1] * (1 + 2e-3) and counts[0] >= counts[1] * (1 - 2e-3), (counts, costs)
    assert all(abs(a - b) <= 1 for a, b in zip(its0, its1)), (its0, its1)
    limit = max(1e-5 + 10 * noise, 5e-5)
    assert dt < limit and dr < limit, (dt, dr, noise)
    assert res0.kernel_launches <= 3 + 4 and res1.kernel_launches > 10 * res0.kernel_launches


@pytest.mark.parametrize("kw", [{}, {"use_pyramid_level_0": False, "use_gradmag": True}], ids=["default", "no_level0_gradmag"])
def test_odometry_deterministic_batch_equals_single_call(odo_mods, kw):
    """In the deterministic mode the batched call (frames as the base) and the _to_frame form give the single call's bits."""
    import torch
    S, DirectBA, O, R = odo_mods
    sc, true_rel, frame = odometry.make_pair(S, "rig_half", base_kf=2)
    ba = DirectBA.from_scene(sc)
    ba.SetDeterministic(True)
    dev = odometry.to_dev(frame)
    base = odometry.to_dev((sc.depth[2], sc.normals[2], None, sc.color[2]))
    init2 = S.se3_exp([0.01, 0.0, 0.0, 0.0, 0.0, 0.0])
    est0, res0 = ba.TrackFramePairwise(None, 2, *dev, odometry.IDENT, init2, num_scales=3, **kw)
    est1, res1 = ba.TrackFramePairwiseToFrame(None, *base, *dev, odometry.IDENT, init2, num_scales=3, **kw)
    ests, results, _ = ba.TrackFramesPairwise(None, [base, dev], [(2, 0, 1, odometry.IDENT, init2), (-1, 0, 1, odometry.IDENT, init2)],
                                              num_scales=3, **kw)
    torch.cuda.synchronize()
    for est in (est1, ests[0], ests[1]):
        assert est.tobytes() == est0.tobytes(), (est, est0)
    for r in (res1, results[0], results[1]):
        assert list(r.iterations)[:3] == list(res0.iterations)[:3]
    assert S.pose_error(est0, true_rel)[0] < S.pose_error(odometry.IDENT, true_rel)[0]


def test_raw_frames_at_half_colour_resolution_feed_bundle_adjustment(mods):
    """162 x 122 raw depth and RGB preprocessed with pyramid_level_for_color = 1: keyframes with 81 x 61 colour, surfel creation
    and a BA (test_gpu_preprocess.py's end-to-end path on this rig)."""
    import torch
    S, DirectBA, O, R = mods
    from badslam_b200.direct_ba import PinholeCamera4f
    sc = rig(S, "rig_half")
    cfg = sc.cfg
    ch, cw = sc.color.shape[1:3]
    cap = 1 << 17
    ba = DirectBA(cap, cfg.raw_to_float_depth, cfg.baseline_fx, cfg.cell,
                  color_camera_initial_estimate=PinholeCamera4f(cw, ch, sc.color_K),
                  depth_camera_initial_estimate=PinholeCamera4f(cfg.width, cfg.height, sc.depth_K), max_keyframes=cfg.num_keyframes)
    ba.SetSurfels(torch.zeros((17, cap), dtype=torch.float32, device="cuda"), 0)
    created = 0
    for k in range(cfg.num_keyframes):
        raw = S.raw_frame(sc, k, noise_raw=1.0)[0]
        rgb = S.raw_frame(sc, k, noise_raw=1.0, scale=2)[1]          # the colour sensor at twice the colour camera's resolution
        assert raw.shape == (cfg.height, cfg.width) and rgb.shape == (2 * ch, 2 * cw, 3)
        kf = ba.CreateKeyframeFromFrame(k, torch.from_numpy(raw.view(np.int16)).cuda(), torch.from_numpy(rgb).cuda(),
                                        sc.poses_init[k], max_depth=6.0, pyramid_level_for_color=1)
        assert tuple(kf.depth_buffer.shape) == (cfg.height, cfg.width) and tuple(kf.color_buffer.shape) == (ch, cw, 4)
        assert 0 < kf.min_depth < kf.max_depth <= 6.0
        created += ba.CreateSurfelsForKeyframe(None, True, kf.id)
    assert created > 1000 and ba.surfels_size() == created
    rgba = ba.GetSurfelsHost()[5].view(np.uint32)
    assert np.count_nonzero(rgba) > 0.9 * created          # the colour row is sampled in the colour image
    r = ba.BundleAdjustment(None, False, False, False, True, True, 3, 3)
    assert r.iterations_done == 3 and r.depth_residual_count > 0.5 * created
    assert 0 < r.descriptor_residual_count // 2 < r.depth_residual_count
    poses = ba.GetKeyframeStates()[0]
    assert np.all(np.isfinite(poses))

    def rel(P, k):
        return S.se3_mul(S.se3_inverse(P[0]), P[k])
    e_init = max(S.pose_error(rel(sc.poses_init, k), rel(sc.poses_true, k))[0] for k in range(1, cfg.num_keyframes))
    e_ba = max(S.pose_error(rel(poses, k), rel(sc.poses_true, k))[0] for k in range(1, cfg.num_keyframes))
    print(f"relative pose error: {e_init:.2e} m before, {e_ba:.2e} m after 3 BA iterations on preprocessed raw frames")
    assert e_ba < e_init
