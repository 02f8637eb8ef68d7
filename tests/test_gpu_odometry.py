"""GPU parity of the image-pair odometry (bba_track_frame_pairwise; SURVEY.md 8(f4)): the sm_90a path through the C ABI against
the reference's own kernels (oracle/_ref: kernel_downsample.cu, cuda_image_processing.cu, kernel_opt_pose.cu:422-1340 behind the
restated host loop of pairwise_frame_tracking.cc) and the CPU oracle (oracle/odometry_oracle.py).

What is demanded:
  * pyramids (u8 intensity, u16 normals, float depth picked from the inputs): identical to the reference's, level by level;
  * one evaluation at a given pose (AccumulatePoseEstimationCoeffsFromImagesCUDA / ComputeCostAndResidualCountFromImagesCUDA):
    residual counts identical, H / b / costs within 1e-4 relative (BASELINE.json north_star; fp32 sums in a different order);
  * the whole coarse-to-fine optimisation: the Gauss-Newton iterations of this path do not settle to a fixed point on every
    level (associations flip between iterations; the reference caps them at 30 per level), so two runs that differ in the last
    bit drift apart like the reference drifts from itself (unordered float atomics): the poses must agree to 1e-5 m / rad plus
    ten times the reference's own run-to-run spread (three extra runs), with identical iteration counts and an equally low cost.
"""
import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

REL = 1e-4
MOTION = [0.02, -0.01, 0.015, 0.01, -0.008, 0.012]          # base_T_frame of the tracked frame (se3 tangent: 2 cm, ~1 degree)
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / (np.max(np.abs(b)) + 1e-30))


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    from oracle import odometry_oracle, ref_golden
    assert ref_golden.available(), "recording needs oracle/_ref/libbadslam_ref.so (oracle/build_ref.sh)"
    return S, DirectBA, odometry_oracle, ref_golden


def make_pair(S, name, base_kf=0, motion=MOTION):
    sc = S.make_scene(S.config_by_name(name))
    true_rel = S.se3_exp(motion)
    frame = S.render_frame(sc, S.se3_mul(sc.poses_true[base_kf], true_rel))
    return sc, true_rel, frame


def to_dev(frame):
    import torch
    d, n, _, c = frame
    return (torch.from_numpy(d.view(np.int16)).cuda(), torch.from_numpy(n.view(np.int16)).cuda(), torch.from_numpy(np.ascontiguousarray(c)).cuda())


def oracle_for(O, sc, **kw):
    return O.Odometry(sc.depth_K, sc.color_K, sc.cfg.raw_to_float_depth, sc.cfg.baseline_fx, sc.cfg.cell, sc.depth_a, sc.cfactor, **kw)


def check_levels(ba, ref, orc, num_scales, first_scale, O=None):
    """Product vs reference: identical on the rows the recorded reference levels hold.  Oracle (when given): level 0 identical
    colour / validity, depth to the fast-math rounding; coarser levels are built by the oracle's downsample() from the
    PRODUCT's finer level (equal to the reference's where recorded) and must agree up to the tie-break of "closest to the
    block mean" (tests/test_oracle_odometry.py::assert_same_up_to_ties: on planar surfaces the four depths of a block are
    pairwise symmetric about their mean); the product's images are then handed to the oracle so that its evaluations run on
    the same pyramid."""
    from test_oracle_odometry import assert_same_up_to_ties
    from oracle.ref_golden import kept_rows
    prev = {}
    for scale in range(num_scales):
        for which in (0, 1):
            if which == 1 and scale < first_scale:
                continue
            d0, n0, c0 = ba.OdometryLevel(which, scale)
            d1, n1, c1 = ref.odometry_level(which, scale)
            assert d0.shape == d1.shape
            rows = kept_rows(d1)   # (recorded reference levels may hold a band of rows only)
            assert np.array_equal(c0[rows], c1[rows]), (which, scale, np.mean(c0[rows] != c1[rows]))
            assert np.array_equal(d0[rows], d1[rows]), (which, scale, np.mean(d0[rows] != d1[rows]))
            v = np.asarray(d1[rows]) > 0
            assert np.array_equal(n0[rows][v], np.asarray(n1[rows])[v]), (which, scale)
            # the product's level equals the reference's: the oracle is checked against it in full
            d1, n1, c1 = d0, n0, c0
            valid = d1 > 0
            if orc is not None:
                wn = "tracked" if which else "base"
                if scale == 0:
                    d2, n2, c2 = orc.levels[0][wn]
                    assert np.array_equal(c2, c1), ("oracle colour", which, scale, np.mean(c2 != c1))
                    # the oracle evaluates exp / divisions in IEEE arithmetic, the kernels with the fast-math approximations
                    assert np.array_equal(d2 > 0, valid) and np.allclose(d2[valid], d1[valid], rtol=2e-6, atol=0), ("oracle depth", which)
                    assert np.array_equal(n2[valid], n1[valid])
                else:
                    d2, n2, c2 = O.downsample(*prev[which])
                    assert np.array_equal(c2, c1), ("oracle colour", which, scale, np.mean(c2 != c1))
                    assert_same_up_to_ties(prev[which][0], d2, d1, ("oracle depth", which, scale))
                    same = valid & (d2 == d1)
                    assert same.mean() > 0.5 and np.array_equal(n2[same], n1[same])
                orc.levels[scale][wn] = (d1, np.where(valid, n1, 0).astype(np.uint16), c1)
            prev[which] = (d1, np.where(valid, n1, 0).astype(np.uint16), c1)


@pytest.mark.parametrize("name,num_scales", [("tiny", 3), ("small", 4)])
def test_pyramids_and_single_evaluation_three_way(mods, name, num_scales):
    S, DirectBA, O, R = mods
    sc, true_rel, frame = make_pair(S, name)
    ba, ref = DirectBA.from_scene(sc), R.RefDirectBA(sc)
    dev = to_dev(frame)
    ba.TrackFramePairwise(None, 0, *dev, IDENT, IDENT, num_scales=num_scales, max_iterations_per_scale=1)
    ref.track_frame_pairwise(0, frame[0], frame[1], frame[3], IDENT, IDENT, num_scales=num_scales)
    orc = oracle_for(O, sc)
    orc.build((sc.depth[0], sc.normals[0], sc.color[0]), (frame[0], frame[1], frame[3]), num_scales=num_scales)
    check_levels(ba, ref, orc, num_scales, 0, O)
    off = S.se3_mul(true_rel, S.se3_exp([0.004, -0.003, 0.002, 0.002, 0.001, -0.002]))
    for scale in range(num_scales):
        for pose_a, pose_b in ((true_rel, off), (off, IDENT)):
            H0, b0, n0, s0, counts0, costs0 = ba.OdometryCoeffs(scale, pose_a, pose_b)
            H1, b1, n1, s1, counts1, costs1 = ref.odometry_coeffs(scale, pose_a, pose_b)
            assert n0 == n1 and n1 > 0, (scale, n0, n1)
            assert np.array_equal(counts0, counts1), (scale, counts0, counts1)
            assert rel(H0, H1) < REL and rel(b0, b1) < REL, (scale, rel(H0, H1), rel(b0, b1))
            assert abs(s0 - s1) < REL * abs(s1) and rel(costs0, costs1) < REL, (scale, s0, s1, costs0, costs1)
            H2, b2, n2, s2 = orc.coeffs(scale, pose_a)
            # the oracle's IEEE arithmetic flips a few association decisions that sit exactly on a threshold
            assert abs(n2 - n1) <= max(2, 2e-4 * n1), (scale, n2, n1)
            assert rel(H2, H1) < 2e-3 and rel(b2, b1) < 2e-3, (scale, rel(H2, H1), rel(b2, b1))


def run_tracking(S, ba, ref, sc, frame, true_rel, init1, init2, **kw):
    dev = to_dev(frame)
    est0, res0 = ba.TrackFramePairwise(None, 0, *dev, init1, init2, **kw)
    est1, res1 = ref.track_frame_pairwise(0, frame[0], frame[1], frame[3], init1, init2, **kw)
    # the reference's own run-to-run spread (unordered float atomics): largest pairwise difference of three more runs
    runs = [est1] + [ref.track_frame_pairwise(0, frame[0], frame[1], frame[3], init1, init2, **kw)[0] for _ in range(3)]
    noise = max(max(S.pose_error(a, b)) for i, a in enumerate(runs) for b in runs[i + 1:])
    dt, dr = S.pose_error(est0, est1)
    return est0, res0, est1, res1, noise, dt, dr


@pytest.mark.parametrize("name,num_scales,kw", [
    ("tiny", 3, {}),
    ("small", 4, {}),
    ("small", 4, {"use_gradmag": True}),
    ("small", 4, {"use_pyramid_level_0": False}),
    ("small", 3, {"test_different_initial_estimates": False}),
])
def test_track_frame_pairwise_against_reference(mods, name, num_scales, kw):
    S, DirectBA, O, R = mods
    sc, true_rel, frame = make_pair(S, name)
    ba, ref = DirectBA.from_scene(sc), R.RefDirectBA(sc)
    init2 = S.se3_exp([0.01, 0.0, 0.0, 0.0, 0.0, 0.0])
    est0, res0, est1, res1, noise, dt, dr = run_tracking(S, ba, ref, sc, frame, true_rel, IDENT, init2, num_scales=num_scales, **kw)
    first = 0 if kw.get("use_pyramid_level_0", True) else 1
    check_levels(ba, ref, None, num_scales, first)
    its0, its1 = list(res0.iterations)[:num_scales], list(res1.iterations)[:num_scales]
    print(f"{name} {kw}: iterations {its0} / reference {its1}; pose difference {dt:.2e} m {dr:.2e} rad, reference run-to-run {noise:.2e}; "
          f"error to the rendered motion {S.pose_error(est0, true_rel)} / {S.pose_error(est1, true_rel)}; launches {res0.kernel_launches} / {res1.kernel_launches}")
    assert list(res0.chose_initial)[:num_scales] == list(res1.chose_initial)[:num_scales]
    # the tracking must have done its job on both sides: closer to the rendered motion than the starting point (much closer
    # when the finest level takes part)
    e_init = S.pose_error(IDENT, true_rel)[0]
    gain = 0.5 if first == 0 else 0.9
    assert S.pose_error(est0, true_rel)[0] < gain * e_init and S.pose_error(est1, true_rel)[0] < gain * e_init
    # equally good optimum: the cost of our result is not worse than the cost of the reference's result, both evaluated on the
    # product's pyramid by the product's cost kernel (equal to the reference's at fixed states: the three-way test above)
    gm = bool(kw.get("use_gradmag", False))
    _, _, _, _, counts, costs = ba.OdometryCoeffs(first, est0, est1, use_gradmag=gm)
    assert costs[0] <= costs[1] * (1 + 2e-3) and counts[0] >= counts[1] * (1 - 2e-3), (counts, costs)
    # Same iteration counts and branch decisions; the poses agree to 1e-5 plus the drift of this non-settling iteration: up to 86
    # capped Gauss-Newton steps amplify last-bit differences of H / b (ours are fp64 sums of per-lane fp32 partials, the
    # reference's unordered fp32 atomics), measured here by the reference's own spread.
    assert all(abs(a - b) <= 1 for a, b in zip(its0, its1)), (its0, its1)   # (equal in every run so far; +-1 for a level that stops at the threshold)
    # (the floor of 5e-5 covers a draw in which the reference's four runs happen to agree closely)
    limit = max(1e-5 + 10 * noise, 5e-5)
    assert dt < limit and dr < limit, (dt, dr, noise)
    assert res0.kernel_launches <= num_scales + 4 and res1.kernel_launches > 10 * res0.kernel_launches


def test_depth_only_and_descriptor_only(mods):
    S, DirectBA, O, R = mods
    sc, true_rel, frame = make_pair(S, "small")
    for use_depth, use_desc in ((True, False), (False, True)):
        ba = DirectBA.from_scene(sc, use_depth_residuals=use_depth, use_descriptor_residuals=use_desc)
        ref = R.RefDirectBA(sc, use_depth=use_depth, use_descriptor=use_desc)
        dev = to_dev(frame)
        ba.TrackFramePairwise(None, 0, *dev, IDENT, IDENT, num_scales=3, max_iterations_per_scale=1)
        ref.track_frame_pairwise(0, frame[0], frame[1], frame[3], IDENT, IDENT, num_scales=3)
        for scale in range(3):
            H0, b0, n0, s0, counts0, costs0 = ba.OdometryCoeffs(scale, true_rel, IDENT)
            H1, b1, n1, s1, counts1, costs1 = ref.odometry_coeffs(scale, true_rel, IDENT)
            assert n0 == n1 and np.array_equal(counts0, counts1) and n1 > 0
            assert rel(H0, H1) < REL and rel(b0, b1) < REL and rel(costs0, costs1) < REL


def test_ragged_size_and_errors(mods):
    """An image size that is not a multiple of the tile (32 x 8) or of 2^scales, and the argument checks."""
    import torch
    S, DirectBA, O, R = mods
    cfg = S.SceneConfig(width=148, height=102, num_keyframes=2, num_surfels=2000, cell=2, seed=21, name="ragged")
    sc = S.make_scene(cfg)
    true_rel = S.se3_exp([0.01, 0.005, -0.01, 0.004, -0.003, 0.002])
    frame = S.render_frame(sc, S.se3_mul(sc.poses_true[1], true_rel))
    ba, ref = DirectBA.from_scene(sc), R.RefDirectBA(sc)
    dev = to_dev(frame)
    est0, res0 = ba.TrackFramePairwise(None, 1, *dev, IDENT, IDENT, num_scales=3)
    est1, res1 = ref.track_frame_pairwise(1, frame[0], frame[1], frame[3], IDENT, IDENT, num_scales=3)
    check_levels(ba, ref, None, 3, 0)
    for scale in range(3):
        H0, b0, n0, s0, counts0, costs0 = ba.OdometryCoeffs(scale, true_rel, IDENT)
        H1, b1, n1, s1, counts1, costs1 = ref.odometry_coeffs(scale, true_rel, IDENT)
        assert n0 == n1 and np.array_equal(counts0, counts1)
        assert rel(H0, H1) < REL and rel(b0, b1) < REL
    from badslam_b200._lib import BadBAError
    with pytest.raises(BadBAError):
        ba.TrackFramePairwise(None, 5, *dev, IDENT, IDENT, num_scales=3)            # no such keyframe
    with pytest.raises(BadBAError):
        ba.TrackFramePairwise(None, 0, *dev, IDENT, IDENT, num_scales=9)            # too many levels
    with pytest.raises(BadBAError):
        ba.TrackFramePairwise(None, 0, *dev, IDENT, IDENT, num_scales=1, use_pyramid_level_0=False)
    with pytest.raises(BadBAError):
        ba.OdometryCoeffs(7, IDENT)                                                  # level not built
    torch.cuda.synchronize()
