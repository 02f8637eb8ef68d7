"""GPU parity at the sizes bench.py measures (BASELINE.json configs 2 and 3): the sm_90a path through the C ABI against the
reference's own CUDA kernels (recorded outputs, tests/golden/ref) on the same seeded scene -- the tile sizes (TILE = 1024 at 3 M surfels), the
8-keyframe work groups of the pose kernel and the 13 keyframe groups of the geometry kernels only exist at these sizes.

Tolerances (BASELINE.json north_star): 1e-4 relative on normal-equation coefficients / residual sums, 1e-5 m / 1e-5 rad on
poses (+ the reference's own run-to-run noise: its float atomics are unordered); counts are integers and must match.
"""
import numpy as np
import pytest

from gpu_checks import REL, check_one_ba_iteration, rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mods():
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    from oracle import cpu_oracle, ref_golden
    assert ref_golden.available(), "recording needs oracle/_ref/libbadslam_ref.so (oracle/build_ref.sh)"
    return S, DirectBA, cpu_oracle, ref_golden


def check_pose_coefficients(S, ba, ref, sc, keyframes):
    for k in keyframes:
        pc = ba.AccumulatePoseEstimationCoeffs(k, sc.poses_init[k])
        H, b, cnt, cost = ref.pose_coeffs(k, sc.poses_init[k])
        assert pc.n_assoc + pc.n_photo == cnt, (k, pc.n_assoc, pc.n_photo, cnt)
        assert pc.n_pair == sc.num_surfels and pc.n_pair >= pc.n_inimg >= pc.n_depthok >= pc.n_assoc >= pc.n_photo > 0
        assert rel(pc.H[:], H) < REL and rel(pc.b[:], b) < REL, (k, rel(pc.H[:], H), rel(pc.b[:], b))
        assert abs(pc.cost_depth + pc.cost_desc1 - cost) < REL * cost, (k, pc.cost_depth + pc.cost_desc1, cost)


def test_cfg2_every_keyframe_and_one_ba_iteration(mods):
    S, DirectBA, O, R = mods
    sc = S.make_scene(S.config_by_name("cfg2"))
    ba, ref, ref2 = DirectBA.from_scene(sc), R.RefDirectBA(sc), R.RefDirectBA(sc)
    check_pose_coefficients(S, ba, ref, sc, range(sc.cfg.num_keyframes))
    check_one_ba_iteration(S, R, ba, ref, ref2, sc)


def test_cfg3_spread_keyframes_and_one_ba_iteration(mods):
    """The benchmarked workload itself: 200 keyframes x 3 M surfels.  Keyframes 0, 7, 8, 63, 100, 129, 150, 191, 192, 199 sit in
    different 8-keyframe work groups of the pose kernel (first / last slot of a group, first / middle / last group)."""
    S, DirectBA, O, R = mods
    sc = S.make_scene(S.config_by_name("cfg3"))
    ba, ref = DirectBA.from_scene(sc), R.RefDirectBA(sc)
    check_pose_coefficients(S, ba, ref, sc, (0, 7, 8, 63, 100, 129, 150, 191, 192, 199))
    ref2 = R.RefDirectBA(sc)
    check_one_ba_iteration(S, R, ba, ref, ref2, sc)


# BASELINE.json configs 4 and 5 (500 keyframes / 4 M surfels with intrinsics + depth deformation; 1280x720, 400 keyframes /
# 8 M surfels).  Scene generation alone takes minutes, so these two only run when BADBA_BIG_CONFIGS=1.  The spot check is the
# one of the benchmarked configuration: association counts, H, b and cost of four keyframes from different work groups against
# the reference's own kernels (their recorded outputs, tests/golden/ref).
import os

big = pytest.mark.skipif(not os.environ.get("BADBA_BIG_CONFIGS"), reason="set BADBA_BIG_CONFIGS=1 (minutes of scene generation)")


@big
@pytest.mark.parametrize("name", ["cfg4", "cfg5"])
def test_big_config_spot_check(mods, name):
    import torch
    S, DirectBA, O, R = mods
    sc = S.make_scene(S.config_by_name(name))
    K = sc.cfg.num_keyframes
    ba, ref = DirectBA.from_scene(sc), R.RefDirectBA(sc)
    check_pose_coefficients(S, ba, ref, sc, (0, K // 3 + 1, 2 * K // 3 + 2, K - 1))
    if name == "cfg4":
        # one intrinsics + depth-deformation step (the cfg4 flags) on both sides from the same state
        ba.OptimizeIntrinsics(True, True)
        ref.optimize_intrinsics(True, True)
        di, ci, a = ba._intrinsics()
        rdi, rci, ra = ref.intrinsics()
        # tolerances of tests/test_gpu_parity.py::test_intrinsics_step_three_way
        assert np.all(np.abs(di - rdi) < REL * np.abs(rdi) + 1e-3) and np.all(np.abs(ci - rci) < REL * np.abs(rci) + 1e-3), (di, rdi, ci, rci)
        assert abs(a - ra) < 1e-5, (a, ra)
        assert np.abs(ba.cfactor_buffer() - ref.cfactor()).max() < 1e-4
        # ... and two iterations of the cfg4 alternation itself (activation, geometry, poses, intrinsics + depth deformation)
        # from that state; tolerances of tests/test_gpu_parity.py::test_bundle_adjustment_with_intrinsics without the
        # second reference run (its noise floor is not measured here: 5x the fixed part instead)
        ba.SetLastBAIterationCount(ba.ba_iteration_count())
        ro = ba.BundleAdjustment(None, True, True, False, True, True, 2, 2, increase_ba_iteration_count=False)
        rr = ref.bundle_adjust(True, True, 2, 2, optimize_depth_intrinsics=True, optimize_color_intrinsics=True, count_residuals=False,
                               end_tasks=False)
        assert ro.iterations_done == rr.iterations_done == 2
        di, ci, a = ba._intrinsics()
        rdi, rci, ra = ref.intrinsics()
        assert np.abs(di - rdi).max() < 2.5e-2 and np.abs(ci - rci).max() < 2.5e-2, (di, rdi, ci, rci)
        assert abs(a - ra) < 0.1, (a, ra)
        worst = max(max(S.pose_error(ba.keyframes()[k].global_T_frame(), ref.pose(k))) for k in range(K))
        assert worst < 1e-3, worst
        print(f"cfg4 after 2 BA iterations with intrinsics: a {a:.5f} / reference {ra:.5f}, fx {di[0]:.4f} / {rdi[0]:.4f}, "
              f"worst pose difference {worst:.2e}")
    free, total = torch.cuda.mem_get_info()
    print(f"{name}: device memory in use {(total - free) / 2**30:.2f} GiB")
