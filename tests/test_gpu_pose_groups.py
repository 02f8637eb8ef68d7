"""GPU: the number of keyframes that share one staged surfel tile in the pose kernel (PoseAccumulateArgs::group, forced with
bba_debug_set_pose_group) decides only which (keyframe, chunk) sub-items are dealt out together, never what a sub-item computes.
So in the deterministic mode every record is the same bits at every group size, and in the default mode only the order of the
fp64 atomics changes: each group size stays within the (n + 1) 2^-53 bound of test_gpu_deterministic_values.py of its own
deterministic result.

On `many` (37 keyframes) every group size below 37 leaves a ragged last group; the work lists of 4, 3 and 1 keyframes lie on both
sides of the chunk-size rule (256-surfel chunks from 4 listed keyframes, 128 below).
"""
import copy

import numpy as np
import pytest

from test_gpu_deterministic_values import compare_pose_records, in_mode
from test_gpu_work_groups import distinct_poses

pytestmark = [pytest.mark.gpu]

GROUPS = (8, 16, 32, 64, 0)   # 0: the library's choice (32 on the sorted stream that a forced PRE variant stages)


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import _lib
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    return S, DirectBA, _lib


@pytest.fixture(scope="module")
def many():
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name("many"))


def same_bits(a, b):
    return all(np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8)) for x, y in zip(a, b))


@pytest.mark.parametrize("surfels", [None, 20_001])
def test_pose_records_do_not_depend_on_the_group(mods, many, surfels):
    """Both PRE instantiations, with and without stats, on work lists of 37 / 4 / 3 / 1 keyframes, at every group size."""
    S, DirectBA, L = mods
    sc = copy.copy(many)
    if surfels is not None:
        sc.num_surfels = surfels
    K = sc.cfg.num_keyframes
    poses = distinct_poses(S, sc)
    ba = DirectBA.from_scene(sc)
    deposits = -(-sc.num_surfels // 128)
    lists = {"all": np.random.default_rng(37).permutation(K), "four": [36, 0, 8, 17], "three": [17, 8, 0], "one": [16]}
    try:
        for v in (L.POSE_VARIANT_256_PRE, L.POSE_VARIANT_512_PRE):
            for lname, ids in lists.items():
                ids = np.asarray(ids)
                costs = None
                for with_stats in (True, False):   # (the costs of the first bound b in both)
                    call = lambda: ba.PoseCoeffsBatch(ids, poses[ids], v, with_stats)
                    reference = None
                    for g in GROUPS:
                        ba.DebugSetPoseGroup(g)
                        tag = (sc.num_surfels, int(v), lname, with_stats, g)
                        det, dflt = in_mode(ba, True, call), call()
                        assert dflt[2][ids, 2].sum() > 0, tag
                        if reference is None:
                            reference = det
                            costs = det[3] if with_stats else costs
                        else:
                            assert same_bits(det, reference), tag
                        compare_pose_records(det, dflt, costs, deposits, tag, True, listed=set(ids.tolist()))
    finally:
        ba.DebugSetPoseGroup(0)


def test_group_out_of_range_is_rejected(mods, many):
    from badslam_b200.direct_ba import BadBAError
    S, DirectBA, L = mods
    ba = DirectBA.from_scene(many)
    for g in (-1, 65):
        with pytest.raises(BadBAError):
            ba.DebugSetPoseGroup(g)


def test_one_deterministic_ba_iteration_at_every_group(mods, many):
    """One deterministic BA iteration (poses only) on `many` with the group forced to 8, left to the library (8 there: 37 x 24 k
    pairs stay below the sort rule, so the pose step stages the caller's order) and forced to 32: the same bits."""
    S, DirectBA, L = mods
    out = []
    for g in (8, 0, 32):
        ba = DirectBA.from_scene(many)
        ba.SetDeterministic(True)
        ba.DebugSetPoseGroup(g)
        r = ba.BundleAdjustment(None, False, False, False, True, False, 1, 1)
        poses, activations = ba.GetKeyframeStates()
        out.append((r, poses, activations))
    (r0, p0, a0) = out[0]
    assert r0.pose_iterations_total > many.cfg.num_keyframes
    for g, (r, p, a) in zip((0, 32), out[1:]):
        assert (r.iterations_done, r.converged, r.pose_iterations_total, r.depth_residual_count, r.descriptor_residual_count) == \
            (r0.iterations_done, r0.converged, r0.pose_iterations_total, r0.depth_residual_count, r0.descriptor_residual_count), g
        assert r.cost == r0.cost, g
        assert same_bits((p, a), (p0, a0)), g
