"""The geometry step in one tile-major launch (GeometryPassKernel): activation, normals, positions and descriptors of each surfel
tile over all keyframes with the sums in registers.  It replaces the two group-major launches (ActivationNormalsKernel,
PositionDescriptorKernel) whenever no surfels were created in the iteration, and must compute what they compute bit for bit: after
alternating BA iterations run once with each path (bba_debug_set_geometry_pass), rows 0-7 of every surfel, the active flags, the
keyframe poses and activations and the residual counts are the same bits,

* on cfg2 (640x480, 20 keyframes) and on the two camera rigs whose colour camera is not the depth camera;
* on surfels placed onto the image borders and around z = 0 of some keyframes (tests/test_gpu_geometry_order.py), where the
  culling box test decides at its slack;
* at surfel counts whose last tile and last 32-surfel sub-step are partial, at every tile size, and with 37 keyframes (two
  visibility words, the second partial);
* with a fixed active-keyframe window (the flags are not re-determined) and through bba_optimize_geometry_iteration.
"""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SPLIT, ONE = 1, 2


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    return S, DirectBA


@pytest.fixture(scope="module")
def many_scene(mods):
    S, _ = mods
    return S.make_scene(S.config_by_name("many"))


def bundle_adjust(DirectBA, sc, pass_, tile_shift=0, iterations=2, window=None, **kw):
    """Alternating BA (poses and geometry, no surfel updates) with the given geometry pass: surfel rows 0-7, flags, poses,
    activations and the last iteration's result."""
    ba = DirectBA.from_scene(sc, **kw)
    ba.SetLastBAIterationCount(ba.ba_iteration_count())   # no end tasks: the surfel set stays as it is
    ba.DebugSetGeometryPass(pass_, tile_shift)
    extra = {} if window is None else dict(active_keyframe_window_start=window[0], active_keyframe_window_end=window[1])
    r = ba.BundleAdjustment(None, False, False, False, True, True, iterations, iterations, increase_ba_iteration_count=False, **extra)
    n = sc.num_surfels
    poses, act = ba.GetKeyframeStates()
    return (np.array(ba.GetSurfelsHost()[:8, :n]), np.array(ba.GetActiveHost()[:n]), np.array(poses), np.array(act),
            (r.depth_residual_count, r.descriptor_residual_count, r.pose_iterations_total, r.iterations_done))


def assert_same(a, b, sc, tag):
    rows_a, flags_a, poses_a, act_a, res_a = a
    rows_b, flags_b, poses_b, act_b, res_b = b
    assert np.array_equal(rows_a.view(np.uint32), rows_b.view(np.uint32)), (tag, int((rows_a.view(np.uint32) != rows_b.view(np.uint32)).sum()))
    assert np.array_equal(flags_a, flags_b), tag
    assert np.array_equal(poses_a.view(np.uint32), poses_b.view(np.uint32)), tag
    assert np.array_equal(act_a, act_b) and res_a == res_b, (tag, res_a, res_b)
    n = sc.num_surfels
    assert 0 < flags_a.sum() <= n, tag
    assert np.abs(rows_a[:3] - sc.surfels[:3, :n]).max() > 1e-5, tag   # the step moved surfels


@pytest.mark.parametrize("name", ["cfg2", "rig_half", "rig_same"])
def test_one_launch_equals_two_launches(mods, name):
    S, DirectBA = mods
    sc = S.make_scene(S.config_by_name(name))
    assert_same(bundle_adjust(DirectBA, sc, SPLIT), bundle_adjust(DirectBA, sc, ONE), sc, name)


@pytest.mark.parametrize("use_depth,use_desc", [(True, False), (False, True), (True, True)])
def test_border_surfels(mods, many_scene, use_depth, use_desc):
    from test_gpu_geometry_order import border_scene
    S, DirectBA = mods
    sc = border_scene(S, many_scene)
    kw = dict(use_depth_residuals=use_depth, use_descriptor_residuals=use_desc)
    assert_same(bundle_adjust(DirectBA, sc, SPLIT, **kw), bundle_adjust(DirectBA, sc, ONE, **kw), sc, (use_depth, use_desc))


@pytest.mark.parametrize("n", [1, 33, 4000, 23_999])
@pytest.mark.parametrize("tile_shift", [5, 6, 7, 8])
def test_partial_tiles_at_every_tile_size(mods, many_scene, n, tile_shift):
    S, DirectBA = mods
    sc = copy.copy(many_scene)   # 37 keyframes: the second visibility word holds 5
    sc.num_surfels = n
    split = bundle_adjust(DirectBA, sc, SPLIT, iterations=1)
    one = bundle_adjust(DirectBA, sc, ONE, tile_shift, iterations=1)
    rows_a, flags_a, poses_a, _, res_a = split
    rows_b, flags_b, poses_b, _, res_b = one
    assert np.array_equal(rows_a.view(np.uint32), rows_b.view(np.uint32)) and np.array_equal(flags_a, flags_b), (n, tile_shift)
    assert np.array_equal(poses_a.view(np.uint32), poses_b.view(np.uint32)) and res_a == res_b, (n, tile_shift)


def test_fixed_keyframe_window(mods, many_scene):
    """Keyframes 4..30 active, the others inactive: the flags are set, not determined, and the keyframe list skips some ids."""
    S, DirectBA = mods
    sc = many_scene
    assert_same(bundle_adjust(DirectBA, sc, SPLIT, window=(4, 30)), bundle_adjust(DirectBA, sc, ONE, window=(4, 30)), sc, "window")


def test_standalone_geometry_iteration(mods, many_scene):
    S, DirectBA = mods
    sc = many_scene
    out = []
    for pass_ in (SPLIT, ONE):
        ba = DirectBA.from_scene(sc)
        ba.DebugSetGeometryPass(pass_)
        ba.keyframes()[1].SetActivation(2)
        ba.keyframes()[2].SetActivation(1)
        ba.UpdateSurfelActivation()
        for _ in range(2):
            ba.OptimizeGeometryIteration()
        out.append((np.array(ba.GetSurfelsHost()[:8, :sc.num_surfels]), np.array(ba.GetActiveHost()[:sc.num_surfels])))
    assert np.array_equal(out[0][0].view(np.uint32), out[1][0].view(np.uint32)) and np.array_equal(out[0][1], out[1][1])
    assert np.abs(out[1][0][:3] - sc.surfels[:3, :sc.num_surfels]).max() > 1e-5


def test_the_switch_rejects_unknown_values(mods, many_scene):
    S, DirectBA = mods
    ba = DirectBA.from_scene(copy.copy(many_scene))
    for pass_, shift in ((3, 0), (-1, 0), (0, 4), (0, 9)):
        with pytest.raises(Exception):
            ba.DebugSetGeometryPass(pass_, shift)
    ba.DebugSetGeometryPass(0, 0)
