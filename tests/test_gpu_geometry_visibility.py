"""The geometry kernels' per-sub-step visibility mask: one lane per keyframe of a 32-keyframe group tests the box of the sub-step's
surfels against that keyframe's view, and the warp walks only the set bits in ascending order (the activation-only kernel also
drops the keyframes that are not kActive).  Against the CPU oracle, which evaluates every (surfel, keyframe) pair:

* keyframe lists of 1, 2, 31, 32, 33 and 37 keyframes, so that the mask of a group has its first and last bits set and cleared
  and the second group holds 1 or 5 keyframes, with covisible-active keyframes at the ends of the list (the activation mask
  clears them), in depth-only, descriptor-only and combined mode;
* surfels that no keyframe can see: every mask is empty, no flag is set and no row changes.
The tolerances are those of tests/test_gpu_geometry_order.py's group-edge test.
"""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MODES = [(True, False), (False, True), (True, True)]


@pytest.fixture(scope="module")
def many_scene():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name("many"))


def run_both(sc, states, use_depth, use_desc):
    """UpdateSurfelActivation and one OptimizeGeometryIteration on the GPU and in the oracle with the given keyframe activations."""
    from badslam_b200.direct_ba import DirectBA
    from oracle import cpu_oracle
    ba = DirectBA.from_scene(sc, use_depth_residuals=use_depth, use_descriptor_residuals=use_desc)
    for k, s in states:
        ba.keyframes()[k].SetActivation(s)
    n = sc.num_surfels
    ba.UpdateSurfelActivation()
    fa = np.array(ba.GetActiveHost()[:n])
    ba.OptimizeGeometryIteration()
    rows, fg = np.array(ba.GetSurfelsHost()[:8, :n]), np.array(ba.GetActiveHost()[:n])
    orc = cpu_oracle.Oracle(sc, use_depth=use_depth, use_descriptor=use_desc)
    for k, s in states:
        orc.activation[k] = s
    orc.update_activation()
    oa = np.array(orc.active[:n])
    orc.optimize_geometry_iteration()
    return (fa, rows, fg), (oa, np.array(orc.surfels[:8, :n]), np.array(orc.active[:n]))


@pytest.mark.parametrize("use_depth,use_desc", MODES)
@pytest.mark.parametrize("listed", [1, 2, 31, 32, 33, 37])
def test_keyframe_lists_against_oracle(many_scene, listed, use_depth, use_desc):
    sc = many_scene
    K = sc.cfg.num_keyframes
    states = [(k, 2) for k in range(listed, K)]                 # inactive: not in the geometry kernels' list
    if listed > 2:
        states += [(0, 1), (listed - 1, 1)]                     # covisible-active: dropped by the activation-only mask
    if listed > 32:
        states += [(31, 1)]                                     # the last bit of the first group
    (fa, a, fg), (oa, c, og) = run_both(sc, states, use_depth, use_desc)
    n = sc.num_surfels
    assert np.array_equal(fa, oa)
    assert 0 < fa.sum() < n
    assert np.array_equal(fg, og)
    assert (a[3].view(np.uint32) != c[3].view(np.uint32)).mean() < 1e-3
    d = np.max(np.abs(a[:3] - c[:3]), axis=0)
    if use_depth:
        assert d.max() < 5e-4
    else:
        # photometric-only position updates are ill-conditioned for low-texture surfels (see test_gpu_parity.py)
        assert np.mean(d) < 2e-5 and (d > 5e-4).mean() < 0.05, (np.mean(d), (d > 5e-4).mean())
    assert np.abs(a[:3] - sc.surfels[:3, :n]).max() > 1e-4


def test_surfels_no_keyframe_sees(many_scene):
    sc = copy.copy(many_scene)
    n = sc.num_surfels
    cols = sc.surfels.copy()
    cols[0:3, :n] += 1e4                                       # far outside every keyframe's view
    sc.surfels = cols
    (fa, a, fg), (oa, c, og) = run_both(sc, [], True, True)
    assert not fa.any() and np.array_equal(fa, oa) and np.array_equal(fg, og)
    assert np.array_equal(a.view(np.uint32), cols[:8, :n].view(np.uint32))
