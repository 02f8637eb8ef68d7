"""The geometry step's spatial order: both geometry kernels visit the surfels sorted by their Morton code (the standalone entry
points always sort) and skip, per 32-surfel warp step, every keyframe whose view the box of the warp's surfels misses.  Neither
may change what is computed:

* on surfels hand-placed onto the image borders and around the plane z = 0 of a keyframe, where the box test decides at its
  slack, the activation flags, rows 0-7 and flags after one geometry iteration equal bit for bit those of the previous kernels
  (caller order, no culling), in depth-only, descriptor-only and combined mode.  tests/golden/geometry_order_border.npz holds
  them for every placed surfel and a seeded sample of the scene's own, recorded with those kernels (commit 5e2691d) through
  activation_and_geometry() below by tools/record_geometry_order_border.py, which documents the command.  (The reference's
  kernels decide a few of the placed surfels differently, before and after this change: their projection rounds differently
  exactly on the borders);
* at the edges of the geometry kernels' 32-keyframe groups (covisible-active keyframes in the last and first slot of a group, an
  inactive one dropped from the list) against the CPU oracle;
* against the reference's kernels (recorded outputs) at ragged surfel counts (a sub-step with 1, 31 or 33 live lanes, a partial
  last tile): activation flags and packed normals exactly, positions and descriptors as in tests/test_gpu_parity.py;
* every surfel sums the same pairs in the same order whatever order the caller keeps its surfels in: shuffled columns give the
  same rows and flags, permuted, bit for bit.
"""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MODES = [(True, False), (False, True), (True, True)]


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    from oracle import ref_golden
    assert ref_golden.available(), "recording needs oracle/_ref/libbadslam_ref.so (oracle/build_ref.sh)"
    return S, DirectBA, ref_golden


@pytest.fixture(scope="module")
def many_scene():
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name("many"))


def with_surfels(sc, cols, n):
    """A copy of the scene whose surfel buffer holds the first n of the [17, m] columns cols."""
    out = copy.copy(sc)
    pitch = (n + 127) // 128 * 128
    buf = np.zeros((cols.shape[0], pitch), np.float32)
    buf[:, :n] = cols[:, :n]
    out.surfels = buf
    out.num_surfels = n
    return out


def border_scene(S, sc):
    """The scene plus, for keyframes 0, 17 and 36, surfels on, just inside and just beyond each image border and around z = 0 of
    the keyframe's camera frame (normals, radii and descriptors copied from existing surfels)."""
    from test_gpu_spatial_order import border_surfels
    rng = np.random.default_rng(91)
    n0 = sc.num_surfels
    cols = [sc.surfels[:, :n0]]
    for k in (0, 17, 36):
        pos = border_surfels(S, sc, k, rng)
        extra = sc.surfels[:, rng.integers(0, n0, pos.shape[1])].copy()
        extra[0:3] = pos
        cols.append(extra)
    cols = np.concatenate(cols, axis=1)
    return with_surfels(sc, cols, cols.shape[1])


def activation_and_geometry(DirectBA, sc, use_depth, use_desc, activations=((1, 2), (2, 1)), prepare=None, **kw):
    """UpdateSurfelActivation and one OptimizeGeometryIteration with the given (keyframe, activation) states (default: keyframe 1
    inactive, keyframe 2 covisible-active): the flags after the activation, and rows 0-7 and the flags after the geometry
    iteration.  kw go to DirectBA.from_scene; prepare(ba) runs before the first call (multi-rank set-up)."""
    ba = DirectBA.from_scene(sc, use_depth_residuals=use_depth, use_descriptor_residuals=use_desc, **kw)
    if prepare is not None:
        prepare(ba)
    for k, a in activations:
        ba.keyframes()[k].SetActivation(a)
    n = sc.num_surfels
    ba.UpdateSurfelActivation()
    flags = np.array(ba.GetActiveHost()[:n])
    ba.OptimizeGeometryIteration()
    return flags, np.array(ba.GetSurfelsHost()[:8, :n]), np.array(ba.GetActiveHost()[:n])


def reference(R, sc, use_depth, use_desc, activations=((1, 2), (2, 1))):
    ref = R.RefDirectBA(sc, use_depth, use_desc)
    for k, a in activations:
        ref.set_activation(k, a)
    ref.update_activation()
    flags = np.array(ref.active())
    ref.optimize_geometry_iteration()
    return flags, np.array(ref.surfels()), np.array(ref.active())


def check_against_reference(R, sc, ours, ref, use_depth, use_desc, tag):
    fa, a, fa2 = ours
    fr, b_, fr2 = ref
    assert R.equal(fa, fr) and R.equal(fa2, fr2), tag
    assert R.equal(a[3].view(np.uint32), b_[3].view(np.uint32)), tag          # packed normals
    assert np.array_equal(a[4:6].view(np.uint32), sc.surfels[4:6, :sc.num_surfels].view(np.uint32)), tag   # radius / colour
    d = np.max(np.abs(a[:3] - b_[:3]), axis=0)
    if use_depth:
        assert d.max() < 2e-6, (tag, d.max())
    else:
        # photometric-only position updates are ill-conditioned for low-texture surfels (see test_gpu_parity.py)
        assert np.mean(d) < 2e-6 and (d > 2e-6).mean() < 0.1 and d.max() < 2e-3, (tag, np.mean(d), d.max())
    if use_desc:
        assert np.max(np.abs(a[6:8] - b_[6:8])) < 2e-3, tag
    else:
        assert np.array_equal(a[6:8].view(np.uint32), sc.surfels[6:8, :sc.num_surfels].view(np.uint32)), tag


@pytest.mark.parametrize("use_depth,use_desc", MODES)
def test_border_surfels_match_the_caller_order_kernels(mods, many_scene, use_depth, use_desc):
    import os
    S, DirectBA, R = mods
    sc = border_scene(S, many_scene)
    fa, rows, fg = activation_and_geometry(DirectBA, sc, use_depth, use_desc)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "geometry_order_border.npz")
    mode = f"{int(use_depth)}{int(use_desc)}"
    with np.load(path) as z:
        cols = z["columns"]
        assert np.array_equal(fa[cols], z[mode + "_flags_act"])
        assert np.array_equal(rows[:, cols].view(np.uint32), z[mode + "_rows"].view(np.uint32))
        assert np.array_equal(fg[cols], z[mode + "_flags"])
    placed = fa[many_scene.num_surfels:]
    assert 0 < placed.sum() < placed.size   # the placed surfels reach the decisions: some are seen, not all of them
    assert np.abs(rows[:3] - sc.surfels[:3, :sc.num_surfels]).max() > 1e-4   # the step did something


@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 257])
def test_ragged_surfel_counts_against_reference(mods, many_scene, n):
    S, DirectBA, R = mods
    sc = copy.copy(many_scene)
    sc.num_surfels = n
    ours = activation_and_geometry(DirectBA, sc, True, True)
    ref = reference(R, sc, True, True)
    check_against_reference(R, sc, ours, ref, True, True, f"{n} surfels")


def test_geometry_group_edges_against_oracle(mods, many_scene):
    """37 keyframes, 5 and 36 inactive: the keyframe list holds 35, keyframes 32 / 33 are the last of the first group and the first
    of the second, both covisible-active (normals only, no activation).  Against the CPU oracle with the tolerances of
    tests/test_gpu_work_groups.py (the reference's activation kernel decides some surfels differently in this set-up, before and
    after this change)."""
    from oracle import cpu_oracle
    S, DirectBA, R = mods
    sc = many_scene
    states = ((5, 2), (32, 1), (33, 1), (36, 2))
    fa, a, fg = activation_and_geometry(DirectBA, sc, True, True, activations=states)
    orc = cpu_oracle.Oracle(sc)
    for k, s in states:
        orc.activation[k] = s
    orc.update_activation()
    n = sc.num_surfels
    assert np.array_equal(fa, orc.active[:n])
    assert 0 < fa.sum() < n
    orc.optimize_geometry_iteration()
    c = orc.surfels[:8, :n]
    assert np.array_equal(fg, orc.active[:n])
    assert np.max(np.abs(a[:3] - c[:3])) < 5e-4 and (a[3].view(np.uint32) != c[3].view(np.uint32)).mean() < 1e-3
    assert np.abs(a[:3] - sc.surfels[:3, :n]).max() > 1e-4


@pytest.mark.parametrize("use_depth,use_desc", MODES)
def test_results_do_not_depend_on_the_callers_surfel_order(mods, many_scene, use_depth, use_desc):
    S, DirectBA, R = mods
    sc = border_scene(S, many_scene)
    n = sc.num_surfels
    perm = np.random.default_rng(6).permutation(n)
    shuffled = with_surfels(sc, sc.surfels[:, :n][:, perm], n)
    f0, rows0, g0 = activation_and_geometry(DirectBA, sc, use_depth, use_desc)
    f1, rows1, g1 = activation_and_geometry(DirectBA, shuffled, use_depth, use_desc)
    assert np.array_equal(f0[perm], f1) and np.array_equal(g0[perm], g1)
    assert np.array_equal(rows0[:, perm].view(np.uint32), rows1.view(np.uint32))
    assert 0 < f0.sum() < n
