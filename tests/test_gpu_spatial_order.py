"""The pose step's spatial order: the PRE instantiations of the pose kernel read the surfels sorted by their Morton code and skip
(keyframe, chunk) pairs whose chunk box lies outside the keyframe's view.  Neither may change what is computed:

* culling is exact -- the per-keyframe stage counts equal those of a non-PRE instantiation, which projects every pair, also on
  surfels hand-placed onto the image borders and around the plane z = 0 of a keyframe;
* results do not depend on the order the caller keeps its surfels in;
* ragged surfel counts (the sort of one surfel, a partial last chunk, a tile with fewer than 32 lanes live).
"""
import copy

import numpy as np
import pytest

from gpu_checks import rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import _lib
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    return S, DirectBA, _lib


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


def border_surfels(S, sc, k, rng, group=300):
    """Positions that keyframe k (at poses_init) sees on, just inside and just beyond each image border, and around z = 0 of its
    camera frame; [3, 6 * group], one spatially compact group per border and one for z = 0."""
    W, H = sc.cfg.width, sc.cfg.height
    fx, fy, cx, cy = [float(v) for v in sc.depth_K]
    R = S.quat_to_R(sc.poses_init[k][:4]).astype(np.float64)
    t = sc.poses_init[k][4:].astype(np.float64)
    offsets = np.array([0.0, 1e-4, -1e-4, 1e-3, -1e-3, 0.25, -0.25, -0.5, -0.99, -1.0, -1.01, -1.5])
    zc = rng.uniform(float(sc.min_depth[k]), float(sc.max_depth[k]), group)
    groups = []
    along_x, along_y = rng.uniform(0, W, group), rng.uniform(0, H, group)
    off = rng.choice(offsets, group)
    for px, py in ((0.0 + off, along_y), (W - 1e-3 - off, along_y), (along_x, 0.0 + off), (along_x, H - 1e-3 - off)):
        groups.append(np.stack([(px - cx) / fx * zc, (py - cy) / fy * zc, zc]))
    # around the camera plane: z of either sign down to 1e-6 m, x / y within a metre
    z0 = rng.choice([1e-6, -1e-6, 1e-4, -1e-4, 1e-2, -1e-2, 0.0], group)
    groups.append(np.stack([rng.uniform(-1, 1, group), rng.uniform(-1, 1, group), z0]))
    # a near-degenerate group: every surfel on the left border plane at px = 0 exactly (in fp64), spread in depth
    groups.append(np.stack([(0.0 - cx) / fx * zc, (along_y - cy) / fy * zc, zc]))
    local = np.concatenate(groups, axis=1)
    return (R @ local + t[:, None]).astype(np.float32)


def check_same(ba, ids, poses, variants, reference_variant, tag):
    """Every PRE variant against the non-PRE reference_variant: stage counts exact, H / b to 1e-5 (other fp32 chunk partials)."""
    H0, b0, c0, _ = ba.PoseCoeffsBatch(ids, poses[ids], reference_variant, with_stats=True)
    for v in variants:
        for stats in (True, False):
            H, b, c, _ = ba.PoseCoeffsBatch(ids, poses[ids], v, with_stats=stats)
            for k in ids:
                want = tuple(c0[k]) if stats else (0, 0, c0[k][2], c0[k][3])
                assert tuple(c[k]) == want, (tag, v, stats, int(k), c[k], c0[k])
                assert rel(H[k], H0[k]) < 1e-5 and rel(b[k], b0[k]) < 1e-5, (tag, v, int(k), rel(H[k], H0[k]), rel(b[k], b0[k]))
    return c0


def test_culling_is_exact_at_image_borders_and_z0(mods, many_scene):
    S, DirectBA, L = mods
    sc = many_scene
    K = sc.cfg.num_keyframes
    rng = np.random.default_rng(90)
    n0 = sc.num_surfels
    cols = [sc.surfels[:, :n0]]
    for k in (0, 17, 36):
        pos = border_surfels(S, sc, k, rng)
        extra = sc.surfels[:, rng.integers(0, n0, pos.shape[1])].copy()   # normals, radii, descriptors of existing surfels
        extra[0:3] = pos
        cols.append(extra)
    cols = np.concatenate(cols, axis=1)
    scb = with_surfels(sc, cols, cols.shape[1])
    ids = np.arange(K)
    poses = sc.poses_init
    pre = (L.POSE_VARIANT_256_PRE, L.POSE_VARIANT_512_PRE)
    base = check_same(DirectBA.from_scene(sc), ids, poses, pre, L.POSE_VARIANT_256, "scene")
    counts = check_same(DirectBA.from_scene(scb), ids, poses, pre, L.POSE_VARIANT_256, "with border surfels")
    placed = cols.shape[1] - n0
    for k in (0, 17, 36):   # the placed surfels do reach the decisions: some project into the image, and not all of them
        added = int(counts[k][0]) - int(base[k][0])
        assert 0 < added < placed, (k, added, placed)
    # short work lists take 128-surfel sub-chunks of the 256-surfel boxes
    check_same(DirectBA.from_scene(scb), np.array([0, 17, 36]), poses, pre, L.POSE_VARIANT_256, "three keyframes")


@pytest.mark.parametrize("n", [1, 255, 256, 257, 513])
def test_culling_is_exact_at_ragged_surfel_counts(mods, many_scene, n):
    S, DirectBA, L = mods
    sc = copy.copy(many_scene)
    sc.num_surfels = n
    ba = DirectBA.from_scene(sc)
    K = sc.cfg.num_keyframes
    counts = check_same(ba, np.arange(K), sc.poses_init, (L.POSE_VARIANT_256_PRE, L.POSE_VARIANT_512_PRE), L.POSE_VARIANT_256,
                        f"{n} surfels")
    assert n == 1 or counts[:, 0].sum() > 0


def test_results_do_not_depend_on_the_callers_surfel_order(mods, many_scene):
    """One alternating BA iteration (geometry, then the pose step in its PRE instantiation) on the scene and on the same scene with
    its surfel columns shuffled: poses to 1e-6, geometry rows and active flags bit for bit, permuted the same way."""
    import torch
    S, DirectBA, L = mods
    sc = many_scene
    n = sc.num_surfels
    perm = np.random.default_rng(5).permutation(n)
    shuffled = with_surfels(sc, sc.surfels[:, :n][:, perm], n)

    def one_iteration(scene):
        ba = DirectBA.from_scene(scene)
        ba.SetLastBAIterationCount(ba.ba_iteration_count())
        res = ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, increase_ba_iteration_count=False)
        torch.cuda.synchronize()
        poses, act = ba.GetKeyframeStates()
        return res, np.asarray(poses), np.asarray(act), ba.GetSurfelsHost(), ba.GetActiveHost()

    # the forced PRE variants always sort (the BA pose step sorts only from 16 M pairs per launch, `many` has 0.9 M)
    ids = np.arange(sc.cfg.num_keyframes)
    for v in (L.POSE_VARIANT_256_PRE, L.POSE_VARIANT_512_PRE):
        H0, b0, c0, _ = DirectBA.from_scene(sc).PoseCoeffsBatch(ids, sc.poses_init, v)
        H1, b1, c1, _ = DirectBA.from_scene(shuffled).PoseCoeffsBatch(ids, sc.poses_init, v)
        assert np.array_equal(c0, c1), v
        for k in ids:
            assert rel(H1[k], H0[k]) < 1e-5 and rel(b1[k], b0[k]) < 1e-5, (v, int(k), rel(H1[k], H0[k]), rel(b1[k], b0[k]))
    r0, p0, a0, rows0, f0 = one_iteration(sc)
    r1, p1, a1, rows1, f1 = one_iteration(shuffled)
    assert r0.depth_residual_count == r1.depth_residual_count and r0.descriptor_residual_count == r1.descriptor_residual_count
    assert r0.depth_residual_count > 0
    for k in range(sc.cfg.num_keyframes):
        dt, dr = S.pose_error(p0[k], p1[k])
        assert dt < 1e-6 and dr < 1e-6, (k, dt, dr)
    assert np.array_equal(a0, a1)
    assert np.array_equal(rows0[:, :n][:, perm].view(np.uint32), rows1[:, :n].view(np.uint32))
    assert np.array_equal(f0[:n][perm], f1[:n])
