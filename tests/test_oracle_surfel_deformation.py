"""CPU: the properties of the surfel deformation's oracle (tests/surfel_deform_oracle.py, DESIGN.md §3.13) on the tiny and small
scenes, and its association test against the C oracle's (orc_pair_residuals bit 0) away from the thresholds.

* identity: with the original poses the inverses of the current ones, nothing moves and every row keeps its bits;
* rigid: when every keyframe moves by one G, every surfel -- the ones without a voter included -- lands at G p and its normal
  at R_G n;
* halves: when the keyframes >= K/2 move by E, the surfels whose voters all moved land at E p and the ones whose voters all
  stayed keep their bits;
* the result of a surfel does not depend on the order of the surfels."""
import numpy as np
import pytest

import surfel_deform_oracle as D

_CACHE = {}


def _scene(name):
    if name not in _CACHE:
        from badslam_b200.scene import config_by_name, make_scene
        _CACHE[name] = make_scene(config_by_name(name))
    return _CACHE[name]


def _inverse(A):
    from oracle.cpu_oracle import se3_inverse
    return se3_inverse(A)


def _compose(A, B):
    from oracle.cpu_oracle import se3_mul
    return se3_mul(A, B)


def _run(sc, current, original):
    inv = np.stack([_inverse(p) for p in current])
    return D.deform_surfels(D.Camera.of_scene(sc), sc.depth, sc.normals, sc.surfels, sc.num_surfels, current, original, inv)


def _G():
    from oracle.cpu_oracle import se3_exp
    return se3_exp(np.array([0.2, -0.15, 0.16, 0.2, -0.2, 0.22], np.float32))   # about 0.3 m and 20 degrees


def _apply(G, p):
    R = D._rot64(G[:4])
    return R @ p.astype(np.float64) + np.asarray(G[4:], np.float64)[:, None]


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_identity(name):
    sc = _scene(name)
    cur = sc.poses_init
    original = np.stack([_inverse(p) for p in cur])
    out, moved, unobserved, voters, _ = _run(sc, cur, original)
    assert moved == 0
    assert out.tobytes() == np.asarray(sc.surfels, np.float32).tobytes()
    assert voters.any(axis=1).mean() > 0.9   # the scene's surfels are observed by the keyframes that made them


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_rigid(name):
    sc = _scene(name)
    n = sc.num_surfels
    G = _G()
    original = np.stack([_inverse(p) for p in sc.poses_init])
    cur = np.stack([_compose(G, p) for p in sc.poses_init])
    out, moved, unobserved, voters, _ = _run(sc, cur, original)
    assert moved == n
    assert unobserved == int((~voters.any(axis=1)).sum())
    np.testing.assert_allclose(out[:3, :n], _apply(G, sc.surfels[:3, :n]), atol=1e-5)
    n_old = D.unpack_normal(sc.surfels[3, :n]).astype(np.float64)
    expect = D.pack_normal((D._rot64(G[:4]) @ n_old).astype(np.float32)).view(np.uint32)
    got = out[3, :n].view(np.uint32)
    steps = np.stack([np.abs(((got >> s) & 0x3ff).astype(np.int32) - ((expect >> s) & 0x3ff).astype(np.int32)) % 1022 for s in (0, 10, 20)])
    assert steps.max() <= 1


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_halves(name):
    sc = _scene(name)
    n = sc.num_surfels
    K = len(sc.poses_init)
    E = _G()
    original = np.stack([_inverse(p) for p in sc.poses_init])
    cur = np.array(sc.poses_init, np.float32, copy=True)
    for k in range(K // 2, K):
        cur[k] = _compose(E, cur[k])
    out, moved, unobserved, voters, _ = _run(sc, cur, original)
    observed = voters.any(axis=1)
    all_moved = observed & ~voters[:, :K // 2].any(axis=1)
    all_still = observed & ~voters[:, K // 2:].any(axis=1)
    assert all_moved.sum() > n // 50 and all_still.sum() > n // 50
    np.testing.assert_allclose(out[:3, :n][:, all_moved], _apply(E, sc.surfels[:3, :n])[:, all_moved], atol=1e-5)
    assert out[:4, :n][:, all_still].tobytes() == np.asarray(sc.surfels[:4, :n][:, all_still], np.float32).tobytes()
    assert out[4:, :n].tobytes() == np.asarray(sc.surfels[4:, :n], np.float32).tobytes()
    assert int(all_moved.sum()) <= moved <= n - int(all_still.sum())


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_surfel_order(name):
    sc = _scene(name)
    n = sc.num_surfels
    K = len(sc.poses_init)
    original = np.stack([_inverse(p) for p in sc.poses_init])
    cur = np.array(sc.poses_init, np.float32, copy=True)
    for k in range(K // 2, K):
        cur[k] = _compose(_G(), cur[k])
    out, moved, unobserved, _, margin = _run(sc, cur, original)
    perm = np.random.default_rng(5).permutation(n)
    shuffled = np.array(sc.surfels, np.float32, copy=True)
    shuffled[:, :n] = sc.surfels[:, perm]
    cam = D.Camera.of_scene(sc)
    inv = np.stack([_inverse(p) for p in cur])
    out2, moved2, unobserved2, _, margin2 = D.deform_surfels(cam, sc.depth, sc.normals, shuffled, n, cur, original, inv)
    assert (moved2, unobserved2) == (moved, unobserved)
    assert out2[:, :n].tobytes() == out[:, perm].tobytes()
    assert np.array_equal(margin2, margin[perm])


def test_association_against_c_oracle():
    """The fp32 association of the numpy oracle equals orc_pair_residuals' on every pair of the tiny scene away from a
    threshold."""
    from oracle.cpu_oracle import Oracle
    sc = _scene("tiny")
    O = Oracle(sc)
    cam = D.Camera.of_scene(sc)
    n = sc.num_surfels
    p = sc.surfels[:3, :n]
    nrm = D.unpack_normal(sc.surfels[3, :n])
    checked = 0
    for k in range(len(sc.poses_init)):
        T = D.quat_to_matrix_f32(_inverse(sc.poses_init[k]))
        assoc, margin = D.associate(cam, T, sc.depth[k], sc.normals[k], p, nrm)
        for i in np.flatnonzero(margin > 1e-3)[::7]:
            flags, *_ = O.pair_residuals(k, sc.surfels[:8, i])
            assert bool(flags & 1) == bool(assoc[i]), (k, i)
            checked += 1
    assert checked > 1000
