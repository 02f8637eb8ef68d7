"""CPU: the properties of the keyframe co-visibility oracle (tests/covisibility_oracle.py, DESIGN.md §3.19) on the tiny and small
scenes: C is symmetric, no pair shares more surfels than either keyframe observes, duplicated keyframes give equal rows, deleted
surfels count nowhere, and the diagonal is the voter count of the surfel deformation's oracle at identity changes."""
import numpy as np
import pytest

import covisibility_oracle as O
import surfel_deform_oracle as D

_CACHE = {}


def _scene(name):
    if name not in _CACHE:
        from badslam_b200.scene import config_by_name, make_scene
        _CACHE[name] = make_scene(config_by_name(name))
    return _CACHE[name]


def _inverses(poses):
    from oracle.cpu_oracle import se3_inverse
    return np.stack([se3_inverse(p) for p in poses]).astype(np.float32)


def _measure(sc, keyframes=None, surfels=None):
    ks = list(range(sc.cfg.num_keyframes)) if keyframes is None else list(keyframes)
    s = sc.surfels if surfels is None else surfels
    return O.covisibility(D.Camera.of_scene(sc), [sc.depth[k] for k in ks], [sc.normals[k] for k in ks], s, sc.num_surfels,
                          _inverses([sc.poses_init[k] for k in ks]))


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_symmetric_and_bounded(name):
    C, near, A, _ = _measure(_scene(name))
    assert np.array_equal(C, C.T) and np.array_equal(near, near.T)
    d = np.diag(C)
    assert (C <= np.minimum(d[:, None], d[None, :])).all()
    assert np.array_equal(d, A.sum(axis=0))
    assert (d > 0).all()
    # evidence: near-threshold surfels are a small share of the pairs' counts
    assert near.sum() <= 0.01 * C.sum(), (near.sum(), C.sum())


def test_duplicated_keyframes_give_equal_rows():
    sc = _scene("tiny")
    K = sc.cfg.num_keyframes
    ks = list(range(K)) + [0, K - 1]
    C, _, _, _ = _measure(sc, ks)
    assert np.array_equal(C[K], C[0]) and np.array_equal(C[K + 1], C[K - 1])
    assert C[0, K] == C[0, 0] and C[K - 1, K + 1] == C[K - 1, K - 1]


def test_deleted_surfels_count_nowhere():
    sc = _scene("tiny")
    C, _, A, _ = _measure(sc)
    s = np.array(sc.surfels, np.float32, copy=True)
    gone = np.flatnonzero(A.any(axis=1))[::3]
    s[0, gone] = np.nan
    C2, _, A2, _ = _measure(sc, surfels=s)
    assert not A2[gone].any()
    Ai = A.astype(np.int64)
    Ai[gone] = 0
    assert np.array_equal(C2, Ai.T @ Ai)


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_diagonal_is_the_deformation_voter_count(name):
    sc = _scene(name)
    C, _, _, _ = _measure(sc)
    cur = np.asarray(sc.poses_init, np.float32)
    inv = _inverses(cur)
    _, moved, _, voters, _ = D.deform_surfels(D.Camera.of_scene(sc), sc.depth, sc.normals, sc.surfels, sc.num_surfels, cur, inv, inv)
    assert moved == 0
    assert np.array_equal(np.diag(C), voters.sum(axis=0))
