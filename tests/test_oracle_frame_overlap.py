"""CPU: the properties of the frame overlap oracle (tests/frame_overlap_oracle.py, DESIGN.md §3.20) on the tiny and small scenes: a
query made of keyframe k's images at k's pose reproduces row k of the co-visibility oracle, new <= uncovered <= valid, a frame that
sees no surfel leaves every valid cell uncovered, and deleted surfels count nowhere."""
import numpy as np
import pytest

import covisibility_oracle as CO
import frame_overlap_oracle as O
import surfel_deform_oracle as D

_CACHE = {}


def _scene(name):
    if name not in _CACHE:
        from badslam_b200.scene import config_by_name, make_scene
        _CACHE[name] = make_scene(config_by_name(name))
    return _CACHE[name]


def _measure(sc, k, pose=None, surfels=None, min_obs=2):
    """Keyframe k's images at `pose` (k's own by default), filtered against every keyframe."""
    from badslam_b200.scene import se3_inverse, se3_mul
    pose = np.asarray(sc.poses_init[k] if pose is None else pose, np.float32)
    covis = [(D.quat_to_matrix_f32(se3_mul(se3_inverse(sc.poses_init[b]), pose).astype(np.float32)), sc.depth[b], sc.normals[b])
             for b in range(sc.cfg.num_keyframes)]
    inv = [se3_inverse(p).astype(np.float32) for p in sc.poses_init]
    return O.frame_overlap(D.Camera.of_scene(sc), sc.depth[k], sc.normals[k], se3_inverse(pose).astype(np.float32),
                           sc.surfels if surfels is None else surfels, sc.num_surfels, covis, min_obs,
                           keyframes=(list(sc.depth), list(sc.normals), np.stack(inv)))


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_a_keyframe_reproduces_its_covisibility_row(name):
    from oracle.cpu_oracle import se3_inverse
    sc = _scene(name)
    inv = np.stack([se3_inverse(p) for p in sc.poses_init]).astype(np.float32)
    C, _, _, _ = CO.covisibility(D.Camera.of_scene(sc), sc.depth, sc.normals, sc.surfels, sc.num_surfels, inv)
    for k in range(sc.cfg.num_keyframes):
        r = _measure(sc, k)
        assert np.array_equal(r["shared"], C[k]), k
        assert r["observed"] == C[k, k] > 0
        assert r["new"] <= r["uncovered"] <= r["valid"]
        assert r["uncovered"] < r["valid"]   # the map covers part of its own keyframe
        assert r["near_observed"] <= 0.01 * r["observed"] + 2


def test_a_frame_that_sees_nothing_is_all_uncovered():
    from badslam_b200.scene import se3_exp, se3_mul
    sc = _scene("tiny")
    far = se3_mul(se3_exp([0, 0, 50.0, 0, 0, 0]), sc.poses_init[0]).astype(np.float32)
    r = _measure(sc, 0, pose=far)
    assert r["observed"] == 0 and not r["shared"].any()
    assert r["uncovered"] == r["valid"] > 0
    assert r["new"] <= r["uncovered"]


def test_the_filter_only_removes():
    sc = _scene("small")
    loose, strict = _measure(sc, 1, min_obs=1), _measure(sc, 1, min_obs=1000)
    assert loose["uncovered"] == strict["uncovered"]
    assert strict["new"] == 0 <= loose["new"] <= loose["uncovered"]


def test_deleted_surfels_count_nowhere():
    sc = _scene("tiny")
    before = _measure(sc, 0)
    s = np.array(sc.surfels, np.float32, copy=True)
    s[0, :] = np.nan
    after = _measure(sc, 0, surfels=s)
    assert after["observed"] == 0 and not after["shared"].any()
    assert after["uncovered"] == after["valid"] == before["valid"]
    assert after["uncovered"] > before["uncovered"]
