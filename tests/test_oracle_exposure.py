"""CPU: the properties of the keyframe exposure oracle (tests/exposure_oracle.py, DESIGN.md §3.21) on synthetic observation tables
and on the tiny scene: known gains are recovered to the Q16 rounding, sum(r) = 0, the gauge choice and disconnected components,
outliers are rejected, and the system does not depend on the surfel order."""
import numpy as np
import pytest

import exposure_oracle as O


def _table(K=12, n=4000, per=8, seed=0, log_gains=None):
    """A synthetic observation table: n surfels of log radiance z_s, each seen by `per` random keyframes, y = round(2^16 (x + z))."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(np.log(0.7), np.log(1.4), K) if log_gains is None else np.asarray(log_gains, np.float64)
    z = rng.uniform(np.log(20), np.log(200), n)
    valid = np.zeros((n, K), bool)
    for s in range(n):
        valid[s, rng.choice(K, per, replace=False)] = True
    y = np.where(valid, np.rint(65536.0 * (x[None, :] + z[:, None])), 0).astype(np.int64)
    return valid, y, x


def test_recovers_known_gains():
    valid, y, x = _table()
    e = O.estimate(valid, y, gauge=0)
    got = e["log"]
    want = x - x[0]
    assert np.abs(got - want).max() < 2e-6, np.abs(got - want).max()
    assert (e["inliers"] == valid.sum(axis=0)).all()
    assert np.array_equal(e["observations"], valid.sum(axis=0))


def test_rhs_sums_to_zero_and_C_symmetric():
    valid, y, _ = _table(seed=3)
    y = y + np.where(valid, np.random.default_rng(4).integers(-5000, 5000, y.shape), 0)
    C, r = O.system(valid, y)
    assert int(r.sum()) == 0
    assert np.array_equal(C, C.T)
    assert np.array_equal(np.diag(C), valid.sum(axis=0))


def test_gauge_choice():
    valid, y, x = _table(seed=5)
    for g in (0, 4, 11):
        e = O.estimate(valid, y, gauge=g)
        assert e["log"][g] == 0.0
        assert np.abs(e["log"] - (x - x[g])).max() < 2e-6


def test_disconnected_components():
    """Keyframes 8..11 share no surfel with 0..7: NaN gains and 0 inliers for them, the first group still recovered."""
    valid, y, x = _table(K=12, seed=6)
    valid[:, 8:] = False
    y[:, 8:] = 0
    rng = np.random.default_rng(7)
    extra = np.zeros((500, 12), bool)
    for s in range(500):
        extra[s, 8 + rng.choice(4, 3, replace=False)] = True
    z = rng.uniform(3, 5, 500)
    ye = np.where(extra, np.rint(65536.0 * (x[None, :] + z[:, None])), 0).astype(np.int64)
    valid, y = np.vstack([valid, extra]), np.vstack([y, ye])
    e = O.estimate(valid, y, gauge=2)
    assert np.isnan(e["gains"][8:]).all() and (e["inliers"][8:] == 0).all()
    assert (e["observations"][8:] > 0).all()
    assert np.abs(e["log"][:8] - (x[:8] - x[2])).max() < 2e-6
    e = O.estimate(valid, y, gauge=9)
    assert np.isnan(e["gains"][:8]).all()
    assert np.abs(e["log"][8:] - (x[8:] - x[9])).max() < 2e-6


def test_outliers_rejected():
    """10 % of the observations scaled by 1.5 or 1 / 1.5 (log +-0.41): the second round drops them and recovers the gains."""
    valid, y, x = _table(K=12, n=6000, per=10, seed=8)
    rng = np.random.default_rng(9)
    obs = np.argwhere(valid)
    bad = obs[rng.random(len(obs)) < 0.10]
    factor = np.where(rng.random(len(bad)) < 0.5, np.log(1.5), -np.log(1.5))
    y[bad[:, 0], bad[:, 1]] += np.rint(65536.0 * factor).astype(np.int64)
    clean = O.estimate(valid, y, gauge=0, outer_iterations=1)
    e = O.estimate(valid, y, gauge=0)
    want = x - x[0]
    assert np.abs(e["log"] - want).max() < 1e-3, np.abs(e["log"] - want).max()
    assert np.abs(clean["log"] - want).max() > 1e-3
    kept = e["member"][bad[:, 0], bad[:, 1]]
    assert kept.mean() < 0.02, kept.mean()
    good = valid.copy()
    good[bad[:, 0], bad[:, 1]] = False
    assert e["member"][good].mean() > 0.97


def test_surfel_permutation():
    valid, y, _ = _table(seed=10)
    y = y + np.where(valid, np.random.default_rng(11).integers(-9000, 9000, y.shape), 0)
    perm = np.random.default_rng(12).permutation(len(valid))
    a = O.estimate(valid, y, gauge=1)
    b = O.estimate(valid[perm], y[perm], gauge=1)
    assert np.array_equal(a["C"], b["C"]) and np.array_equal(a["r"], b["r"])
    assert np.array_equal(a["member"][perm], b["member"])
    assert np.allclose(a["log"], b["log"], rtol=0, atol=1e-12)


def test_log_table():
    assert O.LOG_Q16[1] == 0 and O.LOG_Q16[255] == round(65536 * np.log(255))
    assert (np.diff(O.LOG_Q16[1:]) > 0).all()


def test_compensated_luma():
    v = np.arange(256)
    assert np.array_equal(O.compensated_luma(v, 1.0), v)
    assert O.compensated_luma([200], 0.5)[0] == 255 and O.compensated_luma([100], 2.0)[0] == 50


@pytest.fixture(scope="module")
def tiny():
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name("tiny"))


def _scene_table(sc, color):
    import surfel_deform_oracle as D
    from oracle.cpu_oracle import se3_inverse
    inv = np.stack([se3_inverse(p) for p in sc.poses_init]).astype(np.float32)
    return O.observations(D.Camera.of_scene(sc), sc.depth_K, sc.color_K, sc.depth, sc.normals, color, sc.surfels, sc.num_surfels, inv)[:2]


def test_scene_gains(tiny):
    """tiny with its colours scaled by known gains: the estimate is within 2 % of the true ratios to keyframe 0."""
    K = tiny.cfg.num_keyframes
    g = np.random.default_rng(13).uniform(0.7, 1.4, K)
    # (g / 1.4: no channel clips; a clipped channel changes the luma by other than g, which no gain can represent)
    valid, y = _scene_table(tiny, O.scale_colors(tiny.color, g / 1.4))
    assert valid.sum() > 100
    e = O.estimate(valid, y, gauge=0)
    ok = ~np.isnan(e["gains"])
    assert ok.sum() >= 2
    ratio = e["gains"][ok] / (g[ok] / g[0])
    assert np.abs(ratio - 1).max() < 0.02, ratio
    v0, y0 = _scene_table(tiny, tiny.color)
    e0 = O.estimate(v0, y0, gauge=0)
    assert np.abs(e0["gains"][~np.isnan(e0["gains"])] - 1).max() < 0.02
