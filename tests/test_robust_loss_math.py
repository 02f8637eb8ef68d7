"""CPU-only: the robust loss of the pose terms (bba_host_robust_loss, host_math.hpp RobustLoss) against its closed forms (Ceres'
conventions), its weight against a finite difference of rho, Huber's continuity at s = delta^2, and the exact w = 1 of the
trivial loss and of a Huber inlier, which keeps the results of handles without outliers unchanged bit for bit."""
import ctypes as C

import numpy as np
import pytest

TRIVIAL, HUBER, CAUCHY = 0, 1, 2


def _lib():
    from badslam_b200 import _lib
    return _lib.load()


def loss(kind, scale, s):
    rho, w = C.c_double(), C.c_double()
    _lib().bba_host_robust_loss(kind, scale, s, C.byref(rho), C.byref(w))
    return rho.value, w.value


S = np.r_[0.0, np.geomspace(1e-6, 1e6, 61)]


@pytest.mark.parametrize("scale", [0.05, 1.0, 3.0])
def test_closed_forms(scale):
    d = float(np.float32(scale))
    for s in S:
        rho, w = loss(TRIVIAL, scale, s)
        assert (rho, w) == (s, 1.0)
        rho, w = loss(HUBER, scale, s)
        want = (s, 1.0) if s <= d * d else (2 * d * np.sqrt(s) - d * d, d / np.sqrt(s))
        assert rho == pytest.approx(want[0], rel=1e-14, abs=1e-300) and w == pytest.approx(want[1], rel=1e-14)
        rho, w = loss(CAUCHY, scale, s)
        assert rho == pytest.approx(d * d * np.log1p(s / (d * d)), rel=1e-14, abs=1e-300)
        assert w == pytest.approx(1.0 / (1.0 + s / (d * d)), rel=1e-14)


@pytest.mark.parametrize("kind", [HUBER, CAUCHY])
def test_weight_is_the_derivative_of_rho(kind):
    scale = 0.7
    for s in np.geomspace(1e-3, 1e3, 25):
        h = 1e-6 * s
        if kind == HUBER and abs(s - float(np.float32(scale)) ** 2) < 2 * h:
            continue
        fd = (loss(kind, scale, s + h)[0] - loss(kind, scale, s - h)[0]) / (2 * h)
        assert loss(kind, scale, s)[1] == pytest.approx(fd, rel=1e-6), s


def test_huber_is_continuous_at_delta_squared():
    d = float(np.float32(0.3))
    s0 = d * d
    below, at, above = loss(HUBER, 0.3, np.nextafter(s0, 0)), loss(HUBER, 0.3, s0), loss(HUBER, 0.3, np.nextafter(s0, np.inf))
    assert at == (s0, 1.0)
    assert abs(above[0] - at[0]) <= 1e-15 and abs(below[0] - at[0]) <= 1e-15
    assert abs(above[1] - 1.0) <= 1e-15 and below[1] == 1.0


def test_trivial_and_inlier_huber_weigh_exactly_one():
    for s in S:
        assert loss(TRIVIAL, 1.0, s)[1] == 1.0
        assert loss(TRIVIAL, 0.0, s) == (s, 1.0)   # (the scale of a trivial loss is not read)
        if s <= 1e4:
            assert loss(HUBER, 100.0, s) == (s, 1.0)
    assert loss(7, 1.0, 2.5) == (2.5, 1.0)        # an unknown type counts as trivial on the host
    assert 0.0 < loss(CAUCHY, 1.0, 1e12)[1] < 1e-11 and loss(HUBER, 1.0, 1e12)[1] == pytest.approx(1e-6)
