"""The exact accumulator of the deterministic mode on the host (bba_host_exact_sum, badslam_b200/csrc/exact_sum.cuh): the sum of
fp32 values is computed exactly and rounded once to fp64, so every permutation of the same values gives the same bits, and those
are math.fsum's (a correctly rounded sum).  Non-finite values follow IEEE addition.  No device needed."""
import math

import numpy as np
import pytest

from badslam_b200.direct_ba import exact_sum

FLT_MAX = float(np.finfo(np.float32).max)
FLT_TRUE_MIN = float(np.float32(1e-45))


def arrays():
    """The arrays the device test (tests/test_gpu_deterministic.py) also sums."""
    rng = np.random.default_rng(1234)
    n = 4096
    wide = (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, n)).astype(np.float32)
    cancel = np.concatenate([wide, -wide[: n // 2], np.float32([1e30, 1, -1e30])])
    sub = (rng.integers(-(1 << 23), 1 << 23, 1000) * FLT_TRUE_MIN).astype(np.float32)   # subnormals and zeros
    big = np.full(1000, FLT_MAX, np.float32)
    big_mixed = np.concatenate([big, -big[:999], np.float32([FLT_TRUE_MIN])])
    million = (rng.standard_normal(10 ** 6) * 10.0 ** rng.uniform(-20, 20, 10 ** 6)).astype(np.float32)
    # sums at or above 2^139 in magnitude reach the tenth 32-bit digit of the rounding (ExactFinalize, k == 9)
    top = np.full(4096, FLT_MAX, np.float32)                                             # ~2^140
    top_carry = np.concatenate([top, -top[:4095], np.float32([FLT_TRUE_MIN])])           # from the top digit down to bit 0
    top_edge = np.full(4096, 2.0 ** 127, np.float32)                                     # exactly 2^139: the digit boundary
    neg_tiny = np.full(1 << 20, -FLT_TRUE_MIN, np.float32)                               # a borrow through every word
    return dict(wide=wide, cancel=cancel, subnormal=sub, flt_max=big, flt_max_mixed=big_mixed, million=million,
                three=np.float32([1e30, 1, -1e30]), top_digit=top, top_digit_negative=-top, top_digit_carry=top_carry,
                top_digit_edge=top_edge, negative_tiny=neg_tiny)


def bits(x):
    return np.float64(x).tobytes()


def same(a, b):
    """Equal bits; zeros compared by value (an exact zero is +0.0, fsum may give -0.0)."""
    return (a == 0 and b == 0) or bits(a) == bits(b)


@pytest.mark.parametrize("name", list(arrays()))
def test_every_permutation_gives_the_correctly_rounded_sum(name):
    a = arrays()[name]
    want = math.fsum(a.astype(np.float64))
    rng = np.random.default_rng(7)
    results = [exact_sum(a), exact_sum(a[::-1]), exact_sum(np.sort(a))] + [exact_sum(rng.permutation(a)) for _ in range(3)]
    for r in results:
        assert same(r, want), (name, r, want)
    assert len({bits(r) for r in results}) == 1, name


def test_known_values():
    assert exact_sum([1e30, 1, -1e30]) == 1.0
    assert exact_sum([]) == 0.0 and bits(exact_sum([])) == bits(0.0)
    assert bits(exact_sum([-0.0, -0.0])) == bits(0.0)            # an exact zero is +0.0
    assert bits(exact_sum([1.5, -1.5])) == bits(0.0)
    assert exact_sum([FLT_TRUE_MIN] * 3) == 3 * FLT_TRUE_MIN
    assert exact_sum([FLT_MAX] * 4) == 4 * FLT_MAX                # beyond the fp32 range, exact in fp64
    # rounding to fp64 once: 1 + 2^-60 is not representable and rounds to 1; ties go to even
    assert exact_sum([1.0, 2.0 ** -60]) == 1.0
    assert exact_sum([1.0, 2.0 ** -53]) == 1.0                    # tie, 1 is even
    assert exact_sum([1.0 + 2.0 ** -23, 2.0 ** -53]) == 1.0 + 2.0 ** -23 and \
        exact_sum([1.0, 2.0 ** -52, 2.0 ** -53]) == 1.0 + 2.0 ** -51   # tie to even upwards
    assert exact_sum([1.0, 2.0 ** -53, 2.0 ** -100]) == 1.0 + 2.0 ** -52   # above the tie: up


def test_non_finite_values():
    inf, nan = float("inf"), float("nan")
    assert exact_sum([1.0, inf, 2.0]) == inf
    assert exact_sum([-inf, 1.0, -inf]) == -inf
    assert math.isnan(exact_sum([inf, -inf]))
    assert math.isnan(exact_sum([1.0, nan]))
    assert math.isnan(exact_sum([nan, inf]))
    for a in ([inf, -inf, 3.0], [2.0, nan, -inf]):   # independent of the order
        assert math.isnan(exact_sum(a)) and math.isnan(exact_sum(a[::-1]))
