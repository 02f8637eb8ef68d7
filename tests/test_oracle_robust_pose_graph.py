"""The numpy IRLS oracle of the robust pose terms (tests/robust_pose_oracle.py) on the CPU: with trivial losses it is
pose_graph_oracle's Gauss-Newton, its robust optimum is a stationary point of the robust cost, and on a 200-keyframe circle with
three false loop closures a Cauchy loss keeps the map where the outlier-free optimum is while the trivial loss bends it."""
import numpy as np

import pose_graph_oracle as O
import robust_pose_oracle as R

_I6 = np.eye(6)


def false_loop_circle(K=200, true_loops=((5, 197),), false_loops=((20, 30), (80, 91), (140, 149)), info=1e4):
    """The truth on a circle of K keyframes, the odometry chain at the truth, the true loops and false loops whose Z is the true
    relative pose times exp(0.5 m, 20 degrees); every edge has information `info` (sigma 1 cm / 0.01 rad by default)."""
    truth = O.circle(K)
    L = info * _I6
    terms = O.odometry_chain(truth, L)
    chain = len(terms)
    for a, b in true_loops:
        terms.append(O.Term(a, b, O.mul(O.inv(O.pose(truth, a)), O.pose(truth, b)), L))
    wrong = O.se3_exp(np.r_[0.3, -0.3, 0.3, 0.0, 0.0, np.deg2rad(20.0)])
    assert np.linalg.norm(np.r_[0.3, -0.3, 0.3]) >= 0.5
    for a, b in false_loops:
        terms.append(O.Term(a, b, O.mul(O.mul(O.inv(O.pose(truth, a)), O.pose(truth, b)), wrong), L))
    return truth, terms, chain


def _max_move(P, Q):
    return float(np.max(np.linalg.norm(P[1] - Q[1], axis=1)))


def test_trivial_losses_are_the_plain_oracle():
    truth = O.circle(30)
    start = O.drift(truth, 0.02, 0.01, seed=5)
    terms = O.odometry_chain(start, _I6) + [O.Term(a, b, O.mul(O.inv(O.pose(truth, a)), O.pose(truth, b)), 4 * _I6)
                                            for a, b in [(2, 27), (8, 20)]]
    terms.append(O.Term(4, -1, O.pose(truth, 4), 100 * _I6))
    want, held, cost, its = O.gauss_newton(terms, start, gauge=0)
    got, held_r, cost_r, its_r = R.gauss_newton(terms, [(R.TRIVIAL, 1.0)] * len(terms), start, gauge=0)
    assert its_r == its and np.array_equal(held_r, held)
    assert abs(cost_r - cost) <= 1e-14 * cost   # (rho(s) / 2 of s = r^T L r against r^T L r / 2: rounding only)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_the_robust_optimum_is_stationary():
    truth, terms, chain = false_loop_circle(K=16, true_loops=[(1, 14)], false_loops=[(3, 8)], info=100.0)
    start = O.drift(truth, 0.02, 0.01, seed=2)
    terms = O.odometry_chain(start, 100 * _I6) + terms[chain:]
    terms.append(O.Term(0, -1, O.pose(truth, 0), 400 * _I6))   # a prior fixes the gauge
    losses = [(R.TRIVIAL, 0.0)] * (len(terms) - 3) + [(R.HUBER, 0.5), (R.CAUCHY, 1.0), (R.HUBER, 2.0)]
    opt, held, cost, its = R.gauss_newton(terms, losses, start, gauge=-1)
    assert not held.any()
    g0 = R.cost_gradient(terms, losses, start, held)
    g = R.cost_gradient(terms, losses, opt, held)
    print(f"robust cost {R.total_cost(terms, losses, start):.6g} -> {cost:.6g} in {its} iterations; "
          f"|grad| {np.linalg.norm(g0):.3g} -> {np.linalg.norm(g):.3g}")
    assert np.linalg.norm(g) <= 1e-5 * np.linalg.norm(g0)
    w = R.weights(terms, losses, opt)
    assert w[-2] < 0.1 and np.all(w[:-3] == 1.0)   # the false loop is down-weighted, the trivial terms are not


def test_cauchy_rejects_false_loops_on_the_circle():
    truth, terms, chain = false_loop_circle()
    clean = terms[:chain + 1]
    want, _, _, _ = R.gauss_newton(clean, [(R.TRIVIAL, 0.0)] * len(clean), truth, gauge=0, max_iterations=10)
    trivial, _, _, _ = R.gauss_newton(terms, [(R.TRIVIAL, 0.0)] * len(terms), truth, gauge=0, max_iterations=30)
    losses = [(R.TRIVIAL, 0.0)] * chain + [(R.CAUCHY, 1.0)] * (len(terms) - chain)
    robust, _, _, _ = R.gauss_newton(terms, losses, truth, gauge=0, max_iterations=30)
    d_trivial, d_cauchy = _max_move(trivial, want), _max_move(robust, want)
    print(f"largest keyframe move from the outlier-free optimum: trivial {d_trivial:.4f} m, Cauchy {d_cauchy:.5f} m")
    assert _max_move(want, truth) < 1e-9
    assert d_cauchy < 0.005 and d_trivial > 0.1
    w = R.weights(terms, losses, robust)
    assert np.all(w[chain + 1:] < 1e-2 * w[chain])   # the false loops weigh far less than the true one
