"""The numpy pose-graph oracle (tests/pose_graph_oracle.py) on the CPU: its terms are the library's, its optimum is an
independent optimiser's, and CG preconditioned with the block-tridiagonal part of H needs at most 12 L + 1 iterations (L: the
edges between keyframes that are not consecutive)."""
import ctypes as C

import numpy as np
import pytest
import scipy.optimize

import pose_graph_oracle as O

_IDENTITY = np.eye(6)


def _lib():
    from badslam_b200 import _lib
    return _lib.load()


def _upper(M):
    return np.asarray(M, np.float32)[np.triu_indices(6)]


def _matrix(H, n):
    M = np.zeros((n, n))
    M[np.triu_indices(n)] = H
    return M + np.triu(M, 1).T


def _f32(A):
    return np.asarray(O.to_array(A), np.float32)


def _graph(K, loops, sigma=(0.01, 0.005), seed=0):
    """A drifted circle of K keyframes, the chain at the drifted state and loop constraints from the truth."""
    truth = O.circle(K)
    start = O.drift(truth, *sigma, seed=seed)
    terms = O.odometry_chain(start, _IDENTITY)
    for a, b in loops:
        terms.append(O.Term(a, b, O.mul(O.inv(O.pose(truth, a)), O.pose(truth, b)), _IDENTITY))
    return truth, start, terms


def test_terms_match_the_library():
    lib = _lib()
    rng = np.random.default_rng(3)
    for _ in range(20):
        A = O.se3_exp(rng.normal(0, 0.8, 6))
        B = O.se3_exp(rng.normal(0, 0.8, 6))
        Z = O.mul(O.mul(O.inv(A), B), O.se3_exp(rng.normal(0, 0.05, 6)))
        G = rng.normal(size=(6, 6))
        L = G @ G.T + 0.5 * np.eye(6)
        pa, pb, z, info = _f32(A), _f32(B), _f32(Z), _upper(L)
        # prior on A at Z
        H, b, cost = np.zeros(21), np.zeros(6), C.c_double()
        lib.bba_host_pose_prior_terms(z.ctypes.data, pa.ctypes.data, info.ctypes.data, H.ctypes.data, b.ctypes.data, C.byref(cost))
        t = O.Term(0, -1, z, info)
        Ho, bo, co = O.term_blocks(t, O.from_array(pa))
        assert np.allclose(_matrix(H, 6), Ho, rtol=1e-5, atol=1e-6 * np.abs(Ho).max())
        assert np.allclose(b, bo, rtol=1e-5, atol=1e-6 * np.abs(bo).max())
        assert abs(cost.value - co) <= 1e-6 * co
        # constraint (A, B, Z)
        H, b = np.zeros(78), np.zeros(12)
        lib.bba_host_pose_constraint_terms(z.ctypes.data, pa.ctypes.data, pb.ctypes.data, info.ctypes.data, H.ctypes.data,
                                           b.ctypes.data, C.byref(cost))
        t = O.Term(0, 1, z, info)
        Ho, bo, co = O.term_blocks(t, O.from_array(pa), O.from_array(pb))
        assert np.allclose(_matrix(H, 12), Ho, rtol=1e-5, atol=1e-6 * np.abs(Ho).max())
        assert np.allclose(b, bo, rtol=1e-5, atol=1e-6 * np.abs(bo).max())
        assert abs(cost.value - co) <= 1e-6 * co


def test_noise_free_graph_returns_the_truth():
    K = 24
    truth = O.circle(K)
    start = O.drift(truth, 0.05, 0.03, seed=1)
    # every edge from the truth: the chain and two loops; keyframe 0 starts at its true pose and is the gauge
    terms = O.odometry_chain(truth, _IDENTITY) + [O.Term(a, b, O.mul(O.inv(O.pose(truth, a)), O.pose(truth, b)), _IDENTITY)
                                                  for a, b in ((0, K - 1), (3, 15))]
    poses, held, cost, _ = O.gauss_newton(terms, start, gauge=0)
    assert held.sum() == 1 and held[0]
    assert cost < 1e-20
    assert np.abs(poses[1] - truth[1]).max() < 1e-9 and np.abs(poses[0] - truth[0]).max() < 1e-9


def test_optimum_equals_scipy_least_squares():
    K = 30
    truth, start, terms = _graph(K, [(5, K - 3), (2, 17)], sigma=(0.02, 0.01), seed=2)
    P = O.se3_exp(np.array([0.1, -0.05, 0.02, 0.01, 0.02, -0.01]))
    terms.append(O.Term(K // 2, -1, O.mul(O.pose(truth, K // 2), P), np.diag([4.0] * 3 + [9.0] * 3)))
    poses, held, cost, _ = O.gauss_newton(terms, start, gauge=0)
    fun, unpack, n = O.least_squares_whitened(terms, start, held)
    ls = scipy.optimize.least_squares(fun, np.zeros(n), xtol=1e-14, ftol=1e-14, gtol=1e-14)
    other = unpack(ls.x)
    assert abs(0.5 * np.sum(ls.fun ** 2) - cost) <= 1e-9 * cost
    assert np.abs(other[1] - poses[1]).max() < 1e-6 and np.abs(other[0] - poses[0]).max() < 1e-6


@pytest.mark.parametrize("K", [200, 1000])
@pytest.mark.parametrize("loops", ["one", "random"])
def test_tridiagonal_pcg_iteration_bound(K, loops):
    pairs = [(5, K - 3)] if loops == "one" else O.random_loops(K, 10 if K == 200 else 20, seed=K)
    _, start, terms = _graph(K, pairs, seed=K)
    held = O.held_keyframes(K, terms, 0)
    H, b, _ = O.normal_equations(terms, start, held)
    # the chain is at its optimum at the start: move the right-hand side off zero with the loops' own terms
    assert np.linalg.norm(b) > 0
    L = len(pairs)
    its, x = O.pcg_iterations(H, b, O.block_tridiagonal(H))
    assert its <= 12 * L + 1 + 3, (its, L)
    assert np.linalg.norm(H @ x + b) <= 1e-9 * np.linalg.norm(b)
    if K == 200 and loops == "one":   # block Jacobi on the same system is far slower: the reason for the preconditioner
        its_jacobi, _ = O.pcg_iterations(H, b, O.block_diagonal(H))
        assert its_jacobi > 10 * its, (its_jacobi, its)


def test_chain_only_graph_is_at_its_optimum():
    K = 40
    _, start, terms = _graph(K, [])
    poses, held, cost, _ = O.gauss_newton(terms, start, gauge=0)
    assert cost < 1e-20
    assert np.abs(poses[1] - start[1]).max() < 1e-12 and np.abs(poses[0] - start[0]).max() < 1e-12


def test_held_rule():
    t = [O.Term(1, 2, np.array([0, 0, 0, 1, 1, 0, 0], np.float32), _IDENTITY),
         O.Term(4, 5, np.array([0, 0, 0, 1, 1, 0, 0], np.float32), _IDENTITY),
         O.Term(6, 7, np.array([0, 0, 0, 1, 1, 0, 0], np.float32), _IDENTITY),
         O.Term(7, -1, np.array([0, 0, 0, 1, 0, 0, 0], np.float32), _IDENTITY)]
    held = O.held_keyframes(9, t, gauge=5)
    # 0, 3, 8: untouched; 1: lowest of a component without gauge or prior; 5: the gauge; {6, 7} has a prior
    assert np.nonzero(held)[0].tolist() == [0, 1, 3, 5, 8]
