"""The device pose graph (bba_optimize_pose_graph, DESIGN §3.14) at the keyframe counts where its one-CTA solve changes shape.

PoseGraphSolveKernel walks its blocks in loops strided by its 256 threads: the level-0 copy of the factorisation and H p take a
second pass from K = 257 on, the back sweep at level l from a level size of 257, the even positions of the factorisation and the
forward sweep from 513, the odd positions of the forward sweep from 514 (level sizes n_0 = K, n_(l+1) = ceil(n_l / 2)).  So K
runs over 1, 2, 3, 5 and both sides of those edges up to 2 500 keyframes:

a. M = H, well conditioned: the chain and a prior on every keyframe, both with information I, no gauge.  The block-tridiagonal
   preconditioner is H itself (cond ~ 5), so PCG takes one iteration per Gauss-Newton iteration; a second one means M^-1 is wrong.
b. M = H, a loop closure: the chain and the loop (0, K - 1) with keyframe 0 as the gauge, whose held row drops the loop's coupling.
   cond(H) ~ K^2, so rounding may cost one more PCG iteration.
c. M != H, one Gauss-Newton step (max_iterations = 1) against the oracle's sparse direct step from the same fp32 start (assembly
   and H p), and the PCG iterations against the oracle's block-tridiagonal PCG on the same system (the preconditioner); one full
   solve at 2 500 keyframes with 50 loops.
d. held rows inside the reduction: two constraint components with untouched keyframes between them, the gauge in the second; then
   attitude priors on the second component and no gauge, so its first keyframe is held in translation and yaw only.
e. bits: the deterministic mode and a second handle; a handle whose pose-graph buffers grew between two calls; a handle with room
   for more keyframes than it holds.

The handles hold keyframes that share the two 80x60 images of one tiny scene (test_gpu_pose_graph.make_handle); every oracle result
is computed once per module."""
import functools

import numpy as np
import pytest
import scipy.sparse.linalg as spl

import attitude_prior_oracle as A
import pose_graph_oracle as O
import test_gpu_pose_graph as PG
from gpu_checks import POSE_R, POSE_T

pytestmark = pytest.mark.gpu

SHAPES = [1, 2, 3, 5, 256, 257, 512, 513, 514, 1024, 1025, 1027, 2049, 2053, 2500]
UP = np.array([0.0, 0.0, 1.0])
_I6 = np.eye(6)
_HANDLES = {}


def _handle(K):
    """One handle per K for the module, with no priors, constraints or attitude priors.  K = 1 takes the first keyframe of the
    same scene generated with one keyframe (the shared scene has two)."""
    if K not in _HANDLES:
        if K == 1:
            from badslam_b200.direct_ba import DirectBA
            from badslam_b200.scene import SceneConfig, make_scene
            one = make_scene(SceneConfig(80, 60, 1, 2000, cell=1, seed=41, name="pose_graph_one"))
            _HANDLES[K] = DirectBA.from_scene(one, device="cuda:0", max_keyframes=1)
        else:
            _HANDLES[K] = PG.make_handle(K)
    ba = _HANDLES[K]
    ba.ClearKeyframePosePriors()
    ba.RemoveKeyframePoseConstraints()
    ba.ClearKeyframeAttitudePriors()
    return ba


def _terms(start32, cons=(), priors=(), chain=True):
    """The oracle's terms of a call: priors [(k, pose32, L)], constraints [(a, b, Z32, L)], the chain at start32 with I."""
    S = O.from_array(start32)
    terms = [O.Term(k, -1, P, L) for k, P, L in priors] + [O.Term(a, b, Z, L) for a, b, Z, L in cons]
    if chain:
        terms += [O.Term(k, k + 1, PG._f32(O.mul(O.inv(O.pose(S, k)), O.pose(S, k + 1))), _I6) for k in range(len(start32) - 1)]
    return S, terms


def _constraints(truth, pairs, noise_seed=None):
    """Constraints (a, b, Z, I) with Z the true relative pose, or a noisy measurement of it."""
    if noise_seed is None:
        return [(a, b, PG._relative(truth, a, b), _I6) for a, b in pairs]
    rng = np.random.default_rng(noise_seed)
    return [(a, b, PG._f32(O.mul(O.mul(O.inv(O.pose(truth, a)), O.pose(truth, b)), O.se3_exp(np.r_[rng.normal(0, 0.01, 3),
                                                                                                    rng.normal(0, 0.005, 3)]))),
             _I6) for a, b in pairs]


def _add(ba, cons):
    ba.AddKeyframePoseConstraints([c[0] for c in cons], [c[1] for c in cons], [c[2] for c in cons], _I6)


def _check_optimum(tag, got, r, want, cost, terms=None):
    """The cost within 1e-4 of the oracle's optimum's, and the poses within POSE_T / POSE_R of it -- or, given the terms, within what
    fp32 poses resolve.  Along the softest direction of a long loop (eigenvalue ~ pi^2 / K^2 of H) a step of 1e-5 m lowers the
    cost by ~1e-13, less than rounding the poses to fp32 changes it (~1e-12 at 2 000 keyframes of a 5 m circle).  The rule that a
    step which raises the cost is taken back and ends the call then stops there at random, with converged = 0.  Such poses are
    held to the resolution of that rule: in fp64 they cost no more above the optimum than twice what rounding the optimum itself
    to fp32 costs."""
    dt, dr = PG._worst(got, want)
    note = ""
    if terms is not None and not (dt < POSE_T and dr < POSE_R):
        excess = O.total_cost(terms, O.from_array(got)) - cost
        rounding = O.total_cost(terms, O.from_array(PG._f32(want))) - cost
        note = f"; above POSE_T: fp64 cost {excess:.3g} above the optimum, its fp32 rounding {rounding:.3g}"
    print(f"{tag}: GN {r['iterations']} / PCG {r['linear_iterations']}, converged {r['converged']}, worst pose error "
          f"{dt:.3g} m / {dr:.3g} rad, cost {r['final_cost']:.9g} (oracle {cost:.9g}){note}")
    if note:
        assert excess <= 2 * rounding, (dt, dr, excess, rounding)
    else:
        assert dt < POSE_T and dr < POSE_R, (dt, dr)
    # (1e-12: about the cost of rounding a pose 5 m out to fp32, for K = 1 whose optimum, its prior, costs 0)
    assert abs(r["final_cost"] - cost) <= 1e-4 * cost + 1e-12, (r["final_cost"], cost)


# ---- a. M = H, well conditioned ------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _case_a(K):
    """A drifted circle, the chain at the start and a prior on every keyframe, a noisy measurement of the truth (so that K = 1
    has a step to take too), all with information I; no gauge."""
    truth, start = PG._circle(K, seed=K)
    noise = O.se3_exp(np.random.default_rng(K).normal(0.0, 1.0, (K, 6)) * np.r_[[0.01] * 3, [0.005] * 3])
    priors = [(k, P, _I6) for k, P in enumerate(PG._f32(O.mul(truth, noise)))]
    S, terms = _terms(start, priors=priors)
    want, held, cost, its = O.gauss_newton(terms, S, gauge=-1)
    return start, priors, want, cost


@pytest.mark.parametrize("K", SHAPES)
def test_tridiagonal_graph_takes_one_pcg_iteration(K):
    start, priors, want, cost = _case_a(K)
    ba = _handle(K)
    ba.SetKeyframeStates(start)
    ba.SetKeyframePosePriors([p[0] for p in priors], [p[1] for p in priors], _I6)
    r = ba.OptimizePoseGraph(gauge_keyframe=-1)
    _check_optimum(f"a K={K}", ba.GetKeyframeStates()[0], r, want, cost)
    assert r["converged"] == 1 and r["held_keyframes"] == 0
    # cond(H) ~ 5: one PCG iteration per Gauss-Newton iteration, or M^-1 is not H^-1
    assert 1 <= r["linear_iterations"] <= r["iterations"], r


# ---- b. M = H, a loop closure at the gauge -----------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _case_b(K):
    truth, start = PG._circle(K, seed=K + 1)
    cons = _constraints(truth, [(0, K - 1)])
    S, terms = _terms(start, cons)
    want, held, cost, _ = O.gauss_newton(terms, S, gauge=0)
    return start, cons, terms, want, cost


@pytest.mark.parametrize("K", [257, 513, 1025, 2049, 2500])
def test_loop_at_the_gauge_keeps_m_equal_to_h(K):
    start, cons, terms, want, cost = _case_b(K)
    ba = _handle(K)
    ba.SetKeyframeStates(start)
    _add(ba, cons)
    r = ba.OptimizePoseGraph(gauge_keyframe=0)
    got = ba.GetKeyframeStates()[0]
    _check_optimum(f"b K={K}", got, r, want, cost, terms)
    assert r["held_keyframes"] == 1
    assert np.array_equal(got[0].view(np.uint32), start[0].view(np.uint32))
    # M = H, but cond(H) ~ K^2: rounding may leave the first PCG iterate above the 1e-10 relative residual
    assert r["iterations"] <= r["linear_iterations"] <= 2 * r["iterations"], r


# ---- c. M != H ---------------------------------------------------------------------------------------------------------------
def _loops(K, L):
    return [(5, K - 3)] if L == 1 else O.random_loops(K, L, seed=K + L)


@functools.lru_cache(maxsize=None)
def _case_c(K, L):
    """The oracle's one Gauss-Newton step from the fp32 start (sparse direct) and the block-tridiagonal PCG's iterations on it."""
    truth, start = PG._circle(K, seed=K + 2)
    cons = _constraints(truth, _loops(K, L))
    S, terms = _terms(start, cons)
    held = O.held_keyframes(K, terms, 0)
    H, b, free = O.normal_equations(terms, S, held)
    delta = np.zeros(6 * K)
    delta[free] = spl.spsolve(H.tocsc(), -b)
    its, _ = O.pcg_iterations(H, b, O.block_tridiagonal(H))
    return start, cons, O.mul(S, O.se3_exp(delta.reshape(K, 6))), its


@pytest.mark.parametrize("L", [1, 20])
@pytest.mark.parametrize("K", [513, 1025, 2053, 2500])
def test_one_step_matches_the_direct_solve(K, L):
    start, cons, want, its = _case_c(K, L)
    ba = _handle(K)
    ba.SetKeyframeStates(start)
    _add(ba, cons)
    r = ba.OptimizePoseGraph(gauge_keyframe=0, max_iterations=1)
    dt, dr = PG._worst(ba.GetKeyframeStates()[0], want)
    print(f"c K={K} L={L} one step: PCG {r['linear_iterations']} (oracle {its}), worst pose error {dt:.3g} m / {dr:.3g} rad")
    assert r["iterations"] == 1 and r["final_cost"] < r["initial_cost"], r
    assert dt < POSE_T and dr < POSE_R, (dt, dr)
    # within 12 L + 1 iterations (the bound in exact arithmetic) the counts agree to one; past it CG has lost orthogonality and
    # the count follows the rounding, where two fp64 restatements that sum in different orders agree to 1 %
    slack = 1 if its <= 12 * L + 1 else int(np.ceil(0.01 * its))
    assert abs(r["linear_iterations"] - its) <= slack, (r["linear_iterations"], its)


@functools.lru_cache(maxsize=None)
def _case_c_full(K, L):
    truth, start = PG._circle(K, seed=K + 3)
    cons = _constraints(truth, _loops(K, L))
    S, terms = _terms(start, cons)
    want, held, cost, _ = O.gauss_newton(terms, S, gauge=0)
    return start, cons, terms, want, cost


def test_full_solve_with_50_loops_at_2500():
    K, L = 2500, 50
    start, cons, terms, want, cost = _case_c_full(K, L)
    ba = _handle(K)
    ba.SetKeyframeStates(start)
    _add(ba, cons)
    r = ba.OptimizePoseGraph(gauge_keyframe=0)
    _check_optimum(f"c K={K} L={L} full", ba.GetKeyframeStates()[0], r, want, cost, terms)
    assert r["converged"] == 1 and r["linear_iterations"] <= (12 * L + 4) * r["iterations"], r


# ---- d. held rows inside the reduction --------------------------------------------------------------------------------------
_D_K, _D_GAUGE = 1025, 600
_D_FIRST, _D_SECOND = range(0, 400), range(410, 1025)   # 400-409 untouched


@functools.lru_cache(maxsize=None)
def _case_d():
    """Constraint chains over [0, 399] and [410, 1024] with one loop in each, noisy measurements of the truth; no odometry
    chain."""
    K = _D_K
    truth, start = PG._circle(K, seed=11)
    pairs = [(k, k + 1) for k in _D_FIRST[:-1]] + [(k, k + 1) for k in _D_SECOND[:-1]] + [(5, 395), (415, 1020)]
    return truth, start, _constraints(truth, pairs, noise_seed=12)


def test_held_rows_inside_the_reduction():
    K = _D_K
    truth, start, cons = _case_d()
    S, terms = _terms(start, cons, chain=False)
    want, held, cost, _ = O.gauss_newton(terms, S, gauge=_D_GAUGE)
    assert np.nonzero(held)[0].tolist() == [0] + list(range(400, 410)) + [_D_GAUGE]
    ba = _handle(K)
    ba.SetKeyframeStates(start)
    _add(ba, cons)
    r = ba.OptimizePoseGraph(add_current_state_odometry_constraints=False, gauge_keyframe=_D_GAUGE)
    got = ba.GetKeyframeStates()[0]
    _check_optimum("d held rows", got, r, want, cost, terms)
    assert r["converged"] == 1 and r["held_keyframes"] == int(held.sum())
    for k in np.nonzero(held)[0]:
        assert np.array_equal(got[k].view(np.uint32), start[k].view(np.uint32)), k


def test_partially_held_row_inside_the_reduction():
    """Attitude priors on the second component and no gauge: keyframe 410 is held in translation and yaw (held = 2), 0 and the
    untouched 400-409 fully.  The components are independent, so the oracle solves each on its own: the first with
    pose_graph_oracle, the second re-indexed from 0 with attitude_prior_oracle."""
    K = _D_K
    truth, start, cons = _case_d()
    d_meas = np.array([A.tilt(O.pose(truth, k)[0], UP) for k in range(K)], np.float32)
    L_att = 1e2
    S = O.from_array(start)
    first = [c for c in cons if c[0] in _D_FIRST]
    second = [c for c in cons if c[0] in _D_SECOND]
    want1, held1, cost1, _ = O.gauss_newton(_terms(start, first, chain=False)[1], S, gauge=-1)
    o = _D_SECOND.start
    sub = (S[0][o:], S[1][o:])
    terms2 = [O.Term(a - o, b - o, Z, L) for a, b, Z, L in second]
    atts = [A.Attitude(k - o, np.float32(UP), d_meas[k], np.float32(L_att)) for k in _D_SECOND]
    want2, held2, axes, cost2, _ = A.gauss_newton(terms2, [(0, 0.0)] * len(terms2), atts, sub, gauge=-1)
    assert held2[0] == 2 and not held2[1:].any()
    want = (np.concatenate([want1[0][:o], want2[0]]), np.concatenate([want1[1][:o], want2[1]]))
    ba = _handle(K)
    ba.SetKeyframeStates(start)
    _add(ba, cons)
    ba.SetKeyframeAttitudePriors(list(_D_SECOND), UP, d_meas[o:], L_att)
    r = ba.OptimizePoseGraph(add_current_state_odometry_constraints=False, gauge_keyframe=-1)
    got = ba.GetKeyframeStates()[0]
    _check_optimum("d partially held", got, r, want, cost1 + cost2)
    assert r["converged"] == 1 and r["held_keyframes"] == 11
    for k in [0] + list(range(400, 410)):
        assert np.array_equal(got[k].view(np.uint32), start[k].view(np.uint32)), k
    # keyframe 410 keeps its translation, and its yaw about d_ref moves as the oracle's: every step holds the twist in its own
    # tangent, and the product of such steps turns it at second order (2.6e-6 rad here)
    G = O.from_array(got)
    assert np.max(np.abs(G[1][o] - S[1][o])) <= 1e-6
    assert abs(A.yaw_about(G[0][o], S[0][o], UP) - A.yaw_about(want2[0][0], S[0][o], UP)) <= 1e-6


# ---- e. bits -----------------------------------------------------------------------------------------------------------------
def _bits(ba):
    return ba.GetKeyframeStates()[0].view(np.uint32).copy()


def _loop_graph(K):
    truth, start = PG._circle(K, seed=K + 4)
    return start, _constraints(truth, [(5, K - 3)] + O.random_loops(K, 4, seed=K))


@pytest.mark.parametrize("K", [1025, 2500])
def test_same_bits_across_modes_and_handles(K):
    start, cons = _loop_graph(K)
    outs = []
    for det in (False, True, False):
        ba = PG.make_handle(K, deterministic=det)
        ba.SetKeyframeStates(start)
        _add(ba, cons)
        r = ba.OptimizePoseGraph()
        outs.append((_bits(ba), r))
        del ba
    print(f"e K={K}: {outs[0][1]}")
    assert outs[0][1]["converged"] == 1
    for bits, r in outs[1:]:
        assert np.array_equal(bits, outs[0][0]) and r == outs[0][1]


def test_regrown_buffers_give_the_bits_of_a_fresh_handle():
    """A first call with one constraint reserves the pose graph's buffers for two; 300 more constraints grow them."""
    K = 1025
    start, _ = _loop_graph(K)
    truth = O.circle(K)
    cons = _constraints(truth, O.random_loops(K, 301, seed=5))
    ba = PG.make_handle(K)
    ba.SetKeyframeStates(start)
    _add(ba, cons[:1])
    ba.OptimizePoseGraph(max_iterations=3)
    _add(ba, cons[1:])
    ba.SetKeyframeStates(start)
    r = ba.OptimizePoseGraph(max_iterations=3)
    fresh = PG.make_handle(K)
    fresh.SetKeyframeStates(start)
    _add(fresh, cons)
    rf = fresh.OptimizePoseGraph(max_iterations=3)
    assert r["iterations"] >= 1 and r["final_cost"] < r["initial_cost"], r
    assert np.array_equal(_bits(ba), _bits(fresh)) and r == rf, (r, rf)


def test_room_for_more_keyframes_gives_the_same_bits():
    """prev and the solver's workspace sit at offsets of max_keyframes, not of K."""
    from badslam_b200.direct_ba import DirectBA
    K = 2049
    start, cons = _loop_graph(K)
    outs = []
    for capacity in (K, 2600):
        ba = DirectBA.from_scene(PG._images(), device="cuda:0", max_keyframes=capacity)
        PG._add_keyframes(ba, K)
        ba.SetKeyframeStates(start)
        _add(ba, cons)
        r = ba.OptimizePoseGraph()
        outs.append((_bits(ba), r))
        del ba
    assert outs[0][1]["converged"] == 1
    assert np.array_equal(outs[0][0], outs[1][0]) and outs[0][1] == outs[1][1], (outs[0][1], outs[1][1])
