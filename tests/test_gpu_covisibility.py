"""GPU: keyframe co-visibility (bba_measure_keyframe_covisibility, DESIGN.md §3.19) against the numpy oracle
(tests/covisibility_oracle.py) and its exact invariants.

The kernels decide the association test with fast maths, so a pair within rounding of a threshold may go the other way: every
oracle comparison allows |got - want| <= near[a][b] (the surfels near a threshold for keyframe a or b) and asserts that near is a
small fraction of the evidence.  Everything else is exact:

1. against the oracle on tiny, small, many (37 keyframes: 32 + 5 around the geometry group), rig_half and small after a surfel
   deformation of the drifted halves;
2. C == C^T, C[a][b] <= min(C[a][a], C[b][b]), and rows of subsets and repeated ids equal those of the all-pairs call;
3. the Gram kernel's 64-wide tile edges: 63, 64, 65 and 129 copies of cfg1's keyframes;
4. the same bits for a permutation of the surfels, forced chunks, the deterministic mode, two and three ranks, repeated calls;
5. surfel counts around warp and tile edges, deleted surfels, a keyframe that sees nothing;
6. nothing on the handle changes, a later deterministic BA iteration is the same bits, the launch counts;
7. refused arguments;
8. the place-index loop scene: the loop keyframe shares few surfels with keyframe 0 before the closure and many after it, and the
   candidate filter removes the current keyframe's neighbours but keeps keyframe 0."""
import copy
import ctypes as C

import numpy as np
import pytest

import covisibility_oracle as O
import surfel_deform_oracle as D

pytestmark = pytest.mark.gpu

_CACHE = {}


def _scene(name):
    if name not in _CACHE:
        from badslam_b200 import scene as S
        _CACHE[name] = S.make_scene(S.config_by_name(name))
    return _CACHE[name]


def _lib():
    from badslam_b200 import _lib
    return _lib.load()


def _f32(x):
    return np.ascontiguousarray(x, np.float32)


def _inverse(A):
    out = np.zeros(7, np.float32)
    _lib().bba_host_se3_inverse(_f32(A).ctypes.data, out.ctypes.data)
    return out


def _compose(A, B):
    out = np.zeros(7, np.float32)
    _lib().bba_host_se3_compose(_f32(A).ctypes.data, _f32(B).ctypes.data, out.ctypes.data)
    return out


def _exp(x):
    out = np.zeros(7, np.float32)
    _lib().bba_host_se3_exp(_f32(x).ctypes.data, out.ctypes.data)
    return out


def _make(sc, deterministic=False, **kw):
    from badslam_b200.direct_ba import DirectBA
    ba = DirectBA.from_scene(sc, device="cuda:0", **kw)
    if deterministic:
        ba.SetDeterministic(True)
    return ba


def _oracle(sc, ba, surfels=None, n=None):
    """The oracle at the handle's current poses on the scene's images and surfels."""
    poses = ba.GetKeyframeStates()[0]
    inv = np.stack([_inverse(p) for p in poses])
    s = sc.surfels if surfels is None else surfels
    return O.covisibility(D.Camera.of_scene(sc), sc.depth, sc.normals, s, sc.num_surfels if n is None else n, inv)


def _check_oracle(got, want, near):
    assert got.shape == want.shape
    diff = np.abs(got.astype(np.int64) - want)
    assert (diff <= near).all(), np.argwhere(diff > near)[:10]
    assert near.sum() <= max(4, 0.01 * want.sum()), (near.sum(), want.sum())


def _check_invariants(ba, C_all):
    K = len(C_all)
    assert np.array_equal(C_all, C_all.T)
    d = np.diag(C_all)
    assert (C_all <= np.minimum(d[:, None], d[None, :])).all()
    rng = np.random.default_rng(K)
    for ids in ([K - 1], list(range(K))[::2], list(rng.integers(0, K, 2 * K + 3))):
        assert np.array_equal(ba.MeasureKeyframeCovisibility(ids), C_all[ids])


# ---- 1. + 2. against the oracle, and the exact invariants ----------------------------------------------------------------------

@pytest.mark.parametrize("name", ["tiny", "small", "many", "rig_half"])
def test_against_oracle(name):
    sc = _scene(name)
    ba = _make(sc)
    got = ba.MeasureKeyframeCovisibility()
    want, near, _, _ = _oracle(sc, ba)
    print(f"{name}: K {len(got)}, total count {int(want.sum())}, near {int(near.sum())}, max |got - want| "
          f"{int(np.abs(got.astype(np.int64) - want).max())}")
    _check_oracle(got, want, near)
    _check_invariants(ba, got)


def test_after_deformation():
    """small with the keyframes >= K/2 moved by about 0.3 m and 20 degrees and the map deformed with them."""
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    ba = _make(sc)
    original = ba.RememberKeyframePoses()
    cur = np.array(sc.poses_init, np.float32, copy=True)
    G = _exp([0.2, -0.15, 0.16, 0.2, -0.2, 0.22])
    for k in range(K // 2, K):
        cur[k] = _compose(G, cur[k])
    ba.SetKeyframeStates(cur)
    ba.DeformSurfelsWithKeyframePoseChanges(original)
    got = ba.MeasureKeyframeCovisibility()
    rows = ba.GetSurfelsHost(17)
    want, near, _, _ = _oracle(sc, ba, surfels=rows)
    _check_oracle(got, want, near)
    _check_invariants(ba, got)


# ---- 3. Gram tile edges --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", [63, 64, 65, 129])
def test_gram_tile_edges(K):
    """cfg1's two keyframes added again and again at their own poses: every copy of a keyframe has its row and column, and shares
    all its surfels with the other copies."""
    sc = _scene("cfg1")
    base = sc.cfg.num_keyframes
    ba = _make(sc, max_keyframes=K)
    while ba.KeyframeCount() < K:
        k = ba.KeyframeCount() % base
        ba.AddKeyframeHost(sc.depth[k], sc.normals[k], sc.radius[k], sc.color[k], sc.poses_init[k], sc.min_depth[k], sc.max_depth[k])
    got = ba.MeasureKeyframeCovisibility()
    src = np.arange(K) % base
    for k in range(K):
        assert np.array_equal(got[k], got[src[k]][src]), k
        assert np.array_equal(got[:, k], got[:, src[k]]), k
        assert got[k, src[k]] == got[k, k] == got[src[k], src[k]] > 0
    assert np.array_equal(got[:base, :base], _make(sc).MeasureKeyframeCovisibility())


# ---- 4. independence -----------------------------------------------------------------------------------------------------------

def test_surfel_order():
    sc = _scene("small")
    n = sc.num_surfels
    a = _make(sc).MeasureKeyframeCovisibility()
    shuffled = copy.copy(sc)
    shuffled.surfels = np.array(sc.surfels, np.float32, copy=True)
    shuffled.surfels[:, :n] = sc.surfels[:, np.random.default_rng(9).permutation(n)]
    assert np.array_equal(_make(shuffled).MeasureKeyframeCovisibility(), a)


def test_chunks_modes_and_repeats():
    sc = _scene("many")
    ba = _make(sc)
    want = ba.MeasureKeyframeCovisibility()
    assert np.array_equal(ba.MeasureKeyframeCovisibility(), want)
    for chunk in (32, 4096, 100_000, 0):
        ba.DebugSetCovisibilityChunk(chunk)
        assert np.array_equal(ba.MeasureKeyframeCovisibility(), want), chunk
        assert np.array_equal(ba.MeasureKeyframeCovisibility([3, 36, 3]), want[[3, 36, 3]]), chunk
    det = _make(sc, deterministic=True)
    assert np.array_equal(det.MeasureKeyframeCovisibility(), want)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mode", ["gather", "peer"])
def test_local_group_ranks(world, mode):
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    sc = _scene("small")
    one = _make(sc).MeasureKeyframeCovisibility()
    handles = DirectBA.create_local_ranks(sc, world, ["cuda:0"] * world)
    with LocalGroup(handles, peer_stores=mode == "peer") as group:
        outs = group.run(lambda r, ba: ba.MeasureKeyframeCovisibility())
    for o in outs:
        assert np.array_equal(o, one)


# ---- 5. surfel-count edges -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("count", [1, 31, 32, 33, 255, 256, 257])
def test_surfel_counts(count):
    sc = copy.copy(_scene("small"))
    sc.num_surfels = count
    ba = _make(sc)
    got = ba.MeasureKeyframeCovisibility()
    want, near, _, _ = _oracle(sc, ba)
    assert (np.abs(got.astype(np.int64) - want) <= near).all()


def test_deleted_surfels_and_a_blind_keyframe():
    sc = copy.copy(_scene("small"))
    K = sc.cfg.num_keyframes
    sc.surfels = np.array(sc.surfels, np.float32, copy=True)
    sc.surfels[0, ::3] = np.nan
    sc.poses_init = np.array(sc.poses_init, np.float32, copy=True)
    sc.poses_init[K - 1] = _compose(_exp([0, 0, 50.0, 0, 0, 0]), sc.poses_init[K - 1])   # looks at nothing of the map
    ba = _make(sc)
    got = ba.MeasureKeyframeCovisibility()
    want, near, A, _ = _oracle(sc, ba)
    assert not A[::3].any()
    _check_oracle(got, want, near)
    assert not got[K - 1].any() and not got[:, K - 1].any()
    assert (np.diag(got)[:K - 1] > 0).all()


# ---- 6. nothing changes --------------------------------------------------------------------------------------------------------

def _state(ba):
    p, a = ba.GetKeyframeStates()
    return ba.GetSurfelsHost(17).tobytes(), ba.GetActiveHost().tobytes(), p.tobytes(), a.tobytes()


def test_nothing_changes_and_launch_counts():
    sc = _scene("many")
    ba = _make(sc)
    ba.SetKeyframeStates(activations=np.array([0, 1, 2] * 12 + [0], np.int32))
    before = _state(ba)
    ba.MeasureKeyframeCovisibility()   # (may build the spatial order)
    assert _state(ba) == before
    n = ba.kernel_launch_count()
    ba.MeasureKeyframeCovisibility()
    assert ba.kernel_launch_count() - n == 3   # stream gather, bits, Gram
    chunk = 4096
    ba.DebugSetCovisibilityChunk(chunk)
    n = ba.kernel_launch_count()
    ba.MeasureKeyframeCovisibility([0])
    assert ba.kernel_launch_count() - n == 3 * -(-sc.num_surfels // chunk)
    assert _state(ba) == before


def test_later_ba_is_the_same_bits():
    sc = _scene("small")
    runs = []
    for measure in (False, True):
        ba = _make(sc, deterministic=True)
        if measure:
            ba.MeasureKeyframeCovisibility()
        ba.BundleAdjustment(None, False, False, False, True, True, 1, 1)
        runs.append(_state(ba))
    assert runs[0] == runs[1]


def test_empty_map_launches_nothing():
    sc = copy.copy(_scene("tiny"))
    sc.num_surfels = 0
    ba = _make(sc)
    n = ba.kernel_launch_count()
    got = ba.MeasureKeyframeCovisibility()
    assert got.shape == (sc.cfg.num_keyframes,) * 2 and not got.any()
    assert ba.kernel_launch_count() == n


# ---- 7. refusals ---------------------------------------------------------------------------------------------------------------

def test_refusals():
    from badslam_b200 import _lib as L
    sc = _scene("tiny")
    K = sc.cfg.num_keyframes
    ba = _make(sc)
    before = ba.kernel_launch_count(), _state(ba)
    lib = _lib()
    out = np.zeros((2 * K, K), np.uint32)
    ids = np.array([0, 1], np.int32)
    bad = np.array([0, K], np.int32)
    neg = np.array([-1], np.int32)
    for count, i, kc, o in [(2, ids, K, None), (2, None, K, out), (0, ids, K, out), (-2, ids, K, out), (2, bad, K, out),
                            (1, neg, K, out), (2, ids, K - 1, out), (-1, None, K + 1, out)]:
        st = lib.bba_measure_keyframe_covisibility(ba._h, count, None if i is None else i.ctypes.data, kc,
                                                   None if o is None else o.ctypes.data, None)
        assert st == L.ERR_INVALID_ARGUMENT, (count, i, kc)
        assert (ba.kernel_launch_count(), _state(ba)) == before
    assert not out.any()


# ---- 8. the loop scene ---------------------------------------------------------------------------------------------------------

LOOP_MOTIONS = [   # tests/test_gpu_loop_verification.py
    [-0.04, 0.01, 0.00, 0.000, 0.010, -0.005],
    [-0.02, 0.00, 0.01, 0.008, 0.000, 0.004],
    [0.00, -0.01, 0.00, -0.005, 0.006, 0.000],
    [0.02, 0.01, -0.01, 0.004, -0.008, 0.006],
    [0.04, 0.00, 0.01, -0.006, 0.004, -0.008],
    [0.01, -0.02, 0.02, 0.012, -0.010, 0.015],
]
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
# From the counts this scene gives (DESIGN §3.19): the loop keyframe shares few surfels with keyframe 0 before the closure and
# many after it; a candidate that shares more than SHARED_NEIGHBOUR surfels with the current keyframe is its neighbour.
SHARED_NEIGHBOUR = 0.25   # of the current keyframe's own count


def test_loop_scene():
    """test_gpu_place_index.py's loop on the drifted `small` scene: six loop keyframes rendered around keyframe 0, every keyframe
    from K / 2 on moved rigidly with the map.  The query's candidates for the current (last) loop keyframe are filtered by the
    surfels they share with it; the verified edge, the pose graph and the surfel deformation then close the loop."""
    from badslam_b200 import _lib as L
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import render_frame, se3_exp, se3_inverse, se3_mul
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    loop_truth = [se3_mul(sc.poses_true[0], se3_exp(m)).astype(np.float32) for m in LOOP_MOTIONS]
    truth = np.concatenate([np.asarray(sc.poses_true, np.float32), np.array(loop_truth)])
    n = len(truth)
    current = n - 1
    Dm = se3_exp([0.12, -0.08, 0.06, 0.03, -0.04, 0.05])
    pivot = sc.poses_true[K // 2 - 1]
    move = se3_mul(se3_mul(pivot, Dm), se3_inverse(pivot))
    drifted = np.array([truth[k] if k < K // 2 else se3_mul(move, truth[k]) for k in range(n)], np.float32)
    ba = DirectBA.from_scene(sc, poses=sc.poses_true, device="cuda:0", max_keyframes=n)
    for p in loop_truth:
        d, nrm, r, c = render_frame(sc, p)
        valid = d[(d & 0x8000) == 0] * sc.cfg.raw_to_float_depth
        ba.AddKeyframeHost(d, nrm, r, c, p, float(valid.min()), float(valid.max()))
    original = ba.RememberKeyframePoses()
    ba.SetKeyframeStates(drifted)
    ba.DeformSurfelsWithKeyframePoseChanges(original)

    before = ba.MeasureKeyframeCovisibility([current])[0]
    ba.IndexKeyframes()
    (ids, _), = ba.QueryPlaceIndex([(current, 0, 0, n - 2)], max_matches=8)
    limit = SHARED_NEIGHBOUR * before[current]
    kept = [int(k) for k in ids if before[k] <= limit]
    print(f"before the closure: counts with the current keyframe {list(before)}; candidates {list(ids)}, kept {kept}")
    assert 0 in ids and 0 in kept
    assert all(k >= K or before[k] > limit for k in ids if k not in kept)
    assert any(k >= K for k in ids if k not in kept)   # the current keyframe's own neighbours go

    v, = ba.VerifyLoopClosures(None, [(current, 0, IDENT)], num_scales=5)
    assert v.status == L.LOOP_ACCEPTED, L.LOOP_STATUS_NAMES[v.status]
    ba.AddKeyframePoseConstraints([0], [current], [se3_inverse(np.array(v.cur_T_old, np.float64)).astype(np.float32)],
                                  np.diag([1e4] * 3 + [1e5] * 3))
    remembered = ba.RememberKeyframePoses()
    ba.OptimizePoseGraph()
    ba.DeformSurfelsWithKeyframePoseChanges(remembered)
    after = ba.MeasureKeyframeCovisibility([current])[0]
    print(f"after the closure: counts with the current keyframe {list(after)}")
    assert after[0] > 4 * max(before[0], 1) and after[0] > SHARED_NEIGHBOUR * after[current]
