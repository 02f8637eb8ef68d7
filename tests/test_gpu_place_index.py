"""GPU: the randomized-fern place index (bba_index_keyframes, bba_query_place_index, bba_get_place_index_codes; DESIGN §3.18).

* codes: equal the numpy oracle bit for bit on tiny, small, rig_half, rig_same, cfg1 (exactly 80 x 60) and a 640 x 480 image
  pair with holes in its depth, in the default and the deterministic mode; encoding a frame gives the code of the same images
  added as a keyframe;
* queries: equal the oracle for ranges, ties, max_matches above the candidate count, empty ranges and keyframe and frame queries
  mixed in one call;
* scale: 2 500 keyframes at 80 x 60 and an all-pairs query in one call equal the oracle;
* options: new options reset the index; bba_update_keyframe_host and a re-index change exactly that keyframe's code;
* refused calls change nothing, the launch counter included; successful calls launch what the header says;
* a query on a front-end thread while a BA runs equals the same query on a quiet handle;
* loop closure end to end on the drifted `small` scene with six loop keyframes around keyframe 0: the index's best match of the
  current loop keyframe among the keyframes before the loop is keyframe 0, verification from the identity accepts it, and the
  constraint, pose graph, surfel deformation and BA end as close to the truth as with the true relative pose; the verification
  from the identity of every loop keyframe is reported;
* relocalisation: frames within LOOP_MOTIONS of keyframe 3, lost at keyframe 0's pose, are recovered to 1 cm / 0.5 deg from the
  poses of their best matches as hypotheses, which the lost pose alone does not achieve.
"""
import threading

import numpy as np
import pytest

import loop_verification_oracle as LV
import place_index_oracle as O

pytestmark = pytest.mark.gpu

LOOP_MOTIONS = [   # tests/test_gpu_loop_verification.py
    [-0.04, 0.01, 0.00, 0.000, 0.010, -0.005],
    [-0.02, 0.00, 0.01, 0.008, 0.000, 0.004],
    [0.00, -0.01, 0.00, -0.005, 0.006, 0.000],
    [0.02, 0.01, -0.01, 0.004, -0.008, 0.006],
    [0.04, 0.00, 0.01, -0.006, 0.004, -0.008],
    [0.01, -0.02, 0.02, 0.012, -0.010, 0.015],
]
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)


def to_dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


def scene(name):
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name(name))


def handle(sc, **kw):
    from badslam_b200.direct_ba import DirectBA
    return DirectBA.from_scene(sc, poses=sc.poses_true, device="cuda:0", **kw)


def oracle_codes(depths, colors, F=512, lo=0.5, hi=3.0, raw_to_float=1e-3):
    cells, thr = O.ferns(F, *O.raw_range(lo, hi, raw_to_float))
    return np.stack([O.encode(d, c, cells, thr) for d, c in zip(depths, colors)])


@pytest.mark.parametrize("name", ["tiny", "small", "rig_half", "rig_same", "cfg1"])
@pytest.mark.parametrize("deterministic", [False, True], ids=["default", "deterministic"])
def test_codes_equal_the_oracle(name, deterministic):
    sc = scene(name)
    ba = handle(sc)
    ba.SetDeterministic(deterministic)
    K = len(sc.depth)
    ba.IndexKeyframes(num_ferns=256)
    got = ba.PlaceIndexCodes(np.arange(K))
    want = oracle_codes(sc.depth, sc.color, F=256, raw_to_float=sc.cfg.raw_to_float_depth)
    assert got.shape == want.shape and np.array_equal(got, want)
    # the default options (512 ferns) reset the index and give the oracle's codes too
    ba.IndexKeyframes()
    assert np.array_equal(ba.PlaceIndexCodes(np.arange(K)), oracle_codes(sc.depth, sc.color, raw_to_float=sc.cfg.raw_to_float_depth))


def test_frame_code_equals_keyframe_code_at_640x480_with_holes():
    sc = scene("cfg2")
    ba = handle(sc, max_keyframes=len(sc.depth) + 1)
    rng = np.random.default_rng(5)
    depth = sc.depth[0].copy()
    depth[rng.random(depth.shape) < 0.3] |= 0x8000   # scattered holes
    depth[100:220, 200:400] |= 0x8000                # and a block of whole cells without depth
    kid = ba.AddKeyframeHost(depth, sc.normals[0], sc.radius[0], sc.color[0], sc.poses_true[0], 0.3, 10.0)
    for det in (False, True):
        ba.SetDeterministic(det)
        ba.IndexKeyframes(num_ferns=2048, min_depth=0.3, max_depth=10.0)
        got = ba.PlaceIndexCodes([0, kid])
        want = oracle_codes([sc.depth[0], depth], [sc.color[0], sc.color[0]], F=2048, lo=0.3, hi=10.0)
        assert np.array_equal(got, want)
        # the same images as a frame: difference 0 to the keyframe (and only to it among ties it could have)
        frame = (to_dev(depth), None, to_dev(sc.color[0]))
        (ids, diffs), = ba.QueryPlaceIndex([(-1, 0, 0, kid)], frames=[frame], max_matches=4)
        assert ids[0] == kid and diffs[0] == 0
        assert list(diffs[1:]) == [O.difference(want[1], ba.PlaceIndexCodes([k])[0]) for k in ids[1:]]


class Indexed:
    """`small` with copies of keyframes 1 and 3 appended (ties at difference 0) and renders near keyframes 0 and 2 as frames."""

    def __init__(self):
        from badslam_b200.scene import render_frame, se3_exp, se3_mul
        self.sc = sc = scene("small")
        self.ba = ba = handle(sc, max_keyframes=16)
        for k in (1, 3, 1):
            ba.AddKeyframeHost(sc.depth[k], sc.normals[k], sc.radius[k], sc.color[k], sc.poses_true[k], sc.min_depth[k], sc.max_depth[k])
        self.K = ba.KeyframeCount()
        self.frames, self.frame_codes = [], []
        cells, thr = O.ferns(512, 500, 3000)
        for base, m in [(0, LOOP_MOTIONS[0]), (2, LOOP_MOTIONS[3])]:
            d, n, _, c = render_frame(sc, se3_mul(sc.poses_true[base], se3_exp(m)).astype(np.float32))
            self.frames.append((to_dev(d), to_dev(n), to_dev(c)))
            self.frame_codes.append(O.encode(d, c, cells, thr))
        ba.IndexKeyframes()
        self.codes = ba.PlaceIndexCodes(np.arange(self.K))
        self.indexed = np.ones(self.K, bool)

    def oracle(self, q, max_matches):
        kf, frame, first, last = q
        code = self.codes[kf] if kf >= 0 else self.frame_codes[frame]
        return O.query(self.codes, self.indexed, code, first, last, kf, max_matches)


@pytest.fixture(scope="module")
def indexed():
    return Indexed()


def test_queries_equal_the_oracle(indexed):
    ix = indexed
    K = ix.K
    assert np.array_equal(ix.codes, oracle_codes(list(ix.sc.depth) + [ix.sc.depth[k] for k in (1, 3, 1)],
                                                  list(ix.sc.color) + [ix.sc.color[k] for k in (1, 3, 1)]))
    queries = [
        (1, 0, 0, K - 1),       # ties at 0: keyframes 6 and 8 (copies of 1), by id
        (6, 0, 0, K - 1),       # the copy: 1 and 8 tie
        (3, 0, 2, 7),           # a range
        (0, 0, 1, 1),           # one candidate
        (2, 0, 5, 4),           # empty (first > last)
        (4, 0, 4, 4),           # empty (only itself)
        (-1, 0, 0, K - 1),      # a frame near keyframe 0
        (-1, 1, -10, 1000),     # a frame near keyframe 2, range clipped
        (5, 0, -3, 100),        # clipped
        (-1, 0, 1, K - 1),      # keyframe 0 outside the range
    ]
    for m in (1, 3, 8, 64):
        got = ix.ba.QueryPlaceIndex(queries, frames=ix.frames, max_matches=m)
        for q, (ids, diffs) in zip(queries, got):
            want = ix.oracle(q, m)
            assert np.array_equal(ids, want[0]) and np.array_equal(diffs, want[1]), (q, m, ids, diffs, want)
    got = ix.ba.QueryPlaceIndex(queries[:2], max_matches=3)
    assert list(got[0][0][:2]) == [6, 8] and list(got[1][0][:2]) == [1, 8]
    assert got[0][1][0] == 0 and got[1][1][1] == 0
    # the frames' best matches are the keyframes they revisit
    got = ix.ba.QueryPlaceIndex([(-1, 0, 0, K - 1), (-1, 1, 0, K - 1)], frames=ix.frames, max_matches=2)
    assert got[0][0][0] == 0 and got[1][0][0] == 2
    # one query per call gives the same as all together
    for q in queries:
        one, = ix.ba.QueryPlaceIndex([q], frames=ix.frames, max_matches=8)
        want = ix.oracle(q, 8)
        assert np.array_equal(one[0], want[0]) and np.array_equal(one[1], want[1])


def test_few_ferns_and_huge_ranges(indexed):
    """Rows of fewer words than lanes (8 and 64 ferns) match like the oracle, and a range starting near INT_MAX is empty."""
    ix = indexed
    K = ix.K
    try:
        for F in (8, 64):
            ix.ba.IndexKeyframes(num_ferns=F)
            assert ix.ba.PlaceIndexOptions() == (F, 500, 3000)
            codes = ix.ba.PlaceIndexCodes(np.arange(K))
            assert codes.shape == (K, F // 8)
            assert np.array_equal(codes, oracle_codes(list(ix.sc.depth) + [ix.sc.depth[k] for k in (1, 3, 1)],
                                                      list(ix.sc.color) + [ix.sc.color[k] for k in (1, 3, 1)], F=F))
            queries = [(k, 0, 0, K - 1) for k in range(K)] + [(2, 0, 3, 7)]
            for (ids, diffs), (kf, _, first, last) in zip(ix.ba.QueryPlaceIndex(queries, max_matches=5), queries):
                want = O.query(codes, ix.indexed, codes[kf], first, last, kf, 5)
                assert np.array_equal(ids, want[0]) and np.array_equal(diffs, want[1]), (F, kf)
    finally:
        ix.ba.IndexKeyframes()
    huge = 2 ** 31 - 100
    got = ix.ba.QueryPlaceIndex([(0, 0, huge, 5), (0, 0, huge, 2 ** 31 - 1), (-1, 0, huge, -huge), (1, 0, -huge, huge)],
                                frames=ix.frames)
    assert [len(ids) for ids, _ in got] == [0, 0, 0, 8]
    want = ix.oracle((1, 0, 0, K - 1), 8)
    assert np.array_equal(got[3][0], want[0]) and np.array_equal(got[3][1], want[1])


def test_launch_counts_and_refused_calls(indexed):
    from badslam_b200 import _lib as L
    from badslam_b200._lib import BadBAError
    ix = indexed
    ba, K = ix.ba, ix.K
    n = ba.kernel_launch_count()
    ba.QueryPlaceIndex([(0, 0, 0, K - 1)])
    assert ba.kernel_launch_count() - n == 1                      # matching only
    n = ba.kernel_launch_count()
    ba.QueryPlaceIndex([(0, 0, 0, K - 1), (-1, 1, 0, K - 1), (-1, 0, 0, 3)], frames=ix.frames)
    assert ba.kernel_launch_count() - n == 2                      # one encoding launch for both frames + matching
    n = ba.kernel_launch_count()
    ba.IndexKeyframes(ids=[2, 4])
    assert ba.kernel_launch_count() - n == 1
    n = ba.kernel_launch_count()
    ba.PlaceIndexCodes([0, 1])
    assert ba.kernel_launch_count() == n
    codes = ba.PlaceIndexCodes(np.arange(K))
    assert np.array_equal(codes, ix.codes)

    bad_queries = [
        ([(K, 0, 0, K - 1)], {}),                       # not published
        ([(-2, 0, 0, K - 1)], {}),                      # bad keyframe_id
        ([(-1, 2, 0, K - 1)], dict(frames=ix.frames)),  # frame out of range
        ([(-1, 0, 0, K - 1)], {}),                      # no frames
        ([(0, 0, 0, K - 1)], dict(max_matches=0)),
        ([(0, 0, 0, K - 1)], dict(max_matches=65)),
        ([(0, 0, 0, K - 1), (K + 2, 0, 0, 1)], {}),
    ]

    for qs, kw in bad_queries:
        with pytest.raises(BadBAError):
            ba.QueryPlaceIndex(qs, **kw)
        assert ba.kernel_launch_count() == n, (qs, kw)
    for ids, kw in [([K], {}), ([-1], {}), ([0], dict(num_ferns=12)), ([0], dict(num_ferns=4096)), ([0], dict(min_depth=4.0)),
                    ([0], dict(max_depth=40.0)), ([0], dict(min_depth=float("nan")))]:
        with pytest.raises(BadBAError):
            ba.IndexKeyframes(ids=ids, **kw)
        assert ba.kernel_launch_count() == n, (ids, kw)
    lib = ba._lib
    q = (L.PlaceQuery * 1)()
    out = np.zeros(8, np.int32)
    cnt = np.zeros(1, np.int32)
    assert lib.bba_query_place_index(ba._h, 0, None, 1, None, 8, out.ctypes.data, out.ctypes.data, cnt.ctypes.data, None) == L.ERR_INVALID_ARGUMENT
    assert lib.bba_query_place_index(ba._h, 0, None, 0, q, 8, out.ctypes.data, out.ctypes.data, cnt.ctypes.data, None) == L.ERR_INVALID_ARGUMENT
    assert lib.bba_query_place_index(ba._h, 0, None, 1, q, 8, None, out.ctypes.data, cnt.ctypes.data, None) == L.ERR_INVALID_ARGUMENT
    assert lib.bba_query_place_index(ba._h, -1, None, 1, q, 8, out.ctypes.data, out.ctypes.data, cnt.ctypes.data, None) == L.ERR_INVALID_ARGUMENT
    # frames the encoder could not read with aligned loads, or without an image
    depth, _, color = ix.frames[0]
    fq = (L.PlaceQuery * 1)()
    fq[0].keyframe_id, fq[0].frame, fq[0].first_keyframe, fq[0].last_keyframe = -1, 0, 0, K - 1
    for field, delta in [("color_rgba", 1), ("color_rgba", 2), ("color_pitch", 2), ("depth", 1), ("depth_pitch", 1), ("depth", None),
                         ("color_rgba", None), ("depth_pitch", -2), ("color_pitch", -4)]:
        fb = (L.FrameBuffers * 1)()
        fb[0].depth, fb[0].depth_pitch = depth.data_ptr(), depth.stride(0) * 2
        fb[0].color_rgba, fb[0].color_pitch = color.data_ptr(), color.stride(0)
        setattr(fb[0], field, None if delta is None else getattr(fb[0], field) + delta)
        assert lib.bba_query_place_index(ba._h, 1, fb, 1, fq, 8, out.ctypes.data, out.ctypes.data, cnt.ctypes.data, None) == \
            L.ERR_INVALID_ARGUMENT, (field, delta)
    assert lib.bba_get_place_index_codes(ba._h, 1, np.zeros(1, np.int32).ctypes.data, 32, out.ctypes.data, None) == L.ERR_INVALID_ARGUMENT
    assert lib.bba_index_keyframes(ba._h, None, 0, out.ctypes.data, None) == L.ERR_INVALID_ARGUMENT
    assert lib.bba_index_keyframes(ba._h, None, 1, None, None) == L.ERR_INVALID_ARGUMENT
    assert ba.kernel_launch_count() == n
    # the index is unchanged by every refused call
    assert np.array_equal(ba.PlaceIndexCodes(np.arange(K)), codes)
    # a handle without an index: BBA_ERR_STATE
    other = handle(scene("tiny"))
    n = other.kernel_launch_count()
    with pytest.raises(BadBAError) as e:
        other.QueryPlaceIndex([(0, 0, 0, 3)])
    assert e.value.status == L.ERR_STATE
    with pytest.raises(BadBAError) as e:
        other.PlaceIndexCodes([0])
    assert e.value.status == L.ERR_STATE
    assert other.kernel_launch_count() == n


def test_options_reset_and_reindex():
    from badslam_b200._lib import BadBAError
    sc = scene("small")
    ba = handle(sc)
    K = ba.KeyframeCount()
    ba.IndexKeyframes()
    before = ba.PlaceIndexCodes(np.arange(K))
    ba.IndexKeyframes(ids=[0, 2], num_ferns=512, min_depth=0.5, max_depth=2.0)   # new options: only 0 and 2 are indexed
    with pytest.raises(BadBAError):
        ba.PlaceIndexCodes([1])
    with pytest.raises(BadBAError):
        ba.QueryPlaceIndex([(1, 0, 0, K - 1)])
    (ids, _), = ba.QueryPlaceIndex([(0, 0, 0, K - 1)])
    assert list(ids) == [2]
    want = oracle_codes(sc.depth[[0, 2]], sc.color[[0, 2]], hi=2.0)
    assert np.array_equal(ba.PlaceIndexCodes([0, 2]), want)
    # the same options again keep the index: 0 and 2 stay, 1 joins
    ba.IndexKeyframes(ids=[1], num_ferns=512, min_depth=0.5, max_depth=2.0)
    assert len(ba.QueryPlaceIndex([(0, 0, 0, K - 1)])[0][0]) == 2
    # back to the defaults, then new images for keyframe 4: only its code changes after the re-index
    ba.IndexKeyframes()
    assert np.array_equal(ba.PlaceIndexCodes(np.arange(K)), before)
    ba_host = handle(sc, host_owned=True)
    ba_host.IndexKeyframes()
    assert np.array_equal(ba_host.PlaceIndexCodes(np.arange(K)), before)
    ba_host.UpdateKeyframeHost(4, depth=sc.depth[1], color=sc.color[1])
    assert np.array_equal(ba_host.PlaceIndexCodes(np.arange(K)), before)   # nothing is encoded automatically
    ba_host.IndexKeyframes(ids=[4])
    after = ba_host.PlaceIndexCodes(np.arange(K))
    changed = [k for k in range(K) if not np.array_equal(after[k], before[k])]
    assert changed == [4] and np.array_equal(after[4], before[1])


def test_all_pairs_at_2500_keyframes():
    """2 500 keyframes at 80 x 60 (random images, every tenth a copy of an earlier one) queried all against all in one call."""
    import torch
    sc = scene("cfg1")
    from badslam_b200.direct_ba import DirectBA
    N = 2500
    ba = DirectBA.from_scene(sc, poses=sc.poses_true, device="cuda:0", max_keyframes=N)
    rng = np.random.default_rng(11)
    depths, colors = list(sc.depth), list(sc.color)
    while len(depths) < N:
        k = len(depths)
        if k % 10 == 0:
            j = int(rng.integers(0, k))
            d, c = depths[j], colors[j]
        else:
            d = rng.integers(400, 3200, (60, 80)).astype(np.uint16)
            d[rng.random(d.shape) < 0.2] |= 0x8000
            c = rng.integers(0, 256, (60, 80, 4)).astype(np.uint8)
        ba.AddKeyframeHost(d, sc.normals[0], sc.radius[0], c, sc.poses_true[k % 2], 0.4, 3.2)
        depths.append(d)
        colors.append(c)
    ba.IndexKeyframes()
    codes = ba.PlaceIndexCodes(np.arange(N))
    sample = rng.choice(N, 100, replace=False)
    assert np.array_equal(codes[sample], oracle_codes([depths[k] for k in sample], [colors[k] for k in sample]))
    queries = [(k, 0, 0, N - 1) for k in range(N)]
    n = ba.kernel_launch_count()
    got = ba.QueryPlaceIndex(queries, max_matches=8)
    torch.cuda.synchronize()
    assert ba.kernel_launch_count() - n == 1
    D = O.differences_all_pairs(codes)
    indexed = np.ones(N, bool)
    for k in range(N):
        want = O.query_from_differences(D[k], indexed, 0, N - 1, k, 8)
        assert np.array_equal(got[k][0], want[0]) and np.array_equal(got[k][1], want[1]), k


def test_query_beside_a_running_ba(indexed):
    """A query on a front-end thread and stream while a BA runs on another equals the same query on a quiet handle."""
    import torch
    ix = indexed
    K = ix.K
    queries = [(k, 0, 0, K - 1) for k in range(K)] + [(-1, 0, 0, K - 1), (-1, 1, 0, K - 1)]
    quiet = ix.ba.QueryPlaceIndex(queries, frames=ix.frames, max_matches=8)
    lo, hi = torch.cuda.Stream.priority_range()
    ba_stream, fe_stream = torch.cuda.Stream(priority=lo), torch.cuda.Stream(priority=hi)
    started, results, errors = threading.Event(), [], []

    def progress(it):
        started.set()
        return 1

    def run_ba():
        try:
            ix.ba.BundleAdjustment(ba_stream, False, False, False, True, True, 6, 6, progress_function=progress)
        except Exception as e:   # reported below
            errors.append(e)
        finally:
            started.set()

    t = threading.Thread(target=run_ba)
    t.start()
    assert started.wait(300)
    while t.is_alive() and len(results) < 20:
        results.append(ix.ba.QueryPlaceIndex(queries, frames=ix.frames, max_matches=8, stream=fe_stream))
    t.join(300)
    assert not t.is_alive() and not errors, errors
    results.append(ix.ba.QueryPlaceIndex(queries, frames=ix.frames, max_matches=8, stream=fe_stream))
    for r in results:
        for (a, b), (c, d) in zip(r, quiet):
            assert np.array_equal(a, c) and np.array_equal(b, d)


def _aligned_error(poses, truth):
    from badslam_b200.scene import pose_error, se3_inverse, se3_mul
    align = se3_mul(truth[0], se3_inverse(poses[0]))
    return np.array([pose_error(se3_mul(align, poses[k]), truth[k]) for k in range(len(truth))]).mean(0)


def test_loop_closure_end_to_end_on_small():
    """test_gpu_loop_verification.py's loop (six keyframes rendered within LOOP_MOTIONS of keyframe 0 after `small`'s own) on
    test_gpu_pose_graph.py's drifted scene: every keyframe from K / 2 on, the loop keyframes included, moved rigidly about
    keyframe K / 2 - 1, with the map carried along.  The index finds keyframe 0 for the current (last) loop keyframe among the
    keyframes before the loop; verification from the identity accepts it; the verified edge, the pose graph, the surfel
    deformation and ten BA iterations then end as close to the truth as the same sequence with the true relative pose."""
    from badslam_b200 import _lib as L
    from badslam_b200.scene import render_frame, se3_exp, se3_inverse, se3_mul
    sc = scene("small")
    K = sc.cfg.num_keyframes
    loop_truth = [se3_mul(sc.poses_true[0], se3_exp(m)).astype(np.float32) for m in LOOP_MOTIONS]
    truth = np.concatenate([np.asarray(sc.poses_true, np.float32), np.array(loop_truth)])
    n = len(truth)
    current = n - 1
    D = se3_exp([0.12, -0.08, 0.06, 0.03, -0.04, 0.05])
    pivot = sc.poses_true[K // 2 - 1]
    move = se3_mul(se3_mul(pivot, D), se3_inverse(pivot))
    drifted = np.array([truth[k] if k < K // 2 else se3_mul(move, truth[k]) for k in range(n)], np.float32)
    images = [render_frame(sc, p) for p in loop_truth]

    def setup():
        ba = handle(sc, max_keyframes=n)
        for p, (d, nrm, r, c) in zip(loop_truth, images):
            valid = d[(d & 0x8000) == 0] * sc.cfg.raw_to_float_depth
            ba.AddKeyframeHost(d, nrm, r, c, p, float(valid.min()), float(valid.max()))
        original = ba.RememberKeyframePoses()
        ba.SetKeyframeStates(drifted)
        ba.DeformSurfelsWithKeyframePoseChanges(original)
        return ba

    def close(ba, Z):
        ba.AddKeyframePoseConstraints([0], [current], [Z], np.diag([1e4] * 3 + [1e5] * 3))
        remembered = ba.RememberKeyframePoses()
        r = ba.OptimizePoseGraph()
        assert r["final_cost"] < r["initial_cost"]
        ba.DeformSurfelsWithKeyframePoseChanges(remembered)
        ba.BundleAdjustment(None, False, False, False, True, True, 10, 10)
        return _aligned_error(ba.GetKeyframeStates()[0], truth)

    ba = setup()
    ba.IndexKeyframes()
    (ids, diffs), = ba.QueryPlaceIndex([(current, 0, 0, K - 1)], max_matches=3)
    print(f"loop query: matches {list(ids)}, differences {list(diffs)} of 512")
    assert ids[0] == 0
    # verification from the identity, for every loop keyframe as the current one (a report; the assertion is on the last)
    cands = [(K + j, 0, IDENT) for j in range(len(LOOP_MOTIONS))]
    verified = ba.VerifyLoopClosures(None, cands, num_scales=5)
    for j, v in enumerate(verified):
        true_cur_T_old = se3_mul(se3_inverse(truth[K + j]), truth[0])
        dt, dr = LV.same_pose(v.cur_T_old, true_cur_T_old)
        print(f"identity start, loop keyframe {j} ({LOOP_MOTIONS[j]}): {L.LOOP_STATUS_NAMES[v.status]}, agreement "
              f"{v.translation_difference * 1e3:.1f} mm / {np.degrees(v.angle_difference):.2f} deg, cur_T_old off the truth by "
              f"{dt * 1e3:.1f} mm / {np.degrees(dr):.3f} deg")
    v = verified[-1]
    assert v.status == L.LOOP_ACCEPTED, L.LOOP_STATUS_NAMES[v.status]
    from_index = close(ba, se3_inverse(np.array(v.cur_T_old, np.float64)).astype(np.float32))
    with_truth = close(setup(), se3_mul(se3_inverse(truth[0]), truth[current]).astype(np.float32))
    print(f"mean keyframe error after BA: true relative pose {with_truth}, index + identity + verification {from_index}")
    assert from_index[0] <= with_truth[0] * 1.05 + 1e-5 and from_index[1] <= with_truth[1] * 1.05 + 1e-6, (from_index, with_truth)


def test_relocalisation_on_small():
    """Frames rendered at keyframe 3's pose times each of LOOP_MOTIONS, lost at keyframe 0's pose: the query's best matches give
    the hypotheses of one bba_estimate_frame_poses_for_frames call, the one with the most associations is kept (INTEGRATION.md),
    and it lies within 1 cm / 0.5 deg of the truth; tracking from the lost pose alone does not get there."""
    from badslam_b200.scene import pose_error, render_frame, se3_exp, se3_mul
    sc = scene("small")
    K = sc.cfg.num_keyframes
    ba = handle(sc, max_keyframes=K + 32)
    ba.IndexKeyframes()
    truths, frames = [], []
    for m in LOOP_MOTIONS:
        p = se3_mul(sc.poses_true[3], se3_exp(m)).astype(np.float32)
        d, n, _, c = render_frame(sc, p)
        truths.append(p)
        frames.append((to_dev(d), to_dev(n), to_dev(c)))
    matches = ba.QueryPlaceIndex([(-1, f, 0, ba.KeyframeCount() - 1) for f in range(len(frames))], frames=frames, max_matches=4)
    assert all(ids[0] == 3 for ids, _ in matches), [list(ids) for ids, _ in matches]
    published = ba.GetKeyframeStates()[0]
    hyps = np.concatenate([published[ids] for ids, _ in matches])
    frame_of_entry = np.concatenate([np.full(len(ids), f) for f, (ids, _) in enumerate(matches)])
    est, _, _, at = ba.EstimateFramePosesFromBuffers(None, frames, hyps, frame_of_entry=frame_of_entry, with_coeffs=True)
    lost, _, _ = ba.EstimateFramePosesFromBuffers(None, frames, np.repeat(np.asarray(sc.poses_true[0:1], np.float32), len(frames), 0))
    for f in range(len(frames)):
        rows = np.flatnonzero(frame_of_entry == f)
        best = rows[int(np.argmax([at[r].n_assoc for r in rows]))]
        dt, dr = pose_error(est[best], truths[f])
        lt, lr = pose_error(lost[f], truths[f])
        print(f"frame {f}: hypotheses {list(matches[f][0])}, kept {frame_of_entry[best]}/{best}: {dt * 1e3:.2f} mm / "
              f"{np.degrees(dr):.3f} deg; from the lost pose {lt * 1e3:.1f} mm / {np.degrees(lr):.2f} deg")
        assert dt < 0.01 and dr < np.radians(0.5), (f, dt, dr)
        assert lt > 0.01 or lr > np.radians(0.5), (f, lt, lr)
