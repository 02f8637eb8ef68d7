"""GPU: the frame overlap measurement (bba_measure_frame_overlap, DESIGN.md §3.20) against its defining property, the keyframe
co-visibility call, the numpy oracle (tests/frame_overlap_oracle.py) and its exact invariants:

1. a query made of keyframe k's own images at k's pose gives k's row of MeasureKeyframeCovisibility and its diagonal, and matches
   the oracle within its near counts on tiny and small;
2. the defining property: frames rendered between and beyond the keyframes are measured, then added as keyframes, and surfel
   creation on them creates exactly uncovered_cells surfels unfiltered and new_surfels filtered;
3. repeated frames and queries and the Gram kernel's 64-wide tile edges (63, 64, 65, 129 queries);
4. the same bits for forced chunks, a permutation of the surfels, the deterministic mode, two and three ranks;
5. surfel counts around warp and tile edges, deleted surfels, an empty map, a handle without keyframes;
6. nothing on the handle changes; the launch counts;
7. refused arguments;
8. along a path leaving a keyframe's view, the uncovered share of the frame grows."""
import copy
import dataclasses

import numpy as np
import pytest

import frame_overlap_oracle as O
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


def _make(sc, deterministic=False, **kw):
    from badslam_b200.direct_ba import DirectBA
    ba = DirectBA.from_scene(sc, device="cuda:0", **kw)
    if deterministic:
        ba.SetDeterministic(True)
    return ba


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).cuda()


def _kf_frames(sc):
    """Every keyframe's (depth, normals) as device tensors."""
    return [(_dev(sc.depth[k]), _dev(sc.normals[k])) for k in range(sc.cfg.num_keyframes)]


def _kf_queries(sc, ba):
    poses = ba.GetKeyframeStates()[0]
    return [(k, poses[k], sc.min_depth[k], sc.max_depth[k]) for k in range(sc.cfg.num_keyframes)]


def _depth_range(sc, depth):
    valid = depth[(depth & 0x8000) == 0].astype(np.float32) * np.float32(sc.cfg.raw_to_float_depth)
    return float(valid.min()), float(valid.max())


def _render(sc, pose):
    from badslam_b200.scene import render_frame
    d, n, r, c = render_frame(sc, np.asarray(pose, np.float32))
    return d, n, r, c, _depth_range(sc, d)


def _path_poses(sc, count=6):
    """Poses between consecutive keyframes and beyond the last one."""
    from badslam_b200.scene import se3_exp, se3_mul
    P = np.asarray(sc.poses_true, np.float32)
    out = []
    for i in range(count):
        a, b = P[i % len(P)], P[(i + 1) % len(P)]
        mid = np.concatenate([a[:4], 0.5 * (a[4:] + b[4:])]).astype(np.float32)
        out.append(mid if i % 2 == 0 else se3_mul(b, se3_exp([0.05 * (i - 3), 0.03, -0.04, 0.02, -0.03 * i, 0.01])).astype(np.float32))
    return out


def _tuple(r):
    return (r.observed_surfels.tobytes(), r.valid_cells.tobytes(), r.uncovered_cells.tobytes(), r.new_surfels.tobytes(),
            None if r.shared is None else r.shared.tobytes())


# ---- 1. keyframe queries -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["tiny", "small", "rig_half"])
def test_keyframe_queries_give_covisibility_rows(name):
    sc = _scene(name)
    K = sc.cfg.num_keyframes
    ba = _make(sc)
    C_all = ba.MeasureKeyframeCovisibility()
    r = ba.MeasureFrameOverlap(_kf_frames(sc), _kf_queries(sc, ba))
    assert np.array_equal(r.shared, C_all)
    assert np.array_equal(r.observed_surfels, np.diag(C_all))
    assert (r.new_surfels <= r.uncovered_cells).all() and (r.uncovered_cells <= r.valid_cells).all()
    assert (r.uncovered_cells < r.valid_cells).all()
    if name == "rig_half":
        return
    lib = _lib()
    cam = D.Camera.of_scene(sc)
    poses = ba.GetKeyframeStates()[0]
    Kd = _f32(sc.depth_K)
    counts = ba.min_observation_counts
    min_obs = counts[0] if K + 1 < 5 else counts[1] if K + 1 < 10 else counts[2]
    inv = np.stack([_inverse(p) for p in poses])
    for k in range(K):
        covis = []
        for b in range(K):
            if lib.bba_host_frusta_intersect(Kd.ctypes.data, sc.cfg.width, sc.cfg.height, _f32(poses[k]).ctypes.data, sc.min_depth[k],
                                             sc.max_depth[k], _f32(poses[b]).ctypes.data, sc.min_depth[b], sc.max_depth[b]):
                covis.append((D.quat_to_matrix_f32(_compose(inv[b], poses[k])), sc.depth[b], sc.normals[b]))
        want = O.frame_overlap(cam, sc.depth[k], sc.normals[k], inv[k], sc.surfels, sc.num_surfels, covis, min_obs,
                               keyframes=(list(sc.depth), list(sc.normals), inv))
        got = dict(observed=r.observed_surfels[k], valid=r.valid_cells[k], uncovered=r.uncovered_cells[k], new=r.new_surfels[k])
        print(f"{name} keyframe {k}: device {got}, oracle { {x: want[x] for x in got} }, near new {want['near_new']}")
        assert got["valid"] == want["valid"]
        for x in ("observed", "uncovered", "new"):
            assert abs(int(got[x]) - want[x]) <= want["near_" + ("observed" if x == "observed" else x)], (k, x)
        assert (np.abs(r.shared[k].astype(np.int64) - want["shared"]) <= want["near_shared"]).all(), k


def _inverse(A):
    out = np.zeros(7, np.float32)
    _lib().bba_host_se3_inverse(_f32(A).ctypes.data, out.ctypes.data)
    return out


def _compose(A, B):
    out = np.zeros(7, np.float32)
    _lib().bba_host_se3_compose(_f32(A).ctypes.data, _f32(B).ctypes.data, out.ctypes.data)
    return out


# ---- 2. the defining property --------------------------------------------------------------------------------------------------

def _roomy(name):
    """The scene with half its surfels (many unsupported cells) and room for the surfels one more keyframe creates."""
    sc = copy.copy(_scene(name))
    sc.num_surfels = sc.num_surfels // 2
    sc.surfels = np.pad(sc.surfels, ((0, 0), (0, (sc.cfactor.size + 127) // 128 * 128)))
    return sc


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_creation_creates_what_was_measured(name):
    sc = _roomy(name)
    K = sc.cfg.num_keyframes
    checked = 0
    for pose in _path_poses(sc):
        d, n, rad, c, (lo, hi) = _render(sc, pose)
        ba = _make(sc, max_keyframes=K + 1)
        r = ba.MeasureFrameOverlap([(_dev(d), _dev(n))], [(0, pose, lo, hi)], with_shared=False)
        assert r.shared is None
        for filt, want in ((False, r.uncovered_cells[0]), (True, r.new_surfels[0])):
            fresh = _make(sc, max_keyframes=K + 1)
            k = fresh.AddKeyframeHost(d, n, rad, c, pose, lo, hi)
            created = fresh.CreateSurfelsForKeyframe(None, filt, k)
            print(f"{name}: filter {int(filt)}: measured {int(want)} of {int(r.valid_cells[0])} valid cells, created {created}")
            assert created == want
        checked += int(r.new_surfels[0] > 0)
    assert checked >= 2


# ---- 3. repeats and the Gram tile edges ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("count", [63, 64, 65, 129])
def test_repeats_and_gram_tile_edges(count):
    sc = _scene("small")
    K = sc.cfg.num_keyframes
    ba = _make(sc)
    frames = _kf_frames(sc)
    base = ba.MeasureFrameOverlap(frames, _kf_queries(sc, ba))
    qs = _kf_queries(sc, ba)
    pick = np.random.default_rng(count).integers(0, K, count)
    r = ba.MeasureFrameOverlap(frames + frames[:1], [qs[i] for i in pick])
    for field in ("observed_surfels", "valid_cells", "uncovered_cells", "new_surfels", "shared"):
        assert np.array_equal(getattr(r, field), getattr(base, field)[pick]), field
    lean = ba.MeasureFrameOverlap(frames, [qs[i] for i in pick], with_shared=False)
    assert np.array_equal(lean.observed_surfels, r.observed_surfels) and np.array_equal(lean.new_surfels, r.new_surfels)


# ---- 4. independence -----------------------------------------------------------------------------------------------------------

def _path_call(sc, ba, shared=True):
    frames, queries = [], []
    for i, pose in enumerate(_path_poses(sc)):
        d, n, _, _, (lo, hi) = _render(sc, pose)
        frames.append((_dev(d), _dev(n)))
        queries.append((i, pose, lo, hi))
    return ba.MeasureFrameOverlap(frames, queries, with_shared=shared)


def test_chunks_order_and_modes():
    sc = _scene("small")
    ba = _make(sc)
    want = _tuple(_path_call(sc, ba))
    assert _tuple(_path_call(sc, ba)) == want
    for chunk in (32, 4096, 100_000, 0):
        ba.DebugSetCovisibilityChunk(chunk)
        assert _tuple(_path_call(sc, ba)) == want, chunk
    assert _tuple(_path_call(sc, _make(sc, deterministic=True))) == want
    shuffled = copy.copy(sc)
    shuffled.surfels = np.array(sc.surfels, np.float32, copy=True)
    n = sc.num_surfels
    shuffled.surfels[:, :n] = sc.surfels[:, np.random.default_rng(9).permutation(n)]
    assert _tuple(_path_call(sc, _make(shuffled))) == want


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mode", ["gather", "peer"])
def test_local_group_ranks(world, mode):
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    sc = _scene("small")
    one = _tuple(_make(sc).MeasureFrameOverlap(_kf_frames(sc), _kf_queries(sc, _make(sc))))
    handles = DirectBA.create_local_ranks(sc, world, ["cuda:0"] * world)
    frames = _kf_frames(sc)
    with LocalGroup(handles, peer_stores=mode == "peer") as group:
        outs = group.run(lambda r, ba: _tuple(ba.MeasureFrameOverlap(frames, _kf_queries(sc, ba))))
    for o in outs:
        assert o == one


# ---- 5. surfel-count edges, deleted surfels, empty map, no keyframes -----------------------------------------------------------

@pytest.mark.parametrize("count", [1, 31, 32, 33, 255, 256, 257])
def test_surfel_counts(count):
    sc = copy.copy(_scene("small"))
    sc.num_surfels = count
    ba = _make(sc)
    r = ba.MeasureFrameOverlap(_kf_frames(sc), _kf_queries(sc, ba))
    C_all = ba.MeasureKeyframeCovisibility()
    assert np.array_equal(r.shared, C_all) and np.array_equal(r.observed_surfels, np.diag(C_all))
    assert r.observed_surfels.sum() >= 1 or count < 32
    assert (r.uncovered_cells <= r.valid_cells).all() and (r.valid_cells - r.uncovered_cells <= r.observed_surfels).all()


def test_deleted_surfels():
    sc = copy.copy(_scene("small"))
    sc.surfels = np.array(sc.surfels, np.float32, copy=True)
    sc.surfels[0, ::3] = np.nan
    ba = _make(sc)
    r = ba.MeasureFrameOverlap(_kf_frames(sc), _kf_queries(sc, ba))
    assert np.array_equal(r.shared, ba.MeasureKeyframeCovisibility())
    full = _make(_scene("small"))
    f = full.MeasureFrameOverlap(_kf_frames(sc), _kf_queries(sc, full))
    assert (r.observed_surfels < f.observed_surfels).all() and (r.uncovered_cells >= f.uncovered_cells).all()


def test_empty_map_and_no_keyframes():
    from badslam_b200.direct_ba import DirectBA
    sc = copy.copy(_scene("tiny"))
    sc.num_surfels = 0
    K = sc.cfg.num_keyframes
    ba = _make(sc)
    n0 = ba.kernel_launch_count()
    r = ba.MeasureFrameOverlap(_kf_frames(sc), _kf_queries(sc, ba))
    assert ba.kernel_launch_count() - n0 == 1   # the seed count only
    assert not r.observed_surfels.any() and not r.shared.any() and r.shared.shape == (K, K)
    assert np.array_equal(r.uncovered_cells, r.valid_cells) and (r.valid_cells > 0).all()
    assert (r.new_surfels <= r.uncovered_cells).all()
    # no keyframes: shared is not written, nothing filters a seed but the observation count of the first keyframe (1: itself)
    empty = copy.copy(sc)
    empty.cfg = dataclasses.replace(sc.cfg, num_keyframes=0)
    bare = DirectBA.from_scene(empty, device="cuda:0", max_keyframes=K)
    assert bare.KeyframeCount() == 0
    lib = _lib()
    from badslam_b200 import _lib as L
    frames = _kf_frames(sc)
    bufs = (L.FrameBuffers * 1)()
    bufs[0].depth, bufs[0].depth_pitch = frames[0][0].data_ptr(), frames[0][0].stride(0) * 2
    bufs[0].normals, bufs[0].normals_pitch = frames[0][1].data_ptr(), frames[0][1].stride(0) * 2
    q = (L.FrameOverlapQuery * 1)()
    q[0].frame, q[0].global_T_frame[:], q[0].min_depth, q[0].max_depth = 0, list(map(float, sc.poses_init[0])), sc.min_depth[0], sc.max_depth[0]
    out = (L.FrameOverlap * 1)()
    sentinel = np.full(4, 7, np.uint32)
    assert lib.bba_measure_frame_overlap(bare._h, 1, bufs, 1, q, 0, sentinel.ctypes.data, out, None) == 0
    assert (sentinel == 7).all()
    assert out[0].observed_surfels == 0 and out[0].uncovered_cells == out[0].valid_cells == r.valid_cells[0]
    assert out[0].new_surfels == (out[0].uncovered_cells if ba.min_observation_counts[0] <= 1 else 0)


# ---- 6. nothing changes, launch counts -----------------------------------------------------------------------------------------

def _state(ba):
    p, a = ba.GetKeyframeStates()
    return (ba.GetSurfelsHost(17).tobytes(), ba.GetActiveHost().tobytes(), p.tobytes(), a.tobytes(), ba.covisibility().tobytes(),
            ba.KeyframeCount())


def test_nothing_changes_and_launch_counts():
    sc = _scene("small")
    ba = _make(sc)
    frames, qs = _kf_frames(sc), _kf_queries(sc, ba)
    ba.MeasureFrameOverlap(frames, qs)   # (may build the spatial order)
    before = _state(ba)
    n = ba.kernel_launch_count()
    ba.MeasureFrameOverlap(frames, qs)
    assert ba.kernel_launch_count() - n == 6   # 2 x (stream gather, bits), Gram, seed count
    n = ba.kernel_launch_count()
    ba.MeasureFrameOverlap(frames, qs, with_shared=False)
    assert ba.kernel_launch_count() - n == 4   # stream gather, bits, Gram, seed count
    chunk = 4096
    ba.DebugSetCovisibilityChunk(chunk)
    n = ba.kernel_launch_count()
    ba.MeasureFrameOverlap(frames, qs[:1], with_shared=False)
    assert ba.kernel_launch_count() - n == 3 * -(-sc.num_surfels // chunk) + 1
    assert _state(ba) == before


# ---- 7. refusals ---------------------------------------------------------------------------------------------------------------

def test_refusals():
    from badslam_b200 import _lib as L
    sc = _scene("tiny")
    K = sc.cfg.num_keyframes
    ba = _make(sc)
    frames = _kf_frames(sc)
    lib = _lib()
    ba.MeasureFrameOverlap(frames, _kf_queries(sc, ba))
    before = ba.kernel_launch_count(), _state(ba)

    def bufs(**change):
        b = (L.FrameBuffers * 1)()
        b[0].depth, b[0].depth_pitch = frames[0][0].data_ptr(), frames[0][0].stride(0) * 2
        b[0].normals, b[0].normals_pitch = frames[0][1].data_ptr(), frames[0][1].stride(0) * 2
        for k, v in change.items():
            setattr(b[0], k, v)
        return b

    def query(**change):
        q = (L.FrameOverlapQuery * 1)()
        q[0].frame, q[0].min_depth, q[0].max_depth = 0, sc.min_depth[0], sc.max_depth[0]
        q[0].global_T_frame[:] = list(map(float, sc.poses_init[0]))
        for k, v in change.items():
            if k == "pose":
                q[0].global_T_frame[:] = v
            else:
                setattr(q[0], k, v)
        return q

    out = (L.FrameOverlap * 1)()
    shared = np.zeros(K, np.uint32)
    w = sc.cfg.width
    cases = [
        dict(frames=None), dict(queries=None), dict(out=None), dict(count=0), dict(frame_count=0),
        dict(queries=query(frame=1)), dict(queries=query(frame=-1)),
        dict(frames=bufs(depth=None)), dict(frames=bufs(normals=None)), dict(frames=bufs(depth_pitch=2 * w - 2)),
        dict(frames=bufs(normals_pitch=2 * w - 2)), dict(frames=bufs(depth_pitch=2 * w + 1 + 2 * 64)),
        dict(queries=query(pose=[0, 0, 0, 1, float("nan"), 0, 0])), dict(queries=query(pose=[0, 0, 0, 0, 0, 0, 0])),
        dict(queries=query(pose=[0, 0, 0, 1, float("inf"), 0, 0])), dict(queries=query(min_depth=0.0)),
        dict(queries=query(min_depth=2.0, max_depth=1.0)), dict(queries=query(max_depth=float("nan"))),
        dict(keyframe_count=K - 1), dict(keyframe_count=K + 1),
    ]
    for case in cases:
        a = dict(frame_count=1, frames=bufs(), count=1, queries=query(), keyframe_count=K, out=out)
        a.update(case)
        st = lib.bba_measure_frame_overlap(ba._h, a["frame_count"], a["frames"], a["count"], a["queries"], a["keyframe_count"],
                                           shared.ctypes.data, a["out"], None)
        assert st == L.ERR_INVALID_ARGUMENT, case
        assert (ba.kernel_launch_count(), _state(ba)) == before, case
    assert not shared.any()


# ---- 8. a path leaving a keyframe's view ---------------------------------------------------------------------------------------

# Measured on an H100 80GB HBM3 (DESIGN §3.20): on `small` the uncovered share is 0.613 at keyframe 0's pose and rises step by step
# to 0.902 at the path's end.  Asserted with about half that rise as the margin.
UNCOVERED_RISE = 0.15


def test_uncovered_share_grows_along_a_path_leaving_the_view():
    from badslam_b200.scene import se3_exp, se3_mul
    sc = _scene("small")
    ba = _make(sc, poses=sc.poses_true)
    start = np.asarray(sc.poses_true[0], np.float32)
    poses = [se3_mul(start, se3_exp([0.1 * s, 0.0, -0.05 * s, 0.0, 0.12 * s, 0.0])).astype(np.float32) for s in range(6)]
    frames, queries = [], []
    for i, p in enumerate(poses):
        d, n, _, _, (lo, hi) = _render(sc, p)
        frames.append((_dev(d), _dev(n)))
        queries.append((i, p, lo, hi))
    r = ba.MeasureFrameOverlap(frames, queries)
    share = r.uncovered_cells / np.maximum(r.valid_cells, 1)
    print(f"uncovered share along the path: {np.round(share, 3).tolist()}, new {r.new_surfels.tolist()}, "
          f"observed {r.observed_surfels.tolist()}, shared with keyframe 0 {r.shared[:, 0].tolist()}")
    assert share[-1] >= share[0] + UNCOVERED_RISE
    assert r.shared[-1, 0] < r.shared[0, 0]
