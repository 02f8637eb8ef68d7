"""GPU: the image-pair odometry for many (base, tracked frame) pairs in one call (bba_track_frames_pairwise, DESIGN.md 3.8).

What is demanded:
  * deterministic mode: every entry's pose, iterations, cost-comparison branches, residual count / sum and pass count equal those
    of its own bba_track_frame_pairwise / _to_frame call bit for bit, whatever else the call holds and in whatever order: 1, 2,
    7 and sm_count + 5 entries (more than two chunks), keyframe and buffer bases mixed, frames repeated with other starting
    poses, descriptor and gradient-magnitude residuals, depth only and descriptor only, with and without pyramid level 0, one
    or two initial estimates, 1, 3 and 5 pyramid levels;
  * default mode: iteration counts within one of the single calls', poses within the tolerance tests/test_gpu_odometry.py
    applies against the reference (1e-5 m / rad plus ten times the run-to-run drift of the single calls);
  * 4 + (num_scales - 1) launches per chunk, whatever the entry count, and so per single-pair call of either form;
  * every bad argument is refused before anything is enqueued, by the batch and by both single-pair forms: launch counter and
    keyframe states unchanged;
  * the parity hooks describe the batch's last entry, bit for bit as after a single call on that pair;
  * a batch issued while a bundle adjustment holds at an iteration boundary equals the same batch run alone.
"""
import threading

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

MOTION = np.array([0.02, -0.01, 0.015, 0.01, -0.008, 0.012])   # as tests/test_gpu_odometry.py
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
TIMEOUT = 300.0


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200 import _lib
    from badslam_b200.direct_ba import DirectBA
    return S, DirectBA, _lib


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def to_dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


class Pairs:
    """Frames rendered at small offsets from the keyframes (frame j near keyframe j % K), followed by the keyframes' own buffers
    as frames; entries cycle through them with keyframe bases, keyframe buffers as bases and other rendered frames as bases, each
    round with other starting poses."""

    def __init__(self, S, sc, ba, frames_per_kf=2):
        import torch
        self.S, self.K = S, sc.cfg.num_keyframes
        self.frames = []
        for j in range(self.K * frames_per_kf):
            k = j % self.K
            motion = MOTION * (1.0 - 0.15 * (j // self.K)) * (1 if j % 2 == 0 else -1)
            d, n, _, c = S.render_frame(sc, S.se3_mul(sc.poses_true[k], S.se3_exp(motion)))
            self.frames.append((to_dev(d), to_dev(n), to_dev(c)))
        self.n_rendered = len(self.frames)
        for k in range(self.K):
            kf = ba._keyframes[k]
            self.frames.append((kf.depth_buffer, kf.normals_buffer, kf.color_buffer))
        torch.cuda.synchronize()

    def entries(self, count, seed=0):
        rng = np.random.default_rng(seed)
        out = []
        for i in range(count):
            t = i % self.n_rendered
            k = t % self.K
            p1 = self.S.se3_exp(rng.normal(0, 0.004, 6)).astype(np.float32)
            p2 = self.S.se3_exp(np.array([0.01, 0, 0, 0, 0, 0]) + rng.normal(0, 0.004, 6)).astype(np.float32)
            kind = i % 3
            if kind == 0:
                out.append((k, 0, t, p1, p2))                              # keyframe base
            elif kind == 1:
                out.append((-1, self.n_rendered + k, t, p1, p2))           # the keyframe's buffers as a base
            else:
                other = (t + self.K) % self.n_rendered                     # another frame near the same keyframe
                out.append((-1, other, t, p1, p2))
        return out


def single(ba, pairs, e, **kw):
    kf, bf, tf, p1, p2 = e
    if kf >= 0:
        return ba.TrackFramePairwise(None, kf, *pairs.frames[tf], p1, p2, **kw)
    return ba.TrackFramePairwiseToFrame(None, *pairs.frames[bf], *pairs.frames[tf], p1, p2, **kw)


def bits(est, r):
    return (np.asarray(est, np.float32).tobytes(), list(r.iterations), list(r.chose_initial), r.residual_count,
            np.float32(r.residual_sum).tobytes(), r.passes)


def make(S, DirectBA, name, deterministic=True, **kw):
    sc = S.make_scene(S.config_by_name(name))
    ba = DirectBA.from_scene(sc, **kw)
    ba.SetDeterministic(deterministic)
    return sc, ba, Pairs(S, sc, ba)


OPTION_SETS = {
    "default": dict(num_scales=3),
    "gradmag": dict(num_scales=3, use_gradmag=True),
    "no_level0": dict(num_scales=3, use_pyramid_level_0=False),
    "one_initial": dict(num_scales=3, test_different_initial_estimates=False),
    "one_scale": dict(num_scales=1),
    "one_scale_one_initial": dict(num_scales=1, test_different_initial_estimates=False),
}


@pytest.mark.parametrize("opts", list(OPTION_SETS), ids=list(OPTION_SETS))
def test_deterministic_batch_equals_single_calls(mods, opts):
    S, DirectBA, _ = mods
    kw = OPTION_SETS[opts]
    sc, ba, pairs = make(S, DirectBA, "tiny")
    n_max = sm_count() + 5
    entries = pairs.entries(n_max, seed=1)
    want = [bits(*single(ba, pairs, e, **kw)) for e in entries]
    assert max(max(w[1]) for w in want) > 0 and all(w[3] > 0 for w in want)
    for count in (1, 2, 7, n_max):
        est, res, _ = ba.TrackFramesPairwise(None, pairs.frames, entries[:count], **kw)
        for i in range(count):
            assert bits(est[i], res[i]) == want[i], (opts, count, i)
    # shuffled: the same bits per entry
    perm = np.random.default_rng(2).permutation(n_max)
    est, res, _ = ba.TrackFramesPairwise(None, pairs.frames, [entries[i] for i in perm], **kw)
    for j, i in enumerate(perm):
        assert bits(est[j], res[j]) == want[i], (opts, "shuffled", j, i)


@pytest.mark.parametrize("name,kw", [
    ("small", dict(num_scales=5)),
    ("small", dict(num_scales=5, use_gradmag=True, use_pyramid_level_0=False)),
], ids=["five_scales", "five_scales_gradmag_no_level0"])
def test_deterministic_five_scales(mods, name, kw):
    S, DirectBA, _ = mods
    sc, ba, pairs = make(S, DirectBA, name)
    entries = pairs.entries(9, seed=3)
    want = [bits(*single(ba, pairs, e, **kw)) for e in entries]
    est, res, _ = ba.TrackFramesPairwise(None, pairs.frames, entries, **kw)
    for i in range(len(entries)):
        assert bits(est[i], res[i]) == want[i], (name, kw, i)


@pytest.mark.parametrize("use_depth,use_desc", [(True, False), (False, True)], ids=["depth_only", "descriptor_only"])
def test_deterministic_residual_types(mods, use_depth, use_desc):
    S, DirectBA, _ = mods
    sc, ba, pairs = make(S, DirectBA, "tiny", use_depth_residuals=use_depth, use_descriptor_residuals=use_desc)
    entries = pairs.entries(7, seed=4)
    want = [bits(*single(ba, pairs, e, num_scales=3)) for e in entries]
    est, res, _ = ba.TrackFramesPairwise(None, pairs.frames, entries, num_scales=3)
    for i in range(len(entries)):
        assert bits(est[i], res[i]) == want[i], (use_depth, use_desc, i)


def test_default_mode_against_single_calls(mods):
    S, DirectBA, _ = mods
    sc, ba, pairs = make(S, DirectBA, "tiny", deterministic=False)
    kw = dict(num_scales=3)
    n = sm_count() + 5
    entries = pairs.entries(n, seed=5)
    runs = [[single(ba, pairs, e, **kw) for e in entries] for _ in range(3)]
    est, res, _ = ba.TrackFramesPairwise(None, pairs.frames, entries, **kw)
    worst = 0.0
    for i in range(n):
        noise = max(max(S.pose_error(runs[a][i][0], runs[b][i][0])) for a in range(3) for b in range(a + 1, 3))
        limit = max(1e-5 + 10 * noise, 5e-5)
        dt, dr = S.pose_error(est[i], runs[0][i][0])
        worst = max(worst, dt, dr)
        assert dt < limit and dr < limit, (i, dt, dr, noise)
        its, its1 = list(res[i].iterations)[:3], list(runs[0][i][1].iterations)[:3]
        assert all(abs(a - b) <= 1 for a, b in zip(its, its1)), (i, its, its1)
    print(f"default mode, {n} entries: largest pose difference to the single calls {worst:.2e}")


def test_launches_per_chunk_and_per_single_pair_call(mods):
    S, DirectBA, _lib = mods
    sc, ba, pairs = make(S, DirectBA, "tiny", deterministic=False)
    chunk = _lib.ODOMETRY_CHUNK_ENTRIES
    for num_scales in (1, 3):
        per_chunk = 4 + (num_scales - 1)
        for count in (1, 7, chunk, chunk + 1, 2 * chunk + 3):
            before = ba.kernel_launch_count()
            _, res, launches = ba.TrackFramesPairwise(None, pairs.frames, pairs.entries(count), num_scales=num_scales)
            chunks = -(-count // chunk)
            assert launches == chunks * per_chunk, (num_scales, count, launches)
            assert ba.kernel_launch_count() - before == launches
            assert all(r.kernel_launches == per_chunk for r in res)
    # the single-pair calls are one-entry chunks: the keyframe form and the buffer form (one luma launch for both frames)
    e = pairs.entries(2)
    assert single(ba, pairs, e[0], num_scales=3)[1].kernel_launches == 6
    assert single(ba, pairs, e[1], num_scales=3)[1].kernel_launches == 6


def test_bad_arguments_change_nothing(mods):
    S, DirectBA, _lib = mods
    import ctypes as C
    import torch
    sc, ba, pairs = make(S, DirectBA, "tiny", deterministic=False)
    K, nf = pairs.K, len(pairs.frames)
    good = pairs.entries(3)
    ba.TrackFramesPairwise(None, pairs.frames, good, num_scales=3)
    torch.cuda.synchronize()
    states, launches = ba.GetKeyframeStates(), ba.kernel_launch_count()

    def refused(status, frames, entries, **kw):
        with pytest.raises(_lib.BadBAError) as err:
            ba.TrackFramesPairwise(None, frames, entries, **kw)
        assert err.value.status == status, (err.value, entries[:1], kw)

    e = good[0]
    bad_entries = [
        (K, 0, 0, e[3], e[4]),            # no such keyframe
        (-2, 0, 0, e[3], e[4]),           # keyframe id below -1
        (0, 0, nf, e[3], e[4]),           # tracked frame out of range
        (0, 0, -1, e[3], e[4]),
        (-1, nf, 0, e[3], e[4]),          # base frame out of range
        (-1, -1, 0, e[3], e[4]),
    ]
    for b in bad_entries:
        refused(_lib.ERR_INVALID_ARGUMENT, pairs.frames, good + [b], num_scales=3)
    refused(_lib.ERR_INVALID_ARGUMENT, pairs.frames, [], num_scales=3)                 # count 0
    refused(_lib.ERR_INVALID_ARGUMENT, [], good, num_scales=3)                          # frame_count 0
    refused(_lib.ERR_INVALID_ARGUMENT, pairs.frames, good, num_scales=0)
    refused(_lib.ERR_INVALID_ARGUMENT, pairs.frames, good, num_scales=9)
    refused(_lib.ERR_INVALID_ARGUMENT, pairs.frames, good, num_scales=1, use_pyramid_level_0=False)
    d, n, c = pairs.frames[0]
    narrow = (torch.zeros((d.shape[0], d.shape[1] - 1), dtype=d.dtype, device=d.device), n, c)   # a pitch too small for the image
    refused(_lib.ERR_INVALID_ARGUMENT, [narrow] + pairs.frames[1:], good, num_scales=3)
    # NULL arrays
    o = _lib.OdometryOptions(3, 1, 0, 1, 30)
    bufs = (_lib.FrameBuffers * nf)()
    for b, (dd, nn, cc) in zip(bufs, pairs.frames):
        b.depth, b.depth_pitch, b.normals, b.normals_pitch = dd.data_ptr(), dd.stride(0) * 2, nn.data_ptr(), nn.stride(0) * 2
        b.color_rgba, b.color_pitch = cc.data_ptr(), cc.stride(0)
    ents = (_lib.OdometryEntry * 1)()
    ents[0].base_keyframe_id, ents[0].tracked_frame = 0, 0
    ents[0].base_T_frame_initial_1[:] = IDENT.tolist()
    ents[0].base_T_frame_initial_2[:] = IDENT.tolist()
    out = np.zeros((1, 7), np.float32)
    lib, h = ba._lib, ba._h
    assert lib.bba_track_frames_pairwise(h, None, nf, bufs, 1, ents, out.ctypes.data, None, None, None) == _lib.ERR_INVALID_ARGUMENT
    assert lib.bba_track_frames_pairwise(h, C.byref(o), nf, None, 1, ents, out.ctypes.data, None, None, None) == _lib.ERR_INVALID_ARGUMENT
    assert lib.bba_track_frames_pairwise(h, C.byref(o), nf, bufs, 1, None, out.ctypes.data, None, None, None) == _lib.ERR_INVALID_ARGUMENT
    assert lib.bba_track_frames_pairwise(h, C.byref(o), nf, bufs, 1, ents, None, None, None, None) == _lib.ERR_INVALID_ARGUMENT

    # the single-pair forms refuse the same arguments before anything is enqueued, and what an entry cannot express
    def refused_single(status, kf, frame, base=None, **kw):
        with pytest.raises(_lib.BadBAError) as err:
            if base is None:
                ba.TrackFramePairwise(None, kf, *frame, e[3], e[4], **kw)
            else:
                ba.TrackFramePairwiseToFrame(None, *base, *frame, e[3], e[4], **kw)
        assert err.value.status == status, (err.value, kf, base is None, kw)

    frame = pairs.frames[0]
    for base in (None, pairs.frames[1]):
        refused_single(_lib.ERR_INVALID_ARGUMENT, 0, frame, base, num_scales=8)     # 160x120 has no level 7
        refused_single(_lib.ERR_INVALID_ARGUMENT, 0, frame, base, num_scales=0)
        refused_single(_lib.ERR_INVALID_ARGUMENT, 0, frame, base, num_scales=9)
        refused_single(_lib.ERR_INVALID_ARGUMENT, 0, frame, base, num_scales=1, use_pyramid_level_0=False)
        refused_single(_lib.ERR_INVALID_ARGUMENT, 0, narrow, base, num_scales=3)
    refused_single(_lib.ERR_INVALID_ARGUMENT, 0, frame, narrow, num_scales=3)      # a base frame's pitch
    refused_single(_lib.ERR_INVALID_ARGUMENT, K, frame, num_scales=3)              # no such keyframe
    refused_single(_lib.ERR_INVALID_ARGUMENT, -1, frame, num_scales=3)
    fb = bufs[0]
    p1 = np.ascontiguousarray(e[3], np.float32)
    F = C.POINTER(C.c_float)
    for init1, init2, est in ((None, p1, out), (p1, None, out), (p1, p1, None)):   # test_different_initial_estimates needs init2
        args = (None if init1 is None else init1.ctypes.data_as(F), None if init2 is None else init2.ctypes.data_as(F),
                None if est is None else est.ctypes.data_as(F), None, None)
        frame_args = (fb.depth, fb.depth_pitch, fb.normals, fb.normals_pitch, fb.color_rgba, fb.color_pitch)
        assert lib.bba_track_frame_pairwise(h, C.byref(o), 0, *frame_args, *args) == _lib.ERR_INVALID_ARGUMENT
        assert lib.bba_track_frame_pairwise_to_frame(h, C.byref(o), *frame_args, *frame_args, *args) == _lib.ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert ba.kernel_launch_count() == launches
    assert all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(ba.GetKeyframeStates(), states))

    # the depth / colour pyramid combination the single call rejects: colour neither the depth size nor half of it
    from badslam_b200.direct_ba import PinholeCamera4f
    dcam, ccam = PinholeCamera4f(160, 120, [120, 120, 80, 60]), PinholeCamera4f(100, 76, [75, 75, 50, 38])
    ba2 = DirectBA(1024, 1e-3, 40, 2, color_camera_initial_estimate=ccam, depth_camera_initial_estimate=dcam)
    frame = (torch.zeros((120, 160), dtype=torch.int16, device="cuda"), torch.zeros((120, 160), dtype=torch.int16, device="cuda"),
             torch.zeros((76, 100, 4), dtype=torch.uint8, device="cuda"))
    before = ba2.kernel_launch_count()
    for call in (lambda: ba2.TrackFramesPairwise(None, [frame], [(-1, 0, 0, IDENT, IDENT)], num_scales=3, use_pyramid_level_0=False),
                 lambda: ba2.TrackFramePairwise(None, 0, *frame, IDENT, IDENT, num_scales=3, use_pyramid_level_0=False),
                 lambda: ba2.TrackFramePairwiseToFrame(None, *frame, *frame, IDENT, IDENT, num_scales=3, use_pyramid_level_0=False)):
        with pytest.raises(_lib.BadBAError) as err:
            call()
        assert err.value.status == _lib.ERR_UNSUPPORTED
    assert ba2.kernel_launch_count() == before


@pytest.mark.parametrize("opts", ["default", "no_level0"])
def test_parity_hooks_describe_the_last_entry(mods, opts):
    S, DirectBA, _ = mods
    kw = OPTION_SETS[opts]
    first = 0 if kw.get("use_pyramid_level_0", True) else 1
    sc, ba, pairs = make(S, DirectBA, "tiny")
    pose_a, pose_b = S.se3_exp(MOTION).astype(np.float32), S.se3_exp(0.5 * MOTION).astype(np.float32)

    def hooks():
        # (the normals of a pixel without depth are whatever the pyramid's plane held before: not part of the level)
        levels = [ba.OdometryLevel(which, scale) for scale in range(kw["num_scales"]) for which in (0, 1) if which == 0 or scale >= first]
        levels = [(d, np.where(d > 0, n, 0), c) for d, n, c in levels]
        coeffs = [ba.OdometryCoeffs(scale, pose_a, pose_b) for scale in range(first, kw["num_scales"])]
        return [np.asarray(x).tobytes() for lv in levels for x in lv] + [np.asarray(x).tobytes() for c in coeffs for x in c]

    for last in (0, 1, 2):   # a keyframe base, the keyframe's buffers as base, another frame as base
        entries = pairs.entries(11, seed=6)
        entries = entries[:10] + [pairs.entries(3, seed=7)[last]]
        ba.TrackFramesPairwise(None, pairs.frames, entries, **kw)
        after_batch = hooks()
        single(ba, pairs, entries[-1], **kw)
        assert after_batch == hooks(), (opts, last)


def test_batch_beside_a_held_bundle_adjustment(mods):
    """The BA call holds at the top of iteration 1 while another thread runs a batch on a high-priority stream.  Without the
    intrinsics step the BA call publishes no state the odometry reads, so the batch must equal the same batch run alone."""
    S, DirectBA, _ = mods
    import torch
    sc, ba, pairs = make(S, DirectBA, "small")
    entries = pairs.entries(sm_count() + 5, seed=8)
    kw = dict(num_scales=4)
    alone_est, alone_res, alone_launches = ba.TrackFramesPairwise(None, pairs.frames, entries, **kw)
    lo_pri, hi_pri = torch.cuda.Stream.priority_range()
    lo, hi = torch.cuda.Stream(priority=lo_pri), torch.cuda.Stream(priority=hi_pri)
    go, done = threading.Event(), threading.Event()
    box, held = {}, {}

    def progress(it):
        if it == 1:
            go.set()
            if not done.wait(TIMEOUT):
                held["timeout"] = True
                return False
        return True

    def front_end():
        try:
            assert go.wait(TIMEOUT), "the BA call never reached iteration 1"
            with torch.cuda.stream(hi):
                box["value"] = ba.TrackFramesPairwise(hi, pairs.frames, entries, **kw)
        except BaseException as e:   # reported by the test thread
            box["error"] = e
        finally:
            done.set()

    t = threading.Thread(target=front_end, daemon=True)
    t.start()
    with torch.cuda.stream(lo):
        res = ba.BundleAdjustment(lo, optimize_depth_intrinsics=False, optimize_color_intrinsics=False, do_surfel_updates=False,
                                  optimize_poses=True, optimize_geometry=True, min_iterations=2, max_iterations=2,
                                  progress_function=progress)
    lo.synchronize()
    t.join(TIMEOUT)
    assert not t.is_alive() and "timeout" not in held
    if "error" in box:
        raise box["error"]
    est, results, launches = box["value"]
    assert res.iterations_done == 2
    assert launches == alone_launches
    for i in range(len(entries)):
        assert bits(est[i], results[i]) == bits(alone_est[i], alone_res[i]), i
