"""GPU: the front end (preprocessing, image-pair odometry, the readers) on its own thread and high-priority stream while a bundle
adjustment runs on the same handle on a low-priority stream -- BadSlam's default parallel_ba mode (include/badba.h "Conventions",
INTEGRATION.md section 2, DESIGN.md "Front end beside a running BA").

What is demanded:
  * bba_track_frame_pairwise_to_frame against a frame's buffers equals bba_track_frame_pairwise against the same buffers as a
    keyframe, bit for bit;
  * a front-end call made while the BA call is held at the top of an iteration returns, bit for bit, what the same call returns
    serially on the state published at that point; the BA call's result is not disturbed by it;
  * free-running overlap and keyframes added while the front end tracks: every output equals the serial one, every polled pose
    set is one the BA call published, no call fails.
None of the tests repeats anything to provoke a race; every wait has a timeout.
"""
import threading

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

MOTION = [0.02, -0.01, 0.015, 0.01, -0.008, 0.012]   # base_T_frame of the tracked frame (as tests/test_gpu_odometry.py)
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
TIMEOUT = 300.0   # seconds for any wait on the other thread


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    return S, DirectBA


def streams():
    import torch
    lo, hi = torch.cuda.Stream.priority_range()   # (lowest, highest): a lower number is a higher priority
    return torch.cuda.Stream(priority=lo), torch.cuda.Stream(priority=hi)


def to_dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


class FrontEndInputs:
    """A raw frame to preprocess and a rendered frame (near keyframe 0) to track, as device tensors."""

    def __init__(self, S, sc, ba):
        import torch
        raw, rgb = S.raw_frame(sc, 1, scale=1)
        self.raw, self.rgb = to_dev(raw), to_dev(rgb)
        d, n, _, c = S.render_frame(sc, S.se3_mul(sc.poses_true[0], S.se3_exp(MOTION)))
        self.frame = (to_dev(d), to_dev(n), to_dev(c))
        kf = ba._keyframes[0]
        self.base = (kf.depth_buffer, kf.normals_buffer, kf.color_buffer)
        self.init2 = S.se3_exp([0.01, 0.0, 0.0, 0.0, 0.0, 0.0])
        torch.cuda.synchronize()


def published_state(ba, stream):
    """The readers: keyframe count, poses, activations, intrinsics, a, residual types and cfactor."""
    import ctypes as C
    K = ba._lib.bba_keyframe_count(ba._h)
    p, a = np.zeros((K, 7), np.float32), np.zeros(K, np.int32)
    ba._check(ba._lib.bba_get_keyframe_states(ba._h, K, p.ctypes.data, a.ctypes.data))
    d, c, da = ba._intrinsics()
    ud, uc = C.c_int(), C.c_int()
    ba._check(ba._lib.bba_get_residual_types(ba._h, C.byref(ud), C.byref(uc)))
    return dict(count=K, poses=p, activation=a, depth_K=np.array(d, np.float32), color_K=np.array(c, np.float32),
                a=np.float32(da), residual_types=(ud.value, uc.value), cfactor=ba.cfactor_buffer(stream))


def preprocess(ba, inp, stream):
    import torch
    with torch.cuda.stream(stream):
        d, n, r, c, mn, mx = ba.PreprocessFrame(inp.raw, inp.rgb, median_filter_and_densify_iterations=1, stream=stream)
        u16 = lambda t: t.view(torch.int16).cpu().numpy()
        return dict(depth=u16(d), normals=u16(n), radius=u16(r), rgba=c.cpu().numpy(), min=mn, max=mx)


def tracking(result):
    pose, res = result
    return dict(pose=pose.copy(), iterations=list(res.iterations), chose_initial=list(res.chose_initial),
                residual_count=res.residual_count, residual_sum=res.residual_sum)


def track_by_id(ba, inp, stream, kf=0, **kw):
    import torch
    with torch.cuda.stream(stream):
        return tracking(ba.TrackFramePairwise(stream, kf, *inp.frame, IDENT, inp.init2, num_scales=4, **kw))


def track_to_frame(ba, inp, stream, **kw):
    import torch
    with torch.cuda.stream(stream):
        return tracking(ba.TrackFramePairwiseToFrame(stream, *inp.base, *inp.frame, IDENT, inp.init2, num_scales=4, **kw))


def front_end_calls(ba, inp, stream):
    return dict(preprocess=preprocess(ba, inp, stream), track=track_by_id(ba, inp, stream), to_frame=track_to_frame(ba, inp, stream),
                readers=published_state(ba, stream))


def assert_same(got, want, what=""):
    """Bit-for-bit equality of nested dicts / lists of arrays and scalars (floats compared by their bits)."""
    if isinstance(want, dict):
        assert set(got) == set(want), what
        for k in want:
            assert_same(got[k], want[k], f"{what}.{k}")
    elif isinstance(want, (list, tuple)):
        assert len(got) == len(want), what
        for i, (g, w) in enumerate(zip(got, want)):
            assert_same(g, w, f"{what}[{i}]")
    else:
        g, w = np.asarray(got), np.asarray(want)
        assert g.shape == w.shape and g.dtype == w.dtype and g.tobytes() == w.tobytes(), (what, got, want)


def run_thread(fn):
    """Runs fn() on a daemon thread; returns (thread, box) with box['value'] / box['error'] once it ends."""
    box = {}

    def body():
        try:
            box["value"] = fn()
        except BaseException as e:   # reported by the test thread
            box["error"] = e
    t = threading.Thread(target=body, daemon=True)
    t.start()
    return t, box


def join(t, box):
    t.join(TIMEOUT)
    assert not t.is_alive(), "the other thread did not finish in time"
    if "error" in box:
        raise box["error"]
    return box.get("value")


@pytest.mark.parametrize("name", ["tiny", "small"])
@pytest.mark.parametrize("kw", [{}, {"use_gradmag": True}, {"use_pyramid_level_0": False}], ids=["desc", "gradmag", "no_level0"])
def test_base_as_buffers_equals_base_as_keyframe(mods, name, kw):
    S, DirectBA = mods
    sc = S.make_scene(S.config_by_name(name))
    ba = DirectBA.from_scene(sc)
    inp = FrontEndInputs(S, sc, ba)
    import torch
    st = torch.cuda.current_stream()
    by_id = track_by_id(ba, inp, st, **kw)
    by_buffers = track_to_frame(ba, inp, st, **kw)
    assert_same(by_buffers, by_id, name)
    assert max(by_id["iterations"]) > 0 and by_id["residual_count"] > 0
    # the base frame need not be a keyframe: another frame of the scene as the base, then the same buffers added as a keyframe
    d, n, r, c = S.render_frame(sc, sc.poses_true[1])
    base = (to_dev(d), to_dev(n), to_dev(c))
    inp.base = base
    first = track_to_frame(ba, inp, st, **kw)
    from badslam_b200.direct_ba import Keyframe
    kf = Keyframe(99, float(sc.min_depth[1]), float(sc.max_depth[1]), base[0].view(torch.uint16), base[1].view(torch.uint16),
                  to_dev(r).view(torch.uint16), base[2], sc.poses_true[1])
    ba2 = DirectBA.from_scene(sc, max_keyframes=sc.cfg.num_keyframes + 1)
    kid = ba2.AddKeyframe(kf)
    assert_same(track_by_id(ba2, inp, st, kf=kid, **kw), first, name + " (added afterwards)")


def test_gated_overlap_equals_serial_calls(mods):
    """The BA call holds at the top of iteration 1 (its progress_function waits, with a timeout) while the other thread makes
    every kind of front-end call on a high-priority stream; afterwards the recorded published state is restored and every call
    repeated serially.  The BA call's final state is compared with two undisturbed runs: bit for bit if those agree bit for bit,
    else within their run-to-run tolerance.  On an H100 the undisturbed runs of this setup (surfel updates + depth intrinsics)
    differ in the last bits (pose differences ~5e-10), so the tolerance branch is the one that applies there."""
    S, DirectBA = mods
    import torch
    sc = S.make_scene(S.config_by_name("small"))
    lo, hi = streams()
    kw = dict(optimize_depth_intrinsics=True, optimize_color_intrinsics=False, do_surfel_updates=True, optimize_poses=True,
              optimize_geometry=True, min_iterations=3, max_iterations=3)

    def run_ba(front_end):
        ba = DirectBA.from_scene(sc)
        inp = FrontEndInputs(S, sc, ba)
        recorded, box = {}, {}
        go, done = threading.Event(), threading.Event()

        def progress(it):
            recorded[it] = published_state(ba, lo)
            if front_end and it == 1:
                go.set()
                if not done.wait(TIMEOUT):
                    box["timeout"] = True
                    return False
            return True
        if front_end:
            def fe():
                assert go.wait(TIMEOUT), "the BA call never reached iteration 1"
                try:
                    return front_end_calls(ba, inp, hi)
                finally:
                    done.set()
            t, fbox = run_thread(fe)
        with torch.cuda.stream(lo):
            res = ba.BundleAdjustment(lo, progress_function=progress, **kw)
        lo.synchronize()
        assert "timeout" not in box
        out = join(t, fbox) if front_end else None
        final = dict(state=published_state(ba, lo), surfels=ba.GetSurfelsHost(), active=ba.GetActiveHost(), size=res.surfels_size)
        return ba, inp, recorded, out, final, res

    ba, inp, recorded, concurrent, final, res = run_ba(True)
    assert res.iterations_done == 3 and res.surfels_merged + res.surfels_deleted > 0   # (the surfel lifecycle ran)
    # the front end saw the state published at the top of iteration 1 ...
    assert_same(concurrent["readers"], recorded[1], "readers")
    assert not np.array_equal(recorded[1]["depth_K"], np.asarray(sc.depth_K, np.float32)), "the intrinsics step did not move"
    # ... and computed from it exactly what the same calls compute serially on that state
    K = recorded[1]["count"]
    ba.SetKeyframeStates(recorded[1]["poses"], recorded[1]["activation"])
    ba._set_intrinsics(recorded[1]["depth_K"], recorded[1]["color_K"], recorded[1]["a"])
    ba.SetCFactorBuffer(recorded[1]["cfactor"])
    assert K == sc.cfg.num_keyframes
    serial = front_end_calls(ba, inp, hi)
    assert_same(concurrent, serial, "front end")

    # the BA call itself: as undisturbed runs from the same start
    _, _, rec_a, _, final_a, _ = run_ba(False)
    _, _, rec_b, _, final_b, _ = run_ba(False)
    same = lambda f, g: all(np.asarray(f[k]).tobytes() == np.asarray(g[k]).tobytes() for k in ("surfels", "active", "size")) and \
        all(np.asarray(f["state"][k]).tobytes() == np.asarray(g["state"][k]).tobytes() for k in ("poses", "depth_K", "color_K", "a", "cfactor"))
    if same(final_a, final_b):
        print("undisturbed runs agree bit for bit: the disturbed run must too")
        assert same(final, final_a)
    else:
        noise = max(max(S.pose_error(p, q)) for p, q in zip(final_a["state"]["poses"], final_b["state"]["poses"]))
        print(f"undisturbed runs differ (pose noise {noise:.2e}): run-to-run tolerance")
        assert final["size"] == final_a["size"]
        for p, q in zip(final["state"]["poses"], final_a["state"]["poses"]):
            dt, dr = S.pose_error(p, q)
            assert dt < 1e-5 + 2 * noise and dr < 1e-5 + 2 * noise
        assert np.allclose(final["state"]["depth_K"], final_a["state"]["depth_K"], rtol=1e-4)


def test_free_running_overlap(mods):
    """Five BA iterations on a cfg2-sized scene (no intrinsics) while the other thread runs 20 preprocess + track cycles and polls
    the keyframe states."""
    S, DirectBA = mods
    import torch
    sc = S.make_scene(S.config_by_name("cfg2"))
    lo, hi = streams()
    ba = DirectBA.from_scene(sc)
    inp = FrontEndInputs(S, sc, ba)
    serial = dict(preprocess=preprocess(ba, inp, hi), track=track_by_id(ba, inp, hi))
    published = [published_state(ba, hi)["poses"]]

    def progress(it):
        published.append(published_state(ba, lo)["poses"])
        return True

    def fe():
        outs, polls = [], []
        for _ in range(20):
            outs.append(dict(preprocess=preprocess(ba, inp, hi), track=track_by_id(ba, inp, hi)))
            polls.append(published_state(ba, hi)["poses"])
        return outs, polls
    t, box = run_thread(fe)
    with torch.cuda.stream(lo):
        res = ba.BundleAdjustment(lo, False, False, False, True, True, 5, 5, progress_function=progress)
    lo.synchronize()
    outs, polls = join(t, box)
    published.append(published_state(ba, lo)["poses"])
    assert res.iterations_done == 5
    for i, o in enumerate(outs):
        assert_same(o, serial, f"cycle {i}")
    keys = {p.tobytes() for p in published}
    assert len(keys) > 2, "the poses did not move"
    for i, p in enumerate(polls):
        assert p.tobytes() in keys, f"poll {i} returned a pose set that was never published"


def test_keyframes_added_while_tracking(mods):
    """The BA thread adds 30 keyframes, each followed by surfel creation and one BA iteration, while the front end tracks
    against keyframe 0 by id."""
    S, DirectBA = mods
    import torch
    sc = S.make_scene(S.config_by_name("small"))
    K = sc.cfg.num_keyframes
    lo, hi = streams()
    ba = DirectBA.from_scene(sc, max_keyframes=K + 30)
    inp = FrontEndInputs(S, sc, ba)
    serial = track_by_id(ba, inp, hi)
    stop = threading.Event()

    def fe():
        outs = []
        while not stop.is_set() or not outs:
            outs.append(track_by_id(ba, inp, hi))
            counts = ba._lib.bba_keyframe_count(ba._h)
            assert K <= counts <= K + 30
        return outs
    t, box = run_thread(fe)
    try:
        with torch.cuda.stream(lo):
            for i in range(30):
                k = i % K
                kid = ba.AddKeyframeHost(sc.depth[k], sc.normals[k], sc.radius[k], sc.color[k], sc.poses_init[k], sc.min_depth[k],
                                         sc.max_depth[k], stream=lo)
                assert kid == K + i
                ba.CreateSurfelsForKeyframe(lo, True, kid)
                ba.BundleAdjustment(lo, False, False, False, True, True, 1, 1, increase_ba_iteration_count=False)
        lo.synchronize()
    finally:
        stop.set()
    outs = join(t, box)
    assert len(outs) >= 1
    for i, o in enumerate(outs):
        assert_same(o, serial, f"track {i}")
    # the handle stays usable on both sides
    assert ba._lib.bba_keyframe_count(ba._h) == K + 30
    assert_same(track_by_id(ba, inp, hi), serial, "after")
    with torch.cuda.stream(lo):
        assert ba.BundleAdjustment(lo, False, False, False, True, True, 1, 1).iterations_done == 1
    lo.synchronize()
