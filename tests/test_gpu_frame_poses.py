"""GPU: frame-to-model pose estimation of many entries in one call (bba_estimate_frame_poses_for_frames, DESIGN.md 3.3).  An entry
is one (frame, initial pose) pair; the entries ride through the pose step as temporary entries behind the keyframes, in chunks of
as many entries as there are free keyframe slots.  Every entry must give what its own single-frame call gives (to the BA pose
tolerance: from 4 entries on the pose kernel sums in another order), a batch of one must BE the single-frame call, and the call
must leave no trace in the handle.

Frames are the keyframes' own buffers (so that the keyframe form of the call and the CPU oracle give a second answer) and frames
rendered at poses near the keyframes'.

Launch counts: a pose step enqueues three kernels per Gauss-Newton iteration (the pose kernel's record packing and accumulation,
the solve) and keeps up to three iterations queued ahead of the one running, so a step whose entries stopped after m iterations
launches 3 e kernels with e between m and m + 3 (at least 2, at most 30), depending on how far the GPU has got when the host
polls.  A pose-kernel launch with stats (at_estimate) is two kernels.  The checks below hold the counts to that structure.
"""
import numpy as np
import pytest

from gpu_checks import rel

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-5   # m / rad, the BA pose tolerance
MOTION = [0.02, -0.01, 0.015, 0.01, -0.008, 0.012]
DEPTH = 3         # iterations the pose step keeps queued ahead (RunPoseStep's kDepth)


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import _lib as L
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    from oracle import cpu_oracle as O
    return S, DirectBA, L, O


_scenes = {}


def scene(S, name):
    if name not in _scenes:
        _scenes[name] = S.make_scene(S.config_by_name(name))
    return _scenes[name]


def dev16(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).cuda()


def dev8(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def frames_of(S, sc, rendered=3):
    """The keyframes' buffers, then `rendered` frames at poses a small motion away from keyframes 0, 1, ...  Returns
    (frames, true poses, keyframe id of each frame or -1)."""
    K = sc.cfg.num_keyframes
    frames = [(dev16(sc.depth[k]), dev16(sc.normals[k]), dev8(sc.color[k])) for k in range(K)]
    truth = [sc.poses_init[k] for k in range(K)]
    for r in range(rendered):
        pose = S.se3_mul(sc.poses_true[r % K], S.se3_exp(np.asarray(MOTION) * (1 + 0.3 * r)))
        d, n, _, c = S.render_frame(sc, pose)
        frames.append((dev16(d), dev16(n), dev8(c)))
        truth.append(np.asarray(pose, np.float32))
    return frames, truth, list(range(K)) + [-1] * rendered


def starts(S, truth, frame_of_entry, seed=1, scale=0.002):
    """One start per entry: its frame's pose (keyframes: the perturbed initial pose) moved by a few mm / mrad."""
    rng = np.random.default_rng(seed)
    return np.stack([S.se3_mul(truth[f], S.se3_exp(rng.normal(0, scale, 6))) for f in frame_of_entry]).astype(np.float32)


def single_calls(ba, frames, init, frame_of_entry):
    return [ba.EstimateFramePoseFromBuffers(None, init[i], *frames[f]) for i, f in enumerate(frame_of_entry)]


def step_launches(m):
    """The possible kernel counts of one pose step whose entries stopped after m Gauss-Newton iterations."""
    return {3 * e for e in range(max(m, 2), min(m + DEPTH, 30) + 1)}


def assert_pose_close(S, a, b, tol, what):
    dt, dr = S.pose_error(a, b)
    assert dt < tol and dr < tol, (what, dt, dr)


@pytest.mark.parametrize("name", ["tiny", "small", "many"])
def test_batch_of_one_is_the_single_frame_call(mods, name):
    S, DirectBA, L, O = mods
    sc = scene(S, name)
    ba = DirectBA.from_scene(sc, max_keyframes=sc.cfg.num_keyframes + 1)
    frames, truth, _ = frames_of(S, sc, rendered=1)
    for f in (0, len(frames) - 1):   # a keyframe's buffers, a rendered frame
        init = starts(S, truth, [f])
        c0 = ba.kernel_launch_count()
        pose, it, conv = ba.EstimateFramePoseFromBuffers(None, init[0], *frames[f])
        c1 = ba.kernel_launch_count()
        poses, its, convs = ba.EstimateFramePosesFromBuffers(None, [frames[f]], init)
        c2 = ba.kernel_launch_count()
        assert poses[0].tobytes() == pose.tobytes(), (name, f)
        assert (int(its[0]), bool(convs[0])) == (it, conv), (name, f)
        # the same launches: one luma extraction, one pose step of one entry (no surfel stream below 4 entries); only how many
        # iterations the host had queued ahead when the list ran empty may differ
        allowed = {1 + n for n in step_launches(it)}
        assert c1 - c0 in allowed and c2 - c1 in allowed and (c2 - c1 - (c1 - c0)) % 3 == 0, (name, f, c1 - c0, c2 - c1, it)


@pytest.mark.parametrize("name", ["tiny", "small", "many"])
def test_entries_agree_with_single_calls(mods, name):
    check_entries_agree_with_single_calls(mods, scene(mods[0], name))


def check_entries_agree_with_single_calls(mods, sc, reference=None):
    """37 entries (the keyframes' buffers and rendered frames) in calls of 1 .. 37 entries against the single-frame calls, the
    keyframe form, the oracle and the coefficients at the estimate.  With `reference` (a RefDirectBA of the scene), the keyframe
    entries of the 37-entry call are also held to the reference's EstimateFramePose from the same start, and the reference's own
    run-to-run spread there (a second run) widens the 1e-6 bar to the keyframe form, which sums in another order from 4 entries
    on.  The oracle then has to match only where it took the reference's number of Gauss-Newton iterations: the convergence
    test (|x|^2 < 1e-6 in scaled units, direct_ba_alternating.cc) lets a last step of up to ~1e-3 decide, and the oracle's IEEE
    arithmetic puts that step on the other side of the threshold now and then."""
    S, DirectBA, L, O = mods
    name = sc.cfg.name
    K = sc.cfg.num_keyframes
    ba = DirectBA.from_scene(sc, max_keyframes=K + 37)
    frames, truth, kf_of_frame = frames_of(S, sc)
    frame_of_entry = [i % len(frames) for i in range(37)]
    init = starts(S, truth, frame_of_entry)
    want = single_calls(ba, frames, init, frame_of_entry)
    orc = O.Oracle(sc)
    for count in (1, 3, 4, 8, 9, 37):
        poses, its, convs, coeffs = ba.EstimateFramePosesFromBuffers(None, frames, init[:count], frame_of_entry[:count], with_coeffs=True)
        for i in range(count):
            tag = (name, count, i)
            assert_pose_close(S, poses[i], want[i][0], POSE_TOL, tag)
            assert bool(convs[i]) == want[i][2], tag
            k = kf_of_frame[frame_of_entry[i]]
            if k >= 0:
                kf_pose, kf_its, _ = ba.EstimateFramePose(None, init[i], k)
                spread = 0.0
                if reference is not None and count == 37:
                    rp, rits, _ = reference.estimate_frame_pose(k, init[i])
                    spread = max(S.pose_error(rp, reference.estimate_frame_pose(k, init[i])[0]))
                    assert int(its[i]) == kf_its == rits, ("iterations",) + tag + (int(its[i]), kf_its, rits)
                    assert_pose_close(S, poses[i], rp, POSE_TOL + 2 * spread, ("reference",) + tag)
                assert_pose_close(S, poses[i], kf_pose, 1e-6 + 2 * spread, ("keyframe form",) + tag)
                if count == 37:
                    po, oits, _ = orc.estimate_frame_pose(k, init[i])
                    if reference is None or oits == rits:
                        assert_pose_close(S, poses[i], po, POSE_TOL, ("oracle",) + tag)
                    else:
                        print(f"{tag}: the oracle stopped after {oits} iterations, the reference and this path after {rits}")
                # at_estimate: what bba_accumulate_pose_coeffs returns at the returned pose
                pc = ba.AccumulatePoseEstimationCoeffs(k, poses[i])
                got = coeffs[i]
                assert (got.n_pair, got.n_inimg, got.n_depthok, got.n_assoc, got.n_photo) == \
                       (pc.n_pair, pc.n_inimg, pc.n_depthok, pc.n_assoc, pc.n_photo), tag
                assert got.n_assoc > 0, tag
                assert rel(got.H[:], pc.H[:]) < 1e-4 and rel(got.b[:], pc.b[:]) < 1e-4, tag
                for c in ("cost_depth", "cost_desc1", "cost_desc2"):
                    assert abs(getattr(got, c) - getattr(pc, c)) <= 1e-4 * abs(getattr(pc, c)) + 1e-12, (c,) + tag


def test_several_hypotheses_for_one_frame(mods):
    S, DirectBA, L, O = mods
    sc = scene(S, "small")
    K = sc.cfg.num_keyframes
    ba = DirectBA.from_scene(sc, max_keyframes=K + 8)
    pose = S.se3_mul(sc.poses_true[0], S.se3_exp(MOTION))
    d, n, _, c = S.render_frame(sc, pose)
    frame = (dev16(d), dev16(n), dev8(c))
    near = starts(S, [np.asarray(pose, np.float32)], [0] * 7, seed=4, scale=0.003)
    far_k = max(range(K), key=lambda k: S.pose_error(sc.poses_true[k], pose)[0])
    init = np.concatenate([near, sc.poses_true[far_k][None].astype(np.float32)])
    poses, its, convs, coeffs = ba.EstimateFramePosesFromBuffers(None, [frame], init, [0] * 8, with_coeffs=True)
    for i in range(7):
        single, _, conv = ba.EstimateFramePoseFromBuffers(None, init[i], *frame)
        assert_pose_close(S, poses[i], single, POSE_TOL, i)
        assert bool(convs[i]) == conv, i
    best = max(coeffs[i].n_assoc for i in range(7))
    assert coeffs[7].n_assoc < best, (coeffs[7].n_assoc, best, far_k)


def test_chunks_of_the_free_slots(mods):
    S, DirectBA, L, O = mods
    sc = scene(S, "small")
    K = sc.cfg.num_keyframes
    frames, truth, _ = frames_of(S, sc)
    frame_of_entry = [(3 * i) % len(frames) for i in range(10)]
    init = starts(S, truth, frame_of_entry, seed=7)
    wide, narrow = DirectBA.from_scene(sc, max_keyframes=K + 20), DirectBA.from_scene(sc, max_keyframes=K + 3)
    want, want_its, want_conv = wide.EstimateFramePosesFromBuffers(None, frames, init, frame_of_entry)
    c0 = narrow.kernel_launch_count()
    got, its, conv = narrow.EstimateFramePosesFromBuffers(None, frames, init, frame_of_entry)
    launches = narrow.kernel_launch_count() - c0
    for i in range(10):
        assert_pose_close(S, got[i], want[i], POSE_TOL, i)
    assert np.array_equal(conv, want_conv)
    # four chunks (3 + 3 + 3 + 1 entries): four luma launches and four pose steps, none with the surfel stream (< 4 entries)
    lo = hi = 0
    for b in range(0, 10, 3):
        steps = step_launches(int(its[b:b + 3].max()))
        lo, hi = lo + 1 + min(steps), hi + 1 + max(steps)
    assert lo <= launches <= hi and (launches - 4) % 3 == 0, (launches, lo, hi)
    # no free slot: a loud error, not a silent reallocation
    full = DirectBA.from_scene(sc, max_keyframes=K)
    from badslam_b200._lib import BadBAError
    with pytest.raises(BadBAError) as e:
        full.EstimateFramePosesFromBuffers(None, frames, init, frame_of_entry)
    assert e.value.status == L.ERR_STATE


def test_launch_count_does_not_grow_with_the_entries(mods):
    S, DirectBA, L, O = mods
    sc = scene(S, "many")
    K = sc.cfg.num_keyframes
    ba = DirectBA.from_scene(sc, max_keyframes=K + 37)
    frames, truth, _ = frames_of(S, sc)
    frame_of_entry = [i % len(frames) for i in range(37)]
    init = starts(S, truth, frame_of_entry, seed=9)
    for with_coeffs in (False, True):
        c0 = ba.kernel_launch_count()
        its = ba.EstimateFramePosesFromBuffers(None, frames, init, frame_of_entry, with_coeffs=with_coeffs)[1]
        launches = ba.kernel_launch_count() - c0
        # one luma launch + the surfel stream + one pose step (+ one pose-kernel launch with stats: two kernels)
        allowed = {2 + 2 * int(with_coeffs) + n for n in step_launches(int(its.max()))}
        assert launches in allowed, (with_coeffs, launches, sorted(allowed))
    c0 = ba.kernel_launch_count()
    single_calls(ba, frames, init, frame_of_entry)
    singles = ba.kernel_launch_count() - c0
    assert singles >= 37 * 7 and singles > 4 * launches, (singles, launches)


def handle_state(ba):
    poses, act = ba.GetKeyframeStates()
    return dict(count=ba._lib.bba_keyframe_count(ba._h), poses=poses.tobytes(), act=act.tobytes(), covis=ba.covisibility().tobytes(),
                surfels=ba.GetSurfelsHost().tobytes(), active=ba.GetActiveHost().tobytes(), size=ba.surfels_size())


def test_no_trace_in_the_handle(mods):
    S, DirectBA, L, O = mods
    sc = scene(S, "small")
    K = sc.cfg.num_keyframes
    frames, truth, _ = frames_of(S, sc)
    frame_of_entry = [i % len(frames) for i in range(12)]
    init = starts(S, truth, frame_of_entry, seed=5)
    ba = DirectBA.from_scene(sc, max_keyframes=K + 12)
    before = handle_state(ba)
    first = ba.EstimateFramePosesFromBuffers(None, frames, init, frame_of_entry, with_coeffs=True)
    assert handle_state(ba) == before
    ba.SetDeterministic(True)
    runs = [ba.EstimateFramePosesFromBuffers(None, frames, init, frame_of_entry, with_coeffs=True) for _ in range(2)]
    assert handle_state(ba) == before
    for a, b in zip(runs[0][:3], runs[1][:3]):
        assert a.tobytes() == b.tobytes()
    assert [bytes(c) for c in runs[0][3]] == [bytes(c) for c in runs[1][3]]
    for i in range(12):
        assert_pose_close(S, runs[0][0][i], first[0][i], POSE_TOL, i)

    # a BA after a batch call is the BA of a fresh handle, bit for bit
    def ba_after(batch):
        h = DirectBA.from_scene(sc, max_keyframes=K + 12)
        h.SetDeterministic(True)
        if batch:
            h.EstimateFramePosesFromBuffers(None, frames, init, frame_of_entry, with_coeffs=True)
        r = h.BundleAdjustment(None, False, False, False, True, True, 3, 3)
        assert r.iterations_done == 3
        return handle_state(h)
    assert ba_after(True) == ba_after(False)


def test_error_paths_leave_the_handle_unchanged(mods):
    S, DirectBA, L, O = mods
    sc = scene(S, "tiny")
    K = sc.cfg.num_keyframes
    ba = DirectBA.from_scene(sc, max_keyframes=K + 4)
    frames, truth, _ = frames_of(S, sc, rendered=0)
    bufs = (L.FrameBuffers * K)()
    for b, (d, n, c) in zip(bufs, frames):
        b.depth, b.depth_pitch, b.normals, b.normals_pitch = d.data_ptr(), d.stride(0) * 2, n.data_ptr(), n.stride(0) * 2
        b.color_rgba, b.color_pitch = c.data_ptr(), c.stride(0)
    init = starts(S, truth, list(range(K)))
    out = np.zeros((K, 7), np.float32)
    fmap = np.zeros(K, np.int32)
    lib, h = ba._lib, ba._h

    def call(frame_count=K, frames_=bufs, count=K, fm=None, init_=init, out_=out):
        return lib.bba_estimate_frame_poses_for_frames(h, frame_count, frames_, count, fm, None if init_ is None else init_.ctypes.data,
                                                       None if out_ is None else out_.ctypes.data, None, None, None, None)
    before = handle_state(ba)
    launches = ba.kernel_launch_count()
    assert call(frames_=None) == L.ERR_INVALID_ARGUMENT
    assert call(init_=None) == L.ERR_INVALID_ARGUMENT
    assert call(out_=None) == L.ERR_INVALID_ARGUMENT
    assert call(count=0) == L.ERR_INVALID_ARGUMENT
    assert call(frame_count=0) == L.ERR_INVALID_ARGUMENT
    assert call(frame_count=K - 1) == L.ERR_INVALID_ARGUMENT   # entry i uses frame i without a map
    fmap[1] = K
    assert call(fm=fmap.ctypes.data) == L.ERR_INVALID_ARGUMENT
    fmap[1] = -1
    assert call(fm=fmap.ctypes.data) == L.ERR_INVALID_ARGUMENT
    fmap[1] = 0
    saved = bufs[2].color_pitch
    bufs[2].color_pitch = sc.cfg.width * 4 - 1
    assert call() == L.ERR_INVALID_ARGUMENT
    bufs[2].color_pitch = saved
    saved = bufs[1].normals
    bufs[1].normals = None
    assert call() == L.ERR_INVALID_ARGUMENT
    bufs[1].normals = saved
    assert not out.any()
    assert ba.kernel_launch_count() == launches and handle_state(ba) == before
    assert call(fm=fmap.ctypes.data) == L.OK and out.any()
    assert handle_state(ba) == before
    # more than one rank: refused before anything runs
    from badslam_b200._lib import BadBAError
    multi = DirectBA.from_scene(sc, max_keyframes=K + 4, world_size=2)
    c0 = multi.kernel_launch_count()
    with pytest.raises(BadBAError) as e:
        multi.EstimateFramePosesFromBuffers(None, frames, init)
    assert e.value.status == L.ERR_UNSUPPORTED and multi.kernel_launch_count() == c0
