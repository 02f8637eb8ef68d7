"""GPU: the trajectory deformation on real odometry + BA output (RememberKeyframePoses / ExtrapolateAndInterpolateKeyframePoseChanges
around BundleAdjustment, as BadSlam's BA thread runs them, bad_slam.cc:1267-1301).

What is demanded:
  * on `small` (views brought closer together) with every second scene view a keyframe at its perturbed pose and the views
    between tracked against the preceding keyframe (bba_track_frame_pairwise), the deformed poses after a BA call equal
    oracle/trajectory_oracle.py's on the same read-back arrays bit for bit (the same fp32 host arithmetic), and the tracked
    frames' error against the true poses falls with their keyframes' error;
  * RememberKeyframePoses made on the front-end thread while the BA call runs returns the poses of one publication: every call
    equals the inverse of a pose set the BA call published, never a mix of two.
None of the tests repeats anything to provoke a race; every wait has a timeout.
"""
import dataclasses
import threading

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]

TIMEOUT = 300.0   # seconds for any wait on the other thread


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200 import direct_ba as D
    return S, D


def to_dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


def inverses(lib, poses):
    out = np.empty_like(poses)
    for k in range(len(poses)):
        lib.bba_host_se3_inverse(poses[k].ctypes.data, out[k].ctypes.data)
    return out


def test_deformed_odometry_trajectory(mods):
    S, D = mods
    import torch
    from oracle import trajectory_oracle as T
    # `small`, with its views 0.2 m / 0.1 rad apart instead of 3 m / 0.7 rad: consecutive views are then what a moving camera
    # records, so that image-pair odometry between them and the interpolation between neighbouring keyframes mean something
    sc = S.make_scene(dataclasses.replace(S.config_by_name("small"), pose_spread_t=0.2, pose_spread_r=0.1))
    cfg = sc.cfg
    views = np.arange(cfg.num_keyframes)
    keyframe_views, tracked_views = views[0::2], views[1::2]   # 0 2 4 | 1 3 5: frames between keyframes and one after the last
    cam_d = D.PinholeCamera4f(cfg.width, cfg.height, sc.depth_K)
    cam_c = D.PinholeCamera4f(cfg.width, cfg.height, sc.color_K)
    ba = D.DirectBA(sc.pitch, cfg.raw_to_float_depth, cfg.baseline_fx, cfg.cell, color_camera_initial_estimate=cam_c,
                    depth_camera_initial_estimate=cam_d, max_keyframes=len(keyframe_views))
    for v in keyframe_views:
        ba.AddKeyframeHost(sc.depth[v], sc.normals[v], sc.radius[v], sc.color[v], sc.poses_init[v], sc.min_depth[v], sc.max_depth[v])
    ba.SetSurfelsHost(sc.surfels, sc.num_surfels)
    lib = ba._lib

    # BadSlam::RunOdometry for the views between: tracked against the preceding keyframe, seeded with the perturbed relative pose
    frame_poses = np.zeros((cfg.num_keyframes, 7), np.float32)
    frame_poses[keyframe_views] = sc.poses_init[keyframe_views]
    stream = torch.cuda.current_stream()
    for v in tracked_views:
        kf_id = int(v - 1) // 2
        guess = S.se3_mul(S.se3_inverse(sc.poses_init[v - 1]), sc.poses_init[v])
        base_T_frame, res = ba.TrackFramePairwise(stream, kf_id, to_dev(sc.depth[v]), to_dev(sc.normals[v]), to_dev(sc.color[v]), guess)
        assert res.residual_count > 0
        kf_pose = ba.GetKeyframeStates()[0][kf_id]
        lib.bba_host_se3_compose(kf_pose.ctypes.data, base_T_frame.ctypes.data, frame_poses[v].ctypes.data)

    def errors(poses, which):
        return np.array([S.pose_error(poses[v], sc.poses_true[v]) for v in which])   # [n, 2]: metres, radians

    kf_before, fr_before = errors(frame_poses, keyframe_views), errors(frame_poses, tracked_views)
    original = ba.RememberKeyframePoses()
    assert np.array_equal(original, inverses(lib, sc.poses_init[keyframe_views].copy()))
    r = ba.BundleAdjustment(None, False, False, False, True, True, 1, 10)
    assert r.iterations_done >= 1
    current = ba.GetKeyframeStates()[0]
    before = frame_poses.copy()
    ba.ExtrapolateAndInterpolateKeyframePoseChanges(0, cfg.num_keyframes - 1, original, keyframe_views, frame_poses)

    # the library's deformation is the oracle's on the same arrays, bit for bit; the keyframes' rows are the caller's
    expected = T.deform_trajectory(keyframe_views, original, current, 0, cfg.num_keyframes - 1, before)
    assert frame_poses.tobytes() == expected.tobytes()
    assert np.array_equal(frame_poses[keyframe_views], before[keyframe_views])
    frame_poses[keyframe_views] = current
    kf_after, fr_after = errors(frame_poses, keyframe_views), errors(frame_poses, tracked_views)
    print("keyframes  before", kf_before.tolist(), "after", kf_after.tolist())
    print("tracked    before", fr_before.tolist(), "after", fr_after.tolist())
    # The tracked frames follow their keyframes towards the true trajectory.  Measured on one H100 80GB HBM3 (translation errors
    # in mm, views 0 2 4 | 1 3 5):  keyframes 3.23 3.78 5.37 -> 2.25 2.30 2.30 (mean x0.55),  tracked frames 3.29 3.78 5.40 ->
    # 2.98 2.76 2.29 (mean x0.64); each tracked frame ends within 0.73 mm of its preceding keyframe's error.  Without the
    # deformation the tracked frames would keep their errors.
    kf_ratio, fr_ratio = kf_after[:, 0].mean() / kf_before[:, 0].mean(), fr_after[:, 0].mean() / fr_before[:, 0].mean()
    assert kf_ratio < 0.65 and fr_ratio < 0.75, (kf_ratio, fr_ratio)
    assert fr_after[:, 0].max() < fr_before[:, 0].max()
    assert np.abs(fr_after[:, 0] - kf_after[:, 0]).max() < 1e-3


def test_remember_keyframe_poses_on_the_front_end_thread_reads_one_publication(mods):
    """Five BA iterations (poses and geometry) on a low-priority stream while the front-end thread calls RememberKeyframePoses
    until the call ends; every result is the inverse of a pose set published before the call, at the top of an iteration or at
    its end."""
    S, D = mods
    import torch
    sc = S.make_scene(S.config_by_name("small"))
    lo, _ = torch.cuda.Stream.priority_range()
    lo = torch.cuda.Stream(priority=lo)
    ba = D.DirectBA.from_scene(sc)
    lib = ba._lib
    published = [ba.GetKeyframeStates()[0]]

    def progress(it):
        published.append(ba.GetKeyframeStates()[0])
        return True

    stop, box = threading.Event(), {}

    def front_end():
        polls = []
        try:
            while not stop.is_set() or not polls:
                polls.append(ba.RememberKeyframePoses())
        except BaseException as e:   # reported by the test thread
            box["error"] = e
        box["polls"] = polls
    t = threading.Thread(target=front_end, daemon=True)
    t.start()
    try:
        with torch.cuda.stream(lo):
            res = ba.BundleAdjustment(lo, False, False, False, True, True, 5, 5, progress_function=progress)
        lo.synchronize()
    finally:
        stop.set()
    t.join(TIMEOUT)
    assert not t.is_alive(), "the front-end thread did not finish in time"
    if "error" in box:
        raise box["error"]
    published.append(ba.GetKeyframeStates()[0])
    assert res.iterations_done == 5
    keys = {inverses(lib, p).tobytes() for p in published}
    assert len(keys) > 2, "the poses did not move"
    polls = box["polls"]
    print(f"{len(polls)} polls, {len({p.tobytes() for p in polls})} distinct pose sets, {len(keys)} published")
    for i, p in enumerate(polls):
        assert p.shape == (sc.cfg.num_keyframes, 7)
        assert p.tobytes() in keys, f"poll {i} is not the inverse of one published pose set"
