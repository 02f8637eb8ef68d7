"""A dataset in the reference's input layout -> keyframes -> surfels -> bundle adjustment, entirely through the public API:

    python tools/run_dataset.py --make-synthetic /tmp/synth      # writes a synthetic sequence in the TUM / ETH3D layout
    python tools/run_dataset.py /tmp/synth --trajectory groundtruth.txt --keyframe-interval 1 --raw-to-float-depth 0.001
    python tools/run_dataset.py /path/to/eth3d/sequence --trajectory groundtruth.txt        # 5000 raw units per metre (default)

Every `--keyframe-interval`-th frame becomes a keyframe at its trajectory pose, perturbed by --pose-noise to give BA something to
do: raw depth + colour are uploaded, DirectBA.CreateKeyframeFromFrame preprocesses them on the device (bba_preprocess_frame, or
bba_preprocess_raw_frame with --median-filter-iterations / --pyramid-level-for-depth / --pyramid-level-for-color: the
full-resolution frames are uploaded and filtered or downscaled in the same launch, the cameras are the calibration's
Scaled(0.5 ** level)) and adds the keyframe, surfels are created for it, and BundleAdjustment runs every --ba-interval keyframes.
Prints one JSON line.

With --export-poses PATH every frame gets a pose, as BadSlam computes one: each frame after the first keyframe is preprocessed
and tracked against the last keyframe with the image-pair odometry (bba_track_frame_pairwise), seeded by the motion model
(direct_ba.MotionModel: predict, track, push; rebased when the frame becomes a keyframe), like BadSlam::RunOdometry.  Keyframes
keep their trajectory pose (+ noise).  Every BundleAdjustment call is wrapped in RememberKeyframePoses /
ExtrapolateAndInterpolateKeyframePoseChanges, so the tracked frames move with their keyframes, and the trajectory of all frames
is written in the TUM format of rgbd_dataset.save_poses:

    python tools/run_dataset.py /tmp/synth --keyframe-interval 2 --raw-to-float-depth 0.001 --export-poses /tmp/synth/poses.txt

With --refine-frames (needs --export-poses) the handle gets --refine-headroom free keyframe slots, the preprocessed buffers of every
tracked frame are kept on the device, and after the last BA every frame that is not a keyframe is tracked against the final
surfel map in one call (DirectBA.EstimateFramePosesFromBuffers, bba_estimate_frame_poses_for_frames, which runs in chunks of the
free slots), starting from its deformed pose; the JSON line then also gives the refined frame-pose error and the seconds the
refinement took.  That keeps every frame's buffers resident: about 2.5 MB per 640x480 frame.

With --pose-prior-sigma T,R every keyframe gets a soft pose prior at its trajectory pose (DirectBA.SetKeyframePosePriors) with
the information diag(1/T^2 x3, 1/R^2 x3), T in metres and R in radians, which holds the map in the trajectory's frame.  The JSON
line always gives the keyframes' absolute error against the trajectory ("max_abs_keyframe_error_m_rad"); with the flag it also
repeats the run without priors on the same noisy poses and gives that error as "max_abs_keyframe_error_without_priors_m_rad".

With --attitude-prior-sigma R every keyframe gets an attitude prior (DirectBA.SetKeyframeAttitudePriors): the map-frame direction
d_ref = (0, 0, -1) as measured in the keyframe's camera frame at its trajectory pose, turned by seeded noise of R radians about a
random axis, with the information 1/R^2.  That is what an accelerometer at rest reports as gravity, and it holds the map's roll and
pitch.  The JSON line always gives the keyframes' mean tilt error against the trajectory ("mean_tilt_error_rad"); with the flag it
also repeats the run without attitude priors and gives that error as "mean_tilt_error_without_attitude_priors_rad".  Both flags
together repeat the run without either.

With --keyframe-min-new-fraction F (needs --export-poses) keyframes are chosen by what the map already explains: a tracked frame
becomes a keyframe when the surfels its creation would add cover at least F of its valid sparse cells (new_surfels / valid_cells of
DirectBA.MeasureFrameOverlap, bba_measure_frame_overlap, at its tracked pose), or when --keyframe-interval frames have passed since
the last keyframe, up to --max-keyframes.  A slow camera then adds fewer keyframes and a fast one more.  The JSON line gives the
keyframe count either way.

With --exposure-compensation the gains of every keyframe are estimated from the surfels they share and set before every
BundleAdjustment call (DirectBA.EstimateKeyframeExposures / SetKeyframeExposures, DESIGN §3.21), so that an auto-exposure camera's
brightness changes do not bias the descriptor residuals; a keyframe that shares nothing with keyframe 0 keeps its gain.  The JSON
line gives the smallest and largest gain set ("exposure_gain_min_max").

The views of --make-synthetic lie metres apart (a BA test scene, not a video), so odometry between them fails and only the
keyframe poses of that sequence are meaningful; on a recorded sequence every frame is tracked from its neighbour.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def make_synthetic(folder, name="small"):
    from badslam_b200 import rgbd_dataset as D
    from badslam_b200 import scene as S
    sc = S.make_scene(S.config_by_name(name))
    frames = [S.raw_frame(sc, k, noise_raw=1.0) for k in range(sc.cfg.num_keyframes)]
    stamps = [1000.0 + 0.1 * k for k in range(sc.cfg.num_keyframes)]
    D.write_tum_dataset(folder, sc.depth_K, [f[1] for f in frames], [f[0] for f in frames], stamps, sc.poses_true)
    print(f"wrote {len(frames)} frames ({sc.cfg.width}x{sc.cfg.height}, raw_to_float_depth {sc.cfg.raw_to_float_depth}) to {folder}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("folder", nargs="?")
    ap.add_argument("--make-synthetic", metavar="DIR")
    ap.add_argument("--trajectory", default="groundtruth.txt")
    ap.add_argument("--keyframe-interval", type=int, default=10)       # bad_slam_config.h: keyframe_interval
    ap.add_argument("--max-keyframes", type=int, default=200)
    ap.add_argument("--ba-interval", type=int, default=10, help="run BundleAdjustment after this many new keyframes (and at the end)")
    ap.add_argument("--ba-iterations", type=int, default=10)
    ap.add_argument("--raw-to-float-depth", type=float, default=1.0 / 5000.0)   # bad_slam_config.h: raw_to_float_depth
    ap.add_argument("--max-depth", type=float, default=3.0)
    ap.add_argument("--cell-size", type=int, default=4)
    ap.add_argument("--max-surfels", type=int, default=20_000_000)
    ap.add_argument("--pose-noise", type=float, default=0.002, help="metres / radians added to the trajectory poses")
    ap.add_argument("--median-filter-iterations", type=int, default=0,        # bad_slam_config.h: median_filter_and_densify_iterations
                    help="median densify filter passes over the raw depth (0..8)")
    ap.add_argument("--pyramid-level-for-depth", type=int, default=0, help="downscale the depth by 2^level (0..3)")
    ap.add_argument("--pyramid-level-for-color", type=int, default=0, help="downscale the colour by 2^level (0..3)")
    ap.add_argument("--export-poses", metavar="PATH", default=None,
                    help="track every frame, deform the tracked poses with each BA call and write all frames' poses (TUM format)")
    ap.add_argument("--refine-frames", action="store_true",
                    help="after the last BA, refine every non-keyframe pose against the final map in one call (needs --export-poses)")
    ap.add_argument("--keyframe-min-new-fraction", metavar="F", type=float, default=None,
                    help="make a tracked frame a keyframe when its new surfels would cover at least this fraction of its valid cells, "
                         "or after --keyframe-interval frames (needs --export-poses)")
    ap.add_argument("--refine-headroom", type=int, default=64, help="free keyframe slots the handle keeps for --refine-frames")
    ap.add_argument("--pose-prior-sigma", metavar="T,R", default=None,
                    help="anchor every keyframe to its trajectory pose with a soft prior of these sigmas (metres, radians)")
    ap.add_argument("--attitude-prior-sigma", metavar="RAD", type=float, default=None,
                    help="give every keyframe an attitude prior from its trajectory pose with this sigma (radians)")
    ap.add_argument("--exposure-compensation", action="store_true",
                    help="estimate and set every keyframe's exposure gain before every BundleAdjustment call")
    a = ap.parse_args()
    if a.refine_frames and a.export_poses is None:
        ap.error("--refine-frames needs --export-poses")
    if a.keyframe_min_new_fraction is not None and a.export_poses is None:
        ap.error("--keyframe-min-new-fraction needs --export-poses")
    if a.make_synthetic:
        make_synthetic(a.make_synthetic)
        return 0
    if a.pose_prior_sigma is not None:
        try:
            a.pose_prior_sigma = [float(x) for x in a.pose_prior_sigma.split(",")]
            assert len(a.pose_prior_sigma) == 2 and min(a.pose_prior_sigma) > 0
        except (ValueError, AssertionError):
            ap.error("--pose-prior-sigma takes two positive numbers T,R")
    if a.attitude_prior_sigma is not None and not a.attitude_prior_sigma > 0:
        ap.error("--attitude-prior-sigma takes a positive number RAD")
    if a.pose_prior_sigma is not None or a.attitude_prior_sigma is not None:
        line = run(a, a.pose_prior_sigma, a.attitude_prior_sigma)
        without = run(a, None, None) if line is not None else None
        if without is None:
            return 1
        if a.pose_prior_sigma is not None:
            line["max_abs_keyframe_error_without_priors_m_rad"] = without["max_abs_keyframe_error_m_rad"]
        if a.attitude_prior_sigma is not None:
            line["mean_tilt_error_without_attitude_priors_rad"] = without["mean_tilt_error_rad"]
    else:
        line = run(a, None, None)
    if line is None:
        return 1
    print(json.dumps(line))
    return 0


DOWN = np.array([0.0, 0.0, -1.0])   # d_ref of --attitude-prior-sigma, map frame


def tilt(pose, S):
    """DOWN in the camera frame of global_T_frame `pose`."""
    return S.quat_to_R(np.asarray(pose[:4], np.float64)).T @ DOWN


def run(a, prior_sigma, attitude_sigma):
    """One pass over the sequence; returns the JSON line's fields (None if the poses could not be written)."""
    import torch
    from badslam_b200 import rgbd_dataset as D
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA, MotionModel, PinholeCamera4f
    ds = D.TUMRGBDDataset(a.folder, a.trajectory)
    cam = PinholeCamera4f(ds.width, ds.height, ds.camera_parameters)
    dynamic = a.keyframe_min_new_fraction is not None
    # the keyframes' frame indices: every --keyframe-interval-th frame, or (dynamic) decided frame by frame after tracking
    idx = [] if dynamic else list(range(0, len(ds), a.keyframe_interval))[:a.max_keyframes]
    # main.cc:457-460: the cameras of the handle are the calibration scaled to the pyramid levels
    depth_cam, color_cam = cam.Scaled(0.5 ** a.pyramid_level_for_depth), cam.Scaled(0.5 ** a.pyramid_level_for_color)
    ba = DirectBA(a.max_surfels, a.raw_to_float_depth, 40.0, a.cell_size, color_camera_initial_estimate=color_cam,
                  depth_camera_initial_estimate=depth_cam,
                  max_keyframes=(a.max_keyframes if dynamic else len(idx)) + (a.refine_headroom if a.refine_frames else 0))
    raw_options = dict(median_filter_and_densify_iterations=a.median_filter_iterations,
                       pyramid_level_for_depth=a.pyramid_level_for_depth, pyramid_level_for_color=a.pyramid_level_for_color)
    surfels = torch.zeros((17, a.max_surfels), dtype=torch.float32, device="cuda")
    ba.SetSurfels(surfels, 0)
    rng = np.random.default_rng(0)
    rng_attitude = np.random.default_rng(1)   # (a stream of its own: the pose noise stays that of a run without the flag)
    true_poses, t_pre, t_ba, created, results = [], 0.0, 0.0, 0, []
    export = a.export_poses is not None
    keyframe_frames = set(idx)
    frame_poses = np.zeros((len(ds), 7), np.float32)   # global_T_frame of every frame (--export-poses)
    motion_model, base_kf, tracked, t_odometry = MotionModel(), None, 0, 0.0
    kept = {}   # --refine-frames: frame index -> its preprocessed (depth, normals, rgba)
    n = -1   # keyframes added so far - 1
    last_ba = -1   # n at the last BundleAdjustment
    gain_range = [np.inf, -np.inf]   # --exposure-compensation: the smallest and largest gain set

    def bundle_adjust(i):
        nonlocal t_ba, last_ba
        original = ba.RememberKeyframePoses() if export else None
        t = time.perf_counter()
        if a.exposure_compensation:
            gains = ba.EstimateKeyframeExposures()[0]
            gains = np.where(np.isnan(gains), ba.GetKeyframeExposures(), gains).astype(np.float32)
            ba.SetKeyframeExposures(gains)
            gain_range[0], gain_range[1] = min(gain_range[0], float(gains.min())), max(gain_range[1], float(gains.max()))
        r = ba.BundleAdjustment(None, False, False, True, True, True, 1, a.ba_iterations)
        torch.cuda.synchronize()
        t_ba += time.perf_counter() - t
        results.append((r.iterations_done, int(r.depth_residual_count + r.descriptor_residual_count), r.surfels_size))
        if export:   # bad_slam.cc:1267-1301
            ba.ExtrapolateAndInterpolateKeyframePoseChanges(0, i, original, [k.frame_index for k in ba.keyframes()], frame_poses)
        last_ba = n

    for i in (range(len(ds)) if export else idx):
        overlap = None
        if export and base_kf is not None:
            # BadSlam::RunOdometry: the frame against the last keyframe, seeded by the motion model
            raw = torch.from_numpy(ds.load_depth(i).view(np.int16)).cuda()
            rgb = torch.from_numpy(ds.load_color(i)).cuda()
            torch.cuda.synchronize()
            t = time.perf_counter()
            depth, normals, _, rgba, lo, hi = ba.PreprocessFrame(raw, rgb, max_depth=a.max_depth, want_min_max=dynamic, **raw_options)
            e1, e2 = motion_model.PredictFramePose()
            base_T_frame, _ = ba.TrackFramePairwise(None, base_kf.id, depth, normals, rgba, e1, e2)
            motion_model.Push(base_T_frame)
            ba._lib.bba_host_se3_compose(base_kf.global_T_frame().ctypes.data, base_T_frame.ctypes.data, frame_poses[i].ctypes.data)
            torch.cuda.synchronize()
            t_odometry += time.perf_counter() - t
            tracked += 1
            if dynamic and 0 < lo <= hi:   # what the map already explains of the frame at its tracked pose
                overlap = ba.MeasureFrameOverlap([(depth, normals)], [(0, frame_poses[i], lo, hi)], with_shared=False)
            if dynamic:
                fraction = (float(overlap.new_surfels[0]) / max(1, int(overlap.valid_cells[0]))) if overlap is not None else 0.0
                if len(idx) < a.max_keyframes and (fraction >= a.keyframe_min_new_fraction or i - idx[-1] >= a.keyframe_interval):
                    idx.append(i)
                    keyframe_frames.add(i)
            if a.refine_frames and i not in keyframe_frames:
                kept[i] = (depth, normals, rgba)
        elif dynamic and not idx:
            idx.append(i)   # the first frame
            keyframe_frames.add(i)
        if i not in keyframe_frames:
            continue
        n += 1
        pose = ds.frames[i].depth_global_T_frame
        true_poses.append(pose)
        noisy = S.se3_mul(pose, S.se3_exp(np.concatenate([rng.normal(0, a.pose_noise, 3), rng.normal(0, a.pose_noise, 3)])))
        raw = torch.from_numpy(ds.load_depth(i).view(np.int16)).cuda()
        rgb = torch.from_numpy(ds.load_color(i)).cuda()
        torch.cuda.synchronize()
        t = time.perf_counter()
        kf = ba.CreateKeyframeFromFrame(i, raw, rgb, noisy, max_depth=a.max_depth, **raw_options)
        if prior_sigma is not None:
            ba.SetKeyframePosePriors([kf.id], [pose], np.diag([prior_sigma[0] ** -2] * 3 + [prior_sigma[1] ** -2] * 3))
        if attitude_sigma is not None:
            axis = rng_attitude.normal(size=3)
            noise = S.se3_exp(np.r_[0.0, 0.0, 0.0, rng_attitude.normal(0, attitude_sigma) * axis / np.linalg.norm(axis)])
            measured = tilt(S.se3_mul(pose, noise), S)
            ba.SetKeyframeAttitudePriors([kf.id], DOWN, measured[None], attitude_sigma ** -2)
        created += ba.CreateSurfelsForKeyframe(None, True, kf.id)
        torch.cuda.synchronize()
        t_pre += time.perf_counter() - t
        if export:
            frame_poses[i] = noisy
            if base_kf is not None:
                motion_model.Rebase()   # bad_slam.cc:1057-1068: the frame tracked last became a keyframe
            base_kf = kf
        if (n + 1) % a.ba_interval == 0 or (not dynamic and n + 1 == len(idx)):
            bundle_adjust(i)
    if dynamic and last_ba != n:
        bundle_adjust(len(ds) - 1)
    poses = ba.GetKeyframeStates()[0]
    rel = lambda P, k: S.se3_mul(S.se3_inverse(P[0]), P[k])
    err = [S.pose_error(rel(poses, k), rel(true_poses, k)) for k in range(1, len(idx))]
    line = {"frames": len(ds), "keyframes": len(idx), "image": [ds.width, ds.height],
            "depth_image": [depth_cam.width, depth_cam.height], "surfels_created": created,
            "surfels": ba.surfels_size(), "ba_calls": results, "seconds_preprocess_and_creation": round(t_pre, 3),
            "seconds_bundle_adjustment": round(t_ba, 3),
            "max_relative_pose_error_m_rad": [max(e[0] for e in err), max(e[1] for e in err)] if err else None}
    abs_err = [S.pose_error(poses[k], true_poses[k]) for k in range(len(idx))]
    line["max_abs_keyframe_error_m_rad"] = [max(e[0] for e in abs_err), max(e[1] for e in abs_err)]
    tilts = [np.arccos(np.clip(tilt(poses[k], S) @ tilt(true_poses[k], S), -1.0, 1.0)) for k in range(len(idx))]
    line["mean_tilt_error_rad"] = float(np.mean(tilts))
    if a.exposure_compensation:
        line["exposure_gain_min_max"] = gain_range if np.isfinite(gain_range[0]) else None
    if prior_sigma is not None:
        line["pose_prior_sigma_m_rad"] = prior_sigma
    if attitude_sigma is not None:
        line["attitude_prior_sigma_rad"] = attitude_sigma
    if export:
        frame_poses[idx] = poses
        all_true = [f.depth_global_T_frame for f in ds.frames]
        max_err = lambda P: ([max(e[0] for e in err), max(e[1] for e in err)]
                             if (err := [S.pose_error(rel(P, k), rel(all_true, k)) for k in range(1, len(ds))]) else None)
        line.update({"frames_tracked": tracked, "seconds_odometry": round(t_odometry, 3), "poses_exported": len(ds),
                     "max_relative_frame_pose_error_m_rad": max_err(frame_poses)})
        if a.refine_frames and kept:
            # every tracked frame against the final map, from its deformed pose, in one call
            order = sorted(kept)
            torch.cuda.synchronize()
            t = time.perf_counter()
            refined = ba.EstimateFramePosesFromBuffers(None, [kept[i] for i in order], frame_poses[order])[0]
            torch.cuda.synchronize()
            frame_poses[order] = refined
            line.update({"frames_refined": len(order), "seconds_refinement": round(time.perf_counter() - t, 3),
                         "max_relative_frame_pose_error_refined_m_rad": max_err(frame_poses)})
        if not D.save_poses(a.export_poses, [f.depth_time_string for f in ds.frames], frame_poses):
            print(f"cannot write {a.export_poses}", file=sys.stderr)
            return None
    return line


if __name__ == "__main__":
    sys.exit(main())
