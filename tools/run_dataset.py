"""A dataset in the reference's input layout -> keyframes -> surfels -> bundle adjustment, entirely through the public API:

    python tools/run_dataset.py --make-synthetic /tmp/synth      # writes a synthetic sequence in the TUM / ETH3D layout
    python tools/run_dataset.py /tmp/synth --trajectory groundtruth.txt --keyframe-interval 1 --raw-to-float-depth 0.001
    python tools/run_dataset.py /path/to/eth3d/sequence --trajectory groundtruth.txt        # 5000 raw units per metre (default)

Every `--keyframe-interval`-th frame becomes a keyframe at its trajectory pose (the reference's odometry front-end is out of
scope: poses come from the file, perturbed by --pose-noise to give BA something to do): raw depth + colour are uploaded,
DirectBA.CreateKeyframeFromFrame preprocesses them on the device (bba_preprocess_frame, or bba_preprocess_raw_frame with
--median-filter-iterations / --pyramid-level-for-depth / --pyramid-level-for-color: the full-resolution frames are uploaded and
filtered or downscaled in the same launch, the cameras are the calibration's Scaled(0.5 ** level)) and adds the keyframe,
surfels are created for it, and BundleAdjustment runs every --ba-interval keyframes.  Prints one JSON line.
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
    a = ap.parse_args()
    if a.make_synthetic:
        make_synthetic(a.make_synthetic)
        return 0
    import torch
    from badslam_b200 import rgbd_dataset as D
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA, PinholeCamera4f
    ds = D.TUMRGBDDataset(a.folder, a.trajectory)
    cam = PinholeCamera4f(ds.width, ds.height, ds.camera_parameters)
    idx = list(range(0, len(ds), a.keyframe_interval))[:a.max_keyframes]
    # main.cc:457-460: the cameras of the handle are the calibration scaled to the pyramid levels
    depth_cam, color_cam = cam.Scaled(0.5 ** a.pyramid_level_for_depth), cam.Scaled(0.5 ** a.pyramid_level_for_color)
    ba = DirectBA(a.max_surfels, a.raw_to_float_depth, 40.0, a.cell_size, color_camera_initial_estimate=color_cam,
                  depth_camera_initial_estimate=depth_cam, max_keyframes=len(idx))
    raw_options = dict(median_filter_and_densify_iterations=a.median_filter_iterations,
                       pyramid_level_for_depth=a.pyramid_level_for_depth, pyramid_level_for_color=a.pyramid_level_for_color)
    surfels = torch.zeros((17, a.max_surfels), dtype=torch.float32, device="cuda")
    ba.SetSurfels(surfels, 0)
    rng = np.random.default_rng(0)
    true_poses, t_pre, t_ba, created, results = [], 0.0, 0.0, 0, []
    for n, i in enumerate(idx):
        pose = ds.frames[i].depth_global_T_frame
        true_poses.append(pose)
        noisy = S.se3_mul(pose, S.se3_exp(np.concatenate([rng.normal(0, a.pose_noise, 3), rng.normal(0, a.pose_noise, 3)])))
        raw = torch.from_numpy(ds.load_depth(i).view(np.int16)).cuda()
        rgb = torch.from_numpy(ds.load_color(i)).cuda()
        torch.cuda.synchronize()
        t = time.perf_counter()
        kf = ba.CreateKeyframeFromFrame(i, raw, rgb, noisy, max_depth=a.max_depth, **raw_options)
        created += ba.CreateSurfelsForKeyframe(None, True, kf.id)
        torch.cuda.synchronize()
        t_pre += time.perf_counter() - t
        if (n + 1) % a.ba_interval == 0 or n + 1 == len(idx):
            t = time.perf_counter()
            r = ba.BundleAdjustment(None, False, False, True, True, True, 1, a.ba_iterations)
            torch.cuda.synchronize()
            t_ba += time.perf_counter() - t
            results.append((r.iterations_done, int(r.depth_residual_count + r.descriptor_residual_count), r.surfels_size))
    poses = ba.GetKeyframeStates()[0]
    rel = lambda P, k: S.se3_mul(S.se3_inverse(P[0]), P[k])
    err = [S.pose_error(rel(poses, k), rel(true_poses, k)) for k in range(1, len(idx))]
    print(json.dumps({"frames": len(ds), "keyframes": len(idx), "image": [ds.width, ds.height],
                      "depth_image": [depth_cam.width, depth_cam.height], "surfels_created": created,
                      "surfels": ba.surfels_size(), "ba_calls": results, "seconds_preprocess_and_creation": round(t_pre, 3),
                      "seconds_bundle_adjustment": round(t_ba, 3),
                      "max_relative_pose_error_m_rad": [max(e[0] for e in err), max(e[1] for e in err)] if err else None}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
