"""What the deterministic mode (bba_set_deterministic) costs: default against deterministic, alternating in one process, three runs
of each.

  * one BA iteration on cfg3 (bench.py's step: surfels, poses and activations restored before every step, no end tasks);
  * the same on cfg4 with the depth- and colour-intrinsics steps in every iteration (bench.py --intrinsics);
  * bba_track_frame_pairwise per frame (640x480, 5 scales, RunOdometry's options).
The card's name and power limit are printed with the numbers.

    python tools/deterministic_cost.py [--workloads cfg3,cfg4] [--steps 10] [--warmup 2] [--frames 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

RUNS = 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def ba_iteration(workload, intrinsics, steps, warmup):
    import torch
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import config_by_name, make_scene
    sc = make_scene(config_by_name(workload))
    ba = DirectBA.from_scene(sc)
    surf = ba.surfels()
    backup = surf[:8].clone()
    poses0, act0 = sc.poses_init.copy(), np.zeros(sc.cfg.num_keyframes, np.int32)
    ba.SetLastBAIterationCount(ba.ba_iteration_count())
    cam0 = (ba.depth_camera(), ba.color_camera(), ba.a(), ba.cfactor_buffer().copy())

    def step():
        surf[:8].copy_(backup, non_blocking=True)
        ba.SetKeyframeStates(poses0, act0)
        if intrinsics:
            ba.SetDepthCamera(cam0[0]); ba.SetColorCamera(cam0[1]); ba.SetA(cam0[2]); ba.SetCFactorBuffer(cam0[3])
        return ba.BundleAdjustment(None, intrinsics, intrinsics, False, True, True, 1, 1, increase_ba_iteration_count=False)

    out = {"default": [], "deterministic": []}
    results = {}
    for _ in range(RUNS):
        for mode in ("default", "deterministic"):
            ba.SetDeterministic(mode == "deterministic")
            for _ in range(warmup):
                step()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                res = step()
            e1.record()
            torch.cuda.synchronize()
            out[mode].append(e0.elapsed_time(e1) / steps)
            results[mode] = (res.pose_iterations_total, res.depth_residual_count, res.ms_pose_optimization, res.ms_intrinsics_optimization)
    return out, results


def tracking(frames):
    import torch
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    sc = S.make_scene(S.SceneConfig(width=640, height=480, num_keyframes=2, num_surfels=2000, cell=4, seed=31, name="odometry"))
    depth, normals, _, color = S.render_frame(sc, S.se3_mul(sc.poses_true[0], S.se3_exp([0.02, -0.01, 0.015, 0.01, -0.008, 0.012])))
    dev = (torch.from_numpy(depth.view(np.int16)).cuda(), torch.from_numpy(normals.view(np.int16)).cuda(), torch.from_numpy(color).cuda())
    ident = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
    init2 = S.se3_exp([0.01, 0, 0, 0, 0, 0])
    ba = DirectBA.from_scene(sc)
    out = {"default": [], "deterministic": []}
    for _ in range(RUNS):
        for mode in ("default", "deterministic"):
            ba.SetDeterministic(mode == "deterministic")
            for _ in range(3):
                ba.TrackFramePairwise(None, 0, *dev, ident, init2)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(frames):
                ba.TrackFramePairwise(None, 0, *dev, ident, init2)   # (synchronises: the call returns the estimate)
            out[mode].append((time.perf_counter() - t0) * 1e3 / frames)
    return out


def summary(name, unit, out, extra=None):
    d, t = np.array(out["default"]), np.array(out["deterministic"])
    line = {"measurement": name, "unit": unit, "default": [round(x, 4) for x in d], "deterministic": [round(x, 4) for x in t],
            "median_ratio": round(float(np.median(t) / np.median(d)), 4),
            "default_spread": round(float((d.max() - d.min()) / np.median(d)), 4)}
    if extra:
        line.update(extra)
    print(json.dumps(line), flush=True)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg3,cfg4")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--frames", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(0)}), flush=True)
    for w in [w for w in a.workloads.split(",") if w]:
        intr = w == "cfg4"
        out, res = ba_iteration(w, intr, a.steps, a.warmup)
        summary(f"{w} BA iteration" + (" with intrinsics" if intr else ""), "ms per iteration", out,
                {"last_step (pose iterations, residuals, ms pose, ms intrinsics)": res})
    summary("bba_track_frame_pairwise 640x480, 5 scales", "ms per frame", tracking(a.frames))
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
