"""Measures what the front end (keyframe preprocessing + image-pair odometry of one frame) costs while a bundle adjustment runs
on the same handle -- BadSlam's default parallel_ba mode (INTEGRATION.md section 2) -- and what it costs the BA:

  * preprocess + track latency per frame (host wall time, both calls synchronise) on a high-priority stream, alone and while
    bba_bundle_adjust iterates on a low-priority stream on another thread;
  * BA time per iteration (pose + geometry, no intrinsics), alone and with the front end running beside it.

Each arm runs `--runs` times; the poses and activations are reset before every BA run so that every run does the same work.

    python tools/front_end_latency.py [--workload cfg3] [--iterations 5] [--frames 30] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    import torch
    name = torch.cuda.get_device_name()
    try:
        limit = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=power.limit",
                                "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        limit = "unknown"
    return name, limit or "unknown"


def spread(v):
    v = np.asarray(v, np.float64)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max()), "n": int(v.size)}


def main():
    import torch
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--iterations", type=int, default=5)
    ap.add_argument("--frames", type=int, default=30, help="frames per alone run")
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    name, power_limit = card()
    sc = S.make_scene(S.config_by_name(a.workload))
    ba = DirectBA.from_scene(sc)
    lo_p, hi_p = torch.cuda.Stream.priority_range()
    lo, hi = torch.cuda.Stream(priority=lo_p), torch.cuda.Stream(priority=hi_p)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int16) if x.dtype == np.uint16 else np.ascontiguousarray(x)).cuda()
    raw, rgb = S.raw_frame(sc, 0)
    raw, rgb = dev(raw), dev(rgb)
    d, n, _, c = S.render_frame(sc, S.se3_mul(sc.poses_true[0], S.se3_exp([0.02, -0.01, 0.015, 0.01, -0.008, 0.012])))
    frame = (dev(d), dev(n), dev(c))
    ident = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
    p0, a0 = ba.GetKeyframeStates()

    def one_frame():
        t = time.perf_counter()
        with torch.cuda.stream(hi):
            ba.PreprocessFrame(raw, rgb, stream=hi)            # min / max depth: synchronises hi
            ba.TrackFramePairwise(hi, 0, *frame, ident, ident)  # synchronises hi
        return (time.perf_counter() - t) * 1e3

    def run_ba():
        ba.SetKeyframeStates(p0, a0)
        torch.cuda.synchronize()
        t = time.perf_counter()
        with torch.cuda.stream(lo):
            r = ba.BundleAdjustment(lo, False, False, False, True, True, a.iterations, a.iterations)
        lo.synchronize()
        return (time.perf_counter() - t) * 1e3 / r.iterations_done

    for _ in range(3):   # warm-up: allocations, module load, both paths
        one_frame()
    run_ba()
    alone, ba_alone, concurrent, ba_concurrent, frames_concurrent = [], [], [], [], []
    for _ in range(a.runs):
        alone.append(float(np.median([one_frame() for _ in range(a.frames)])))
        ba_alone.append(run_ba())
        lat, done = [], threading.Event()

        def front_end():
            while not done.is_set():
                lat.append(one_frame())
        t = threading.Thread(target=front_end, daemon=True)
        t.start()
        try:
            ba_concurrent.append(run_ba())
        finally:
            done.set()
        t.join(600)
        assert not t.is_alive(), "front-end thread did not stop"
        lat = lat[:-1] if len(lat) > 1 else lat   # (the last frame may have run after the BA call ended)
        concurrent.append(float(np.median(lat)))
        frames_concurrent.append(len(lat))
    out = {"workload": a.workload, "gpu": name, "power_limit": power_limit, "ba_iterations": a.iterations,
           "front_end_ms_per_frame_alone": spread(alone), "front_end_ms_per_frame_beside_ba": spread(concurrent),
           "frames_beside_ba_per_run": frames_concurrent,
           "ba_ms_per_iteration_alone": spread(ba_alone), "ba_ms_per_iteration_with_front_end": spread(ba_concurrent)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
