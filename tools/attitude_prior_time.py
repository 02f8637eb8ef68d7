"""What attitude priors cost (DESIGN §3.17): an attitude prior on every keyframe against none, the two arms alternating on one
handle, three runs of each.

* The pose graph (bba_optimize_pose_graph) on the circle graphs of tools/pose_graph_time.py at K = 200 and K = 2500 with 50 random
  loops and the odometry chain, gauge keyframe 0; every call starts from the same drifted poses and is timed alone with CUDA
  events.  The attitude priors measure the truth's gravity direction with sigma 0.01 rad.  Gauss-Newton iterations are printed
  beside the times.
* One cfg3 BA iteration in the alternating and in the PCG scheme, as bench.py's step (surfels, poses and activations restored
  before every step), with attitude priors from the true poses (sigma 0.01 rad) on all 200 keyframes against none.

The card's name, power limit and SM clock are printed with the numbers.

    python tools/attitude_prior_time.py [--calls 10] [--steps 10] [--warmup 2] [--runs 3] [--no-cfg3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def events(torch, fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        last = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, last


def summary(out):
    t, c = np.array(out["none"]), np.array(out["attitude"])
    return {"none": [round(x, 4) for x in t], "attitude": [round(x, 4) for x in c],
            "median_ratio": round(float(np.median(c) / np.median(t)), 4),
            "none_spread": round(float((t.max() - t.min()) / np.median(t)), 4)}


def measured(poses32):
    """d_meas = R_k^-1 (0, 0, 1) of fp32 poses."""
    import pose_graph_oracle as O
    return np.array([O.from_array(p)[0].T @ UP for p in poses32], np.float32)


UP = np.array([0.0, 0.0, 1.0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--no-cfg3", action="store_true")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "attitude_prior_time.py needs a GPU"
    import pose_graph_oracle as O
    import test_gpu_pose_graph as T
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(0)}), flush=True)
    for K in (200, 2500):
        ba = T.make_handle(K)
        truth, start = T._circle(K)
        pairs = O.random_loops(K, 50, seed=7)
        ba.AddKeyframePoseConstraints([p for p, _ in pairs], [q for _, q in pairs], [T._relative(truth, p, q) for p, q in pairs],
                                      np.eye(6))
        d_meas = measured(T._f32(truth))
        out, last = {"none": [], "attitude": []}, {}

        def call():
            ba.SetKeyframeStates(start)
            return ba.OptimizePoseGraph()
        for _ in range(a.runs):
            for arm in ("none", "attitude"):
                if arm == "none":
                    ba.ClearKeyframeAttitudePriors()
                else:
                    ba.SetKeyframeAttitudePriors(np.arange(K), UP, d_meas, 1e4)
                events(torch, call, a.warmup)
                times = []
                for _ in range(a.calls):
                    ms, r = events(torch, call, 1)
                    times.append(ms)
                out[arm].append(float(np.median(times)))
                last[arm] = {"gauss_newton_iterations": r["iterations"], "pcg_iterations": r["linear_iterations"],
                             "converged": r["converged"]}
        print(json.dumps({"measurement": f"pose graph, {K} keyframes, 50 loops + chain, attitude priors on all vs none, median of {a.calls} calls per run",
                          "unit": "ms per call", **summary(out), "last_call": last}), flush=True)
        del ba
    if a.no_cfg3:
        print(json.dumps({"card_after": card()}), flush=True)
        return
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import config_by_name, make_scene
    sc = make_scene(config_by_name("cfg3"))
    K = sc.cfg.num_keyframes
    d_meas = measured(sc.poses_true)
    for scheme in ("alternating", "pcg"):
        ba = DirectBA.from_scene(sc)
        surf = ba.surfels()
        backup = surf[:8].clone()
        poses0, act0 = sc.poses_init.copy(), np.zeros(K, np.int32)
        ba.SetLastBAIterationCount(ba.ba_iteration_count())

        def step():
            surf[:8].copy_(backup, non_blocking=True)
            ba.SetKeyframeStates(poses0, act0)
            if scheme == "pcg":
                return ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, use_pcg=True, pcg_gauge_keyframe=0,
                                           increase_ba_iteration_count=False)
            return ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, increase_ba_iteration_count=False)
        out, last = {"none": [], "attitude": []}, {}
        for _ in range(a.runs):
            for arm in ("none", "attitude"):
                if arm == "none":
                    ba.ClearKeyframeAttitudePriors()
                else:
                    ba.SetKeyframeAttitudePriors(np.arange(K), UP, d_meas, 1e4)
                events(torch, step, a.warmup)
                ms, res = events(torch, step, a.steps)
                out[arm].append(ms)
                last[arm] = (res.pose_iterations_total, res.pcg_inner_iterations_total, res.kernel_launches)
        print(json.dumps({"measurement": f"cfg3 BA iteration ({scheme}), attitude priors on {K} keyframes vs none",
                          "unit": "ms per iteration", **summary(out),
                          "last_step (pose iterations, pcg inner iterations, launches)": last}), flush=True)
        del ba, surf, backup
        torch.cuda.empty_cache()
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
