"""What soft relative pose constraints cost: one cfg3 BA iteration (bench.py's step: surfels, poses and activations restored before
every step, no end tasks) in the alternating and in the PCG scheme, with constraints against none, on one handle, the two arms
alternating, three runs of each.  The constrained arm has a constraint between every consecutive keyframe pair and 50 seeded
random pairs, all with the true relative poses and sigma 1 cm / 0.01 rad; the arm without constraints removes them.  The card's
name and power limit are printed with the numbers.

    python tools/pose_constraint_time.py [--workload cfg3] [--steps 10] [--warmup 2] [--runs 3] [--random-pairs 50]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    import torch
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import config_by_name, make_scene, se3_inverse, se3_mul
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--random-pairs", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(0)}), flush=True)
    sc = make_scene(config_by_name(a.workload))
    K = sc.cfg.num_keyframes
    rng = np.random.default_rng(0)
    pairs = [(k, k + 1) for k in range(K - 1)]
    while len(pairs) < K - 1 + a.random_pairs:
        i, j = (int(x) for x in rng.choice(K, 2, replace=False))
        pairs.append((i, j))
    ca = np.array([p[0] for p in pairs])
    cb = np.array([p[1] for p in pairs])
    Z = np.array([se3_mul(se3_inverse(sc.poses_true[i]), sc.poses_true[j]) for i, j in pairs], np.float32)
    info = np.diag([1e4] * 6).astype(np.float32)
    results = {}
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

        out = {"none": [], "constrained": []}
        last = {}
        for _ in range(a.runs):
            for arm in ("none", "constrained"):
                if arm == "constrained":
                    ba.AddKeyframePoseConstraints(ca, cb, Z, info)
                else:
                    ba.RemoveKeyframePoseConstraints()
                for _ in range(a.warmup):
                    step()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    res = step()
                e1.record()
                torch.cuda.synchronize()
                out[arm].append(e0.elapsed_time(e1) / a.steps)
                last[arm] = (res.pose_iterations_total, res.pcg_inner_iterations_total, res.kernel_launches)
            ba.RemoveKeyframePoseConstraints()
        n, c = np.array(out["none"]), np.array(out["constrained"])
        results[scheme] = {"none": [round(x, 4) for x in n], "constrained": [round(x, 4) for x in c],
                           "median_ratio": round(float(np.median(c) / np.median(n)), 4),
                           "none_spread": round(float((n.max() - n.min()) / np.median(n)), 4),
                           "last_step (pose iterations, pcg inner iterations, launches)": last}
        del ba, surf, backup
        torch.cuda.empty_cache()
    print(json.dumps({"measurement": f"{a.workload} BA iteration, {len(pairs)} constraints vs none", "unit": "ms per iteration",
                      **results}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
