"""What soft pose priors cost: one cfg3 BA iteration (bench.py's step: surfels, poses and activations restored before every step, no
end tasks) with a prior on every keyframe against none, on one handle, the two arms alternating, three runs of each.  The priors
sit on the true poses with sigma 1 cm / 0.01 rad; the arm without priors clears them.  The card's name and power limit are
printed with the numbers.

    python tools/pose_prior_time.py [--workload cfg3] [--steps 10] [--warmup 2] [--runs 3]
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
    from badslam_b200.scene import config_by_name, make_scene
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(0)}), flush=True)
    sc = make_scene(config_by_name(a.workload))
    K = sc.cfg.num_keyframes
    ba = DirectBA.from_scene(sc)
    surf = ba.surfels()
    backup = surf[:8].clone()
    poses0, act0 = sc.poses_init.copy(), np.zeros(K, np.int32)
    ba.SetLastBAIterationCount(ba.ba_iteration_count())
    info = np.diag([1e4] * 6).astype(np.float32)

    def step():
        surf[:8].copy_(backup, non_blocking=True)
        ba.SetKeyframeStates(poses0, act0)
        return ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, increase_ba_iteration_count=False)

    out = {"none": [], "all": []}
    last = {}
    for _ in range(a.runs):
        for arm in ("none", "all"):
            if arm == "all":
                ba.SetKeyframePosePriors(np.arange(K), sc.poses_true, info)
            else:
                ba.ClearKeyframePosePriors()
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
            last[arm] = (res.pose_iterations_total, res.ms_pose_optimization, res.kernel_launches)
    n, p = np.array(out["none"]), np.array(out["all"])
    print(json.dumps({"measurement": f"{a.workload} BA iteration, priors on {K} keyframes vs none", "unit": "ms per iteration",
                      "none": [round(x, 4) for x in n], "all": [round(x, 4) for x in p],
                      "median_ratio": round(float(np.median(p) / np.median(n)), 4),
                      "none_spread": round(float((n.max() - n.min()) / np.median(n)), 4),
                      "last_step (pose iterations, ms pose, launches)": last}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
