"""What estimating many frame poses in one call (bba_estimate_frame_poses_for_frames) saves over one
bba_estimate_frame_pose_for_frame call per frame.

On a cfg3 map (200 keyframes, 3 M surfels) with as many free keyframe slots as --free-slots, every entry count of --entries runs
as one batch call and as a loop of single-frame calls, alternating, --runs times each after one warm-up of each.  Entry i tracks
keyframe i's own buffers (given as a frame that is not a keyframe) from its initial pose moved by a few mm / mrad.  Each arm is
timed with the host clock around work that ends in a device synchronise.  The poses of the two arms must agree to 1e-5 m / rad.
The card's name and power limit are printed with the numbers.

    python tools/frame_pose_batch_time.py [--workload cfg3] [--entries 8,64,200] [--free-slots 200] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    import torch
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--entries", default="8,64,200")
    ap.add_argument("--free-slots", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(0)}), flush=True)
    sc = S.make_scene(S.config_by_name(a.workload))
    K = sc.cfg.num_keyframes
    ba = DirectBA.from_scene(sc, max_keyframes=K + a.free_slots)
    up16 = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int16)).cuda()
    frames = [(up16(sc.depth[k]), up16(sc.normals[k]), torch.from_numpy(np.ascontiguousarray(sc.color[k])).cuda()) for k in range(K)]
    rng = np.random.default_rng(0)
    for count in [int(c) for c in a.entries.split(",") if c]:
        fmap = [i % K for i in range(count)]
        init = np.stack([S.se3_mul(sc.poses_init[f], S.se3_exp(rng.normal(0, 0.002, 6))) for f in fmap]).astype(np.float32)

        def batch():
            out = ba.EstimateFramePosesFromBuffers(None, frames, init, fmap)
            torch.cuda.synchronize()
            return out

        def loop():
            out = [ba.EstimateFramePoseFromBuffers(None, init[i], *frames[f]) for i, f in enumerate(fmap)]
            torch.cuda.synchronize()
            return np.stack([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out])

        arms = {"batch": batch, "loop": loop}
        times = {k: [] for k in arms}
        launches = {}
        results = {k: fn() for k, fn in arms.items()}   # warm-up
        for _ in range(a.runs):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                c0 = ba.kernel_launch_count()
                t0 = time.perf_counter()
                results[name] = fn()
                times[name].append((time.perf_counter() - t0) * 1e3)
                launches[name] = ba.kernel_launch_count() - c0
        worst = max(max(S.pose_error(p, q)) for p, q in zip(results["batch"][0], results["loop"][0]))
        b, l = np.array(times["batch"]), np.array(times["loop"])
        print(json.dumps({"workload": a.workload, "keyframes": K, "surfels": sc.num_surfels, "free_slots": a.free_slots,
                          "entries": count, "unit": "ms per call / loop", "batch_ms": [round(x, 3) for x in b],
                          "loop_ms": [round(x, 3) for x in l], "speedup_median": round(float(np.median(l) / np.median(b)), 2),
                          "kernel_launches": launches, "max_gauss_newton_iterations": int(results["batch"][1].max()),
                          "converged": int(results["batch"][2].sum()), "worst_pose_difference_m_rad": float(worst),
                          "poses_agree_1e-5": bool(worst < 1e-5)}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
