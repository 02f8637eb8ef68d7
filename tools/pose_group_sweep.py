"""GPU timing of the batched pose kernel (bba_debug_pose_coeffs_batch) at several keyframe-group sizes G (keyframes that share one
staged surfel tile, bba_debug_set_pose_group), with and without stats, on BASELINE configs.

Every keyframe is evaluated at poses_init in one work list, in the instantiation the BA pose step picks for it (512/PRE on cfg3,
the caller-order stream below the sort rule on cfg2), as in tools/pose_kernel_time.py.  The group sizes are visited in turn,
`--repeats` rounds each, so that every G's spread is measured across the same stretch of the session; CUDA events around
`--calls` back-to-back calls per window.  G = 0 is the library's own choice.  Prints the card, its power limit and the SM clock
sampled after each window with the numbers (one JSON line per config, stats and G, then a summary line per config and stats).

    python tools/pose_group_sweep.py [cfg3 cfg3_rank8 cfg2 ...] [--groups 8 16 24 32 64] [--calls N] [--repeats R]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_state():
    """Card name, power limit and current SM clock from nvidia-smi (read only); None where it is not available."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"card": out[0], "power_limit_w": float(out[1]), "sm_clock_mhz": int(out[2])}
    except Exception:   # noqa: BLE001 -- the timing stands without it
        return {"card": None, "power_limit_w": None, "sm_clock_mhz": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["cfg3", "cfg3_rank8", "cfg2"])
    ap.add_argument("--groups", type=int, nargs="+", default=[8, 16, 24, 32, 64])
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "pose_group_sweep.py needs a GPU"
    from badslam_b200 import _lib
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA

    for name in args.configs:
        sc = S.make_scene(S.config_by_name(name))
        ba = DirectBA.from_scene(sc)
        ids = np.arange(sc.cfg.num_keyframes)
        poses = sc.poses_init[ids]
        for stats in (False, True):
            times = {g: [] for g in args.groups}
            for rep in range(args.repeats):
                for g in args.groups:
                    ba.DebugSetPoseGroup(g)
                    for _ in range(args.warmup):
                        ba.PoseCoeffsBatch(ids, poses, _lib.POSE_VARIANT_AUTO, with_stats=stats)
                    torch.cuda.synchronize()
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                    for _ in range(args.calls):
                        _, _, counts, _ = ba.PoseCoeffsBatch(ids, poses, _lib.POSE_VARIANT_AUTO, with_stats=stats)
                    ev1.record()
                    torch.cuda.synchronize()
                    ms = ev0.elapsed_time(ev1) / args.calls
                    times[g].append(ms)
                    print(json.dumps({"config": name, "stats": stats, "group": g, "round": rep, "keyframes": len(ids),
                                      "surfels": int(sc.num_surfels), "ms_per_call": round(ms, 4),
                                      "assoc_pairs": int(counts[:, 2].sum()), **gpu_state()}), flush=True)
            print(json.dumps({"config": name, "stats": stats, "summary": {
                str(g): {"median_ms": round(float(np.median(t)), 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4)}
                for g, t in times.items()}}), flush=True)
        ba.DebugSetPoseGroup(0)


if __name__ == "__main__":
    main()
