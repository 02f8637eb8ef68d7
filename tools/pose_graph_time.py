"""What the keyframe pose graph (bba_optimize_pose_graph, DESIGN §3.14) costs.

Circle graphs (radius 5 m, the drift of tests/test_gpu_pose_graph.py) at K = 200 (cfg3's keyframe count) and K = 2500
(pcg_max_keyframes' default), with one loop (5, K - 3) and with 50 random loops, plus the odometry chain: every call starts from
the same drifted poses and is timed alone with CUDA events (the call synchronises once at its end).  Prints the median and the
range of the calls with the Gauss-Newton and PCG iteration counts, and, in a run of its own under torch.profiler, the device time
of each of the four kernels.  Then, on cfg3, the loop-closure sequence: the pose graph, bba_deform_surfels and one BA iteration,
each timed the same way, so that the pose graph's share is stated.  Also prints the card's name and power limit and the registers
and spills ptxas reported for the four kernels.

    python tools/pose_graph_time.py [--calls N] [--warmup W] [--no-cfg3]
"""
import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KERNELS = ("PoseGraphLinearizeKernel", "PoseGraphAssembleKernel", "PoseGraphSolveKernel", "PoseGraphUpdateKernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def registers():
    log = os.path.join(ROOT, "badslam_b200", "_obj", "pose_graph.cu.log")
    if not os.path.exists(log):
        return "no build log"
    text = open(log).read()
    out = {}
    for k in KERNELS:
        m = re.search(r"Function properties for \S*" + k + r"\S*\n\s*(.*?spill loads)\n.*?(Used \d+ registers)", text)
        out[k] = f"{m.group(2)}, {m.group(1).strip()}" if m else "not found"
    return out


def timed(torch, fn, before=None, calls=10, warmup=2):
    out, last = [], None
    for i in range(warmup + calls):
        if before:
            before()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        last = fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            out.append(e0.elapsed_time(e1))
    return {"median_ms": round(float(np.median(out)), 4), "min_ms": round(min(out), 4), "max_ms": round(max(out), 4)}, last


def kernel_split(torch, fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {k: [0.0, 0] for k in KERNELS}
    for ev in prof.events():
        for k in KERNELS:
            if k in ev.name and ev.device_type.name == "CUDA":
                split[k][0] += ev.device_time_total / 1000.0
                split[k][1] += 1
    return {k: {"ms": round(v[0], 4), "launches": v[1]} for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-cfg3", action="store_true")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "pose_graph_time.py needs a GPU"
    import pose_graph_oracle as O
    import test_gpu_pose_graph as T
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(0), "registers": registers()}), flush=True)
    for K in (200, 2500):
        ba = T.make_handle(K)
        truth, start = T._circle(K)
        for loops in (1, 50):
            pairs = [(5, K - 3)] if loops == 1 else O.random_loops(K, 50, seed=7)
            ba.RemoveKeyframePoseConstraints()
            ba.AddKeyframePoseConstraints([a for a, _ in pairs], [b for _, b in pairs], [T._relative(truth, a, b) for a, b in pairs],
                                          np.eye(6))
            restore = lambda: ba.SetKeyframeStates(start)   # noqa: E731
            row, r = timed(torch, ba.OptimizePoseGraph, restore, args.calls, args.warmup)
            restore()
            split = kernel_split(torch, ba.OptimizePoseGraph)
            print(json.dumps({"keyframes": K, "loops": loops, **row, "gauss_newton_iterations": r["iterations"],
                              "pcg_iterations": r["linear_iterations"], "converged": r["converged"], "kernels": split}), flush=True)
        del ba
    if args.no_cfg3:
        return
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    sc = S.make_scene(S.config_by_name("cfg3"))
    K = sc.cfg.num_keyframes
    ba = DirectBA.from_scene(sc)
    original = ba.RememberKeyframePoses()
    E = S.se3_exp([0.05, -0.04, 0.03, 0.02, -0.02, 0.03])
    drifted = np.array(sc.poses_init, np.float32, copy=True)
    for k in range(K // 2, K):
        drifted[k] = S.se3_mul(E, drifted[k]).astype(np.float32)
    ba.SetKeyframeStates(drifted)
    ba.DeformSurfelsWithKeyframePoseChanges(original)
    Z = S.se3_mul(S.se3_inverse(sc.poses_true[0]), sc.poses_true[K - 1])
    ba.AddKeyframePoseConstraints([0], [K - 1], [Z], np.diag([1e4] * 3 + [1e5] * 3))
    surfels = ba.SurfelsDeviceView()
    saved = surfels.clone()
    remembered = ba.RememberKeyframePoses()
    restore = lambda: ba.SetKeyframeStates(drifted)   # noqa: E731
    rows = {}
    rows["optimize_pose_graph"], r = timed(torch, ba.OptimizePoseGraph, restore, args.calls, args.warmup)
    rows["deform_surfels"], _ = timed(torch, lambda: ba.DeformSurfelsWithKeyframePoseChanges(remembered),
                                      lambda: surfels.copy_(saved), args.calls, args.warmup)
    rows["ba_iteration"], _ = timed(torch, lambda: ba.BundleAdjustment(None, False, False, False, True, True, 1, 1),
                                    lambda: (restore(), surfels.copy_(saved)), 3, 1)
    total = sum(v["median_ms"] for v in rows.values())
    for call, v in rows.items():
        print(json.dumps({"config": "cfg3", "call": call, "keyframes": K, **v, "share": round(v["median_ms"] / total, 4),
                          **({"gauss_newton_iterations": r["iterations"], "pcg_iterations": r["linear_iterations"]}
                             if call == "optimize_pose_graph" else {})}), flush=True)


if __name__ == "__main__":
    main()
