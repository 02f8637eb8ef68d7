"""What bba_verify_loop_closures costs (DESIGN §3.16): one call with k = 1, 21 and 64 candidates on cfg3 (200 keyframes, 640x480)
against the same work as 3 k single bba_track_frame_pairwise calls (the old keyframe's buffers given as the tracked frame) plus
the host agreement test and average, which is what a caller had to do before.  The two arms alternate, ten calls each per k.

The candidates all have the newest keyframe as the current one; their matches are the keyframes whose camera centres lie nearest
to it (ids with two neighbours only), each from the true relative pose.  Both arms track the same 3 k pairs from the same initial
estimates; the necessity test runs in the first arm only (the old way had no device equivalent).  The card's name, power limit
and SM clock are printed with the numbers.

    python tools/loop_verification_time.py [--calls 10] [--counts 1,21,64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--counts", default="1,21,64")
    ap.add_argument("--scene", default="cfg3")
    a = ap.parse_args()
    import ctypes as C
    import torch
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    from badslam_b200 import _lib
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import config_by_name, make_scene, se3_inverse, se3_mul
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(0)}), flush=True)
    sc = make_scene(config_by_name(a.scene))
    K = sc.cfg.num_keyframes
    ba = DirectBA.from_scene(sc, poses=sc.poses_true, device="cuda:0")
    lib = ba._lib
    current = K - 1
    centres = np.array([p[4:7] for p in sc.poses_true])
    order = [int(k) for k in np.argsort(np.linalg.norm(centres - centres[current], axis=1)) if 0 <= k < K - 3]
    F = C.POINTER(C.c_float)

    def host(fn, *args):
        out = np.zeros(7, np.float32)
        getattr(lib, fn)(*[np.ascontiguousarray(x, np.float32).ctypes.data for x in args], out.ctypes.data)
        return out

    def old_way(cands):
        refined_all = []
        for cur, matched, init in cands:
            ids = (matched, matched + 1, matched - 1 if matched > 0 else matched + 2)
            refined = np.zeros((3, 7), np.float32)
            for i, k in enumerate(ids):
                m = np.array([0, 0, 0, 1, 0, 0, 0], np.float32) if i == 0 else host(
                    "bba_host_se3_compose", host("bba_host_se3_inverse", sc.poses_true[matched]), sc.poses_true[k])
                e = host("bba_host_se3_compose", host("bba_host_se3_inverse", init), m)
                kf = ba._keyframes[k]
                est, _ = ba.TrackFramePairwise(None, cur, kf.depth_buffer, kf.normals_buffer, kf.color_buffer, e, e,
                                               test_different_initial_estimates=False)
                refined[i] = host("bba_host_se3_inverse", host("bba_host_se3_compose", m, host("bba_host_se3_inverse", est)))
            avg = np.zeros(7, np.float32)
            ang, tr = C.c_float(), C.c_float()
            lib.bba_host_loop_agreement(refined.ctypes.data, 0.0, 0.0, avg.ctypes.data, C.byref(ang), C.byref(tr))
            refined_all.append(refined)
        return refined_all

    for count in [int(c) for c in a.counts.split(",")]:
        cands = []
        for j in range(count):
            matched = order[j % len(order)]
            cands.append((current, matched, se3_mul(se3_inverse(sc.poses_true[matched]), sc.poses_true[current]).astype(np.float32)))
        ba.VerifyLoopClosures(None, cands)   # warm-up of both arms
        old_way(cands[:1])
        times = {"verify": [], "single_calls": []}
        launches = {}
        for _ in range(a.calls):
            before = ba.kernel_launch_count()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = ba.VerifyLoopClosures(None, cands)
            torch.cuda.synchronize()
            times["verify"].append((time.perf_counter() - t0) * 1e3)
            launches["verify"] = ba.kernel_launch_count() - before
            before = ba.kernel_launch_count()
            t0 = time.perf_counter()
            old_way(cands)
            torch.cuda.synchronize()
            times["single_calls"].append((time.perf_counter() - t0) * 1e3)
            launches["single_calls"] = ba.kernel_launch_count() - before
        statuses = [_lib.LOOP_STATUS_NAMES[v.status] for v in out]
        res = {"measurement": f"{a.scene}, {count} candidates ({3 * count} tracked pairs), host clock around a synchronised call, "
                              f"{a.calls} calls per arm, alternating",
               "launches": launches,
               "statuses": {s: statuses.count(s) for s in set(statuses)},
               "mean_iterations_level0": float(np.mean([v.tracking[i].iterations[0] for v in out for i in range(3)]))}
        for arm, t in times.items():
            t = np.array(t)
            res[arm] = {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3), "max_ms": round(float(t.max()), 3)}
        res["speedup"] = round(res["single_calls"]["median_ms"] / res["verify"]["median_ms"], 3)
        print(json.dumps(res), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
