"""What the place index costs (DESIGN §3.18): bba_index_keyframes for 200 keyframes at 640x480 in one call, a one-frame query
against 200 and against 2 500 indexed keyframes, and the 2 500 x 2 500 all-pairs query in one call.  Ten calls each; the median
and range of the host time around each call (every call ends in a synchronise, the index call by one added here).  The card's
name, power limit and SM clock are printed with the numbers.

The 200 keyframes are cfg2's 20 keyframes (640x480) added ten times each; the 2 500 keyframes are random 80x60 images on a cfg1
handle.  The encoding cost depends on the image size and the fern count, not on the content.

    python tools/place_index_time.py [--calls 10]
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


def timed(fn, calls):
    import torch
    fn()   # warm-up
    torch.cuda.synchronize()
    ms = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": round(float(np.median(ms)), 4), "min_ms": round(min(ms), 4), "max_ms": round(max(ms), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import config_by_name, make_scene
    print("card:", card(), flush=True)
    out = {}

    sc = make_scene(config_by_name("cfg2"))
    ba = DirectBA.from_scene(sc, poses=sc.poses_true, device="cuda:0", max_keyframes=200)
    while ba.KeyframeCount() < 200:
        k = ba.KeyframeCount() % len(sc.depth)
        ba.AddKeyframeHost(sc.depth[k], sc.normals[k], sc.radius[k], sc.color[k], sc.poses_true[k], sc.min_depth[k], sc.max_depth[k])
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int16) if x.dtype == np.uint16 else np.ascontiguousarray(x)).cuda()
    frame = (dev(sc.depth[3]), None, dev(sc.color[3]))
    out["index_200_kf_640x480"] = timed(lambda: ba.IndexKeyframes(), a.calls)
    out["query_1_frame_vs_200"] = timed(lambda: ba.QueryPlaceIndex([(-1, 0, 0, 199)], frames=[frame]), a.calls)
    out["query_1_keyframe_vs_200"] = timed(lambda: ba.QueryPlaceIndex([(3, 0, 0, 199)]), a.calls)
    del ba

    N = 2500
    sc1 = make_scene(config_by_name("cfg1"))
    ba = DirectBA.from_scene(sc1, poses=sc1.poses_true, device="cuda:0", max_keyframes=N)
    rng = np.random.default_rng(1)
    while ba.KeyframeCount() < N:
        d = rng.integers(400, 3200, (60, 80)).astype(np.uint16)
        c = rng.integers(0, 256, (60, 80, 4)).astype(np.uint8)
        ba.AddKeyframeHost(d, sc1.normals[0], sc1.radius[0], c, sc1.poses_true[0], 0.4, 3.2)
    ba.IndexKeyframes()
    frame = (dev(d), None, dev(c))
    out["index_2500_kf_80x60"] = timed(lambda: ba.IndexKeyframes(), a.calls)
    out["query_1_frame_vs_2500"] = timed(lambda: ba.QueryPlaceIndex([(-1, 0, 0, N - 1)], frames=[frame]), a.calls)
    queries = [(k, 0, 0, N - 1) for k in range(N)]
    out["all_pairs_2500"] = timed(lambda: ba.QueryPlaceIndex(queries, max_matches=8), a.calls)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
