"""What the frame overlap measurement costs (bba_measure_frame_overlap, DESIGN §3.20): calls of 1, 8 and 64 queries with and
without the keyframes' side (shared), their kernels separately, and bba_measure_keyframe_covisibility and
bba_create_surfels_for_keyframe on the same map, in the same session.

Workloads: cfg3 and cfg2 at poses_init.  A query is keyframe k's images at k's pose (query i uses keyframe i mod K), the case of a
tracked frame that looks at mapped surfaces.  Each call is timed on the host around the call (it ends in a synchronise).  The
creation runs on a map without spare capacity, so it counts, seeds and filters every call and appends nothing.  The kernel split
comes from a torch.profiler run of its own.  Prints the median and the range of every call, the card's name, power limit and
clock, and the registers and spills ptxas reported for the new kernels when the build log is present.

    python tools/frame_overlap_time.py [cfg3 cfg2] [--calls N] [--out results.json]
"""
import argparse
import json
import os
import re
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


def registers():
    logs = [os.path.join(ROOT, "badslam_b200", "_obj", f) for f in ("kernels.cu.log", "lifecycle.cu.log")]
    if not all(os.path.exists(p) for p in logs):
        return "no build log"
    text = "".join(open(p).read() for p in logs)
    out = {}
    for k in ("CovisibilityBitsKernelILb1", "CovisibilityGramKernel", "FrameSeedCountKernel"):
        m = re.search(r"Function properties for \S*" + k + r"\S*\n\s*(.*?spill loads)\n.*?(Used \d+ registers[^\n]*)", text)
        out[k] = f"{m.group(2)}, {m.group(1).strip()}" if m else "not found"
    return out


def stats(ms):
    return {"median_ms": round(float(np.median(ms)), 4), "min_ms": round(float(min(ms)), 4), "max_ms": round(float(max(ms)), 4)}


def host_timed(torch, fn, calls):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return stats(ms)


def event_timed(torch, fn, calls):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return stats(ms)


KERNELS = ("CovisibilityBitsKernel", "CovisibilityGramKernel", "GeometryStreamKernel", "FrameSeedCountKernel", "SupportLevel0Kernel",
           "SeedKernel", "FilterSeedsKernel", "ScanCountKernel", "CompactScanBlocksKernel", "ScanApplyKernel")


def kernel_split(torch, fn, calls):
    """Mean device time per call of each kernel of KERNELS a call runs, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for key in KERNELS:
            if key in e.key and (key != "SeedKernel" or "FrameSeedCountKernel" not in e.key):
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                out[key] = round(out.get(key, 0.0) + t / 1e3 / calls, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["cfg3", "cfg2"])
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import config_by_name, make_scene
    print("card:", card(), flush=True)
    print("registers:", registers(), flush=True)
    result = {"card": card(), "registers": registers()}
    for name in a.configs:
        sc = make_scene(config_by_name(name))
        K, n = sc.cfg.num_keyframes, sc.num_surfels
        ba = DirectBA.from_scene(sc, device="cuda:0")
        dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int16)).cuda()
        frames = [(dev(sc.depth[k]), dev(sc.normals[k])) for k in range(K)]
        poses = ba.GetKeyframeStates()[0]
        queries = [(i % K, poses[i % K], sc.min_depth[i % K], sc.max_depth[i % K]) for i in range(64)]
        r = {"keyframes": K, "surfels": n}
        for count in (1, 8, 64):
            for shared in (True, False):
                call = lambda: ba.MeasureFrameOverlap(frames, queries[:count], with_shared=shared)
                res = call()
                key = f"{count}_queries_{'shared' if shared else 'lean'}"
                r[key] = host_timed(torch, call, a.calls)
                if count == 1:
                    r[key]["counts"] = [int(res.observed_surfels[0]), int(res.valid_cells[0]), int(res.uncovered_cells[0]),
                                        int(res.new_surfels[0])]
        for count, shared in ((1, True), (1, False), (64, True)):
            r[f"kernels_ms_{count}_{'shared' if shared else 'lean'}"] = kernel_split(
                torch, lambda: ba.MeasureFrameOverlap(frames, queries[:count], with_shared=shared), max(3, a.calls // 2))
        r["keyframe_covisibility_call"] = host_timed(torch, ba.MeasureKeyframeCovisibility, a.calls)
        r["kernels_ms_keyframe_covisibility"] = kernel_split(torch, ba.MeasureKeyframeCovisibility, max(3, a.calls // 2))
        create = lambda: ba.CreateSurfelsForKeyframe(None, True, 0)
        r["create_surfels_call"] = host_timed(torch, create, a.calls)
        r["kernels_ms_create_surfels"] = kernel_split(torch, create, max(3, a.calls // 2))
        print(name, json.dumps(r), flush=True)
        result[name] = r
        del ba
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
