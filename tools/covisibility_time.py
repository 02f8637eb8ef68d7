"""What keyframe co-visibility costs (bba_measure_keyframe_covisibility, DESIGN §3.19): one all-pairs call, its bits and Gram
kernels separately, and the surfel deformation and the activation pass on the same map, in the same session.

Workloads: cfg3, cfg2, cfg3_rank8 (every keyframe active at poses_init) and 2 500 keyframes at cfg1's 80x60 image size over a
1 M-surfel map (three chunks of the 128 MiB budget).  Each call is timed on the host around the call (it ends in a synchronise);
the deformation (identity changes: it walks every pair and moves nothing) and the activation pass with CUDA events.  The kernel
split comes from a torch.profiler run of its own.  Prints the median and the range of every call, the chunks, the card's name and
power limit, and the registers and spills ptxas reported for the two kernels when the build log is present.

    python tools/covisibility_time.py [cfg3 cfg2 cfg3_rank8 kf2500] [--calls N] [--out results.json]
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
    log = os.path.join(ROOT, "badslam_b200", "_obj", "kernels.cu.log")
    if not os.path.exists(log):
        return "no build log"
    text = open(log).read()
    out = {}
    for k in ("CovisibilityBitsKernel", "CovisibilityGramKernel"):
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


def kernel_split(torch, fn, calls):
    """Mean device time per call of each co-visibility kernel and of the stream gather, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for key in ("CovisibilityBitsKernel", "CovisibilityGramKernel", "GeometryStreamKernel"):
            if key in e.key:
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                out[key] = round(t / 1e3 / calls, 4)
    return out


def scene(name):
    from badslam_b200.scene import SceneConfig, config_by_name, make_scene
    if name == "kf2500":
        return make_scene(SceneConfig(80, 60, 2500, 1_000_000, cell=1, seed=1, name="kf2500"))
    return make_scene(config_by_name(name))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["cfg3", "cfg2", "cfg3_rank8", "kf2500"])
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    from badslam_b200.direct_ba import DirectBA
    print("card:", card(), flush=True)
    print("registers:", registers(), flush=True)
    result = {"card": card(), "registers": registers()}
    for name in a.configs:
        sc = scene(name)
        K, n = sc.cfg.num_keyframes, sc.num_surfels
        ba = DirectBA.from_scene(sc, device="cuda:0")
        C = ba.MeasureKeyframeCovisibility()
        chunk = max(256, (128 << 20) * 8 // K // 256 * 256)
        r = {"keyframes": K, "surfels": n, "chunks": -(-n // chunk),
             "bit_row_MB": round(K * -(-min(chunk, n) // 32) * 4 / 1e6, 1),
             "pairs_sharing": int((C > 0).sum()), "mean_diagonal": round(float(np.diag(C).mean()), 1)}
        r["all_pairs_call"] = host_timed(torch, ba.MeasureKeyframeCovisibility, a.calls)
        r["kernels_ms_per_call"] = kernel_split(torch, ba.MeasureKeyframeCovisibility, max(3, a.calls // 2))
        original = ba.RememberKeyframePoses()
        r["deform_surfels"] = event_timed(torch, lambda: ba.DeformSurfelsWithKeyframePoseChanges(original), a.calls)
        r["update_surfel_activation"] = event_timed(torch, ba.UpdateSurfelActivation, a.calls)
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
