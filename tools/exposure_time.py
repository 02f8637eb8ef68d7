"""What keyframe exposure estimation costs (bba_estimate_keyframe_exposures, DESIGN §3.21): the estimate over every keyframe at
one and two rounds, setting every keyframe's gain (bba_set_keyframe_exposures, one luma re-extraction each), and one all-pairs
co-visibility call on the same map for comparison, in the same session.

Workloads: cfg3 (200 keyframes, 3 M surfels) and 2 000 keyframes at cfg1's 80x60 image size over a 1 M-surfel map.  Each call
is timed on the host around the call (the estimate ends in a synchronise; the set is followed by one); the kernel split of the
two-round estimate comes from a torch.profiler run of its own.  Prints the median and range of every call, the card's name, power
limit and maximum SM clock, and the registers and spills ptxas reported for the new kernels when the build logs are present.

    python tools/exposure_time.py [cfg3 kf2000] [--calls N] [--out results.json]
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

KERNELS = ("ExposureWalkKernel", "CovisibilityGramKernel", "ExposureSolveKernel", "GeometryStreamKernel", "ExtractLumaKernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def registers():
    out = {}
    for unit, names in (("kernels.cu", ("ExposureWalkKernelILb0", "ExposureWalkKernelILb1")), ("exposure.cu", ("ExposureSolveKernel",))):
        log = os.path.join(ROOT, "badslam_b200", "_obj", unit + ".log")
        if not os.path.exists(log):
            out[unit] = "no build log"
            continue
        text = open(log).read()
        for k in names:
            m = re.search(r"Function properties for \S*" + k + r"\S*\n\s*(.*?spill loads)\n.*?(Used \d+ registers[^\n]*)", text)
            out[k] = f"{m.group(2)}, {m.group(1).strip()}" if m else "not found"
    return out


def host_timed(torch, fn, calls):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": round(float(np.median(ms)), 3), "min_ms": round(float(min(ms)), 3), "max_ms": round(float(max(ms)), 3)}


def kernel_split(torch, fn, calls):
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
            if key in e.key:
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                out[key] = round(out.get(key, 0.0) + t / 1e3 / calls, 4)
    return out


def scene(name):
    from badslam_b200.scene import SceneConfig, config_by_name, make_scene
    if name == "kf2000":
        return make_scene(SceneConfig(80, 60, 2000, 1_000_000, cell=1, seed=1, name="kf2000"))
    return make_scene(config_by_name(name))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["cfg3", "kf2000"])
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    from badslam_b200.direct_ba import DirectBA
    result = {"card": card(), "registers": registers()}
    print("card:", result["card"], flush=True)
    print("registers:", result["registers"], flush=True)
    for name in a.configs:
        sc = scene(name)
        K, n = sc.cfg.num_keyframes, sc.num_surfels
        ba = DirectBA.from_scene(sc, device="cuda:0")
        gains, obs, inl = ba.EstimateKeyframeExposures()
        r = {"keyframes": K, "surfels": n, "observations": int(obs.sum()), "inliers": int(inl.sum()),
             "unreached": int(np.isnan(gains).sum()),
             "gain_range": [float(np.nanmin(gains)), float(np.nanmax(gains))]}
        r["estimate_1_round"] = host_timed(torch, lambda: ba.EstimateKeyframeExposures(outer_iterations=1), a.calls)
        r["estimate_2_rounds"] = host_timed(torch, lambda: ba.EstimateKeyframeExposures(outer_iterations=2), a.calls)
        ones = np.ones(K, np.float32)
        r["set_all"] = host_timed(torch, lambda: ba.SetKeyframeExposures(ones), a.calls)
        r["covisibility_all_pairs"] = host_timed(torch, ba.MeasureKeyframeCovisibility, a.calls)
        r["kernels_ms_per_2_round_estimate"] = kernel_split(torch, lambda: ba.EstimateKeyframeExposures(outer_iterations=2),
                                                            max(3, a.calls // 2))
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
