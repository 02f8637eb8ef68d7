"""What the surfel deformation (bba_deform_surfels, DESIGN §3.13) costs, next to the activation pass and a geometry iteration in
the same session.

Per config: every keyframe active at poses_init; the keyframes >= K/2 then move by one change (0.3 m, 20 degrees), the loop-closure
case.  Each timed deformation starts from the same map (restored by a device copy outside the timed window) and is timed alone with
CUDA events, without the counters (no synchronise inside the call).  The activation pass and the geometry iteration are timed the
same way.  Prints the median and the spread (min .. max) of every call, the card's name and power limit, and the registers and
spills ptxas reported for DeformSurfelsKernel when the build log is present.

    python tools/surfel_deform_time.py [cfg3 cfg2 ...] [--calls N] [--warmup W]
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def registers():
    log = os.path.join(ROOT, "badslam_b200", "_obj", "kernels.cu.log")
    if not os.path.exists(log):
        return "no build log"
    text = open(log).read()
    m = re.search(r"Function properties for \S*DeformSurfelsKernel\S*\n\s*(.*?spill loads)\n.*?(Used \d+ registers)", text)
    return f"{m.group(2)}, {m.group(1).strip()}" if m else "not found"


def timed(torch, fn, before=None, calls=10, warmup=2):
    out = []
    for i in range(warmup + calls):
        if before:
            before()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            out.append(e0.elapsed_time(e1))
    return {"median_ms": round(float(np.median(out)), 4), "min_ms": round(min(out), 4), "max_ms": round(max(out), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["cfg3", "cfg2"])
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "surfel_deform_time.py needs a GPU"
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(0), "DeformSurfelsKernel": registers()}), flush=True)
    for name in args.configs:
        sc = S.make_scene(S.config_by_name(name))
        K = sc.cfg.num_keyframes
        ba = DirectBA.from_scene(sc)
        lib, h = ba._lib, ba._h
        original = ba.RememberKeyframePoses()
        E = S.se3_exp([0.2, -0.15, 0.16, 0.2, -0.2, 0.22])
        cur = np.array(sc.poses_init, np.float32, copy=True)
        for k in range(K // 2, K):
            cur[k] = S.se3_mul(E, cur[k]).astype(np.float32)
        surfels = ba.SurfelsDeviceView()
        saved = surfels.clone()
        ba.SetKeyframeStates(cur)
        moved, unobserved = ba.DeformSurfelsWithKeyframePoseChanges(original)
        orig = np.ascontiguousarray(original, np.float32)
        stream = torch.cuda.current_stream().cuda_stream

        def deform():
            assert lib.bba_deform_surfels(h, K, orig.ctypes.data, None, None, stream) == 0
        rows = {"deform_surfels": timed(torch, deform, lambda: surfels.copy_(saved), args.calls, args.warmup)}
        surfels.copy_(saved)
        ba.SetKeyframeStates(sc.poses_init)
        rows["update_surfel_activation"] = timed(torch, ba.UpdateSurfelActivation, None, args.calls, args.warmup)
        rows["optimize_geometry_iteration"] = timed(torch, ba.OptimizeGeometryIteration, lambda: surfels.copy_(saved), args.calls,
                                                    args.warmup)
        for call, r in rows.items():
            print(json.dumps({"config": name, "call": call, "keyframes": K, "surfels": int(sc.num_surfels), **r,
                              **({"moved": moved, "unobserved": unobserved} if call == "deform_surfels" else {})}), flush=True)


if __name__ == "__main__":
    main()
