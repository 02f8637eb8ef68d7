"""GPU timing of the alternating BA iteration's geometry step in its two forms (bba_debug_set_geometry_pass): the two group-major
launches (ActivationNormalsKernel + PositionDescriptorKernel, each after its own stream gather) and the one tile-major launch
(GeometryPassKernel after one gather), the latter at every tile size.

The step is bench.py's: surfels and keyframe states restored, then one iteration of BundleAdjustment (poses and geometry, no surfel
updates).  Per step the result's two geometry event times are summed (split: activation + normals stage and position + descriptor
stage; one launch: the gather and the kernel), the forms alternating step by step so that drift hits all of them alike.  A second,
separate run under torch.profiler gives the device time of every geometry kernel launch.  Achieved bandwidth of the one launch:
the bytes it must move per surfel -- stream rows x y z, normal, radius^2, d1, d2, flags (32 B), the order (4 B) and the result
stores (active flag 1 B, normal, x y z, d1, d2: 21 B) -- over its kernel time; the keyframe-image gathers are not counted.

    python tools/geometry_pass_time.py [cfg3 cfg3_rank8 cfg2 ...] [--steps N] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SPLIT, ONE = 1, 2
BYTES_PER_SURFEL = 32 + 4 + 21
FORMS = [("split", SPLIT, 0), ("one", ONE, 0), ("one_t5", ONE, 5), ("one_t6", ONE, 6), ("one_t7", ONE, 7), ("one_t8", ONE, 8)]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable: {type(e).__name__}"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["cfg3", "cfg3_rank8", "cfg2"])
    ap.add_argument("--steps", type=int, default=6, help="timed steps per form")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="directory for the profiler traces")
    args = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    assert torch.cuda.is_available(), "geometry_pass_time.py needs a GPU"
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA

    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name in args.configs:
        sc = S.make_scene(S.config_by_name(name))
        ba = DirectBA.from_scene(sc)
        surf = ba.surfels()
        backup = surf[:8].clone()
        K = sc.cfg.num_keyframes
        act0 = np.zeros(K, np.int32)
        ba.SetLastBAIterationCount(ba.ba_iteration_count())

        def step(pass_, shift):
            surf[:8].copy_(backup, non_blocking=True)
            ba.SetKeyframeStates(sc.poses_init, act0)
            ba.DebugSetGeometryPass(pass_, shift)
            r = ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, increase_ba_iteration_count=False)
            return r.ms_surfel_activation + r.ms_geometry_optimization, r.ms_surfel_activation, r.ms_geometry_optimization

        for _ in range(args.warmup):
            for _, p, t in FORMS:
                step(p, t)
        times = {f: [] for f, _, _ in FORMS}
        parts = {f: np.zeros(2) for f, _, _ in FORMS}
        for _ in range(args.steps):
            for f, p, t in FORMS:
                total, a, b = step(p, t)
                times[f].append(total)
                parts[f] += [a, b]
        for f, _, _ in FORMS:
            v = np.array(times[f])
            print(json.dumps({"config": name, "form": f, "surfels": int(sc.num_surfels), "keyframes": K,
                              "geometry_ms_median": round(float(np.median(v)), 4), "min": round(float(v.min()), 4),
                              "max": round(float(v.max()), 4), "first_stage_ms": round(float(parts[f][0] / args.steps), 4),
                              "second_stage_ms": round(float(parts[f][1] / args.steps), 4)}), flush=True)

        # per-launch device times (a separate run: tracing slows the host)
        for f, p, t in FORMS:
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    step(p, t)
                torch.cuda.synchronize()
            out_dir = args.out or tempfile.mkdtemp()
            os.makedirs(out_dir, exist_ok=True)
            path = os.path.join(out_dir, f"geometry_{name}_{f}.pt.trace.json")
            prof.export_chrome_trace(path)
            with open(path) as fh:
                events = [e for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel"]
            if not args.out:
                os.remove(path)
            per = {}
            for e in events:
                if any(k in e["name"] for k in ("Geometry", "ActivationNormals", "PositionDescriptor")):
                    key = e["name"].split("(")[0].replace("void ", "")
                    per.setdefault(key, []).append(e["dur"] / 1e3)
            rec = {"config": name, "form": f, "kernel_ms": {k: round(float(np.median(v)), 4) for k, v in per.items()}}
            one = [np.median(v) for k, v in per.items() if "GeometryPassKernel" in k]
            if one:
                rec["pass_kernel_GBps"] = round(sc.num_surfels * BYTES_PER_SURFEL / (one[0] * 1e-3) / 1e9, 1)
            print(json.dumps(rec), flush=True)
        del ba, surf, backup
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
