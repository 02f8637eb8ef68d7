"""Where the geometry step's time goes on a BASELINE config: per-kernel device time and the (sub-step, keyframe) visibility.

1. Kernel times.  After one `bba_update_surfel_activation`, `bba_optimize_geometry_iteration` (normals launch + position / descriptor launch, each with its
   geometry-stream gather and memsets) under torch.profiler with CUDA activity, after warm-up calls that also put the surfels
   into spatial order; device time summed per kernel name over --calls calls.
2. Visibility.  The surfels at their scene positions are put into the library's spatial order (MortonKeysKernel's 10-bit
   quantisation over the finite bounds, in fp32, and a stable sort of the 30-bit keys, as the CUB radix sort is) and cut into
   the kernels' 32-surfel sub-steps.  Each sub-step's box is tested against every keyframe's view at poses_init with the plane
   tests of PlanesOutside (kernels.cu), every surfel counted live.  Prints the fraction of (sub-step, keyframe) pairs whose box
   may reach the view: the keyframe iterations left after culling, out of all.  The host's fp32 division can differ from the
   kernel's -use_fast_math one in the last bit, which moves a surfel on a quantisation boundary by one cell.

    python tools/geometry_breakdown.py [cfg3 cfg3_rank8 ...] [--calls N]
"""
import argparse
import collections
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def spread3(q):
    q = q & 0x3FF
    q = (q | (q << 16)) & 0x030000FF
    q = (q | (q << 8)) & 0x0300F00F
    q = (q | (q << 4)) & 0x030C30C3
    q = (q | (q << 2)) & 0x09249249
    return q


def visible_fraction(sc, torch, device, sub=32):
    P = torch.as_tensor(sc.surfels[:3], dtype=torch.float32, device=device)   # [3, n]
    key = torch.zeros(P.shape[1], dtype=torch.int64, device=device)
    for a in range(3):
        c = P[a]
        fin = torch.isfinite(c)
        q = torch.zeros_like(key)
        if bool(fin.any()):
            lo, hi = c[fin].min(), c[fin].max()
            scale = (torch.tensor(1024.0, device=device) / (hi - lo)) if bool(hi > lo) else torch.tensor(0.0, device=device)
            t = (c - lo) * scale
            t = torch.nan_to_num(t, nan=0.0)
            q = torch.clamp(t, 0.0, 1023.0).to(torch.int64)
        key |= spread3(q) << a
    order = torch.sort(key, stable=True).indices
    P = P[:, order]
    n = P.shape[1]
    nb = (n + sub - 1) // sub
    pad = nb * sub - n
    if pad:
        P = torch.cat([P, torch.full((3, pad), float("nan"), device=device)], 1)
    B = P.view(3, nb, sub)
    fin = torch.isfinite(B)
    lo = torch.where(fin, B, torch.full_like(B, float("inf"))).amin(2)   # [3, nb]
    hi = torch.where(fin, B, torch.full_like(B, float("-inf"))).amax(2)
    none = ~fin.any(2)
    lo[none] = float("nan")
    hi[none] = float("nan")
    corners = torch.stack([torch.stack([hi[ax] if (c >> ax) & 1 else lo[ax] for ax in range(3)]) for c in range(8)])   # [8, 3, nb]
    fx, fy, cx, cy = (float(v) for v in sc.depth_K)
    W, H = sc.cfg.width, sc.cfg.height
    lx, rx, ly, ry = cx + 1.0, cx - W - 1.0, cy + 1.0, cy - H - 1.0
    e = 1e-5
    from badslam_b200 import scene as S
    import numpy as np
    visible = 0
    for pose in sc.poses_init:
        T = torch.as_tensor(np.linalg.inv(S.se3_matrix(pose))[:3], dtype=torch.float32, device=device)
        v = [T[r, 0] * corners[:, 0] + T[r, 1] * corners[:, 1] + T[r, 2] * corners[:, 2] + T[r, 3] for r in range(3)]
        A = [(T[r, 0] * corners[:, 0]).abs() + (T[r, 1] * corners[:, 1]).abs() + (T[r, 2] * corners[:, 2]).abs() + T[r, 3].abs()
             for r in range(3)]
        outside = ((v[2] < -e * A[2]).all(0)
                   | (fx * v[0] + lx * v[2] < -e * (fx * A[0] + abs(lx) * A[2])).all(0)
                   | (fx * v[0] + rx * v[2] > e * (fx * A[0] + abs(rx) * A[2])).all(0)
                   | (fy * v[1] + ly * v[2] < -e * (fy * A[1] + abs(ly) * A[2])).all(0)
                   | (fy * v[1] + ry * v[2] > e * (fy * A[1] + abs(ry) * A[2])).all(0))
        visible += int((~outside).sum())
    return nb, len(sc.poses_init), visible / (nb * len(sc.poses_init))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["cfg3", "cfg3_rank8"])
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "geometry_breakdown.py needs a GPU"
    from torch.profiler import ProfilerActivity, profile
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA

    dev = torch.cuda.get_device_properties(0)
    for name in args.configs:
        sc = S.make_scene(S.config_by_name(name))
        nb, nk, frac = visible_fraction(sc, torch, "cuda")
        print(json.dumps({"config": name, "gpu": dev.name, "sub_steps": nb, "keyframes": nk, "visible_fraction": round(frac, 4)}),
              flush=True)
        ba = DirectBA.from_scene(sc)
        ba.UpdateSurfelActivation()   # the kernels update active surfels only
        for _ in range(args.warmup):
            ba.OptimizeGeometryIteration()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.calls):
                ba.OptimizeGeometryIteration()
            torch.cuda.synchronize()
        per = collections.defaultdict(lambda: [0.0, 0])
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                k = ev.name.replace("(anonymous namespace)::", "").split("(")[0][:80]
                per[k][0] += ev.device_time_total / 1000.0
                per[k][1] += 1
        for k, (ms, cnt) in sorted(per.items(), key=lambda kv: -kv[1][0]):
            print(json.dumps({"config": name, "kernel": k, "ms_per_call": round(ms / args.calls, 4), "launches_per_call": cnt / args.calls}),
                  flush=True)
        del ba


if __name__ == "__main__":
    main()
