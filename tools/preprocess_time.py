"""Times the fused keyframe preprocessing (bba_preprocess_frame) against the reference's five kernels on one GPU, and the
raw-frame stage 0 (bba_preprocess_raw_frame): 640x480 with 1 and 4 median densify iterations, 1280x960 -> 640x480 at depth and
colour pyramid level 1.

    python tools/preprocess_time.py [--size 640x480] [--iters 200]

Product: cudaEvents around `iters` back-to-back calls on the current stream (inputs resident, no min/max read-back, so no sync
inside the loop), preceded by an L2 flush buffer write between calls when --flush is given.  Reference: wall time of
oracle/_ref's ref_preprocess_frame, which includes its allocations and host copies -- an upper bound, reported as such.
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="640x480")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--flush", action="store_true")
    a = ap.parse_args()
    w, h = [int(v) for v in a.size.split("x")]
    sc = S.blank_scene(w, h)
    raw, rgb = S.random_raw_frame(w, h, seed=1, hole_fraction=0.01)
    ba = DirectBA.from_scene(sc)
    d_raw = torch.from_numpy(raw.view(np.int16)).cuda()
    d_rgb = torch.from_numpy(rgb).cuda()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda") if a.flush else None
    for _ in range(5):
        ba.PreprocessFrame(d_raw, d_rgb, want_min_max=False)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    if flush is None:
        e0.record()
        for _ in range(a.iters):
            ba.PreprocessFrame(d_raw, d_rgb, want_min_max=False)
        e1.record()
        torch.cuda.synchronize()
        total = e0.elapsed_time(e1)
    else:
        for _ in range(a.iters):
            flush.fill_(1)
            e0.record()
            ba.PreprocessFrame(d_raw, d_rgb, want_min_max=False)
            e1.record()
            torch.cuda.synchronize()
            total += e0.elapsed_time(e1)
    us = 1e3 * total / a.iters
    bytes_alg = 15.0 * w * h
    print(f"fused preprocessing {w}x{h}: {us:.1f} us per frame (2 launches, output tensors allocated per call), "
          f"{bytes_alg / us * 1e-3:.1f} GB/s algorithmic")
    # raw-frame stage 0, same event timing without flush (the same blank 640x480 camera; the 2x frame is the random surface at
    # twice the resolution)
    sc6 = S.blank_scene(640, 480)
    ba6 = DirectBA.from_scene(sc6)
    raw6, rgb6 = S.random_raw_frame(640, 480, seed=1, hole_fraction=0.3)
    raw12, rgb12 = S.random_raw_frame(1280, 960, seed=2, hole_fraction=0.3)
    cases = [("640x480, no stage 0 (bba_preprocess_frame)", raw6, rgb6, {}),
             ("640x480, median_filter_and_densify_iterations 1", raw6, rgb6, dict(median_filter_and_densify_iterations=1)),
             ("640x480, median_filter_and_densify_iterations 4", raw6, rgb6, dict(median_filter_and_densify_iterations=4)),
             ("1280x960 -> 640x480, pyramid_level_for_depth 1 + pyramid_level_for_color 1", raw12, rgb12,
              dict(pyramid_level_for_depth=1, pyramid_level_for_color=1))]
    for name, r, c, opts in cases:
        d_r, d_c = torch.from_numpy(r.view(np.int16)).cuda(), torch.from_numpy(c).cuda()
        for _ in range(5):
            ba6.PreprocessFrame(d_r, d_c, want_min_max=False, **opts)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.iters):
            ba6.PreprocessFrame(d_r, d_c, want_min_max=False, **opts)
        e1.record()
        torch.cuda.synchronize()
        print(f"raw frame {name}: {e0.elapsed_time(e1) / a.iters:.4f} ms per frame")
    try:
        from oracle import ref_cuda as R
        if R.available():
            ref = R.RefDirectBA(sc)
            ref.preprocess_frame(raw, rgb)
            t = time.perf_counter()
            n = max(a.iters // 10, 5)
            for _ in range(n):
                ref.preprocess_frame(raw, rgb)
            print(f"reference kernels (5 launches + allocations + host copies, wall): {1e6 * (time.perf_counter() - t) / n:.1f} us per frame")
    except Exception as e:   # noqa: BLE001
        print("reference arm unavailable:", e)


if __name__ == "__main__":
    main()
