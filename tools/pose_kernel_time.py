"""GPU timing of the batched pose kernel (bba_debug_pose_coeffs_batch) on a BASELINE config, with and without stats.

Every keyframe is evaluated at poses_init in one work list, in the instantiation the BA pose step picks for it (512/PRE on
cfg3): the kernel-level yardstick for changes to PoseAccumulateKernel.  One call also packs the work records, zeroes the
accumulators and reads the result back, so the per-call time is an upper bound of the kernel's own time; CUDA events around
many back-to-back calls.

    python tools/pose_kernel_time.py [cfg3 cfg2 ...] [--calls N]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["cfg3", "cfg2"])
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "pose_kernel_time.py needs a GPU"
    from badslam_b200 import _lib
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA

    dev = torch.cuda.get_device_properties(0)
    for name in args.configs:
        sc = S.make_scene(S.config_by_name(name))
        ba = DirectBA.from_scene(sc)
        ids = np.arange(sc.cfg.num_keyframes)
        poses = sc.poses_init[ids]
        for stats in (False, True):
            for _ in range(args.warmup):
                ba.PoseCoeffsBatch(ids, poses, _lib.POSE_VARIANT_AUTO, with_stats=stats)
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(args.calls):
                _, _, counts, _ = ba.PoseCoeffsBatch(ids, poses, _lib.POSE_VARIANT_AUTO, with_stats=stats)
            ev1.record()
            torch.cuda.synchronize()
            ms = ev0.elapsed_time(ev1) / args.calls
            pairs = int(counts[:, 2].sum())
            print(json.dumps({"config": name, "gpu": dev.name, "stats": stats, "keyframes": len(ids), "surfels": int(sc.num_surfels),
                              "ms_per_call": round(ms, 4), "assoc_pairs": pairs, "assoc_pairs_per_s": pairs / (ms * 1e-3)}), flush=True)


if __name__ == "__main__":
    main()
