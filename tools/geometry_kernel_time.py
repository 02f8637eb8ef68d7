"""GPU timing of the geometry step (bba_update_surfel_activation, bba_optimize_geometry_iteration) on a BASELINE config.

Every keyframe active, the surfels of the config at poses_init: the kernel-level yardstick for changes to ActivationNormalsKernel
and PositionDescriptorKernel.  The standalone entry points put the surfels into spatial order when it is not current (the first
call) and gather each launch's geometry stream, so the per-call time includes the gathers but not the sort.  CUDA events around
many back-to-back calls; the geometry iteration is the normals launch followed by the position / descriptor launch.

    python tools/geometry_kernel_time.py [cfg3 cfg2 ...] [--calls N] [--residuals both|depth|desc]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("configs", nargs="*", default=["cfg3", "cfg2"])
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--residuals", default="both", choices=["both", "depth", "desc"])
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "geometry_kernel_time.py needs a GPU"
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA

    dev = torch.cuda.get_device_properties(0)
    for name in args.configs:
        sc = S.make_scene(S.config_by_name(name))
        ba = DirectBA.from_scene(sc, use_depth_residuals=args.residuals != "desc", use_descriptor_residuals=args.residuals != "depth")
        for label, call in (("activation", ba.UpdateSurfelActivation), ("geometry_iteration", ba.OptimizeGeometryIteration)):
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(args.calls):
                call()
            ev1.record()
            torch.cuda.synchronize()
            ms = ev0.elapsed_time(ev1) / args.calls
            print(json.dumps({"config": name, "gpu": dev.name, "call": label, "residuals": args.residuals, "keyframes": int(sc.cfg.num_keyframes),
                              "surfels": int(sc.num_surfels), "ms_per_call": round(ms, 4)}), flush=True)


if __name__ == "__main__":
    main()
