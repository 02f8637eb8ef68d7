"""GPU timing of the bundle-adjustment step with local groups (bba_local_group_create): the ranks of a job as threads of one
process, exchanging through the library's own all-reduce / all-gather.

    python tools/local_group_time.py [--configs cfg2,cfg3] [--steps 10] [--warmup 3]

For each config: one rank; two ranks in one process on one GPU; two ranks on two GPUs (when there are two).  A step is one
outer BA iteration as bench.py times it (BundleAdjustment(1 iteration), host wall clock; the call synchronises).  With two or
more GPUs the same step of the multi-process NCCL path is taken from `bench.py --gpus 2` for comparison.  Then the exchange
of a PCG vector (the unknown count of the config's PCG system, U = 6 (K - 1) + 3 n + 5) through bba_debug_collective: CUDA
event time on rank 0's stream around the whole exchange (event waits, the rank-order sum kernel, the copy back), and the
bytes that rank moves (world U reads + U writes by the kernel, U reads + U writes by the copy).  Two ranks on one GPU are a
correctness configuration: they share the SMs, so they are not expected to be faster than one rank."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from badslam_b200 import _lib  # noqa: E402
from badslam_b200.direct_ba import DirectBA, LocalGroup  # noqa: E402
from badslam_b200.scene import config_by_name, make_scene  # noqa: E402


def _step(ba):
    return ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, increase_ba_iteration_count=False)


def _timed(ba, steps, warmup):
    for _ in range(warmup):
        _step(ba)
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        _step(ba)
        times.append(1e3 * (time.perf_counter() - t0))
    return times


def _summary(times):
    return {"median_ms": float(np.median(times)), "min_ms": float(np.min(times)), "max_ms": float(np.max(times))}


def _exchange(group, count, reps=20):
    """Event time of one all-reduce of `count` floats on rank 0 (median over reps), and the bytes rank 0 moves."""
    world = len(group.handles)
    bufs = [torch.ones(count, dtype=torch.float32, device=ba.device) for ba in group.handles]
    torch.cuda.synchronize()

    def body(rank, ba):
        out = []
        for i in range(reps + 2):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ba.DebugCollective(_lib.COLLECTIVE_ALLREDUCE_SUM, bufs[rank], count)
            e1.record()
            e1.synchronize()
            if i >= 2:
                out.append(e0.elapsed_time(e1))
        return out
    ms = float(np.median(group.run(body)[0]))
    nbytes = 4 * count * (world + 1) + 4 * count * 2
    return {"count": count, "world": world, "median_ms": ms, "bytes_rank0": nbytes, "GB_per_s": nbytes / (ms * 1e-3) / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="cfg2,cfg3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("local_group_time.py needs a GPU")
    gpus = torch.cuda.device_count()
    props = torch.cuda.get_device_properties(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": props.name, "gpus": gpus, "nvidia_smi": power}), flush=True)
    for name in args.configs.split(","):
        sc = make_scene(config_by_name(name))
        n, K = sc.num_surfels, sc.cfg.num_keyframes
        ba = DirectBA.from_scene(sc, host_owned=True)
        one = _timed(ba, args.steps, args.warmup)
        ba.close()
        del ba
        print(json.dumps({"config": name, "setup": "1 rank", **_summary(one)}), flush=True)
        setups = [("2 ranks, 1 GPU", ["cuda:0", "cuda:0"])]
        if gpus >= 2:
            setups.append(("2 ranks, 2 GPUs", ["cuda:0", "cuda:1"]))
        for label, devices in setups:
            handles = DirectBA.create_local_ranks(sc, len(devices), devices, host_owned=True)
            with LocalGroup(handles) as group:
                times = group.run(lambda rank, b: _timed(b, args.steps, args.warmup))
                print(json.dumps({"config": name, "setup": label, **_summary(times[0])}), flush=True)
                U = 6 * (K - 1) + 3 * n + 5
                print(json.dumps({"config": name, "setup": label, "exchange": "PCG vector all-reduce", **_exchange(group, U)}),
                      flush=True)
            for b in handles:
                b.close()
            torch.cuda.empty_cache()
        if gpus >= 2:
            run = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "2", "--steps", str(args.steps),
                                  "--warmup", str(args.warmup), "--workload", name], capture_output=True, text=True, cwd=ROOT)
            line = run.stdout.strip().splitlines()[-1] if run.stdout.strip() else run.stderr[-300:]
            print(json.dumps({"config": name, "setup": "bench.py --gpus 2 (NCCL, one process per GPU)", "output": line}), flush=True)


if __name__ == "__main__":
    main()
