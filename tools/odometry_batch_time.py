"""Times the image-pair odometry for many pairs in one call (bba_track_frames_pairwise) against a loop of single calls
(bba_track_frame_pairwise) on the same pairs: frames rendered at small offsets from keyframe poses, as tools/odometry_time.py
builds its pair, tracked against 1 to 4 distinct base keyframes.

Each arm is timed with a host clock around work that ends in a synchronise (both calls synchronise their stream), after one
warm-up call of each arm; the arms alternate, three rounds each.

    python tools/odometry_batch_time.py [--size 640x480] [--scales 5] [--counts 1,8,64,200] [--bases 1,2,4] [--rounds 3]
"""
import argparse
import multiprocessing
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:   # (a read-only query)
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def render(sc, global_T_frame):
    """(depth, normals, colour) of a rendered frame as the arrays the device tensors are made from (u16 viewed as i16)."""
    from badslam_b200 import scene as S
    d, n, _, c = S.render_frame(sc, global_T_frame)
    return tuple(np.ascontiguousarray(x).view(np.int16) if x.dtype == np.uint16 else np.ascontiguousarray(x) for x in (d, n, c))


def main():
    import torch
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="640x480")
    ap.add_argument("--scales", type=int, default=5)
    ap.add_argument("--counts", default="1,8,64,200")
    ap.add_argument("--bases", default="1,2,4")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    w, h = [int(v) for v in a.size.split("x")]
    counts = [int(v) for v in a.counts.split(",")]
    bases = [int(v) for v in a.bases.split(",")]
    K = max(bases)
    sc = S.make_scene(S.SceneConfig(width=w, height=h, num_keyframes=K, num_surfels=2000, cell=4, seed=31, name="odometry"))
    rng = np.random.default_rng(0)
    base_motion = np.array([0.02, -0.01, 0.015, 0.01, -0.008, 0.012])
    init2 = S.se3_exp([0.01, 0, 0, 0, 0, 0]).astype(np.float32)
    ident = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
    # entry i of a run with B base keyframes tracks frame (i % B, i // B): the (i // B)-th frame rendered near keyframe i % B
    need = [max((-(-max(counts) // B) for B in bases if k < B), default=0) for k in range(K)]
    jobs = [(k, m, base_motion * rng.uniform(0.5, 1.0) * rng.choice([-1, 1], 6)) for k in range(K) for m in range(need[k])]
    with multiprocessing.get_context("fork").Pool(min(16, os.cpu_count() or 1)) as pool:
        rendered = pool.starmap(render, [(sc, S.se3_mul(sc.poses_true[k], S.se3_exp(motion))) for k, m, motion in jobs])
    frames = {(k, m): tuple(torch.from_numpy(x).cuda() for x in f) for (k, m, _), f in zip(jobs, rendered)}

    def pairs(count, B):
        return [(i % B, (i % B, i // B)) for i in range(count)]

    ba = DirectBA.from_scene(sc)
    name, limit = card()
    print(f"{name}, power limit {limit}; {w}x{h}, {a.scales} pyramid levels, {a.rounds} rounds per arm, host clock, ms per call")
    print("| entries | base keyframes | loop of single calls (ms) | one batch call (ms) | speed-up |")
    print("|---|---|---|---|---|")
    for count in counts:
        for B in bases:
            P = pairs(count, B)
            tracked = sorted({j for _, j in P})
            local = {j: i for i, j in enumerate(tracked)}
            flist = [frames[j] for j in tracked]
            entries = [(k, 0, local[j], ident, init2) for k, j in P]

            def loop():
                for k, j in P:
                    ba.TrackFramePairwise(None, k, *frames[j], ident, init2, num_scales=a.scales)

            def batch():
                ba.TrackFramesPairwise(None, flist, entries, num_scales=a.scales)

            torch.cuda.synchronize()
            loop()
            batch()
            t_loop, t_batch = [], []
            for _ in range(a.rounds):
                for arm, out in ((batch, t_batch), (loop, t_loop)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    arm()
                    torch.cuda.synchronize()
                    out.append((time.perf_counter() - t0) * 1e3)
            ml, mb = float(np.median(t_loop)), float(np.median(t_batch))
            print(f"| {count} | {B} | {min(t_loop):.2f}-{max(t_loop):.2f} ({ml:.2f}) | {min(t_batch):.2f}-{max(t_batch):.2f} ({mb:.2f}) "
                  f"| {ml / mb:.2f}x |", flush=True)


if __name__ == "__main__":
    main()
