"""GPU: the deterministic mode (bba_set_deterministic, DESIGN.md 3.10).  With the mode on, the pose kernel's and the intrinsics
step's scheduling-dependent sums go through the exact accumulator and the odometry kernel sums its per-CTA totals in CTA order, so
that the same inputs give the same bits in every run -- also with the front end running beside a BA call on another stream.  The
results stay within the default mode's tolerances of it.  Every configuration runs a fixed two or three times; nothing loops.
"""
import dataclasses
import math
import threading

import numpy as np
import pytest

from gpu_checks import rel
from test_exact_sum import arrays, bits, same
from test_gpu_concurrent_front_end import (IDENT, FrontEndInputs, assert_same, join, preprocess, run_thread, streams, track_by_id,
                                           track_to_frame)

pytestmark = [pytest.mark.gpu]

POSE_TOL = 1e-5   # m / rad, the BA parity tolerance


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import _lib
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA, exact_sum
    return S, DirectBA, _lib, exact_sum


def test_device_exact_sum_equals_host_and_fsum(mods):
    import torch
    S, DirectBA, _, exact_sum = mods
    ba = DirectBA.from_scene(S.make_scene(S.config_by_name("tiny")))
    rng = np.random.default_rng(3)
    for name, a in arrays().items():
        want = math.fsum(a.astype(np.float64))
        for perm in (a, rng.permutation(a)):
            got = ba.DebugExactSum(torch.from_numpy(np.ascontiguousarray(perm)).cuda())
            host = exact_sum(perm)
            assert bits(got) == bits(host) and same(got, want), (name, got, host, want)
    for a in ([1.0, float("inf")], [float("inf"), float("-inf")], [float("nan"), 2.0]):
        got, host = ba.DebugExactSum(torch.tensor(a, dtype=torch.float32).cuda()), exact_sum(a)
        assert bits(got) == bits(host), (a, got, host)


def test_pose_coeffs_batch_every_variant(mods):
    S, DirectBA, L, _ = mods
    sc = S.make_scene(S.config_by_name("many"))
    ba = DirectBA.from_scene(sc)
    ids = np.arange(sc.cfg.num_keyframes)
    poses = sc.poses_init
    variants = [L.POSE_VARIANT_256_PRE, L.POSE_VARIANT_512_PRE, L.POSE_VARIANT_256, L.POSE_VARIANT_512, L.POSE_VARIANT_1024]
    for with_stats in (True, False):
        for v in variants:
            H0, b0, c0, _ = ba.PoseCoeffsBatch(ids, poses, v, with_stats)
            ba.SetDeterministic(True)
            runs = [ba.PoseCoeffsBatch(ids, poses, v, with_stats) for _ in range(2)]
            ba.SetDeterministic(False)
            (H1, b1, c1, k1), (H2, b2, c2, k2) = runs
            tag = (v, with_stats)
            assert H1.tobytes() == H2.tobytes() and b1.tobytes() == b2.tobytes() and k1.tobytes() == k2.tobytes(), tag
            assert np.array_equal(c1, c2) and np.array_equal(c1, c0), tag
            assert c0[:, 2].sum() > 0, tag
            for k in ids:
                if c0[k, 2]:
                    # (H: 1.5e-8 measured on an H100 in the instantiations without the precomputed frames, bit-equal with them;
                    #  tests/test_gpu_deterministic_values.py holds every slot to its own scale)
                    assert rel(H1[k], H0[k]) < 1e-7 and rel(b1[k], b0[k]) < 5e-7, (tag, k, rel(H1[k], H0[k]), rel(b1[k], b0[k]))


BA_KW = dict(optimize_depth_intrinsics=True, optimize_color_intrinsics=True, do_surfel_updates=True, optimize_poses=True,
             optimize_geometry=True, min_iterations=3, max_iterations=3)


def run_ba(S, DirectBA, sc, deterministic, front_end=False, kw=BA_KW):
    """Alternating BA on a fresh handle built from the scene (the same starting state every time); with front_end, preprocessing
    and odometry run on another thread and stream for the whole call.  Returns the final state."""
    import torch
    lo, hi = streams()
    ba = DirectBA.from_scene(sc)
    ba.SetDeterministic(deterministic)
    if front_end:
        inp = FrontEndInputs(S, sc, ba)
        started, stop = threading.Event(), threading.Event()

        def fe():
            n = 0
            started.set()
            while not stop.is_set() or n == 0:
                preprocess(ba, inp, hi)
                track_by_id(ba, inp, hi)
                n += 1
            return n
        t, box = run_thread(fe)
        assert started.wait(300)
    try:
        with torch.cuda.stream(lo):
            res = ba.BundleAdjustment(lo, **kw)
        lo.synchronize()
    finally:
        if front_end:
            stop.set()
    if front_end:
        assert join(t, box) >= 1
    poses, act = ba.GetKeyframeStates()
    d, c, a = ba._intrinsics()
    n = res.surfels_size
    result = {k: v for k, v in dataclasses.asdict(res).items() if not k.startswith("ms_")}
    return dict(poses=poses, depth_K=np.asarray(d, np.float32), color_K=np.asarray(c, np.float32), a=np.float32(a),
                cfactor=ba.cfactor_buffer(lo), surfels=ba.GetSurfelsHost()[:, :n], active=ba.GetActiveHost()[:n], size=n,
                result=result)


def test_alternating_ba_is_reproducible(mods):
    S, DirectBA, _, _ = mods
    sc = S.make_scene(S.config_by_name("small"))
    first = run_ba(S, DirectBA, sc, True)
    assert first["result"]["iterations_done"] == 3 and first["result"]["surfels_merged"] + first["result"]["surfels_deleted"] > 0
    assert not np.array_equal(first["depth_K"], np.asarray(sc.depth_K, np.float32)), "the intrinsics step did not move"
    assert_same(run_ba(S, DirectBA, sc, True), first, "second run")
    assert_same(run_ba(S, DirectBA, sc, True, front_end=True), first, "run with the front end beside it")
    # against the default mode.  With the intrinsics steps the default mode's fp32 per-cell atomics round after every one of tens of
    # thousands of pairs per cell while the exact sums round once; the cfactors carry that difference into the poses (measured on
    # an H100: 2.4e-5 m / 1.4e-5 rad after three iterations), so the poses are held to the BA tolerance without the intrinsics
    # steps and to five times it with them.
    default = run_ba(S, DirectBA, sc, False)
    for k in ("iterations_done", "pose_iterations_total", "surfels_size", "surfels_created", "surfels_merged", "surfels_deleted"):
        assert default["result"][k] == first["result"][k], (k, default["result"][k], first["result"][k])
    assert np.allclose(first["depth_K"], default["depth_K"], rtol=1e-4) and np.allclose(first["color_K"], default["color_K"], rtol=1e-4)
    for p, q in zip(first["poses"], default["poses"]):
        dt, dr = S.pose_error(p, q)
        assert dt < 5 * POSE_TOL and dr < 5 * POSE_TOL, (dt, dr)
    no_intr = dict(BA_KW, optimize_depth_intrinsics=False, optimize_color_intrinsics=False)
    det, default = (run_ba(S, DirectBA, sc, d, kw=no_intr) for d in (True, False))
    for k in ("iterations_done", "pose_iterations_total", "surfels_size"):
        assert default["result"][k] == det["result"][k], (k, default["result"][k], det["result"][k])
    for p, q in zip(det["poses"], default["poses"]):
        dt, dr = S.pose_error(p, q)
        assert dt < POSE_TOL and dr < POSE_TOL, ("without intrinsics", dt, dr)


def test_frame_tracking_is_reproducible(mods):
    import torch
    S, DirectBA, _, _ = mods
    sc = S.make_scene(S.config_by_name("small"))
    ba = DirectBA.from_scene(sc, max_keyframes=sc.cfg.num_keyframes + 1)   # (the frame pose estimate needs a free slot)
    inp = FrontEndInputs(S, sc, ba)
    st = torch.cuda.current_stream()
    init = S.se3_mul(sc.poses_init[0], S.se3_exp([0.003, -0.002, 0.001, 0.002, 0.0, -0.001]))

    def calls():
        est = ba.EstimateFramePoseFromBuffers(None, init, *inp.frame)
        out = dict(estimate=dict(pose=est[0], iterations=est[1], converged=est[2]), track=track_by_id(ba, inp, st),
                   to_frame=track_to_frame(ba, inp, st))
        out["coeffs"] = list(ba.OdometryCoeffs(1, out["to_frame"]["pose"], IDENT))
        return out
    default = calls()
    ba.SetDeterministic(True)
    first, second = calls(), calls()
    assert_same(second, first, "deterministic")
    assert first["estimate"]["iterations"] == default["estimate"]["iterations"]
    for k in ("track", "to_frame"):
        assert first[k]["iterations"] == default[k]["iterations"], k
        assert first[k]["residual_count"] == default[k]["residual_count"], k
    for k, p in (("estimate", first["estimate"]["pose"]), ("track", first["track"]["pose"]), ("to_frame", first["to_frame"]["pose"])):
        q = default[k]["pose"]
        dt, dr = S.pose_error(p, q)
        assert dt < POSE_TOL and dr < POSE_TOL, (k, dt, dr)


def test_setter_semantics(mods):
    import torch
    S, DirectBA, L, _ = mods
    from badslam_b200._lib import BadBAError
    sc = S.make_scene(S.config_by_name("tiny"))
    ba = DirectBA.from_scene(sc)
    assert not ba.deterministic()
    ba.SetDeterministic(True)
    assert ba.deterministic()
    # the PCG solver is refused, and the handle is left as it was
    before = (ba.GetKeyframeStates()[0].tobytes(), ba.GetSurfelsHost().tobytes(), ba.surfels_size())
    with pytest.raises(BadBAError) as e:
        ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, use_pcg=True, pcg_gauge_keyframe=0)
    assert e.value.status == L.ERR_UNSUPPORTED
    with pytest.raises(BadBAError) as e:
        ba.PCGDebug()
    assert e.value.status == L.ERR_UNSUPPORTED
    assert (ba.GetKeyframeStates()[0].tobytes(), ba.GetSurfelsHost().tobytes(), ba.surfels_size()) == before
    assert ba.deterministic()
    # a front-end call made after the setter runs in the mode it set: on again after off gives the same bits as before
    inp = FrontEndInputs(S, sc, ba)
    st = torch.cuda.current_stream()
    on = track_by_id(ba, inp, st)
    ba.SetDeterministic(False)
    assert not ba.deterministic()
    track_by_id(ba, inp, st)
    ba.SetDeterministic(True)
    assert_same(track_by_id(ba, inp, st), on, "on again")
    ba.SetDeterministic(False)
    assert ba.BundleAdjustment(None, False, False, False, True, True, 1, 1, use_pcg=True, pcg_gauge_keyframe=0).iterations_done == 1
