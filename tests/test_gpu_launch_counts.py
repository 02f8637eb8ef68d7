"""Kernel launch counts against what the device ran.  Each call runs under torch.profiler with CUDA activity; the kernels of its
trace must equal the change of bba_kernel_launch_count and, for BA and tracking calls, the result's kernel_launches.  A CUB radix
sort counts as one launch: its kernels are folded into one per MortonKeysKernel (one per sort).  Memsets and copies are not
kernels on either side.  Nothing but library calls runs inside a profiled window: inputs are uploaded before it."""
import copy
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MOTION = [0.02, -0.01, 0.015, 0.01, -0.008, 0.012]
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    return S, DirectBA


class Traced:
    """Runs library calls under the profiler and compares the kernels of each trace with the library's counters."""

    def __init__(self, ba, trace_dir):
        self.ba, self.dir, self.calls = ba, trace_dir, 0

    def kernels(self, fn):
        """(fn(), kernels in the trace with one per radix sort, change of kernel_launch_count)"""
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        before = self.ba.kernel_launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        counted = self.ba.kernel_launch_count() - before
        path = self.dir / f"trace_{self.calls}.json"
        self.calls += 1
        prof.export_chrome_trace(str(path))
        with open(path) as f:
            names = [e["name"] for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
        sorts = sum("MortonKeysKernel" in n for n in names)
        cub = sum("cub::" in n or "DeviceRadixSort" in n for n in names)
        assert (cub > 0) == (sorts > 0), names
        return out, len(names) - cub + sorts, counted

    def check(self, what, fn, reported=None):
        """Asserts that the trace of fn() holds as many kernels as the library counted (and as reported(fn()) says, if given)."""
        out, traced, counted = self.kernels(fn)
        assert counted == traced, (what, counted, traced)
        if reported is not None:
            assert reported(out) == traced, (what, reported(out), traced)
        return out


def half_map(S, name):
    """The scene with the first half of its surfels, the true poses and room for the surfels that creation adds."""
    sc = copy.copy(S.make_scene(S.config_by_name(name)))
    sc.poses_init = sc.poses_true.copy()
    sc.num_surfels = sc.num_surfels // 2
    cells = sc.cfactor.size * sc.cfg.num_keyframes
    sc.surfels = np.pad(sc.surfels, ((0, 0), (0, (cells + 127) // 128 * 128)))
    return sc


def dev16(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).cuda()


def dev8(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def calibrated(ba, tmp_path, S, sc):
    """A tracer that has seen the two kernels of bba_preprocess_frame: a trace that misses the library's kernels fails here."""
    t = Traced(ba, tmp_path)
    raw, rgb = S.raw_frame(sc, 0)
    raw, rgb = dev16(raw), dev8(rgb)
    _, traced, counted = t.kernels(lambda: ba.PreprocessFrame(raw, rgb))
    assert traced == counted == 2, (traced, counted)
    return t


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_bundle_adjustment(mods, tmp_path, name):
    S, DirectBA = mods
    sc = half_map(S, name)
    ba = DirectBA.from_scene(sc)
    t = calibrated(ba, tmp_path, S, sc)
    launches = lambda r: r.kernel_launches
    for updates in (True, False, True):   # a keyframe's first BA block creates surfels, later ones merge and compact them
        t.check(("alternating", updates), lambda: ba.BundleAdjustment(None, True, True, updates, True, True, 1, 2), launches)
    ba = t.ba = DirectBA.from_scene(sc)
    t.check("pcg", lambda: ba.BundleAdjustment(None, True, True, True, True, True, 1, 2, use_pcg=True, pcg_gauge_keyframe=0),
            launches)
    for step in (0, 1):
        t.check(("pcg_debug", step), lambda: ba.PCGProbe(step, optimize_depth_intrinsics=True, optimize_color_intrinsics=True))


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_surfel_lifecycle(mods, tmp_path, name):
    S, DirectBA = mods
    sc = half_map(S, name)
    K = sc.cfg.num_keyframes
    t = calibrated(DirectBA.from_scene(sc), tmp_path, S, sc)
    for with_active in (True, False):
        # unfiltered creation from every keyframe leaves near-duplicates for the merges to mark
        ba = t.ba = DirectBA.from_scene(sc)
        for k in range(K):
            t.check(("create", k), lambda: ba.CreateSurfelsForKeyframe(None, False, k))
        merged = sum(t.check(("merge", k), lambda: ba.MergeSurfelsForKeyframe(k)) for k in range(K))
        assert merged > 0
        t.check(("compact", with_active), lambda: ba.CompactSurfels(merged, with_active))
    ba = t.ba = DirectBA.from_scene(sc)
    assert sum(t.check(("create filtered", k), lambda: ba.CreateSurfelsForKeyframe(None, True, k)) for k in range(K)) > 0
    t.check("update activation", lambda: ba.UpdateSurfelActivation())
    t.check("geometry iteration", lambda: ba.OptimizeGeometryIteration())
    t.check("intrinsics", lambda: ba.OptimizeIntrinsics(True, True))
    t.check("end tasks", lambda: ba.PerformBASchemeEndTasks())
    # an empty map: the support pass has no surfel to launch for
    empty = copy.copy(sc)
    empty.num_surfels = 0
    for filt in (False, True):
        ba = t.ba = DirectBA.from_scene(empty)
        assert t.check(("create on an empty map", filt), lambda: ba.CreateSurfelsForKeyframe(None, filt, 0)) > 0


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_frame_pose_tracking_and_preprocessing(mods, tmp_path, name):
    S, DirectBA = mods
    sc = S.make_scene(S.config_by_name(name))
    K = sc.cfg.num_keyframes
    ba = DirectBA.from_scene(sc, max_keyframes=K + 1)
    t = calibrated(ba, tmp_path, S, sc)
    k = K - 1
    depth, normals, color = dev16(sc.depth[k]), dev16(sc.normals[k]), dev8(sc.color[k])
    t.check("frame pose of a keyframe", lambda: ba.EstimateFramePose(None, sc.poses_init[k], k))
    t.check("frame pose of buffers", lambda: ba.EstimateFramePoseFromBuffers(None, sc.poses_init[k], depth, normals, color))
    d, n, _, c = S.render_frame(sc, S.se3_mul(sc.poses_true[0], S.se3_exp(MOTION)))
    d, n, c = dev16(d), dev16(n), dev8(c)
    b_depth, b_normals, b_color = dev16(sc.depth[0]), dev16(sc.normals[0]), dev8(sc.color[0])
    launches = lambda r: r[1].kernel_launches
    for kw in (dict(), dict(num_scales=4, use_pyramid_level_0=False, use_gradmag=True)):
        t.check(("track", kw), lambda: ba.TrackFramePairwise(None, 0, d, n, c, IDENT, **kw), launches)
        t.check(("track to frame", kw), lambda: ba.TrackFramePairwiseToFrame(None, b_depth, b_normals, b_color, d, n, c, IDENT, **kw),
                launches)
    raw, rgb = S.raw_frame(sc, 1)
    raw, rgb = dev16(raw), dev8(rgb)
    t.check("preprocess", lambda: ba.PreprocessFrame(raw, rgb))
    t.check("preprocess without colour", lambda: ba.PreprocessFrame(raw, None))
    t.check("raw preprocess", lambda: ba.PreprocessFrame(raw, rgb, median_filter_and_densify_iterations=1))
