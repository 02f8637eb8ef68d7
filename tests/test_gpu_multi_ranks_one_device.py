"""Two and three ranks on one H100 (every process on device 0, gloo): the sharded passes of the multi-GPU path against one rank.

A multi-rank job shards the geometry, intrinsics, PCG-product and end-task passes by 256-surfel granules dealt round-robin, and
deals the pose step's keyframes out to the ranks; sum all-reduces and all-gathers through bba_set_collective make the replicas
equal again.  Every rank here registers a recording variant of tests/test_gpu_multi_one_device.py's host-staged collective: for
each call it keeps the op, the count, this rank's contribution (copied before the collective) and the result, so that the
tests see every rank's partial sums without a hook in the library.  Every test asserts that all ranks received the same
collective results, and compares against the one-rank run of the same call with a bound derived from how the number is summed:

* intrinsics normal equations (bba_debug_intrinsics_coeffs), depth / colour / both, then two OptimizeIntrinsics steps;
* the first PcgInit / PcgStep1 products of a PCG bundle adjustment, and its end result, in both exchange modes;
* the alternating BA's pose step: which rank packs each keyframe's 17-float slot (round-robin on the first step, then
  bba_balance_keyframes of the costs the previous slots give), counts, cost and poses;
* do_surfel_updates with moving poses on tests/test_gpu_multi.py's half map (a ragged granule count: LocalCountBelow);
* a 300-surfel map at world 3 (two granules: rank 2 owns no surfel), and the geometry step of
  tests/test_gpu_multi_geometry_order.py at world 3.

The differences measured against one rank are printed (pytest -s)."""
import copy
import hashlib
import os
import pickle

import numpy as np
import pytest

import test_gpu_multi as M
import test_gpu_multi_geometry_order as G
from gpu_checks import POSE_R, POSE_T
from test_gpu_multi_one_device import _set_host_staged_collective

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24
GAUGE = 1
DIAG5 = [0, 5, 9, 12, 14]       # diagonal of the 5x5 upper triangle among the 34 intrinsics sums
INTR_MODES = ((True, False), (False, True), (True, True))
PCG_RUNS = (("small", False, "gather"), ("small", False, "peer"), ("distorted", True, "gather"), ("many", False, "gather"))


def _many():
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name("many"))


def _map300():
    """`small` cut down to 300 surfels: two granules, the second with 44 surfels, so that rank 2 of three owns none."""
    sc = copy.copy(M._small())
    sc.num_surfels = 300
    return sc


def _small_kf1_alone():
    """`small` with every keyframe but 1 moved 100 m away: no frustum meets keyframe 1's, so that a window of keyframe 1 alone
    puts one keyframe into the pose step's work list (on `small` every keyframe is covisible with every other)."""
    sc = copy.copy(M._small())
    sc.poses_init = sc.poses_init.copy()
    sc.poses_init[np.arange(sc.cfg.num_keyframes) != 1, 4] += 100.0
    return sc


SCENES = {"small": M._small, "distorted": M._distorted_small, "many": _many, "half": M._half_small, "map300": _map300,
          "kf1_alone": _small_kf1_alone}
# (residual options per scene: the 300-surfel map also runs with depth residuals only)
OPTIONS = {"map300_depth": ("map300", {"use_descriptor_residuals": False})}


# ---- recording collective ------------------------------------------------------------------------------------------------

def _device_to_host(ba, ptr, nbytes, stream):
    """A host copy of nbytes at device address ptr, ordered behind the work queued on the library's stream."""
    import torch

    class _Raw:
        pass
    raw = _Raw()
    raw.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2, "strides": None}
    st = torch.cuda.ExternalStream(stream, device=ba.device) if stream else torch.cuda.default_stream(ba.device)
    with torch.cuda.stream(st):
        return torch.as_tensor(raw, device=ba.device).cpu().numpy().copy()


def _set_recording_collective(ba, log, snapshot=None):
    """The host-staged collective, recording every call into `log`: all-reduces as float arrays (this rank's contribution and
    the result), all-gathers as digests of this rank's slice and of the gathered buffer.  snapshot(stream) is called once,
    before the first all-reduce of more than two floats, and its value is logged as {"op": "snapshot", "snapshot": value}."""
    import torch.distributed as dist
    from badslam_b200 import _lib
    _set_host_staged_collective(ba)
    inner = ba._collective_cb
    rank, world = dist.get_rank(), dist.get_world_size()
    state = {"snapped": snapshot is None}

    def digest(a):
        return hashlib.sha256(a.tobytes()).hexdigest()

    def cb(user, op, ptr, count, stream):
        if op == _lib.COLLECTIVE_ALLGATHER:
            mine = _device_to_host(ba, ptr + rank * count, count, stream)
            inner(user, op, ptr, count, stream)
            log.append({"op": "allgather", "count": count, "mine": digest(mine),
                        "result": digest(_device_to_host(ba, ptr, count * world, stream))})
            return
        if not state["snapped"] and count > 2:
            state["snapped"] = True
            log.append({"op": "snapshot", "count": 0, "snapshot": snapshot(stream)})
        mine = _device_to_host(ba, ptr, 4 * count, stream).view(np.float32)
        inner(user, op, ptr, count, stream)
        log.append({"op": "allreduce", "count": count, "mine": mine,
                    "result": _device_to_host(ba, ptr, 4 * count, stream).view(np.float32)})

    ba._recording_cb = ba._collective_cb = _lib.COLLECTIVE_FN(cb)   # keep alive
    ba._recorded_inner = inner
    ba._check(ba._lib.bba_set_collective(ba._h, ba._collective_cb, None))


def _surfel_snapshot(ba):
    """All 17 rows of the replica (the full pitch) and the active flags, read on the library's stream."""
    import torch

    def snap(stream):
        st = torch.cuda.ExternalStream(stream, device=ba.device) if stream else torch.cuda.default_stream(ba.device)
        with torch.cuda.stream(st):
            return ba.surfels().cpu().numpy().copy(), ba.active_surfels().cpu().numpy().copy()
    return snap


def _calls(log, count):
    return [e for e in log if e["op"] == "allreduce" and e["count"] == count]


def _check_same_results(logs):
    """Every rank made the same sequence of collective calls and received the same results."""
    seqs = [[e for e in log if e["op"] != "snapshot"] for log in logs]
    for r, seq in enumerate(seqs[1:], 1):
        assert [(e["op"], e["count"]) for e in seq] == [(e["op"], e["count"]) for e in seqs[0]], r
        for a, b in zip(seq, seqs[0]):
            if a["op"] == "allgather":
                assert a["result"] == b["result"], (r, a["count"])
            else:
                assert a["result"].tobytes() == b["result"].tobytes(), (r, a["count"])


def _bits(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _same(a, b):
    return np.asarray(a).shape == np.asarray(b).shape and np.array_equal(_bits(a), _bits(b))


class Held:
    """Collects measured values against their limits, prints them, and fails at the end with every bound that did not hold."""

    def __init__(self, title):
        self.title, self.bad = title, []

    def __call__(self, name, value, limit):
        value = float(value)
        print(f"[{self.title}] {name}: {value:.3g} (limit {limit:.3g})")
        if not value <= limit:
            self.bad.append((name, value, limit))

    def done(self):
        assert not self.bad, (self.title, self.bad)


# ---- the workers ---------------------------------------------------------------------------------------------------------

def _init(rank, world, port):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)


def _make(scene, **kw):
    from badslam_b200.direct_ba import DirectBA
    name, opts = OPTIONS.get(scene, (scene, {}))
    return DirectBA.from_scene(SCENES[name](), device="cuda:0", **opts, **kw)


def _handle(scene, rank, world, peers, log, snapshot=False):
    ba = _make(scene, rank=rank, world_size=world)
    _set_recording_collective(ba, log, _surfel_snapshot(ba) if snapshot else None)
    if peers:
        assert ba.EnablePeerExchange() == world - 1
    return ba


def _result(r):
    return np.array([r.iterations_done, int(r.converged), r.depth_residual_count, r.descriptor_residual_count, r.pose_iterations_total,
                     r.pcg_inner_iterations_total, r.surfels_created, r.surfels_merged, r.surfels_deleted, r.surfels_size], np.int64)


def _state(ba):
    d, c, a = ba._intrinsics()
    poses, act = ba.GetKeyframeStates()
    return {"poses": poses, "act": act, "surfels": ba.GetSurfelsHost(), "active": ba.GetActiveHost(),
            "intr": np.concatenate([d, c, [np.float32(a)]]).astype(np.float32), "cf": ba.cfactor_buffer()}


def run_intrinsics_coeffs(ba):
    return {(d, c): ba.IntrinsicsCoeffs(d, c) for d, c in INTR_MODES}


# check_intrinsics_step's starting state (tests/gpu_checks.py): a non-zero deformation model
A_INIT = 0.02


def _cf_init(shape):
    return (np.random.default_rng(5).standard_normal(shape) * 0.003).astype(np.float32)


def run_intrinsics_steps(ba):
    ba.SetA(A_INIT)
    ba.SetCFactorBuffer(_cf_init(ba.cfactor_buffer().shape))
    out = []
    for _ in range(2):
        ba.OptimizeIntrinsics(True, True)
        d, c, a = ba._intrinsics()
        out.append(np.concatenate([d, c, [np.float32(a)], ba.cfactor_buffer().ravel()]).astype(np.float32))
    return out


def run_pcg(ba, intr):
    r = ba.BundleAdjustment(None, intr, intr, False, True, True, 2, 2, use_pcg=True, pcg_max_inner_iterations=6, pcg_gauge_keyframe=GAUGE)
    return dict(_state(ba), res=_result(r), rnorm=np.float32(r.pcg_last_r_norm))


def run_pose(ba):
    r = ba.BundleAdjustment(None, False, False, False, True, True, 3, 3)
    return dict(_state(ba), res=_result(r), cost=np.float64(r.cost))


def run_lifecycle(ba):
    """test_gpu_multi.py::_lifecycle_worker, plus the replica at the top of the first call's second iteration: creation, the
    split activation launches, the geometry step, merging and compaction have run once, the poses have not yet been used."""
    import torch
    top = {}

    def progress(it):
        if it == 1 and not top:
            torch.cuda.synchronize()
            n = ba.surfels_size()
            top["surfels"] = ba.surfels()[:, :n].cpu().numpy().copy()
            top["active"] = ba.active_surfels()[:n].cpu().numpy().copy()
        return True
    r = ba.BundleAdjustment(None, False, False, True, True, True, 2, 2, progress_function=progress)
    r2 = ba.BundleAdjustment(None, False, False, True, True, True, 1, 1)
    counts = np.array([r.surfels_created, r.surfels_merged, r.surfels_deleted, r.surfels_size, r2.surfels_created, r2.surfels_size,
                       r.pose_iterations_total], np.int64)
    return dict(_state(ba), counts=counts, top_surfels=top["surfels"], top_active=top["active"])


def run_window(ba):
    """Two iterations with the window of keyframe 1 alone: a work list of one keyframe, so that every other rank packs none."""
    r = ba.BundleAdjustment(None, False, False, False, True, True, 2, 2, active_keyframe_window_start=1, active_keyframe_window_end=1)
    return dict(_state(ba), res=_result(r), cost=np.float64(r.cost))


def run_edge(ba):
    r = ba.BundleAdjustment(None, True, True, False, True, True, 1, 1)
    return dict(_state(ba), res=_result(r), cost=np.float64(r.cost))


def run_geometry_only(ba):
    """The first iteration of run_edge without its pose and intrinsics steps: the replica its pose step reads.  (Without the
    end tasks, which a call that does not advance the BA iteration count runs first while the two counters differ.)"""
    ba.SetLastBAIterationCount(ba.ba_iteration_count())
    ba.BundleAdjustment(None, False, False, False, False, True, 1, 1, increase_ba_iteration_count=False)
    return ba.GetSurfelsHost(), ba.GetActiveHost()


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    _init(rank, world, port)
    out = {}

    def run(key, scene, fn, peers=False, snapshot=False):
        log = []
        value = fn(_handle(scene, rank, world, peers, log, snapshot))
        out[key] = {"log": log, "out": value}

    for scene in ("distorted", "many"):
        run(("coeffs", scene), scene, run_intrinsics_coeffs)
    run(("intr_steps",), "distorted", run_intrinsics_steps)
    for scene, intr, mode in PCG_RUNS:
        run(("pcg", scene, intr, mode), scene, lambda ba, intr=intr: run_pcg(ba, intr), peers=mode == "peer", snapshot=True)
    for mode in ("gather", "peer"):
        run(("pose", mode), "small", run_pose, peers=mode == "peer")
        run(("life", mode), "half", run_lifecycle, peers=mode == "peer")
        run(("window", mode), "kf1_alone", run_window, peers=mode == "peer")
    if world == 3:
        for scene in ("map300", "map300_depth"):
            run(("edge", scene), scene, run_edge, snapshot=True)
    with open(os.path.join(out_dir, f"rank{rank}.pkl"), "wb") as f:
        pickle.dump(out, f)
    dist.barrier()
    dist.destroy_process_group()


_RUNS = {}


def ranks(world, tmp_path_factory):
    """Every scenario of _worker, run once per world size: [rank] -> {key: {"log": ..., "out": ...}}."""
    if world not in _RUNS:
        import time
        import torch.multiprocessing as mp
        out_dir = tmp_path_factory.mktemp(f"world{world}")
        t0 = time.time()
        _RUNS[world] = None   # (a failed run fails every test of this world size once, not again)
        mp.spawn(_worker, args=(world, G._free_port(), str(out_dir)), nprocs=world, join=True)
        print(f"world {world}: every scenario on {world} ranks in {time.time() - t0:.1f} s")
        runs = []
        for r in range(world):
            with open(out_dir / f"rank{r}.pkl", "rb") as f:
                runs.append(pickle.load(f))
        _RUNS[world] = runs
    assert _RUNS[world] is not None, f"the {world}-rank run failed"
    return _RUNS[world]


_ONE = {}


def one_rank(key, fn):
    """The one-rank run of the same call (cached across world sizes)."""
    if key not in _ONE:
        _ONE[key] = fn()
    return _ONE[key]


def _one(scene, fn):
    return fn(_make(scene))


def _entries(runs, key):
    _check_same_results([z[key]["log"] for z in runs])
    return [z[key]["log"] for z in runs], [z[key]["out"] for z in runs]


# ---- 1. intrinsics normal equations ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("scene", ["distorted", "many"])
def test_intrinsics_normal_equations(world, scene, tmp_path_factory):
    """Each rank accumulates its surfel shard; one sum all-reduce of [34 sums as fp32 | B | D | b2 | obs] completes them.
    The one-rank fp64 sums add fp32 warp totals whose exponents span far less than 29 bits, so fp64 adds them exactly in any
    order (test_gpu_deterministic_values.py measured zero): a rank's fp64 partial is exact, and what the sharded path adds
    is one fp32 rounding of each partial plus the fp32 sum over the ranks, together at most world 2^-24 sum_r |partial_r|."""
    logs, outs = _entries(ranks(world, tmp_path_factory), ("coeffs", scene))
    want = one_rank(("coeffs", scene), lambda: _one(scene, run_intrinsics_coeffs))
    again = _one(scene, run_intrinsics_coeffs)
    held = Held(f"intrinsics coefficients, {scene}, world {world}")
    P = want[(True, True)][1].shape[1]
    n = 64 + 8 * P
    for mode_index, mode in enumerate(INTR_MODES):
        sums1, cells1 = want[mode]
        assert again[mode][0].tobytes() == sums1.tobytes(), mode   # fp64 reassociation of the global sums: exactly zero
        calls = [_calls(log, n) for log in logs]
        assert all(len(c) == len(INTR_MODES) for c in calls), [len(c) for c in calls]
        mine = np.stack([c[mode_index]["mine"] for c in calls]).astype(np.float64)
        res = calls[0][mode_index]["result"]
        # what every rank got back is the fp64 widening of the collective's fp32 sums, and the cell rows of the collective
        for o in outs:
            assert o[mode][0].tobytes() == res[:34].astype(np.float64).tobytes(), mode
            assert _same(o[mode][1], res[64:].reshape(8, P)), mode
        # observation counts: every (surfel, keyframe) pair on exactly one rank
        assert np.array_equal(mine[:, 64 + 7 * P:].sum(0), cells1[7].astype(np.float64)), mode
        # the 34 global sums
        S = np.abs(mine[:, :34]).sum(0)
        diff = np.abs(res[:34].astype(np.float64) - sums1)
        assert np.all(diff[S == 0] == 0) and np.all(sums1[S == 0] == 0), mode
        used = S > 0
        assert used.any()
        held(f"{mode} global sums, units of 2^-24 sum_r |partial_r|", np.max(diff[used] / (U24 * S[used])), world)
        held(f"{mode} global sums, relative to |one rank|", np.max(diff[used] / np.abs(sums1[used])), 1.0)
        cells = res[64:].reshape(8, P).astype(np.float64)
        if not mode[0]:
            assert not mine[:, 64:].any() and not cells1.any(), mode
            continue
        # cell rows: fp32 atomics on both sides, (obs + 1) 2^-24 of a bound on the running sums per cell and side, plus the
        # fp32 sum over the ranks
        obs = cells1[7].astype(np.float64)
        seen = obs > 0
        assert not cells[:7, ~seen].any() and not cells1[:7, ~seen].any(), mode
        unit = (2 * obs[seen] + 1 + world) * U24
        D1 = cells1[5, seen].astype(np.float64)
        held(f"{mode} D per cell, units of (2 obs + 1 + world) 2^-24 D", np.max(np.abs(cells[5, seen] - D1) / (unit * D1)), 1.0)
        for r in range(5):
            scale = np.sqrt(sums1[DIAG5[r]] * D1)
            diff = np.abs(cells[r, seen] - cells1[r, seen])
            assert not diff[scale == 0].any(), (mode, r)   # (a row that is zero on one side: d/da at a = 0)
            held(f"{mode} B{r} per cell, units of (2 obs + 1 + world) 2^-24 sqrt(A_rr D)",
                 np.max(diff[scale > 0] / (unit[scale > 0] * scale[scale > 0]), initial=0.0), 1.0)
        b2 = np.abs(cells1[6]).max()
        held(f"{mode} b2 per cell, units of (2 obs + 1 + world) 2^-24 max |b2|", np.max(np.abs(cells[6, seen] - cells1[6, seen]) / unit) / b2, 1.0)
    held.done()


def reference_intrinsics_spread():
    """|K| and |a| differences between the reference's two runs of check_intrinsics_step (depth and colour, `small`, two steps
    from a = 0.02 and seeded cfactors), played back from tests/golden/ref: the reference's own run-to-run spread."""
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref", "test_gpu_parity",
                             "test_intrinsics_step_three_way[True-True].npz"))
    run = [np.concatenate([z[f"{i}|3|intrinsics.0:array"], z[f"{i}|3|intrinsics.1:array"]]).astype(np.float64) for i in (0, 1)]
    a = [float(z[f"{i}|3|intrinsics.2:scalar"]) for i in (0, 1)]
    return np.abs(run[1] - run[0]), abs(a[1] - a[0])


@pytest.mark.parametrize("world", [2, 3])
def test_intrinsics_steps(world, tmp_path_factory):
    """Two OptimizeIntrinsics(True, True) steps from check_intrinsics_step's state: K, a and the cfactors bit-identical on every
    rank.  Against one rank the sharded step adds the fp32 rounding of the 34 sums (test_intrinsics_normal_equations); it must
    not move K or a further than the reference moves them between two runs of the same step (unordered fp32 atomics on the cell
    rows), and K by no more than one fp32 ulp more.  The reference records no second cfactor buffer: the cfactors, the per-cell
    part of the same depth deformation, are held to the spread of `a`."""
    logs, outs = _entries(ranks(world, tmp_path_factory), ("intr_steps",))
    for o in outs[1:]:
        assert all(_same(a, b) for a, b in zip(o, outs[0]))
    want = one_rank(("intr_steps",), lambda: _one("distorted", run_intrinsics_steps))
    again = _one("distorted", run_intrinsics_steps)
    ref_K, ref_a = reference_intrinsics_spread()
    assert ref_a > 0
    held = Held(f"intrinsics steps, world {world}")
    for step in range(2):
        got, w, w2 = (x[step].astype(np.float64) for x in (outs[0], want, again))
        for name, sl in (("K", slice(0, 8)), ("a", slice(8, 9)), ("cfactors", slice(9, None))):
            print(f"[intrinsics steps, world {world}] step {step + 1} {name}: {np.abs(got[sl] - w[sl]).max():.3g} from one rank, "
                  f"one rank run to run {np.abs(w2[sl] - w[sl]).max():.3g}")
    ulp = np.spacing(np.abs(want[1][:8]).astype(np.float32)).astype(np.float64)
    held("K after two steps, units of (reference spread + 1 ulp)", np.max(np.abs(got[:8] - w[:8]) / (ref_K + ulp)), 1.0)
    held(f"a after two steps, units of the reference spread {ref_a:.3g}", abs(got[8] - w[8]) / ref_a, 1.0)
    held("cfactors after two steps, units of the reference spread of a", np.abs(got[9:] - w[9:]).max() / ref_a, 1.0)
    held.done()


# ---- 2. PCG products -------------------------------------------------------------------------------------------------------

def _pcg_one(scene, intr, snapshot):
    """PCGDebug on one rank from the replica the sharded run's first PcgInit saw (after the PCG iteration's normals update)."""
    from badslam_b200.direct_ba import DirectBA
    sc = copy.copy(SCENES[scene]())
    sc.surfels = snapshot
    ba = DirectBA.from_scene(sc, device="cuda:0")
    return ba.PCGDebug(True, True, intr, intr, gauge_keyframe=GAUGE)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("run", PCG_RUNS, ids=["-".join(map(str, r)) for r in PCG_RUNS])
def test_pcg_products(world, run, tmp_path_factory):
    """The first PcgInit (r, M) and PcgStep1 (g + this rank's alpha_d as a (hi, lo) float pair) contributions of every rank.
    Surfel unknowns: exactly 0.0 off the rank's granules; on them r and M equal one rank bit for bit with one 16-keyframe group
    (one RED per unknown), within the reassociation of three fp32 terms with three (`many`).  Pose and intrinsics segments: the
    sum over the ranks within 5e-5 of the segment's largest entry (check_pcg_building_blocks' tolerance against the reference)."""
    from badslam_b200 import _lib
    scene, intr, mode = run
    logs, outs = _entries(ranks(world, tmp_path_factory), ("pcg",) + run)
    snaps = [[e["snapshot"] for e in log if e["op"] == "snapshot"] for log in logs]
    assert all(len(s) == 1 for s in snaps)
    snaps = [s[0] for s in snaps]
    for s in snaps[1:]:   # the rows the products read are the same in every replica (rows 8-16 are per-rank scratch)
        assert _same(s[0][:8], snaps[0][0][:8]) and np.array_equal(s[1], snaps[0][1])
    r1, M1, p1, g1, (alpha_n1, alpha_d1) = _pcg_one(scene, intr, snaps[0][0])
    U = len(r1)
    sc = SCENES[scene]()
    K, n = sc.cfg.num_keyframes, sc.num_surfels
    s0, s1 = 6 * (K - 1), 6 * (K - 1) + 3 * n
    held = Held(f"PCG products, {'-'.join(map(str, run))}, world {world}")
    init = [_calls(log, U) for log in logs]
    step1 = [_calls(log, U + 2) for log in logs]
    assert all(len(c) >= 2 for c in init) and all(len(c) >= 1 for c in step1)
    lib = _lib.load()
    owner = np.array([lib.bba_shard_surfel_owner(i, world) for i in range(0, n, 256)])[np.arange(n) >> 8]
    three_groups = K > 16
    for name, want, contrib in (("r", r1, [c[0]["mine"] for c in init]), ("M", M1, [c[1]["mine"] for c in init]),
                                ("g", g1, [c[0]["mine"][:U] for c in step1])):
        seg_w = want[s0:s1].reshape(n, 3)
        scale = np.abs(seg_w).max()
        worst = 0.0
        for rank, c in enumerate(contrib):
            seg = c[s0:s1].reshape(n, 3)
            assert not seg[owner != rank].any(), (name, rank)          # exactly 0.0 where the rank owns nothing
            mine = owner == rank
            d = np.abs(seg[mine].astype(np.float64) - seg_w[mine])
            if name != "g" and not three_groups:
                assert _same(seg[mine], seg_w[mine]), (name, rank, int((d > 0).sum()))
            worst = max(worst, float(d.max()) if d.size else 0.0)
        if name == "M" and three_groups:   # non-negative terms: two roundings of the running sum
            held("M surfel entries (3 groups), units of 2^-23 max M", worst / (2 * U24 * scale), 1.0)
        elif name == "r" and three_groups:
            held("r surfel entries (3 groups), units of 2^-23 max |r|", worst / (2 * U24 * scale), 1.0)
        elif name == "g":   # p differs from one rank in its pose / intrinsics entries (all-reduced r and M)
            held("g surfel entries, relative to max |g|", worst / scale, 5e-5)
        total = np.sum([c.astype(np.float64) for c in contrib], axis=0)
        for seg_name, lo, hi in (("pose", 0, s0), ("intrinsics", s1, U)):
            if hi > lo:
                held(f"{name} {seg_name} segment, sum over ranks, relative to its max",
                     np.abs(total[lo:hi] - want[lo:hi]).max() / np.abs(want[lo:hi]).max(), 5e-5)
    # alpha_d: every rank's (hi, lo) pair is its part of p^T J^T W J p; with the lambda / prior term of PcgInit2 (recomputed
    # here from p) they add up to the one-rank alpha_d
    pairs = np.array([c[0]["mine"][U:U + 2] for c in step1], np.float32)
    for hi, lo in pairs:
        assert hi > 0 and abs(lo) <= U24 * hi, (hi, lo)
    # (a part that fp32 holds exactly has lo = 0; every rank's at once, at 2^-29 or less each, is not a legitimate outcome)
    assert pairs[:, 1].any(), pairs
    extra = np.full(U, 1e-8, np.float32)
    if intr:
        extra[s1 + 4] += np.float32(100.0)
    eps = float(np.sum(((extra * p1) * p1).astype(np.float64))) * K
    parts = float(np.sum(pairs[:, 0].astype(np.float64) + pairs[:, 1].astype(np.float64)))
    held("alpha_d, sum of the ranks' parts + lambda / prior term, relative", abs(parts + eps - alpha_d1) / alpha_d1, 1e-6)
    # what the ranks receive: the fp32 sums of the hi and of the lo floats; the hi sum rounds once per add (world - 1 times)
    hi_r, lo_r = (float(x) for x in step1[0][0]["result"][U:U + 2])
    bound = (world - 1) * U24 * float(np.abs(pairs).astype(np.float64).sum())
    held("alpha_d received, units of (world - 1) 2^-24 sum |hi| against the parts", abs(hi_r + lo_r - parts) / bound, 1.0)
    held("alpha_d received + lambda / prior term, relative to one rank", abs(hi_r + lo_r + eps - alpha_d1) / alpha_d1, 1e-6)
    held.done()


@pytest.mark.parametrize("world", [2, 3])
def test_pcg_end_to_end(world, tmp_path_factory):
    """The PCG BAs above: replicas bit-identical; equal to one rank within test_gpu_multi.py's PCG tolerances."""
    from badslam_b200.scene import pose_error
    runs = ranks(world, tmp_path_factory)
    for run in PCG_RUNS:
        scene, intr, mode = run
        _, outs = _entries(runs, ("pcg",) + run)
        for o in outs[1:]:
            for key in ("poses", "surfels", "intr", "cf", "res", "rnorm", "act", "active"):
                assert _same(o[key], outs[0][key]), (run, key)
        want = one_rank(("pcg_e2e", scene, intr), lambda: _one(scene, lambda ba: run_pcg(ba, intr)))
        got = outs[0]
        assert got["res"][0] == want["res"][0] and abs(int(got["res"][5]) - int(want["res"][5])) <= 2, (run, got["res"], want["res"])
        assert abs(float(got["rnorm"]) - float(want["rnorm"])) < 5e-2 * max(1.0, float(want["rnorm"])), run
        worst = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(len(want["poses"])))
        ds = float(np.mean(np.abs(got["surfels"][:3] - want["surfels"][:3])))
        print(f"[PCG end to end, {'-'.join(map(str, run))}, world {world}] worst pose difference {worst:.2e}, mean surfel position "
              f"difference {ds:.2e}, inner iterations {int(got['res'][5])} / {int(want['res'][5])}")
        assert worst < 2e-4 and ds < 1e-5, (run, worst, ds)
        if intr:
            assert np.abs(got["intr"][:8] - want["intr"][:8]).max() < 2e-2 and abs(got["intr"][8] - want["intr"][8]) < 5e-3, run
            assert np.abs(got["cf"] - want["cf"]).max() < 1e-3, run


# ---- 3. pose step ----------------------------------------------------------------------------------------------------------

def check_pose_owners(logs, world, K, N):
    """Each pose step's 17-float slots: a keyframe's slot is non-zero on exactly one rank, the result is that rank's slot, and
    the rank is the round-robin deal on the handle's first step, then bba_balance_keyframes of the costs pose_step.cu derives
    from the previous slots.  Returns the number of keyframes each rank packed, per step."""
    from badslam_b200 import _lib
    lib = _lib.load()
    calls = [_calls(log, 17 * K) for log in logs]
    assert len(calls[0]) >= 1 and all(len(c) == len(calls[0]) for c in calls)
    kf_cost = np.zeros(K, np.float32)
    per_step = []
    for step in range(len(calls[0])):
        mine = np.stack([c[step]["mine"].reshape(K, 17) for c in calls])
        res = calls[0][step]["result"].reshape(K, 17)
        nz = (mine != 0).any(axis=2)
        ids = np.flatnonzero(nz.any(axis=0))
        assert len(ids) > 0 and np.all(nz[:, ids].sum(axis=0) == 1), (step, nz)
        owner = nz[:, ids].argmax(axis=0)
        assert _same(res[ids], mine[owner, ids]) and not res[~nz.any(axis=0)].any(), step
        want = np.zeros(len(ids), np.int32)
        cost = np.ascontiguousarray(kf_cost[ids])
        lib.bba_balance_keyframes(cost.ctypes.data, len(ids), world, want.ctypes.data)
        if step == 0:
            assert np.array_equal(want, np.arange(len(ids)) % world)
        assert np.array_equal(owner, want), (step, ids, owner, want, cost)
        for kf in ids:
            kf_cost[kf] = np.float32(max(1, int(res[kf, 7] + 0.5)) * (0.06 * N + float(res[kf, 14])))
        per_step.append(np.bincount(owner, minlength=world))
    return per_step


def check_pose_run(runs, key, want, world, title):
    from badslam_b200.scene import pose_error
    logs, outs = _entries(runs, key)
    for o in outs[1:]:
        for k in ("poses", "act", "surfels", "active", "res", "cost"):
            assert _same(o[k], outs[0][k]), (key, k)
    sc = SCENES["small"]()
    K = sc.cfg.num_keyframes
    per_step = check_pose_owners(logs, world, K, sc.num_surfels)
    got = outs[0]
    held = Held(f"{title}, world {world}")
    print(f"[{title}, world {world}] keyframes packed per rank and step: {[list(map(int, c)) for c in per_step]}")
    # iterations done, converged, residual counts, GN iterations; activations
    assert np.array_equal(got["res"][:5], want["res"][:5]), (got["res"][:5], want["res"][:5])
    assert np.array_equal(got["act"], want["act"])
    held("cost, units of K 2^-24 relative", abs(got["cost"] - want["cost"]) / (K * U24 * want["cost"]), 1.0)
    worst = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(K))
    held("worst pose difference", worst, min(POSE_T, POSE_R))
    held.done()
    return per_step


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mode", ["gather", "peer"])
def test_pose_step(world, mode, tmp_path_factory):
    """test_gpu_multi.py::_worker's 3-iteration alternating BA (keyframe split of the pose step, one all-reduce of the slots)."""
    want = one_rank(("pose",), lambda: _one("small", run_pose))
    check_pose_run(ranks(world, tmp_path_factory), ("pose", mode), want, world, f"pose step, {mode}")


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mode", ["gather", "peer"])
def test_pose_step_window_of_one_keyframe(world, mode, tmp_path_factory):
    """active_keyframe_window_start = end = 1 with no keyframe covisible with keyframe 1: a work list of one keyframe, so that
    every other rank runs the pose step with n_local = 0 and contributes an all-zero slot buffer."""
    want = one_rank(("window",), lambda: _one("kf1_alone", run_window))
    per_step = check_pose_run(ranks(world, tmp_path_factory), ("window", mode), want, world, f"pose step, window of one, {mode}")
    assert len(per_step) == 2 and all(c.sum() == 1 and (c == 0).sum() == world - 1 for c in per_step), per_step


# ---- 4. surfel updates with moving poses -----------------------------------------------------------------------------------

@pytest.mark.parametrize("world", [2, 3])
def test_surfel_updates(world, tmp_path_factory):
    """test_gpu_multi.py::test_two_rank_surfel_updates_match_single_gpu on one device.  The half map has 15,000 surfels, a
    ragged last granule, so the split activation launches of the in-loop creation go through LocalCountBelow; the replica at
    the top of the second iteration (poses not yet used) must equal one rank bit for bit."""
    from badslam_b200.scene import pose_error
    runs = ranks(world, tmp_path_factory)
    want = one_rank(("life",), lambda: _one("half", run_lifecycle))
    sc = SCENES["half"]()
    assert sc.num_surfels % 256 != 0
    assert want["counts"][0] > 0 and want["counts"][1] > 0
    for mode in ("gather", "peer"):
        _, outs = _entries(runs, ("life", mode))
        for o in outs[1:]:
            for key in ("counts", "poses", "surfels", "active", "top_surfels", "top_active"):
                assert _same(o[key], outs[0][key]), (mode, key)
        got = outs[0]
        assert _same(got["top_surfels"], want["top_surfels"]) and np.array_equal(got["top_active"], want["top_active"]), mode
        c, w = got["counts"], want["counts"]
        assert c[0] == w[0] and np.all(np.abs(c[1:6] - w[1:6]) <= np.maximum(3, 0.002 * w[1:6])), (mode, c, w)
        worst = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(sc.cfg.num_keyframes))
        print(f"[surfel updates, {mode}, world {world}] counts {list(c)} / {list(w)}, worst pose difference {worst:.2e}")
        assert worst < 2e-5, (mode, worst)
    assert _same(_entries(runs, ("life", "peer"))[1][0]["surfels"], _entries(runs, ("life", "gather"))[1][0]["surfels"])


# ---- 5. edge shapes --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("scene", ["map300", "map300_depth"])
def test_rank_without_surfels(scene, tmp_path_factory):
    """300 surfels at world 3: rank 2 owns no granule.  One alternating iteration with the intrinsics step, then the end tasks,
    with depth and descriptor residuals and with depth residuals only.  The replica the pose step reads equals one rank bit for
    bit, counts and activations equal it exactly, rank 2's surfel-sharded contributions are zero.

    A keyframe's pose normal equations depend on the work list it is launched with, on one rank too: at the start poses the H
    of the ranks' two-keyframe lists differ from those of the one six-keyframe list by ~1e-7 of max |H| (asserted non-zero
    below).  Six poses constrained by 300 surfels amplify that over the Gauss-Newton iterations, with the poses and the
    intrinsics step after them: with depth and descriptor residuals the result is held to test_gpu_multi.py's PCG end-to-end
    tolerances; with depth residuals only it is further off, and test_rank_without_surfels_depth_only_matches_one_rank records
    that as an open difference.  The measured differences are printed."""
    from badslam_b200 import _lib
    from badslam_b200.scene import pose_error
    world = 3
    lib = _lib.load()
    assert {lib.bba_shard_surfel_owner(i, world) for i in range(300)} == {0, 1}
    logs, outs = _entries(ranks(world, tmp_path_factory), ("edge", scene))
    for o in outs[1:]:
        for key in ("poses", "act", "surfels", "active", "intr", "cf", "res", "cost"):
            assert _same(o[key], outs[0][key]), key
    sc = SCENES["map300"]()
    K, P = sc.cfg.num_keyframes, sc.cfactor.size
    intr_calls = [_calls(log, 64 + 8 * P) for log in logs]
    deleted_calls = [_calls(log, 2) for log in logs]
    assert len(intr_calls[2]) == 1 and len(deleted_calls[2]) == 1
    assert not intr_calls[2][0]["mine"].any() and not deleted_calls[2][0]["mine"].any()
    assert intr_calls[0][0]["mine"][64 + 7 * P:].sum() > 0 and intr_calls[1][0]["mine"][64 + 7 * P:].sum() > 0
    check_pose_owners(logs, world, K, sc.num_surfels)
    # the replica at the pose step's slot all-reduce (the first all-reduce of more than two floats) against one rank's geometry step
    snap = [e["snapshot"] for e in logs[0] if e["op"] == "snapshot"][0]
    rows1, active1 = one_rank(("geometry", scene), lambda: _one(scene, run_geometry_only))
    differ = [(r, int(np.count_nonzero(_bits(snap[0][r, :300]) != _bits(rows1[r])))) for r in range(8)]
    assert _same(snap[0][:8, :300], rows1) and np.array_equal(snap[1][:300], active1), (
        differ, int(np.count_nonzero(snap[1][:300] != active1)), snap[0][:8, :4], rows1[:, :4])
    want = one_rank(("edge", scene), lambda: _one(scene, run_edge))
    again = _one(scene, run_edge)
    got = outs[0]
    assert np.array_equal(got["res"], want["res"]) and np.array_equal(got["act"], want["act"]), (got["res"], want["res"])
    # the pose kernel over the one rank's work list and over each rank's (round-robin) list, at the start poses
    ba = _make(scene)
    H_all = ba.PoseCoeffsBatch(np.arange(K), sc.poses_init[:K])[0]
    H_split = np.zeros_like(H_all)
    for r in range(world):
        ids = np.arange(r, K, world)
        H_split[ids] = ba.PoseCoeffsBatch(ids, sc.poses_init[ids])[0][ids]
    dH = float(np.max(np.abs(H_split - H_all)) / np.abs(H_all).max())
    pose_d = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(K))
    spread = max(max(pose_error(again["poses"][k], want["poses"][k])) for k in range(K))
    title = f"300 surfels, {scene}, world 3"
    print(f"[{title}] H of the split work lists against one list: {dH:.3g} of max |H|; worst pose difference {pose_d:.3g}, "
          f"one rank run to run {spread:.3g}; K {np.abs(got['intr'][:8] - want['intr'][:8]).max():.3g}, "
          f"a {abs(float(got['intr'][8]) - float(want['intr'][8])):.3g}, cfactors {np.abs(got['cf'] - want['cf']).max():.3g}")
    held = Held(title)
    held("cost, units of K 2^-24 relative", abs(got["cost"] - want["cost"]) / (K * U24 * want["cost"]), 1.0)
    held("surfel positions after the end tasks, max", np.abs(got["surfels"][:3] - want["surfels"][:3]).max(), 0.0)
    assert dH > 0 and spread == 0   # one rank is reproducible; the split of the work list changes H
    if scene == "map300":
        held("worst pose difference", pose_d, 2e-4)
        held("depth / colour K", np.abs(got["intr"][:8] - want["intr"][:8]).max(), 5e-3)
        held("a", abs(float(got["intr"][8]) - float(want["intr"][8])), 1e-5)
        held("cfactors", np.abs(got["cf"] - want["cf"]).max(), 1e-3)
    held.done()


@pytest.mark.xfail(strict=True, reason="open: with depth residuals only, the 300-surfel map at world 3 ends 2.4e-3 from one rank in "
                                      "the poses, 0.55 px in K and 0.016 in the cfactors, from bit-identical replicas and counts")
def test_rank_without_surfels_depth_only_matches_one_rank(tmp_path_factory):
    """The depth-only run of test_rank_without_surfels against one rank within the bounds of the other tests: poses within
    POSE_T / POSE_R, K within the reference's run-to-run spread + 1 ulp, a and the cfactors within its spread of a."""
    from badslam_b200.scene import pose_error
    _, outs = _entries(ranks(3, tmp_path_factory), ("edge", "map300_depth"))
    got, want = outs[0], one_rank(("edge", "map300_depth"), lambda: _one("map300_depth", run_edge))
    ref_K, ref_a = reference_intrinsics_spread()
    ulp = np.spacing(np.abs(want["intr"][:8]).astype(np.float32)).astype(np.float64)
    K = len(want["poses"])
    assert max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(K)) < min(POSE_T, POSE_R)
    assert np.all(np.abs(got["intr"][:8] - want["intr"][:8]) <= ref_K + ulp)
    assert abs(float(got["intr"][8]) - float(want["intr"][8])) <= ref_a and np.abs(got["cf"] - want["cf"]).max() <= ref_a


def _geometry_worker(rank, world, port, out_dir):
    from badslam_b200.direct_ba import DirectBA
    log = []
    DirectBA.SetCollective = lambda ba, group=None: _set_recording_collective(ba, log)   # (this worker process only)
    G._worker(rank, world, port, out_dir, backend="gloo", device_of_rank=[0] * world)
    with open(os.path.join(out_dir, f"log{rank}.pkl"), "wb") as f:
        pickle.dump(log, f)


def test_three_rank_geometry_on_one_device_matches_one_rank(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_geometry_worker, args=(3, G._free_port(), str(tmp_path)), nprocs=3, join=True)
    logs = []
    for r in range(3):
        with open(tmp_path / f"log{r}.pkl", "rb") as f:
            logs.append(pickle.load(f))
    assert any(e["op"] == "allgather" for e in logs[0])
    _check_same_results(logs)
    G.check_ranks_against_single_gpu(str(tmp_path), 3)
