"""Local groups (bba_local_group_create): the ranks of a multi-GPU job as handles of one process, each driven by its own thread,
exchanging through the library's own all-reduce and all-gather.  Two and three ranks on device 0, and two GPUs when present.

* the primitive, through bba_debug_collective: every rank's all-reduce equals, bit for bit, the fp32 sum taken sequentially in
  rank order (NaN where it is NaN: the device's NaN bits are its own), with +-0, inf and NaN mixed in, for counts that leave every
  tail of the 128-bit path and for a buffer that is not 16-byte aligned; all-gathers equal the concatenation; the bytes around
  the buffers stay untouched;
* the sharded passes of tests/test_gpu_multi_ranks_one_device.py, driven through LocalGroup.run in both exchange modes: every
  rank's replica, flags, poses, a, cfactor and result counters are bit-identical, and the results hold the bounds that file
  derives against one rank;
* two independent one-rank handles in deterministic mode, each on its own thread at the same time, give the bits of the same
  calls run one after the other;
* argument checks leave the members as they were.
The poisoned state is host logic and is tested on the CPU (test_local_group_rendezvous.py)."""
import ctypes as C
import threading

import numpy as np
import pytest

import test_gpu_multi_ranks_one_device as R
from gpu_checks import POSE_R, POSE_T

pytestmark = pytest.mark.gpu

WORLDS = ["2", "3", "2gpu"]
CANARY = 0xA5
PAD = 64


def _devices(world):
    import torch
    if world == "2gpu":
        if torch.cuda.device_count() < 2:
            pytest.skip("needs two GPUs")
        return ["cuda:0", "cuda:1"]
    return ["cuda:0"] * int(world)


def _group(scene, world, peers=False):
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    devices = _devices(world)
    name, opts = R.OPTIONS.get(scene, (scene, {}))
    handles = DirectBA.create_local_ranks(R.SCENES[name](), len(devices), devices, **opts)
    return LocalGroup(handles, peer_stores=peers)


# ---- the primitive ---------------------------------------------------------------------------------------------------------

def _special_values(rng, n):
    x = rng.standard_normal(n).astype(np.float32) * np.float32(1e3)
    pick = rng.random(n)
    x[pick < 0.03] = np.float32(0.0)
    x[(pick >= 0.03) & (pick < 0.06)] = np.float32(-0.0)
    x[(pick >= 0.06) & (pick < 0.07)] = np.float32(np.inf)
    x[(pick >= 0.07) & (pick < 0.08)] = np.float32(-np.inf)
    x[(pick >= 0.08) & (pick < 0.09)] = np.float32(np.nan)
    x[(pick >= 0.09) & (pick < 0.10)] = np.float32(1e-40)   # denormal
    return x


def _padded(dev, nbytes, offset):
    """A device byte buffer with PAD canary bytes in front of `offset` extra bytes and PAD behind the payload."""
    import torch
    buf = torch.full((PAD + offset + nbytes + PAD,), CANARY, dtype=torch.uint8, device=dev)
    return buf, buf[PAD + offset:PAD + offset + nbytes]


def _check_canaries(buf, nbytes, offset):
    b = buf.cpu().numpy()
    assert np.all(b[:PAD + offset] == CANARY) and np.all(b[PAD + offset + nbytes:] == CANARY)


@pytest.mark.parametrize("world", WORLDS)
def test_allreduce_is_the_rank_order_sum(world):
    import torch
    from badslam_b200 import _lib
    counts = [1, 2, 3, 5, 17 * 6, 17 * 1024 + 1, (1 << 20) + 3]
    with _group("small", world) as group:
        n = len(group.handles)
        for count in counts:
            for offset in (0, 4):   # 16-byte aligned (128-bit path + scalar tail) and 4-byte aligned (scalar path)
                rng = np.random.default_rng(count * 10 + offset)
                xs = [_special_values(rng, count) for _ in range(n)]
                bufs = []
                for r, ba in enumerate(group.handles):
                    buf, view = _padded(ba.device, 4 * count, offset)
                    view.copy_(torch.from_numpy(xs[r].view(np.uint8)).to(ba.device))
                    bufs.append((buf, view))
                torch.cuda.synchronize()
                group.run(lambda r, ba: ba.DebugCollective(_lib.COLLECTIVE_ALLREDUCE_SUM, bufs[r][1], count))
                want = xs[0].copy()
                with np.errstate(invalid="ignore", over="ignore"):
                    for r in range(1, n):
                        want = (want + xs[r]).astype(np.float32)
                got = [v.cpu().numpy().view(np.float32) for _, v in bufs]
                nan = np.isnan(want)
                for r in range(n):
                    assert got[r].tobytes() == got[0].tobytes(), (count, offset, r)
                    assert np.array_equal(np.isnan(got[r]), nan), (count, offset, r)
                    assert np.array_equal(got[r][~nan].view(np.uint32), want[~nan].view(np.uint32)), (count, offset, r)
                    _check_canaries(bufs[r][0], 4 * count, offset)


@pytest.mark.parametrize("world", WORLDS)
def test_allgather_is_the_concatenation(world):
    import torch
    from badslam_b200 import _lib
    with _group("small", world) as group:
        n = len(group.handles)
        for count in (1, 7, 4097):
            rng = np.random.default_rng(count)
            slices = [rng.integers(0, 256, count, dtype=np.uint8) for _ in range(n)]
            bufs = []
            for r, ba in enumerate(group.handles):
                host = np.full(n * count, 0xEE, np.uint8)
                host[r * count:(r + 1) * count] = slices[r]
                buf, view = _padded(ba.device, n * count, 0)
                view.copy_(torch.from_numpy(host).to(ba.device))
                bufs.append((buf, view))
            torch.cuda.synchronize()
            group.run(lambda r, ba: ba.DebugCollective(_lib.COLLECTIVE_ALLGATHER, bufs[r][1], count))
            want = np.concatenate(slices)
            for r in range(n):
                assert np.array_equal(bufs[r][1].cpu().numpy(), want), (count, r)
                _check_canaries(bufs[r][0], n * count, 0)


# ---- the sharded passes ----------------------------------------------------------------------------------------------------

_RUNS = {}


def _ranks(scene, world, mode, fn):
    """fn(ba) on every rank of a local group (cached per scene, world, mode and function)."""
    key = (scene, world, mode, fn.__name__)
    if key not in _RUNS:
        with _group(scene, world, peers=mode == "peer") as group:
            if mode == "peer":
                assert all(ba._lib.bba_peer_count(ba._h) == len(group.handles) - 1 for ba in group.handles)
            _RUNS[key] = group.run(lambda r, ba: fn(ba))
    return _RUNS[key]


def _identical(outs, keys):
    for o in outs[1:]:
        for k in keys:
            assert R._same(o[k], outs[0][k]), k


def run_pcg_small(ba):
    return R.run_pcg(ba, False)


def run_pcg_distorted(ba):
    return R.run_pcg(ba, True)


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("mode", ["gather", "peer"])
def test_alternating_ba(world, mode):
    """R.run_pose: the 3-iteration alternating BA on `small`, against one rank with R.check_pose_run's bounds."""
    from badslam_b200.scene import pose_error
    outs = _ranks("small", world, mode, R.run_pose)
    _identical(outs, ("poses", "act", "surfels", "active", "intr", "cf", "res", "cost"))
    want = R.one_rank(("pose",), lambda: R._one("small", R.run_pose))
    got = outs[0]
    K = len(want["poses"])
    assert np.array_equal(got["res"][:5], want["res"][:5]), (got["res"][:5], want["res"][:5])
    assert np.array_equal(got["act"], want["act"])
    held = R.Held(f"local group, alternating BA, {mode}, world {world}")
    held("cost, units of K 2^-24 relative", abs(got["cost"] - want["cost"]) / (K * R.U24 * want["cost"]), 1.0)
    held("worst pose difference", max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(K)), min(POSE_T, POSE_R))
    held.done()


@pytest.mark.parametrize("world", ["2", "3"])
@pytest.mark.parametrize("mode", ["gather", "peer"])
def test_surfel_updates(world, mode):
    """R.run_lifecycle (do_surfel_updates with moving poses on the half map): the replica at the top of the second iteration
    equals one rank bit for bit, the rest holds R.test_surfel_updates' bounds."""
    from badslam_b200.scene import pose_error
    outs = _ranks("half", world, mode, R.run_lifecycle)
    _identical(outs, ("counts", "poses", "surfels", "active", "top_surfels", "top_active", "intr", "cf"))
    want = R.one_rank(("life",), lambda: R._one("half", R.run_lifecycle))
    got = outs[0]
    assert R._same(got["top_surfels"], want["top_surfels"]) and np.array_equal(got["top_active"], want["top_active"])
    c, w = got["counts"], want["counts"]
    assert c[0] == w[0] and np.all(np.abs(c[1:6] - w[1:6]) <= np.maximum(3, 0.002 * w[1:6])), (c, w)
    worst = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(len(want["poses"])))
    assert worst < 2e-5, worst


@pytest.mark.parametrize("world", ["2", "3"])
@pytest.mark.parametrize("run", [("small", "gather"), ("small", "peer"), ("distorted", "gather")], ids=lambda r: "-".join(r))
def test_pcg(world, run):
    """R.run_pcg, with the intrinsics on the distorted scene: replicas bit-identical, R.test_pcg_end_to_end's bounds."""
    from badslam_b200.scene import pose_error
    scene, mode = run
    intr = scene == "distorted"
    outs = _ranks(scene, world, mode, run_pcg_distorted if intr else run_pcg_small)
    _identical(outs, ("poses", "surfels", "intr", "cf", "res", "rnorm", "act", "active"))
    want = R.one_rank(("pcg_e2e", scene, intr), lambda: R._one(scene, lambda ba: R.run_pcg(ba, intr)))
    got = outs[0]
    assert got["res"][0] == want["res"][0] and abs(int(got["res"][5]) - int(want["res"][5])) <= 2, (got["res"], want["res"])
    assert abs(float(got["rnorm"]) - float(want["rnorm"])) < 5e-2 * max(1.0, float(want["rnorm"]))
    worst = max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(len(want["poses"])))
    ds = float(np.mean(np.abs(got["surfels"][:3] - want["surfels"][:3])))
    assert worst < 2e-4 and ds < 1e-5, (worst, ds)
    if intr:
        assert np.abs(got["intr"][:8] - want["intr"][:8]).max() < 2e-2 and abs(got["intr"][8] - want["intr"][8]) < 5e-3
        assert np.abs(got["cf"] - want["cf"]).max() < 1e-3


@pytest.mark.parametrize("mode", ["gather", "peer"])
def test_rank_without_surfels(mode):
    """The 300-surfel map at world 3 (rank 2 owns no granule): one alternating iteration with the intrinsics step and the end
    tasks, against one rank with R.test_rank_without_surfels' bounds."""
    from badslam_b200.scene import pose_error
    outs = _ranks("map300", "3", mode, R.run_edge)
    _identical(outs, ("poses", "act", "surfels", "active", "intr", "cf", "res", "cost"))
    want = R.one_rank(("edge", "map300"), lambda: R._one("map300", R.run_edge))
    got = outs[0]
    K = len(want["poses"])
    assert np.array_equal(got["res"], want["res"]) and np.array_equal(got["act"], want["act"]), (got["res"], want["res"])
    held = R.Held(f"local group, 300 surfels, {mode}, world 3")
    held("cost, units of K 2^-24 relative", abs(got["cost"] - want["cost"]) / (K * R.U24 * want["cost"]), 1.0)
    held("surfel positions after the end tasks, max", np.abs(got["surfels"][:3] - want["surfels"][:3]).max(), 0.0)
    held("worst pose difference", max(max(pose_error(got["poses"][k], want["poses"][k])) for k in range(K)), 2e-4)
    held("depth / colour K", np.abs(got["intr"][:8] - want["intr"][:8]).max(), 5e-3)
    held("a", abs(float(got["intr"][8]) - float(want["intr"][8])), 1e-5)
    held("cfactors", np.abs(got["cf"] - want["cf"]).max(), 1e-3)
    held.done()


# ---- handles side by side --------------------------------------------------------------------------------------------------

def test_independent_handles_on_concurrent_threads():
    """Two world_size = 1 handles in deterministic mode, each running an alternating BA with the intrinsics step and surfel
    updates on its own thread at the same time, give the bits of the same calls made one after the other."""
    import torch

    def make(scene):
        ba = R._make(scene)
        ba.SetDeterministic(True)
        return ba

    def work(ba):
        r = ba.BundleAdjustment(None, True, True, True, True, True, 2, 2)
        return dict(R._state(ba), res=R._result(r), cost=np.float64(r.cost))

    scenes = ("small", "half")
    alone = [work(make(s)) for s in scenes]
    handles = [make(s) for s in scenes]
    outs, errors = [None, None], []

    def body(i):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                outs[i] = work(handles[i])
        except BaseException as e:  # noqa: B036
            errors.append(e)

    threads = [threading.Thread(target=body, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for a, b in zip(outs, alone):
        for k in ("poses", "act", "surfels", "active", "intr", "cf", "res", "cost"):
            assert R._same(a[k], b[k]), k


# ---- argument checks -------------------------------------------------------------------------------------------------------

def test_argument_checks_leave_the_members_unchanged(tiny_scene):
    import copy

    import torch
    from badslam_b200 import _lib
    from badslam_b200.direct_ba import DirectBA, LocalGroup
    lib = _lib.load()
    ranks = DirectBA.create_local_ranks(tiny_scene, 2)
    three = DirectBA.create_local_ranks(tiny_scene, 3)
    fewer = copy.copy(tiny_scene)
    fewer.num_surfels = tiny_scene.num_surfels - 100
    other = DirectBA.from_scene(fewer, rank=1, world_size=2)
    buf = torch.zeros(8, dtype=torch.float32, device="cuda:0")

    def create(handles, count=None, peers=0):
        arr = (C.c_void_p * len(handles))(*[h._h.value if h is not None else None for h in handles])
        g = C.c_void_p()
        return lib.bba_local_group_create(arr, len(handles) if count is None else count, peers, C.byref(g))

    def unchanged(handles):   # still no exchange registered, no peers mapped
        for ba in handles:
            assert lib.bba_debug_collective(ba._h, _lib.COLLECTIVE_ALLREDUCE_SUM, C.c_void_p(buf.data_ptr()), 8, None) == _lib.ERR_STATE
            assert lib.bba_peer_count(ba._h) == 0

    assert create(three[:2]) == _lib.ERR_INVALID_ARGUMENT                   # world size 3, count 2
    assert create([ranks[0], ranks[0]]) == _lib.ERR_INVALID_ARGUMENT        # duplicate rank 0
    assert create([ranks[1], ranks[0]]) == _lib.ERR_INVALID_ARGUMENT        # ranks out of order
    assert create([three[0], three[1], three[1]]) == _lib.ERR_INVALID_ARGUMENT   # rank 2 missing
    assert create([ranks[0], None]) == _lib.ERR_INVALID_ARGUMENT            # NULL member
    assert lib.bba_local_group_create(None, 2, 0, C.byref(C.c_void_p())) == _lib.ERR_INVALID_ARGUMENT
    arr = (C.c_void_p * 2)(ranks[0]._h.value, ranks[1]._h.value)
    assert lib.bba_local_group_create(arr, 2, 0, None) == _lib.ERR_INVALID_ARGUMENT
    assert create([ranks[0]] * 10) == _lib.ERR_UNSUPPORTED                  # more than 9 ranks
    assert create([ranks[0], other], peers=1) == _lib.ERR_INVALID_ARGUMENT  # peer stores, different surfels_size
    unchanged(ranks + three + [other])
    with LocalGroup(ranks) as group:
        with pytest.raises(_lib.BadBAError) as e:   # a member of two groups
            LocalGroup(ranks)
        assert e.value.status == _lib.ERR_STATE
        noop = _lib.COLLECTIVE_FN(lambda *a: None)
        for ba in ranks:
            assert lib.bba_set_collective(ba._h, noop, None) == _lib.ERR_STATE
            ph = (_lib.PeerHandle * 2)()
            assert lib.bba_peer_import(ba._h, ph, 2) == _lib.ERR_STATE
        # the group is still in service
        xs = [torch.full((5,), float(r + 1), device="cuda:0") for r in range(2)]
        group.run(lambda r, ba: ba.DebugCollective(_lib.COLLECTIVE_ALLREDUCE_SUM, xs[r], 5))
        assert all(np.array_equal(x.cpu().numpy(), np.full(5, 3.0, np.float32)) for x in xs)
    unchanged(ranks)   # destroy restored "no collective"
