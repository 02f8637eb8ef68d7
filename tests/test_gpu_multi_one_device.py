"""Two ranks on one H100 (both processes on device 0, gloo): the surfel exchanges of the multi-GPU path run on a one-GPU box.

* The geometry step of tests/test_gpu_multi_geometry_order.py in both exchange modes (pack / all-gather / unpack through the
  spatial order, and stores into the peer replica).
* The end tasks' observation pass: on the half map of tests/test_gpu_multi.py, a BA call with surfel updates that advances the BA
  iteration count (its end tasks run at the end of the call), then PerformBASchemeEndTasks, in both exchange modes.  The poses
  stay fixed, so that every step is per surfel or replicated and the result does not depend on how the work is split.

Every rank's rows 0-7, active flags, surfel count and deleted counts must equal the one-rank run bit for bit.  Gloo runs the
all-gather only on host tensors, so the ranks register a collective that stages the library's device buffers through host
memory instead of DirectBA.SetCollective's."""
import os

import numpy as np
import pytest

import test_gpu_multi_geometry_order as G

pytestmark = pytest.mark.gpu

WORLD = 2


def _set_host_staged_collective(ba, group=None):
    """bba_set_collective with every collective on a host copy of the buffer, ordered behind the work queued on the stream."""
    import torch
    import torch.distributed as dist
    from badslam_b200 import _lib
    rank, world = dist.get_rank(group), dist.get_world_size(group)

    def device_bytes(ptr, nbytes):
        class _Raw:
            pass
        raw = _Raw()
        raw.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2, "strides": None}
        return torch.as_tensor(raw, device=ba.device)

    def cb(user, op, ptr, count, stream):
        st = torch.cuda.ExternalStream(stream, device=ba.device) if stream else torch.cuda.default_stream(ba.device)
        with torch.cuda.stream(st):
            if op == _lib.COLLECTIVE_ALLGATHER:
                buf = device_bytes(ptr, count * world)
                host = buf.cpu()
                dist.all_gather_into_tensor(host, host[rank * count:(rank + 1) * count].clone(), group=group)
            else:
                buf = device_bytes(ptr, count * 4)
                host = buf.cpu().view(torch.float32)
                dist.all_reduce(host, group=group)
            buf.copy_(host.view(torch.uint8))

    ba._collective_cb = _lib.COLLECTIVE_FN(cb)   # keep alive
    ba._check(ba._lib.bba_set_collective(ba._h, ba._collective_cb, None))


def _init(rank, port):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)


def _geometry_worker(rank, port, out_dir):
    from badslam_b200.direct_ba import DirectBA
    DirectBA.SetCollective = _set_host_staged_collective   # (this worker process only)
    G._worker(rank, WORLD, port, out_dir, backend="gloo", device_of_rank=[0] * WORLD)


def test_two_rank_geometry_on_one_device_matches_one_rank(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_geometry_worker, args=(G._free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    G.check_ranks_against_single_gpu(str(tmp_path), WORLD)


def end_tasks(prepare=None, **kw):
    from badslam_b200.direct_ba import DirectBA
    from test_gpu_multi import _half_small
    ba = DirectBA.from_scene(_half_small(), device="cuda:0", **kw)
    if prepare is not None:
        prepare(ba)
    r = ba.BundleAdjustment(None, False, False, True, False, True, 2, 2, increase_ba_iteration_count=True)
    deleted, size = ba.PerformBASchemeEndTasks(do_surfel_updates=True)
    counts = np.array([r.surfels_created, r.surfels_merged, r.surfels_deleted, r.surfels_size, deleted, size], np.int64)
    return {"rows": ba.GetSurfelsHost(), "active": ba.GetActiveHost(), "counts": counts}


def _end_tasks_worker(rank, port, out_dir):
    import torch.distributed as dist
    _init(rank, port)

    def peers(ba):
        _set_host_staged_collective(ba)
        assert ba.EnablePeerExchange() == WORLD - 1

    out = {}
    for tag, prepare in (("gather", _set_host_staged_collective), ("peer", peers)):
        for key, v in end_tasks(prepare, rank=rank, world_size=WORLD).items():
            out[f"{tag}_{key}"] = v
    np.savez(os.path.join(out_dir, f"end{rank}.npz"), **out)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_end_tasks_on_one_device_match_one_rank(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_end_tasks_worker, args=(G._free_port(), str(tmp_path)), nprocs=WORLD, join=True)
    want = end_tasks()
    c = want["counts"]
    assert c[0] > 0 and c[1] > 0, c   # surfels were created and merged
    for r in range(WORLD):
        z = np.load(tmp_path / f"end{r}.npz")
        for tag in ("gather", "peer"):
            assert np.array_equal(z[f"{tag}_counts"], c), (r, tag, z[f"{tag}_counts"], c)
            assert np.array_equal(z[f"{tag}_rows"].view(np.uint32), want["rows"].view(np.uint32)), (r, tag)
            assert np.array_equal(z[f"{tag}_active"], want["active"]), (r, tag)
