"""Multi-GPU geometry step (needs >= 2 GPUs).  The standalone activation and geometry-iteration entry points always sort, so with
the host-collective exchange every rank owns 256-surfel granules of sorted positions, rebuilds the order from its replica before
each launch, stores its results to caller index perm[s] and exchanges them by pack / all-gather / unpack through perm.  With peer
stores into the other replica the launches keep the caller's order.  In both modes every rank's rows 0-7 and flags must equal the
single-GPU run bit for bit, on the border scene of tests/test_gpu_geometry_order.py, in all three residual modes.  (_worker takes
a backend and a rank -> device map so that the same check can run with both ranks on one device over gloo.)"""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_dir, backend="nccl", device_of_rank=None):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if device_of_rank is None else device_of_rank[rank]
    torch.cuda.set_device(dev)
    kw = {"device_id": torch.device("cuda", dev)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    import test_gpu_geometry_order as T
    sc = T.border_scene(S, S.make_scene(S.config_by_name("many")))

    def collective(ba):
        ba.SetCollective()

    def peers(ba):
        ba.SetCollective()
        assert ba.EnablePeerExchange() == world - 1

    out = {}
    for tag, prepare in (("gather", collective), ("peer", peers)):
        for use_depth, use_desc in T.MODES:
            f, rows, g = T.activation_and_geometry(DirectBA, sc, use_depth, use_desc, prepare=prepare, device=f"cuda:{dev}",
                                                   rank=rank, world_size=world)
            key = f"{tag}_{int(use_depth)}{int(use_desc)}"
            out[key + "_flags_act"], out[key + "_rows"], out[key + "_flags"] = f, rows, g
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
    dist.barrier()
    dist.destroy_process_group()


def check_ranks_against_single_gpu(out_dir, world):
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    import test_gpu_geometry_order as T
    sc = T.border_scene(S, S.make_scene(S.config_by_name("many")))
    ranks = [np.load(os.path.join(out_dir, f"rank{r}.npz")) for r in range(world)]
    for use_depth, use_desc in T.MODES:
        f, rows, g = T.activation_and_geometry(DirectBA, sc, use_depth, use_desc, device="cuda:0")
        assert 0 < f.sum() < f.size
        for r, z in enumerate(ranks):
            for tag in ("gather", "peer"):
                key = f"{tag}_{int(use_depth)}{int(use_desc)}"
                assert np.array_equal(z[key + "_flags_act"], f), (r, key)
                assert np.array_equal(z[key + "_rows"].view(np.uint32), rows.view(np.uint32)), (r, key)
                assert np.array_equal(z[key + "_flags"], g), (r, key)


def test_two_rank_geometry_in_spatial_order_matches_single_gpu(tmp_path):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    check_ranks_against_single_gpu(str(tmp_path), 2)
