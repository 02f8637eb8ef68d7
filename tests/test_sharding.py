"""Host-side logic of the multi-GPU path on CPU: the surfel / keyframe partition exposed by the C ABI and the two
exchange patterns (in-place all-gather of shards, sum all-reduce over disjoint slots), exercised with world_size 2
over the gloo backend."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def owners(lib, n, world):
    idx = np.arange(n, dtype=np.uint32)
    own = np.array([lib.bba_shard_surfel_owner(int(i), world) for i in idx[::256]], np.int64).repeat(256)[:n]
    return idx, own


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 1000, 200_000, 3_000_000])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_surfel_granules_partition_the_surfels(n, world):
    """256-surfel granules dealt round-robin: every surfel has exactly one owner, the shards are balanced to one granule,
    and (owner, local index) is a bijection into the exchange slices."""
    from badslam_b200 import _lib
    lib = _lib.load()
    idx, own = owners(lib, n, world)
    assert np.array_equal(own, (idx >> 8) % world if world > 1 else np.zeros(n, np.int64))
    counts = np.bincount(own, minlength=world) if n else np.zeros(world, np.int64)
    assert counts.sum() == n and counts.max() - counts.min() <= 256
    slice_len = lib.bba_shard_slice_length(n, world)
    assert slice_len % 256 == 0 and slice_len * world >= n and (n == 0 or slice_len >= counts.max())
    for i in (0, 1, 255, 256, 257, n // 2, n - 1):
        if 0 <= i < n:
            loc = lib.bba_shard_surfel_local_index(i, world)
            assert loc < slice_len
            g = i >> 8
            assert loc == (((g // world) << 8) | (i & 255) if world > 1 else i)


def test_keyframe_work_list_is_dealt_round_robin():
    from badslam_b200 import _lib
    lib = _lib.load()
    for world in (1, 2, 8):
        owners = [lib.bba_shard_keyframe_owner(i, world) for i in range(37)]
        assert owners == [i % world if world > 1 else 0 for i in range(37)]
        counts = np.bincount(owners, minlength=world)
        assert counts.max() - counts.min() <= 1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, n, K, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from badslam_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(0)                      # identical replicated state on every rank
    rows = rng.normal(size=(7, n)).astype(np.float32)
    new_rows = rng.normal(size=(7, n)).astype(np.float32)   # what a full (single-rank) geometry step would produce
    idx, own = owners(lib, n, world)
    loc = np.array([lib.bba_shard_surfel_local_index(int(i), world) for i in idx], np.int64)
    mine = own == rank
    local = rows.copy()
    local[:, mine] = new_rows[:, mine]                  # this rank only updates its shard
    # exchange buffer: world slices of [7][shard_len] in local index order (kernels.cu PackShardKernel / UnpackShardsKernel)
    shard_len = lib.bba_shard_slice_length(n, world)
    buf = torch.zeros(world * 7 * shard_len)
    sl = buf.view(world, 7, shard_len)
    sl[rank][:, torch.from_numpy(loc[mine])] = torch.from_numpy(local[:, mine])
    dist.all_gather_into_tensor(buf, buf.view(world, -1)[rank].clone())
    merged = local.copy()
    for r in range(world):
        if r != rank:
            theirs = own == r
            merged[:, theirs] = buf.view(world, 7, shard_len)[r][:, torch.from_numpy(loc[theirs])].numpy()
    assert np.array_equal(merged, new_rows)             # every replica equals the single-rank result, bit for bit

    # pose slots: each keyframe of the work list is owned by exactly one rank; sum over disjoint slots == gather
    work = list(range(0, K, 2)) + [1]                    # some non-inactive keyframes
    truth = rng.normal(size=(K, 17)).astype(np.float32)
    slots = torch.zeros(K, 17)
    for i, kf in enumerate(work):
        if lib.bba_shard_keyframe_owner(i, world) == rank:
            slots[kf] = torch.from_numpy(truth[kf])
    dist.all_reduce(slots)
    for kf in work:
        assert np.array_equal(slots[kf].numpy(), truth[kf])
    untouched = [k for k in range(K) if k not in work]
    assert not slots[untouched].any()
    open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    dist.destroy_process_group()


@pytest.mark.parametrize("world,n", [(2, 1000), (4, 5000), (8, 9001)])
def test_exchange_patterns_gloo(tmp_path, world, n):
    """One process per rank over gloo: the surfel-granule all-gather and the keyframe-slot all-reduce reassemble the same state on
    every rank (world 2, and world 4 with surfel counts that leave ranks with uneven granule counts)."""
    port = _free_port()
    mp.spawn(_worker, args=(world, port, n, 9, str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))


def test_keyframe_balancing_rule():
    """bba_balance_keyframes: longest-first onto the least loaded rank; deterministic; round-robin without statistics."""
    from badslam_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(1)
    for world in (2, 3, 8):
        n = 200
        cost = (rng.random(n) ** 3 * 100 + 1).astype(np.float32)      # skewed work, like Gauss-Newton iterations x visible pairs
        owner = np.full(n, -1, np.int32)
        lib.bba_balance_keyframes(cost.ctypes.data, n, world, owner.ctypes.data)
        assert owner.min() >= 0 and owner.max() < world
        load = np.bincount(owner, weights=cost, minlength=world)
        assert load.max() - load.min() <= cost.max()                     # LPT bound: within one item of each other
        rr = np.bincount(np.arange(n) % world, weights=cost, minlength=world)
        assert load.max() <= rr.max() + 1e-3                             # never worse than round-robin here
        again = np.full(n, -1, np.int32)
        lib.bba_balance_keyframes(cost.ctypes.data, n, world, again.ctypes.data)
        assert np.array_equal(owner, again)                              # every rank computes the same assignment
        # unknown entries take the mean of the known ones; no statistics at all -> round-robin
        partial = cost.copy()
        partial[::3] = 0
        lib.bba_balance_keyframes(partial.ctypes.data, n, world, owner.ctypes.data)
        assert np.bincount(owner, minlength=world).min() > 0
        zeros = np.zeros(n, np.float32)
        lib.bba_balance_keyframes(zeros.ctypes.data, n, world, owner.ctypes.data)
        assert np.array_equal(owner, np.arange(n) % world)
    lib.bba_balance_keyframes(cost.ctypes.data, n, 1, owner.ctypes.data)
    assert not owner.any()


def _worker_round2(rank, world, port, n, K, out_dir):
    """The exchange patterns added in round 2 (bundle_adjust.cu BundleAdjustPCG / PerformEndTasks with world_size > 1), with the same
    arithmetic on the host: (1) PCG products -- every rank sums over ITS surfels only, one fp32 sum all-reduce of the vector with the
    rank's fp64 part of alpha_d appended as a (high, low) float pair; (2) end tasks -- the two result rows of a rank's shard through
    the all-gather, the deleted count as two exactly representable floats through a sum all-reduce."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from badslam_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(3)
    idx, own = owners(lib, n, world)
    mine = own == rank

    # (1) unknown vector = [6 (K - 1) pose | 3 n surfel | 5 + P intrinsics]: a surfel's entries are produced by its owner only, pose
    # and intrinsics entries are partial sums over the owner's surfels
    P = 12
    per_surfel_pose = rng.normal(size=(n, 6 * (K - 1))).astype(np.float32) * 1e-3    # contribution of surfel i to the pose entries
    per_surfel_intr = rng.normal(size=(n, 5 + P)).astype(np.float32) * 1e-3
    surfel_entries = rng.normal(size=(n, 3)).astype(np.float32)
    per_surfel_alpha = rng.random(n)                                                 # fp64 contributions to p^T A p
    g = np.zeros(6 * (K - 1) + 3 * n + 5 + P + 2, np.float32)
    g[:6 * (K - 1)] = per_surfel_pose[mine].sum(0, dtype=np.float32)
    g[6 * (K - 1) + 3 * np.nonzero(mine)[0][:, None] + np.arange(3)] = surfel_entries[mine]
    g[6 * (K - 1) + 3 * n:-2] = per_surfel_intr[mine].sum(0, dtype=np.float32)
    alpha_mine = float(per_surfel_alpha[mine].sum())
    hi = np.float32(alpha_mine)
    g[-2], g[-1] = hi, np.float32(alpha_mine - float(hi))                             # PcgPackAlphaDKernel
    t = torch.from_numpy(g.copy())
    dist.all_reduce(t)
    got = t.numpy()
    assert np.array_equal(got[6 * (K - 1):6 * (K - 1) + 3 * n].reshape(n, 3), surfel_entries)     # gather of disjoint entries: exact
    assert np.allclose(got[:6 * (K - 1)], per_surfel_pose.sum(0, dtype=np.float64), rtol=0, atol=1e-5)
    assert np.allclose(got[6 * (K - 1) + 3 * n:-2], per_surfel_intr.sum(0, dtype=np.float64), rtol=0, atol=1e-5)
    alpha = float(got[-2]) + float(got[-1])                                           # PcgUnpackAlphaDKernel
    assert abs(alpha - per_surfel_alpha.sum()) < 1e-6 * per_surfel_alpha.sum()        # (fp32 alone would be off by ~1e-4 relative here)
    # every rank holds the same bits afterwards: hash all-gathered
    digest = torch.tensor(list(got.tobytes()[:64]) + [int(got.view(np.uint32).sum() % 251)], dtype=torch.int64)
    both = [torch.empty_like(digest) for _ in range(world)]
    dist.all_gather(both, digest)
    assert all(torch.equal(b, both[0]) for b in both)

    # (2) end tasks: rows x (deletion marker) and radius^2 of the shard, deleted count split into (low 12 bits, rest)
    rows = rng.normal(size=(2, n)).astype(np.float32)
    new_rows = rows.copy()
    deleted = rng.random(n) < 0.1
    new_rows[0, deleted] = np.uint32(0x7fffffff).view(np.float32)
    new_rows[1, ~deleted] = rng.random((~deleted).sum()).astype(np.float32)
    loc = np.array([lib.bba_shard_surfel_local_index(int(i), world) for i in idx], np.int64)
    shard_len = lib.bba_shard_slice_length(n, world)
    buf = torch.zeros(world * 2 * shard_len)
    local = rows.copy()
    local[:, mine] = new_rows[:, mine]
    buf.view(world, 2, shard_len)[rank][:, torch.from_numpy(loc[mine])] = torch.from_numpy(local[:, mine])
    dist.all_gather_into_tensor(buf, buf.view(world, -1)[rank].clone())
    merged = local.copy()
    for r in range(world):
        if r != rank:
            theirs = own == r
            merged[:, theirs] = buf.view(world, 2, shard_len)[r][:, torch.from_numpy(loc[theirs])].numpy()
    assert np.array_equal(merged.view(np.uint32), new_rows.view(np.uint32))
    count_mine = int(deleted[mine].sum()) + (1 << 22) * 3                              # (made large: past fp32's 2^24 when summed naively)
    pair = torch.tensor([float(count_mine & 0xfff), float(count_mine >> 12)])
    dist.all_reduce(pair)
    total = int(pair[0].item() + 0.5) + (int(pair[1].item() + 0.5) << 12)
    assert total == int(deleted.sum()) + world * (1 << 22) * 3
    open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    dist.destroy_process_group()


@pytest.mark.parametrize("world,n", [(2, 1000), (4, 3000), (8, 7001)])
def test_round2_exchange_patterns_gloo(tmp_path, world, n):
    port = _free_port()
    mp.spawn(_worker_round2, args=(world, port, n, 5, str(tmp_path)), nprocs=world, join=True)
    assert all((tmp_path / f"ok{r}").exists() for r in range(world))
