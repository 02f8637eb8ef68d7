"""GPU checks of the batch handoff inside the pose kernel's PRE instantiations (the ones the BA pose step runs at 4 or more
keyframes): producer warps pack each sub-item's associated pairs into 32-pair batches, and a consumer warp sums them.

The surfel sets are built from copies of one surfel of `many`, so that every keyframe that associates it has a sub-item with
exactly c associated pairs (0 for the others): c = 1, 31, 32 and 33 straddle the batch boundary, 256 fills a whole chunk, and
an interleaving with a surfel that a keyframe does not associate spreads the pairs over several 32-surfel steps.  Every
keyframe is in the work list.  Checked against the single-keyframe path (which sums the same pairs in another order), against
c times the one-pair sums, and across calls: without stats only the order of the fp64 atomics may differ between two calls.
"""
import copy

import numpy as np
import pytest

from gpu_checks import rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import _lib
    from badslam_b200.direct_ba import DirectBA
    from badslam_b200.scene import config_by_name, make_scene
    return _lib, DirectBA, make_scene(config_by_name("many"))


def with_surfels(sc, columns):
    """A copy of `sc` whose surfels are the given columns of its surfel buffer, in that order."""
    out = copy.copy(sc)
    n = len(columns)
    out.surfels = np.zeros((sc.surfels.shape[0], max(128, -(-n // 128) * 128)), np.float32)
    out.surfels[:, :n] = sc.surfels[:, columns]
    out.num_surfels = n
    return out


def pre_variants(L):
    return {"auto": L.POSE_VARIANT_AUTO, "512/PRE": L.POSE_VARIANT_512_PRE}


def check_list(ba, ids, poses, variant, tag):
    """The batched sums against the single-keyframe path, with and without stats, and twice without stats in a row.
    Returns the batched (H, b, counts) with stats."""
    H, b, cnt, _ = ba.PoseCoeffsBatch(ids, poses[ids], variant, with_stats=True)
    H0, b0, cnt0, _ = ba.PoseCoeffsBatch(ids, poses[ids], variant, with_stats=False)
    H1, b1, cnt1, _ = ba.PoseCoeffsBatch(ids, poses[ids], variant, with_stats=False)
    for k in ids:
        pc = ba.AccumulatePoseEstimationCoeffs(int(k), poses[k])
        t = (tag, int(k))
        assert tuple(cnt[k]) == (pc.n_inimg, pc.n_depthok, pc.n_assoc, pc.n_photo), (t, cnt[k], pc.n_assoc)
        assert tuple(cnt0[k]) == tuple(cnt1[k]) == (0, 0, pc.n_assoc, pc.n_photo), (t, cnt0[k], cnt1[k])
        if pc.n_assoc == 0:
            assert not H[k].any() and not b[k].any() and not H0[k].any() and not b0[k].any(), t
            continue
        assert rel(H[k], pc.H[:]) < 1e-5 and rel(b[k], pc.b[:]) < 1e-5, (t, rel(H[k], pc.H[:]), rel(b[k], pc.b[:]))
        assert rel(H0[k], H[k]) < 1e-9 and rel(b0[k], b[k]) < 1e-9, (t, rel(H0[k], H[k]), rel(b0[k], b[k]))
        assert rel(H1[k], H0[k]) < 1e-12 and rel(b1[k], b0[k]) < 1e-12, (t, rel(H1[k], H0[k]), rel(b1[k], b0[k]))
    return H, b, cnt


def seen_by(ba, ids, poses):
    """Keyframes of `ids` that associate the (single) surfel of `ba`."""
    return [k for k in ids if ba.AccumulatePoseEstimationCoeffs(int(k), poses[k]).n_assoc > 0]


def test_ragged_pair_counts_per_sub_item(env):
    L, DirectBA, sc = env
    K = sc.cfg.num_keyframes
    ids = np.arange(K)
    poses = sc.poses_init
    # a surfel that some keyframes associate and others do not, and one that at least one of the former does not associate
    one = DirectBA.from_scene(with_surfels(sc, [0]))
    a_seen = seen_by(one, ids, poses)
    assert 0 < len(a_seen) < K, a_seen
    H1, b1, _, _ = one.PoseCoeffsBatch(ids, poses, L.POSE_VARIANT_256_PRE, with_stats=False)
    # (surfels are stored in blocks by the keyframe that created them: one candidate per block)
    step = sc.num_surfels // K
    b_col = next(i for i in range(step, sc.num_surfels, step)
                 if set(a_seen) - set(seen_by(DirectBA.from_scene(with_surfels(sc, [i])), a_seen, poses)))
    for c in (1, 31, 32, 33, 256):
        ba = DirectBA.from_scene(with_surfels(sc, [0] * c))
        for vname, v in pre_variants(L).items():
            H, b, cnt = check_list(ba, ids, poses, v, (c, vname))
            assert sorted(np.flatnonzero(cnt[:, 2])) == a_seen and np.all(cnt[a_seen, 2] == c), (c, vname, cnt[:, 2])
            # c copies of one pair: c times its sums
            for k in a_seen:
                assert rel(H[k], c * H1[k]) < 1e-5 and rel(b[k], c * b1[k]) < 1e-5, (c, vname, k, rel(H[k], c * H1[k]))
    # 33 copies of the first surfel interleaved with 33 of the second: a keyframe that associates only the first gets its 33
    # pairs from every other lane of three 32-surfel steps
    ba = DirectBA.from_scene(with_surfels(sc, [0, b_col] * 33))
    for vname, v in pre_variants(L).items():
        _, _, cnt = check_list(ba, ids, poses, v, ("interleaved", vname))
        assert any(cnt[k, 2] == 33 for k in a_seen), (vname, cnt[:, 2])


def test_work_list_of_four_keyframes(env):
    """The smallest work list the BA pose step runs the PRE instantiations for, on all surfels of `many`."""
    L, DirectBA, sc = env
    ba = DirectBA.from_scene(sc)
    for ids in ([0, 1, 2, 3], [36, 17, 8, 0]):
        for vname, v in pre_variants(L).items():
            _, _, cnt = check_list(ba, np.asarray(ids), sc.poses_init, v, (tuple(ids), vname))
            assert np.all(cnt[ids, 2] > 0), (ids, vname, cnt[ids, 2])
