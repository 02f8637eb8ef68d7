"""GPU: the handoff between the producer and consumer warps of the pose kernel's PRE instantiations.  A producer hands every
32-surfel step that has an associated lane to its consumer as one slot (lane L's record at position L, an associated-lane mask in
the header) and hands a sub-item's last slot over only once the sub-item has ended, also when its last steps have no associated
lane.  Here the associated lanes of each 256-surfel chunk are placed on purpose: only the first step, only the last step, only
lane 0 or only lane 31 of one step, none, or all.

The surfels are copies of one surfel, so that they share one Morton key and the (stable) spatial sort keeps the order they are
given in; a copy with its normal flipped is back-facing to the keyframes that associate the surfel: in the image, not
associated.  Counts must equal the CPU oracle's and the non-PRE instantiation's exactly, H agree with both and b with the non-PRE
one within the pose tolerances, and the deterministic mode gives the same bits in two runs and at keyframe groups of 8 and 32.
"""
import copy

import numpy as np
import pytest

from gpu_checks import REL, rel
from test_gpu_deterministic_values import in_mode

pytestmark = pytest.mark.gpu

STEP = 32
CHUNK = 256
NORMAL_ROW = 3   # the packed normal (kRowNormal)
# per chunk: the surfel positions (0..255) that keep the surfel's normal, i.e. associate
PATTERNS = {
    "first step": range(0, STEP),
    "last step": range(CHUNK - STEP, CHUNK),
    "lane 0 of step 3": [3 * STEP],
    "lane 31 of step 4": [4 * STEP + 31],
    "none": [],
    "all": range(CHUNK),
}


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import _lib
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    from oracle import cpu_oracle
    return S, DirectBA, _lib, cpu_oracle


@pytest.fixture(scope="module")
def many():
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name("many"))


def with_columns(sc, cols):
    out = copy.copy(sc)
    n = cols.shape[1]
    out.surfels = np.zeros((sc.surfels.shape[0], max(128, -(-n // 128) * 128)), np.float32)
    out.surfels[:, :n] = cols
    out.num_surfels = n
    return out


def flipped(S, col):
    """The surfel column with its packed normal negated."""
    out = col.copy()
    n = S.unpack_surfel_normal(out[NORMAL_ROW : NORMAL_ROW + 1].view(np.uint32))[0]
    out[NORMAL_ROW] = S.pack_surfel_normal(-n).view(np.float32)
    return out


def pick_surfel(S, O, sc):
    """A surfel column and a keyframe that associates it at poses_init, while its flipped copy lies in that keyframe's image
    without associating."""
    for s in range(0, sc.num_surfels, 211):
        col = sc.surfels[:, s].copy()
        orc, orc_f = O.Oracle(with_columns(sc, col[:, None])), O.Oracle(with_columns(sc, flipped(S, col)[:, None]))
        for k in range(sc.cfg.num_keyframes):
            st, st_f = orc.pose_coeffs(k), orc_f.pose_coeffs(k)
            if st.n_assoc == 1 and st.n_photo == 1 and st_f.n_inimg == 1 and st_f.n_assoc == 0:
                return col, k
    raise AssertionError("no surfel of the scene associates with a keyframe")


@pytest.fixture(scope="module")
def placed(mods, many):
    S, DirectBA, L, O = mods
    col, k = pick_surfel(S, O, many)
    off = flipped(S, col)
    chunks = []
    for keep in PATTERNS.values():
        c = np.repeat(off[:, None], CHUNK, axis=1)
        c[:, list(keep)] = col[:, None]
        chunks.append(c)
    sc = with_columns(many, np.concatenate(chunks, axis=1))
    return sc, k, sum(len(v) for v in PATTERNS.values())


@pytest.mark.parametrize("lname", ["all", "one"])
def test_placed_lanes_against_oracle_and_non_pre(mods, placed, lname):
    """Both PRE instantiations, with and without stats; the one-keyframe list runs 128-surfel sub-items, whose halves of the
    chunks above put the last step of a sub-item, or all of its steps, without associated lanes."""
    S, DirectBA, L, O = mods
    sc, k0, n_assoc = placed
    K = sc.cfg.num_keyframes
    ids = np.arange(K) if lname == "all" else np.array([k0])
    poses = sc.poses_init
    orc = O.Oracle(sc)
    ba = DirectBA.from_scene(sc)
    H0, b0, c0, _ = ba.PoseCoeffsBatch(ids, poses[ids], L.POSE_VARIANT_256, with_stats=True)
    assert c0[k0][2] == n_assoc, (c0[k0], n_assoc)
    # H against the oracle as in test_gpu_parity.py; not b: every pair here is the same surfel's, so b is one pair's term, whose
    # fp32 rounding the 322 copies do not average out (1.2e-4 of the oracle's on an H100)
    for k in ids:
        st = orc.pose_coeffs(int(k))
        assert tuple(c0[k]) == (st.n_inimg, st.n_depthok, st.n_assoc, st.n_photo), (int(k), c0[k])
        if st.n_assoc:
            assert rel(H0[k], st.H[:]) < REL, (int(k), rel(H0[k], st.H[:]))
    for v in (L.POSE_VARIANT_256_PRE, L.POSE_VARIANT_512_PRE):
        for stats in (True, False):
            H, b, c, _ = ba.PoseCoeffsBatch(ids, poses[ids], v, with_stats=stats)
            for k in ids:
                tag = (lname, int(v), stats, int(k))
                assert tuple(c[k]) == (tuple(c0[k]) if stats else (0, 0, c0[k][2], c0[k][3])), (tag, c[k], c0[k])
                if c0[k][2] == 0:
                    assert not H[k].any() and not b[k].any(), tag
                    continue
                assert rel(H[k], H0[k]) < 1e-5 and rel(b[k], b0[k]) < 1e-5, (tag, rel(H[k], H0[k]), rel(b[k], b0[k]))


def same_bits(a, b):
    return all(np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8)) for x, y in zip(a, b))


def test_placed_lanes_deterministic(mods, placed):
    """Deterministic mode: the same bits in two runs, and at keyframe groups of 8 and 32."""
    S, DirectBA, L, O = mods
    sc, k0, _ = placed
    ids = np.arange(sc.cfg.num_keyframes)
    ba = DirectBA.from_scene(sc)
    try:
        for v in (L.POSE_VARIANT_256_PRE, L.POSE_VARIANT_512_PRE):
            for stats in (True, False):
                runs = []
                for g in (8, 8, 32):
                    ba.DebugSetPoseGroup(g)
                    runs.append(in_mode(ba, True, lambda: ba.PoseCoeffsBatch(ids, sc.poses_init, v, stats)))
                assert runs[0][2][k0][2] > 0
                assert same_bits(runs[0], runs[1]) and same_bits(runs[0], runs[2]), (int(v), stats)
    finally:
        ba.DebugSetPoseGroup(0)
