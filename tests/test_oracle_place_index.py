"""CPU-only: the randomized-fern place index (DESIGN §3.18) -- bba_host_place_ferns against the oracle's generator, codes of
hand-built images (thresholds on either side, cells without valid depth, ragged cells at 81 x 61 and 151 x 110), the (D, id)
order of a query, refused options, and the recognition property on `small` with the default encoding: a view within
LOOP_MOTIONS of a keyframe differs from it in fewer ferns than the GPU tests' own-keyframe bound and from every other keyframe
in more than their other-keyframe bound."""
import numpy as np
import pytest

import place_index_oracle as O

# tests/test_gpu_loop_verification.py LOOP_MOTIONS
LOOP_MOTIONS = [
    [-0.04, 0.01, 0.00, 0.000, 0.010, -0.005],
    [-0.02, 0.00, 0.01, 0.008, 0.000, 0.004],
    [0.00, -0.01, 0.00, -0.005, 0.006, 0.000],
    [0.02, 0.01, -0.01, 0.004, -0.008, 0.006],
    [0.04, 0.00, 0.01, -0.006, 0.004, -0.008],
    [0.01, -0.02, 0.02, 0.012, -0.010, 0.015],
]
# Of 512 ferns (0.5 - 3.0 m), on `small`: a revisit of a keyframe differs from it in at most OWN_MAX ferns and from every other
# keyframe in at least OTHER_MIN (measured: 74 - 294 and at least 377)
OWN_MAX, OTHER_MIN = 320, 350


def _lib():
    from badslam_b200 import _lib
    return _lib.load()


def host_ferns(F, lo, hi):
    cells = np.zeros((F, 2), np.int32)
    thr = np.zeros((F, 4), np.int32)
    st = _lib().bba_host_place_ferns(F, lo, hi, cells.ctypes.data, thr.ctypes.data)
    return st, cells, thr


@pytest.mark.parametrize("F,lo,hi", [(8, 1, 1), (512, 500, 3000), (512, 1, 0x7FFF), (2048, 2500, 2600), (64, 1000, 1001)])
def test_host_ferns_equal_the_oracle(F, lo, hi):
    st, cells, thr = host_ferns(F, lo, hi)
    assert st == 0
    c, t = O.ferns(F, lo, hi)
    assert np.array_equal(cells, c) and np.array_equal(thr, t)
    assert cells[:, 0].max() < 80 and cells[:, 1].max() < 60 and thr[:, :3].max() < 256
    assert thr[:, 3].min() >= lo and thr[:, 3].max() <= hi


@pytest.mark.parametrize("F,lo,hi", [(0, 500, 3000), (12, 500, 3000), (2056, 500, 3000), (-8, 500, 3000), (512, 0, 3000),
                                     (512, 3000, 500), (512, 500, 0x8000)])
def test_refused_options(F, lo, hi):
    cells = np.full((max(F, 8), 2), 7, np.int32)
    thr = np.full((max(F, 8), 4), 7, np.int32)
    assert _lib().bba_host_place_ferns(F, lo, hi, cells.ctypes.data, thr.ctypes.data) != 0
    assert (cells == 7).all() and (thr == 7).all()
    assert not O.valid_options(F, lo, hi)


def test_raw_range():
    assert O.raw_range(0.5, 3.0, 1e-3) == (500, 3000)
    assert O.raw_range(0.5, 3.0, 1.0 / 5000) == (2500, 15000)
    assert O.raw_range(0.5, 10.0, 1e-3) == (500, 10000)


def _constant_pair(w, h, cw, ch, rgb, d):
    depth = np.full((h, w), d, np.uint16)
    color = np.zeros((ch, cw, 4), np.uint8)
    color[..., :3] = rgb
    color[..., 3] = 99   # luma is not read
    return depth, color


@pytest.mark.parametrize("size", [(80, 60, 80, 60), (81, 61, 81, 61), (151, 110, 81, 61), (320, 240, 151, 110)])
def test_constant_images_on_either_side_of_the_thresholds(size):
    F = 64
    cells, thr = O.ferns(F, 500, 3000)
    # every threshold pair: an image one above and one at the threshold of fern 0's channels gives bits 1 and 0
    for f in range(4):
        for above in (True, False):
            rgb = [int(thr[f, c]) + (1 if above else 0) for c in range(3)]
            if any(v > 255 for v in rgb):
                continue
            depth, color = _constant_pair(*size, rgb, int(thr[f, 3]) + (1 if above else 0))
            code = O.nibbles(O.encode(depth, color, cells, thr))
            assert code[f] == (15 if above else 0), (f, above, code[f])
    # a cell without valid depth has bit 3 clear, whatever the threshold
    depth, color = _constant_pair(*size, [255, 255, 255], 0x8000 | 4000)
    code = O.nibbles(O.encode(depth, color, cells, thr))
    assert (code & 8 == 0).all() and ((code & 7) == np.where(thr[:, :3].max(1) < 255, 7, code & 7)).all()


def test_ragged_cells_sum_exactly():
    """81 x 61 and 151 x 110: the cells have one or two columns / rows; a gradient image's code equals a direct per-cell sum."""
    rng = np.random.default_rng(3)
    F = 256
    cells, thr = O.ferns(F, 1, 0x7FFF)
    for (w, h) in [(81, 61), (151, 110)]:
        depth = rng.integers(0, 0x10000, (h, w)).astype(np.uint16)
        color = rng.integers(0, 256, (h, w, 4)).astype(np.uint8)
        code = O.nibbles(O.encode(depth, color, cells, thr))
        for f in range(F):
            cx, cy = cells[f]
            x0, x1 = cx * w // 80, (cx + 1) * w // 80
            y0, y1 = cy * h // 60, (cy + 1) * h // 60
            assert x1 - x0 in (1, 2) and y1 - y0 in (1, 2)
            box = color[y0:y1, x0:x1].reshape(-1, 4).astype(np.int64)
            d = depth[y0:y1, x0:x1].ravel().astype(np.int64)
            v = d[(d & 0x8000) == 0]
            want = sum(1 << c for c in range(3) if box[:, c].sum() > thr[f, c] * len(box)) | (8 if v.sum() > thr[f, 3] * len(v) else 0)
            assert code[f] == want, f


def test_difference_counts_nibbles():
    a = np.array([0x00000000, 0xFFFFFFFF], np.uint32)
    b = np.array([0x10000001, 0xFFFFFFF0], np.uint32)
    assert O.difference(a, b) == 3
    assert O.difference(a, a) == 0
    assert O.difference(np.zeros(1, np.uint32), np.array([0x88888888], np.uint32)) == 8


def test_query_order_and_ties():
    rng = np.random.default_rng(0)
    K, W = 40, 2
    codes = rng.integers(0, 2 ** 32, (K, W), dtype=np.uint64).astype(np.uint32)
    codes[10] = codes[3]
    codes[30] = codes[3]
    codes[20] = codes[3]
    indexed = np.ones(K, bool)
    indexed[20] = False
    ids, d = O.query(codes, indexed, codes[3], 0, K - 1, -1, 5)
    assert list(ids[:3]) == [3, 10, 30] and list(d[:3]) == [0, 0, 0]
    assert all((d[i], ids[i]) < (d[i + 1], ids[i + 1]) for i in range(len(ids) - 1))
    ids, d = O.query(codes, indexed, codes[3], 0, K - 1, 3, 2)
    assert list(ids) == [10, 30]
    ids, _ = O.query(codes, indexed, codes[3], 11, 8, -1, 5)
    assert len(ids) == 0
    ids, _ = O.query(codes, indexed, codes[3], -5, 100, -1, 64)
    assert len(ids) == K - 1
    D = O.differences_all_pairs(codes)
    assert all(D[a, b] == O.difference(codes[a], codes[b]) for a in range(K) for b in range(K))
    for q in (0, 3, 17):
        for (first, last, m) in [(0, K - 1, 8), (5, 25, 3), (30, 10, 4), (-3, 1000, 64)]:
            a = O.query(codes, indexed, codes[q], first, last, q, m)
            b = O.query_from_differences(D[q], indexed, first, last, q, m)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_recognition_on_small(small_scene):
    from badslam_b200.scene import render_frame, se3_exp, se3_mul
    sc = small_scene
    cells, thr = O.ferns(512, *O.raw_range(0.5, 3.0, sc.cfg.raw_to_float_depth))
    codes = [O.encode(sc.depth[k], sc.color[k], cells, thr) for k in range(len(sc.depth))]
    own, other = [], []
    for base in range(3):
        for m in LOOP_MOTIONS:
            d, _, _, c = render_frame(sc, se3_mul(sc.poses_true[base], se3_exp(m)).astype(np.float32))
            code = O.encode(d, c, cells, thr)
            diffs = [O.difference(code, ck) for ck in codes]
            own.append(diffs[base])
            other.append(min(x for k, x in enumerate(diffs) if k != base))
    print(f"revisits of keyframes 0-2: own keyframe {min(own)}-{max(own)} ferns, other keyframes >= {min(other)} of 512")
    assert max(own) <= OWN_MAX and min(other) >= OTHER_MIN
