"""numpy restatement of the randomized-fern place index (DESIGN §3.18, csrc/place_index.cu): the fern generator, the encoding of a
depth + colour image pair, the difference of two codes and the ordering of a query's candidates.  Python integers throughout,
so every value is exact."""
import math

import numpy as np

FERN_SEED = 0x5EED0F3E4B5A11CE   # place_index.cu kPlaceFernSeed
GRID_W, GRID_H = 80, 60
MAX_FERNS = 2048
MAX_MATCHES = 64
INVALID_DEPTH_BIT = 0x8000
MASK64 = (1 << 64) - 1


def splitmix64(i, seed=FERN_SEED):
    """Draw i (0-based) of splitmix64 seeded with `seed`."""
    z = (seed + (i + 1) * 0x9E3779B97F4A7C15) & MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
    return z ^ (z >> 31)


def ferns(num_ferns, min_raw, max_raw):
    """(cells [F, 2] = (cx, cy), thresholds [F, 4] = (t_r, t_g, t_b, t_d)), int32."""
    cells = np.zeros((num_ferns, 2), np.int32)
    thr = np.zeros((num_ferns, 4), np.int32)
    for f in range(num_ferns):
        d = [splitmix64(6 * f + j) for j in range(6)]
        cells[f] = (d[0] % GRID_W, d[1] % GRID_H)
        thr[f] = (d[2] % 256, d[3] % 256, d[4] % 256, min_raw + d[5] % (max_raw - min_raw + 1))
    return cells, thr


def raw_range(min_depth, max_depth, raw_to_float_depth):
    """The options' depth range in raw units: llround(m / raw_to_float_depth) in fp64 (the scale is the config's float)."""
    s = float(np.float32(raw_to_float_depth))
    return int(math.floor(float(min_depth) / s + 0.5)), int(math.floor(float(max_depth) / s + 0.5))


def valid_options(num_ferns, min_raw, max_raw):
    return num_ferns % 8 == 0 and 8 <= num_ferns <= MAX_FERNS and 0 < min_raw <= max_raw <= 0x7FFF


def _integral(a):
    """Summed-area table with a zero row and column in front (int64)."""
    s = np.zeros((a.shape[0] + 1, a.shape[1] + 1), np.int64)
    s[1:, 1:] = a.astype(np.int64).cumsum(0).cumsum(1)
    return s


def _box(sat, x0, x1, y0, y1):
    return sat[y1, x1] - sat[y0, x1] - sat[y1, x0] + sat[y0, x0]


def cell_bounds(c, size, grid):
    return c * size // grid, (c + 1) * size // grid


def encode(depth, color, cells, thr):
    """The code of one image pair: depth u16 [h, w] (raw, 0x8000 = invalid), colour u8 [ch, cw, 4]; returns uint32 [F / 8]."""
    depth = np.asarray(depth).view(np.uint16)
    color = np.asarray(color, np.uint8)
    dh, dw = depth.shape
    ch, cw = color.shape[:2]
    valid = (depth & INVALID_DEPTH_BIT) == 0
    sat_d = _integral(np.where(valid, depth, 0))
    sat_n = _integral(valid)
    sat_c = [_integral(color[..., c]) for c in range(3)]
    F = len(cells)
    words = np.zeros(F // 8, np.uint32)
    for f in range(F):
        cx, cy = int(cells[f, 0]), int(cells[f, 1])
        x0, x1 = cell_bounds(cx, cw, GRID_W)
        y0, y1 = cell_bounds(cy, ch, GRID_H)
        n = (x1 - x0) * (y1 - y0)
        code = 0
        for c in range(3):
            if int(_box(sat_c[c], x0, x1, y0, y1)) > int(thr[f, c]) * n:
                code |= 1 << c
        x0, x1 = cell_bounds(cx, dw, GRID_W)
        y0, y1 = cell_bounds(cy, dh, GRID_H)
        if int(_box(sat_d, x0, x1, y0, y1)) > int(thr[f, 3]) * int(_box(sat_n, x0, x1, y0, y1)):
            code |= 8
        words[f // 8] |= np.uint32(code << (4 * (f % 8)))
    return words


def nibbles(code):
    """The F fern values of a code."""
    code = np.asarray(code, np.uint32)
    return ((code[:, None] >> (4 * np.arange(8, dtype=np.uint32))[None, :]) & 0xF).reshape(-1)


def difference(a, b):
    """The number of ferns whose nibbles differ."""
    return int((nibbles(a) != nibbles(b)).sum())


def query(codes, indexed, code, first, last, exclude, max_matches):
    """The matches of one query: codes [K, F / 8] of the published keyframes, indexed [K] bools, the query code, the range
    [first, last] (clipped to [0, K - 1]), the excluded keyframe (-1: none).  Returns (ids, differences) ordered by (D, id)."""
    K = len(codes)
    cand = [k for k in range(max(first, 0), min(last, K - 1) + 1) if indexed[k] and k != exclude]
    scored = sorted((difference(code, codes[k]), k) for k in cand)[:max_matches]
    return np.array([k for _, k in scored], np.int32), np.array([d for d, _ in scored], np.int32)


def differences_all_pairs(codes):
    """D between every pair of codes [K, F / 8] (vectorised): int32 [K, K]."""
    codes = np.asarray(codes, np.uint32)
    K = len(codes)
    out = np.zeros((K, K), np.int32)
    for k in range(K):
        x = codes ^ codes[k]
        x = (x | (x >> 1) | (x >> 2) | (x >> 3)) & np.uint32(0x11111111)
        out[k] = np.bitwise_count(x).sum(1)
    return out


def query_from_differences(D_row, indexed, first, last, exclude, max_matches):
    """query() given the row of differences of the query against every keyframe."""
    K = len(D_row)
    ks = np.arange(max(first, 0), min(last, K - 1) + 1)
    ks = ks[np.asarray(indexed, bool)[ks] & (ks != exclude)] if len(ks) else ks
    order = np.lexsort((ks, D_row[ks]))[:max_matches]
    return ks[order].astype(np.int32), D_row[ks][order].astype(np.int32)
