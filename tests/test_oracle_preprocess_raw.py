"""CPU-only: the host stages in front of keyframe preprocessing (bad_slam.cc:649-689) that bba_preprocess_raw_frame runs as
stage 0 of the fused kernel.

* the oracle's restatements (oracle/preprocess_raw_oracle.c) of MedianFilterAndDensifyDepthMap (preprocessing.cc:40-85),
  Image::DownscaleUsingMedianWhileExcluding (libvis image.h:1003-1053) and DownscaleToHalfSize (image.h:929-948) against an
  independent numpy restatement (np.sort + the tie rule) and hand-built cases.  The reference's versions are host code on
  libvis::Image, which needs Eigen, so they cannot be built into oracle/_ref: these checks are their anchor;
* the tile program's stage 0 (badslam_b200/csrc/preprocess_tile.cuh), executed on the host by harness_preprocess_raw_frame
  (tests/harness/preprocess_raw_host.cpp), against the oracle's stage 0 followed by its whole-image passes, bit for bit.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from badslam_b200 import scene as S
from oracle import cpu_oracle as O
from oracle import preprocess_raw_oracle as R

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def harness():
    src = os.path.join(HERE, "harness", "preprocess_raw_host.cpp")
    hdr = os.path.join(HERE, "..", "badslam_b200", "csrc", "preprocess_tile.cuh")
    out_dir = os.path.join(HERE, "_build")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, "libpreprocess_raw_host.so")
    if not os.path.exists(so) or max(os.path.getmtime(src), os.path.getmtime(hdr)) > os.path.getmtime(so):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", src, "-o", so])
    return C.CDLL(so)


# -- independent numpy restatements -------------------------------------------------------------------------------------
def np_median(values):
    """Sort, middle value; even count: the lower middle one if strictly closer to the fp32 mean, else the upper one."""
    v = np.sort(np.asarray(values, np.uint16))
    n = v.size
    if n % 2:
        return int(v[n // 2])
    mean = np.float32(v.astype(np.float32).sum(dtype=np.float32)) / np.float32(n)
    lo, hi = np.float32(v[n // 2 - 1]), np.float32(v[n // 2])
    return int(lo) if abs(lo - mean) < abs(hi - mean) else int(hi)


def np_median_densify(img):
    h, w = img.shape
    out = img.copy()
    for y in range(h):
        for x in range(w):
            win = img[max(y - 1, 0):y + 2, max(x - 1, 0):x + 2].ravel()
            nz = win[win != 0]
            if nz.size >= 2:
                out[y, x] = np_median(nz)
    return out


def np_downscale(img, w, h):
    H, W = img.shape
    out = np.zeros((h, w), np.uint16)
    for y in range(h):
        for x in range(w):
            box = img[(H * y) // h:(H * (y + 1)) // h, (W * x) // w:(W * (x + 1)) // w].ravel()
            nz = box[box != 0]
            out[y, x] = np_median(nz) if nz.size else 0
    return out


def np_halve(rgb):
    q = rgb // 4
    return (q[0::2, 0::2].astype(np.int32) + q[0::2, 1::2] + q[1::2, 0::2] + q[1::2, 1::2]).astype(np.uint8)


def sparse_depth(shape, zero_fraction, seed):
    rng = np.random.default_rng(seed)
    d = rng.integers(1, 4000, shape).astype(np.uint16)
    d[rng.random(shape) < zero_fraction] = 0
    return d


# -- the restatements ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("zero_fraction", [0.3, 0.5, 0.7])
def test_median_densify_matches_numpy(zero_fraction):
    img = sparse_depth((37, 53), zero_fraction, seed=int(zero_fraction * 10))
    want = img
    for it in range(3):
        want = np_median_densify(want)
        assert np.array_equal(R.median_filter_and_densify(img, it + 1), want), it


def test_median_densify_hand_built_cases():
    z = np.zeros((5, 5), np.uint16)
    lone = z.copy(); lone[2, 2] = 1234
    out = R.median_filter_and_densify(lone)
    assert out[2, 2] == 1234 and np.count_nonzero(out) == 1          # a lone valid pixel survives, nothing is densified from it
    hole = z.copy(); hole[2, 1] = 100; hole[2, 3] = 200
    out = R.median_filter_and_densify(hole)
    assert out[2, 2] == 200                                            # {100, 200}: mean equidistant -> the upper value
    assert out[1, 2] == 200 and out[3, 2] == 200                       # every pixel seeing both is filled the same way
    assert out[2, 0] == 0 and out[2, 4] == 0                           # a hole that sees one valid value stays a hole
    assert out[2, 1] == 100 and out[2, 3] == 200                       # ... and so does a valid pixel: it keeps its value
    tie = z.copy(); tie[1, 1], tie[1, 2], tie[1, 3], tie[2, 1] = 100, 101, 300, 102
    # window of (2, 2): {100, 101, 300, 102} -> sorted 100 101 102 300, mean 150.75: |101 - mean| > |102 - mean| -> 102
    assert R.median_filter_and_densify(tie)[2, 2] == 102
    low = z.copy(); low[1, 1], low[1, 2], low[1, 3], low[2, 1] = 10, 20, 30, 1000
    # {10, 20, 30, 1000}: mean 265 -> |20 - 265| > |30 - 265| -> 30
    assert R.median_filter_and_densify(low)[2, 2] == 30
    corner = z.copy(); corner[0, 1] = 500; corner[1, 0] = 700
    assert R.median_filter_and_densify(corner)[0, 0] == 700           # the clamped window at the image corner


def test_even_count_tie_rule():
    assert np_median([10, 11, 40, 41]) == 40               # mean 25.5: 14.5 from both middle values -> the upper one
    assert np_median([1, 2, 3, 1000]) == 3                 # mean 251.5: the upper one is closer
    assert np_median([1, 2, 100, 101, 102, 103]) == 100    # mean 68.17: the lower one is strictly closer
    img = np.array([[1, 2, 100], [101, 102, 103]], np.uint16)
    assert R.downscale_depth(img, 1, 1)[0, 0] == 100
    img = np.array([[1, 2, 100], [0, 101, 0]], np.uint16)
    assert R.downscale_depth(img, 1, 1)[0, 0] == 100       # {1, 2, 100, 101}: middle pair (2, 100), both 49 from the mean 51 -> upper


@pytest.mark.parametrize("zero_fraction", [0.3, 0.7])
@pytest.mark.parametrize("src,level", [((739, 458), 1), ((160, 120), 1), ((160, 120), 2), ((160, 120), 3), ((83, 61), 1),
                                       ((84, 62), 2)])
def test_downscale_matches_numpy(src, level, zero_fraction):
    W, H = src
    w, h = R.scaled_size(W, level), R.scaled_size(H, level)
    img = sparse_depth((H, W), zero_fraction, seed=W + level)
    assert np.array_equal(R.downscale_depth(img, w, h), np_downscale(img, w, h))


def test_downscale_box_mapping_and_hand_built_boxes():
    # 739 -> 370 and 458 -> 229 (Camera::Scaled(0.5)): boxes of 1 and 2 pixels, from the reference's integer mapping
    assert (R.scaled_size(739, 1), R.scaled_size(458, 1)) == (370, 229)
    starts = [(739 * x) // 370 for x in range(371)]
    widths = np.diff(starts)
    assert set(widths) == {1, 2} and widths.sum() == 739 and widths[0] == 1 and widths[-1] == 2
    ramp = np.tile(np.arange(1, 740, dtype=np.uint16), (458, 1))
    out = R.downscale_depth(ramp, 370, 229)
    # a 1-pixel-wide box is its own value; a 2-pixel one is {a, a + 1}: mean equidistant -> the upper value
    for x in range(370):
        a, b = starts[x], starts[x + 1]
        assert out[0, x] == (a + 1 if b - a == 1 else a + 2), x
    img = np.array([[0, 0, 7, 0], [0, 0, 0, 0]], np.uint16)            # boxes with 0 and 1 valid value
    assert list(R.downscale_depth(img, 2, 1)[0]) == [0, 7]
    img = np.array([[100, 200], [0, 0]], np.uint16)
    assert R.downscale_depth(img, 1, 1)[0, 0] == 200                   # even count, equidistant: upper


def test_color_halving_follows_the_libvis_test_with_u8_truncation():
    # libvis/src/libvis/test/image.cc:136-150 (float: 1.5, 2.5, 5, 5), here u8 with a/4 + b/4 + c/4 + d/4
    data = np.array([[1, 1, 2, 2], [2, 2, 3, 3], [4, 4, 5, 5], [6, 6, 5, 5]], np.uint8)
    rgb = np.repeat(data[..., None], 3, axis=2)
    got = R.downscale_color(rgb, 1)
    assert np.array_equal(got[..., 0], np.array([[0, 0], [4, 4]], np.uint8))      # every quarter truncates: 1/4 = 0, 6/4 = 1
    # the same image x 40 (every value a multiple of 4): no truncation, the libvis test's result x 40
    scaled = np.repeat((data.astype(np.int32) * 40)[..., None], 3, axis=2).astype(np.uint8)
    assert np.array_equal(R.downscale_color(scaled, 1)[..., 1], np.array([[60, 100], [200, 200]], np.uint8))
    # level 2 halves twice: a constant 3 becomes 0, which one 4x4 average (3) does not give
    assert np.all(R.downscale_color(np.full((4, 4, 3), 3, np.uint8), 2) == 0)
    assert np.all(np.full((4, 4), 3).mean() == 3)
    rng = np.random.default_rng(3)
    rgb = rng.integers(0, 256, (64, 96, 3), dtype=np.uint8)
    assert np.array_equal(R.downscale_color(rgb, 2), np_halve(np_halve(rgb)))
    with pytest.raises(ValueError):
        R.downscale_color(rng.integers(0, 256, (6, 10, 3), dtype=np.uint8), 2)   # 5x3 at the second level


# -- the tile program's stage 0 against the oracle -----------------------------------------------------------------------
def run_raw_harness(lib, sc, orc, raw, rgb, n=0, ld=0, lc=0, sigma_xy=1.5, sigma_inv=0.005, radius_factor=2.0, max_depth=3.0):
    m = orc.model
    w, h = m.depth_w, m.depth_h
    cw, ch = m.color_w, m.color_h
    depth, normals, radius = (np.zeros((h, w), np.uint16) for _ in range(3))
    rgba = np.zeros((ch, cw, 4), np.uint8)
    mm = np.zeros(2, np.float32)
    K = (C.c_float * 4)(*[float(v) for v in sc.depth_K])
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    raw = np.ascontiguousarray(raw, np.uint16)
    rgb = np.ascontiguousarray(rgb, np.uint8)
    assert rgb.shape == (ch << lc, cw << lc, 3)
    tiles = lib.harness_preprocess_raw_frame(
        C.c_int(w), C.c_int(h), K, C.c_float(m.raw_to_float_depth), C.c_float(m.a), C.c_int(m.cell), C.c_int(m.cf_w),
        p(orc.cfactor, C.c_float), C.c_float(sigma_xy), C.c_float(sigma_inv), C.c_float(radius_factor), C.c_float(max_depth),
        C.c_int(n), C.c_int(ld), C.c_int(lc), C.c_int(raw.shape[1]), C.c_int(raw.shape[0]),
        p(raw, C.c_uint16), p(depth, C.c_uint16), p(normals, C.c_uint16), p(radius, C.c_uint16),
        C.c_int(cw), C.c_int(ch), p(rgb, C.c_uint8), p(rgba, C.c_uint8), p(mm, C.c_float))
    assert tiles == -(-w // 32) * -(-h // 32)
    return depth, normals, radius, rgba, float(mm[0]), float(mm[1])


def oracle_raw(orc, raw, rgb, n=0, ld=0, lc=0, **kw):
    m = orc.model
    d0, c0 = R.raw_frame_stage0(raw, rgb, (m.depth_w, m.depth_h), n, ld, lc)
    return orc.preprocess_frame(d0, c0, **kw)


def assert_identical(got, want, what):
    gd, gn, gr, gc, gmin, gmax = got
    wd, wn, wr, wc, wmin, wmax = want
    valid = (wd & 0x8000) == 0
    assert np.array_equal(gd, wd), what
    assert np.array_equal(gn, wn), what
    assert np.array_equal(gr[valid], wr[valid]) and np.all(gr[~valid] == 0), what
    assert gmin == wmin and gmax == wmax, what
    assert np.array_equal(gc[..., :3], wc[..., :3]), what
    dl = np.abs(gc[..., 3].astype(np.int32) - wc[..., 3].astype(np.int32))
    assert dl.max() <= 1 and np.mean(dl != 0) < 1e-2, what      # FMA contraction of the luma (oracle) vs none (host build)
    return valid


def upscaled(raw, rgb, level, seed):
    """A 2^level x larger frame whose boxes hold 0 - 2^(2 level) distinct values (rendered frames upsampled + fresh noise)."""
    rng = np.random.default_rng(seed)
    f = 1 << level
    big = np.repeat(np.repeat(raw, f, 0), f, 1).astype(np.int32)
    big = np.where(big > 0, big + rng.integers(-3, 4, big.shape), 0)
    big[rng.random(big.shape) < 0.3] = 0
    crgb = np.repeat(np.repeat(rgb, f, 0), f, 1).astype(np.int32) + rng.integers(0, 4, (rgb.shape[0] * f, rgb.shape[1] * f, 3))
    return np.clip(big, 0, 65535).astype(np.uint16), np.clip(crgb, 0, 255).astype(np.uint8)


@pytest.fixture(scope="module")
def small():
    sc = S.make_scene(S.config_by_name("small"))
    return sc, O.Oracle(sc)


@pytest.mark.parametrize("n", list(range(1, 9)))
def test_tile_program_median_stage_matches_the_oracle(harness, small, n):
    sc, orc = small
    raw, rgb = S.raw_frame(sc, 1)
    rng = np.random.default_rng(n)
    raw[rng.random(raw.shape) < 0.4] = 0                  # holes for the densify filter
    raw[:40, :40] = 0
    sigma_xy = 8.0 if n == 8 else 1.5                      # n = 8 with the largest filter radius (16): the largest halo
    got = run_raw_harness(harness, sc, orc, raw, rgb, n=n, sigma_xy=sigma_xy)
    want = oracle_raw(orc, raw, rgb, n=n, sigma_xy=sigma_xy)
    valid = assert_identical(got, want, n)
    assert valid.mean() > 0.3


@pytest.mark.parametrize("ld,lc", [(1, 1), (2, 2), (3, 3), (1, 0), (0, 2)])
def test_tile_program_pyramid_stage_matches_the_oracle(harness, small, ld, lc):
    sc, orc = small
    raw, rgb = S.raw_frame(sc, 2)
    big = upscaled(raw, rgb, ld, seed=ld)[0] if ld else raw
    _, big_rgb = upscaled(raw, rgb, lc, seed=10 + lc)
    got = run_raw_harness(harness, sc, orc, big, big_rgb, ld=ld, lc=lc)
    want = oracle_raw(orc, big, big_rgb, ld=ld, lc=lc)
    valid = assert_identical(got, want, (ld, lc))
    assert valid.mean() > 0.3


@pytest.mark.parametrize("W,H,n,ld,lc", [(70, 45, 3, 0, 0), (33, 31, 8, 0, 1), (8, 5, 2, 0, 0), (1, 1, 1, 0, 0),
                                          (139, 97, 0, 1, 1), (141, 99, 0, 1, 0), (65, 33, 0, 1, 0), (71, 47, 0, 2, 0),
                                          (135, 95, 0, 3, 0), (66, 34, 0, 0, 1)])
def test_tile_program_stage0_on_ragged_and_tiny_images(harness, W, H, n, ld, lc):
    """Sizes that are not multiples of the tile, where tiles' grown halos and boxes cross the image edge."""
    w, h = R.scaled_size(W, ld), R.scaled_size(H, ld)
    assert W <= w << ld and H <= h << ld
    sc = S.blank_scene(w, h)
    orc = O.Oracle(sc)
    raw, _ = S.random_raw_frame(W, H, seed=W * 100 + H, hole_fraction=0.4)
    _, rgb = S.random_raw_frame(w << lc, h << lc, seed=W + H)
    got = run_raw_harness(harness, sc, orc, raw, rgb, n=n, ld=ld, lc=lc)
    want = oracle_raw(orc, raw, rgb, n=n, ld=ld, lc=lc)
    assert_identical(got, want, (W, H, n, ld, lc))


def test_tile_program_stage0_is_clean_under_address_sanitizer(tmp_path):
    """Every global / shared-memory index of stage 0 (grown halo, ping-pong buffers, box reads of the full-resolution depth,
    colour blocks) on ragged sizes, all median counts / levels and filter radii 0 / 3 / 16, with exactly sized buffers."""
    exe = str(tmp_path / "asan_raw_test")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-omit-frame-pointer", "-x", "c++",
           os.path.join(HERE, "harness", "preprocess_raw_host.cpp"), os.path.join(HERE, "harness", "preprocess_raw_asan_main.cpp"),
           "-o", exe]
    built = subprocess.run(cmd, capture_output=True, text=True)
    if built.returncode != 0:
        pytest.skip("no sanitizer runtime for this g++: " + built.stderr[-200:])
    run = subprocess.run([exe], capture_output=True, text=True, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
    assert run.returncode == 0 and "runtime error" not in run.stderr and "AddressSanitizer" not in run.stderr, run.stderr[-2000:]
    assert "70x45 -> 9x6 n 0 depth level 3 colour level 3 sigma 8.0: 1 tiles" in run.stdout
    assert "139x97 -> 139x97 n 8 depth level 0 colour level 0 sigma 8.0: 20 tiles" in run.stdout


def test_cpp_adaptor_raw_frame_overload_compiles(tmp_path):
    """include/badba_direct_ba.hpp: the PreprocessFrame overload with BadSlamConfig's median / pyramid options compiles and
    links against the library next to the existing one."""
    import shutil
    gxx = shutil.which("g++")
    if gxx is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("no host compiler / CUDA headers")
    root = os.path.dirname(HERE)
    src = tmp_path / "adaptor_raw.cpp"
    src.write_text(r'''
#include "badba_direct_ba.hpp"
struct SE3 { float d[7]; float* data() { return d; } const float* data() const { return d; } };
struct Cam { int w, h; float p[4]; int width() const { return w; } int height() const { return h; } const float* parameters() const { return p; } };
int main(int argc, char**) {
  Cam c{64, 48, {30, 30, 32, 24}};
  try {
    badba::DirectBA<SE3, Cam> ba(1000, 1e-3f, 40.f, 4, 0.8f, 1, 2, 3, c, c, 0, true, true);
    if (argc > 100) {
      float mn, mx;
      ba.PreprocessFrame(nullptr, 1.5f, 0.005f, 2.f, 3.f, 0, 1, 1, {nullptr, 0}, 128, 96, {nullptr, 0}, 128, 96, {nullptr, 0},
                         {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, &mn, &mx);
      ba.PreprocessFrame(nullptr, 1.5f, 0.005f, 2.f, 3.f, {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, {nullptr, 0},
                         {nullptr, 0}, &mn, &mx);
    }
  }
  catch (const badba::Error& e) { return e.status == BBA_ERR_NO_DEVICE ? 42 : 1; }
  return 0;
}''')
    libdir = os.path.join(root, "badslam_b200")
    subprocess.check_call([gxx, "-std=c++17", "-I", os.path.join(root, "include"), "-I", "/usr/local/cuda/include", str(src), "-o",
                           str(tmp_path / "adaptor_raw"), "-L", libdir, "-lbadba_b200", f"-Wl,-rpath,{libdir}"])
