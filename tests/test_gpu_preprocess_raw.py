"""GPU: keyframe preprocessing of a frame as the sensor delivers it (bba_preprocess_raw_frame): the median densify filter and the
depth / colour pyramid levels that the reference runs on the host (bad_slam.cc:649-689), as stage 0 of the fused kernel.

Stage 0 is integer-exact, so it is pinned bit for bit without any fast-math tolerance: the CPU oracle's stage 0
(oracle/preprocess_raw_oracle.c) on the host, then the device's bba_preprocess_frame on its result, must equal
bba_preprocess_raw_frame on the raw frame -- depth, normals, radius, rgba, min and max depth.  The CPU suite
(tests/test_oracle_preprocess_raw.py) anchors the oracle's stage 0 to an independent numpy restatement."""
import ctypes as C

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    from oracle import preprocess_raw_oracle
    return S, DirectBA, preprocess_raw_oracle


@pytest.fixture(scope="module")
def scenes(mods):
    S, DirectBA, R = mods
    out = {}
    for name in ("small", "cfg2"):
        sc = S.make_scene(S.config_by_name(name))
        out[name] = (sc, DirectBA.from_scene(sc))
    return out


def dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()


def host(outs):
    import torch
    torch.cuda.synchronize()
    d, n, r, c, mn, mx = outs
    u16 = lambda t: t.view(torch.int16).cpu().numpy().view(np.uint16)
    return u16(d), u16(n), u16(r), None if c is None else c.cpu().numpy(), mn, mx


def assert_bit_identical(got, want, what):
    for i, name in enumerate(("depth", "normals", "radius", "rgba")):
        if want[i] is None:
            assert got[i] is None, (what, name)
            continue
        assert got[i].shape == want[i].shape and np.array_equal(got[i], want[i]), (what, name)
    assert got[4] == want[4] and got[5] == want[5], (what, got[4:], want[4:])


def frame(S, sc, k, scale_depth, scale_color):
    raw, rgb = S.raw_frame(sc, k, scale=scale_depth)
    if scale_color != scale_depth:
        rgb = S.raw_frame(sc, k, scale=scale_color)[1]
    return raw, rgb


# (scene, keyframe, median iterations, depth level, colour level, extra filter options)
CASES = [("small", 0, 1, 0, 0, {}), ("small", 1, 2, 0, 1, {}), ("small", 2, 8, 0, 0, dict(bilateral_filter_sigma_xy=8.0)),
         ("small", 3, 0, 1, 1, {}), ("small", 4, 0, 2, 2, {}), ("small", 5, 0, 3, 0, {}), ("small", 0, 0, 0, 2, {}),
         ("cfg2", 3, 0, 1, 1, {}), ("cfg2", 5, 2, 0, 1, {})]


@pytest.mark.parametrize("name,k,n,ld,lc,opts", CASES)
def test_stage0_is_the_oracle_stage0_followed_by_preprocess_frame(mods, scenes, name, k, n, ld, lc, opts):
    S, DirectBA, R = mods
    sc, ba = scenes[name]
    raw, rgb = frame(S, sc, k, 1 << ld, 1 << lc)
    if n:
        rng = np.random.default_rng(k)
        raw[rng.random(raw.shape) < 0.3] = 0                 # holes for the densify filter to fill
    d0, c0 = R.raw_frame_stage0(raw, rgb, (sc.cfg.width, sc.cfg.height), n, ld, lc)
    want = host(ba.PreprocessFrame(dev(d0), dev(c0), **opts))
    n0 = ba.kernel_launch_count()
    got = host(ba.PreprocessFrame(dev(raw), dev(rgb), median_filter_and_densify_iterations=n, pyramid_level_for_depth=ld,
                                  pyramid_level_for_color=lc, **opts))
    assert ba.kernel_launch_count() - n0 == 2                     # still one fused launch + the min / max initialisation
    assert_bit_identical(got, want, (name, n, ld, lc))
    valid = (got[0] & 0x8000) == 0
    assert valid.mean() > 0.3 and got[4] < got[5]
    # depth only
    got_d = host(ba.PreprocessFrame(dev(raw), None, median_filter_and_densify_iterations=n, pyramid_level_for_depth=ld,
                                    pyramid_level_for_color=lc, **opts))
    assert_bit_identical(got_d[:3] + (None,) + got_d[4:], want[:3] + (None,) + want[4:], (name, n, ld, lc, "depth only"))


def raw_call(ba, raw, rgb, n=0, ld=0, lc=0, raw_size=None, rgb_size=None, out_size=None, color_size=None):
    """bba_preprocess_raw_frame through the C ABI with explicit sizes -> (status, outputs)."""
    import torch
    from badslam_b200 import _lib
    h, w = out_size or (ba.depth_height, ba.depth_width)
    ch, cw = color_size or (ba.color_height, ba.color_width)
    d, nn, r = (torch.zeros((h, w), dtype=torch.int16, device="cuda") for _ in range(3))
    c = torch.zeros((ch, cw, 4), dtype=torch.uint8, device="cuda")
    o = _lib.RawFrameOptions(_lib.PreprocessOptions(1.5, 0.005, 2.0, 3.0), n, ld, lc)
    rh, rw = raw_size or raw.shape
    gh, gw = rgb_size or rgb.shape[:2]
    mn, mx = C.c_float(), C.c_float()
    st = ba._lib.bba_preprocess_raw_frame(ba._h, C.byref(o), raw.data_ptr(), raw.stride(0) * 2, rw, rh, rgb.data_ptr(),
                                          rgb.stride(0), gw, gh, d.data_ptr(), d.stride(0) * 2, nn.data_ptr(), nn.stride(0) * 2,
                                          r.data_ptr(), r.stride(0) * 2, c.data_ptr(), c.stride(0), C.byref(mn), C.byref(mx), None)
    return st, host((d.view(torch.uint16), nn.view(torch.uint16), r.view(torch.uint16), c, mn.value, mx.value))


def test_all_options_zero_is_preprocess_frame(mods, scenes):
    S, DirectBA, R = mods
    sc, ba = scenes["small"]
    raw, rgb = S.raw_frame(sc, 1)
    want = host(ba.PreprocessFrame(dev(raw), dev(rgb)))
    st, got = raw_call(ba, dev(raw), dev(rgb))
    assert st == 0
    assert_bit_identical(got, want, "all options 0")


def test_argument_errors_launch_nothing(mods):
    S, DirectBA, R = mods
    from badslam_b200 import _lib
    sc = S.blank_scene(160, 120)
    ba = DirectBA.from_scene(sc)
    raw1, rgb1 = (dev(a) for a in S.random_raw_frame(160, 120, seed=1))
    raw2, rgb2 = (dev(a) for a in S.random_raw_frame(320, 240, seed=2))
    raw4, rgb4 = (dev(a) for a in S.random_raw_frame(640, 480, seed=4))
    raw_odd, _ = (dev(a) for a in S.random_raw_frame(641, 481, seed=5))
    INV, UNS = _lib.ERR_INVALID_ARGUMENT, _lib.ERR_UNSUPPORTED
    cases = [
        ((raw1, rgb1, 0, 0, 0, (120, 161)), INV),                  # raw depth size is not the depth camera's
        ((raw2, rgb1, 0, 2, 0), INV),                              # 320x240 is level 1 of 160x120, not level 2
        ((raw1, rgb1, 1, 0, 0, (240, 320)), INV),                  # median filter: raw size = camera size
        ((raw1, rgb2, 0, 0, 0), INV),                              # rgb size without a colour level
        ((raw1, rgb1, 0, 0, 1), INV),                              # colour level 1 needs 320x240
        ((raw1, rgb2, 0, 0, 1, None, (239, 320)), INV),            # odd / mismatched colour size at a level
        ((raw1, rgb1, 9, 0, 0), UNS),                              # n > 8
        ((raw2, rgb1, 0, 4, 0), UNS),                              # depth level > 3
        ((raw1, rgb1, 0, 0, 4), UNS),                              # colour level > 3
        ((raw1, rgb1, -1, 0, 0), INV), ((raw1, rgb1, 0, -1, 0), INV), ((raw1, rgb1, 0, 0, -1), INV),
        ((raw2, rgb1, 1, 1, 0), UNS),                              # median filter together with downscaling
        ((raw_odd, rgb1, 0, 2, 0), UNS),                           # 641 = 4 * 160 + 1: a box of 5 pixels
    ]
    for args, status in cases:
        n0 = ba.kernel_launch_count()
        st, _ = raw_call(ba, *args)
        assert st == status, (args[2:], st, ba._lib.bba_last_error(ba._h))
        assert ba.kernel_launch_count() == n0
    raw_call(ba, raw2, rgb1, 1, 1, 0)
    assert b"Simultaneous downscaling and median filtering of depth maps is not implemented." in ba._lib.bba_last_error(ba._h)
    # ... and the valid neighbours of those calls run
    for args in [(raw2, rgb2, 0, 1, 1), (raw4, rgb4, 0, 2, 2), (raw1, rgb4, 8, 0, 2)]:
        st, got = raw_call(ba, *args)
        assert st == 0 and got[0].shape == (120, 160) and got[3].shape == (120, 160, 4)


def test_keyframes_from_2x_raw_frames_feed_bundle_adjustment(mods):
    """Raw frames of a sensor with twice the resolution -> PreprocessFrame at pyramid level 1 (depth and colour) -> AddKeyframe ->
    surfel creation -> BA, with the handle's cameras built from the full-resolution calibration by Scaled(0.5)."""
    import torch
    S, DirectBA, R = mods
    from badslam_b200.direct_ba import PinholeCamera4f
    sc = S.make_scene(S.config_by_name("small"))
    cfg = sc.cfg
    full = PinholeCamera4f(2 * cfg.width, 2 * cfg.height, 2 * np.asarray(sc.depth_K, np.float32))
    cam = full.Scaled(0.5)
    assert (cam.width, cam.height) == (cfg.width, cfg.height) and np.array_equal(cam.parameters, sc.depth_K)
    cap = 1 << 18
    ba = DirectBA(cap, cfg.raw_to_float_depth, cfg.baseline_fx, cfg.cell, color_camera_initial_estimate=cam,
                  depth_camera_initial_estimate=cam, max_keyframes=cfg.num_keyframes)
    surf = torch.zeros((17, cap), dtype=torch.float32, device="cuda")
    ba.SetSurfels(surf, 0)
    created = 0
    for k in range(cfg.num_keyframes):
        raw, rgb = S.raw_frame(sc, k, noise_raw=1.0, scale=2)
        kf = ba.CreateKeyframeFromFrame(k, dev(raw), dev(rgb), sc.poses_init[k], max_depth=6.0, pyramid_level_for_depth=1,
                                        pyramid_level_for_color=1)
        assert kf.depth_buffer.shape == (cfg.height, cfg.width) and kf.color_buffer.shape == (cfg.height, cfg.width, 4)
        assert 0 < kf.min_depth < kf.max_depth <= 6.0
        created += ba.CreateSurfelsForKeyframe(None, True, kf.id)
    assert created > 1000 and ba.surfels_size() == created
    r = ba.BundleAdjustment(None, False, False, False, True, True, 3, 3)
    assert r.iterations_done == 3 and r.depth_residual_count > 0.5 * created
    poses = ba.GetKeyframeStates()[0]
    assert np.all(np.isfinite(poses))

    def rel(P, k):
        return S.se3_mul(S.se3_inverse(P[0]), P[k])
    e_init = max(S.pose_error(rel(sc.poses_init, k), rel(sc.poses_true, k))[0] for k in range(1, cfg.num_keyframes))
    e_ba = max(S.pose_error(rel(poses, k), rel(sc.poses_true, k))[0] for k in range(1, cfg.num_keyframes))
    print(f"relative pose error: {e_init:.2e} m before, {e_ba:.2e} m after 3 BA iterations on 2x raw frames at level 1")
    assert e_ba < 1.5 * e_init + 1e-3
