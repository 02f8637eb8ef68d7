"""CPU: the camera-rig scenes (badslam_b200/scene.py rig_half / rig_same / rig_half1) before they are used to judge the GPU path
(tests/test_gpu_camera_rigs.py).  They are deterministic, their colour images come through the colour camera at its size, the
default scenes are unchanged, and the oracles see what the rigs are for: pairs that lose their descriptor residual to the colour
image bounds, and odometry that converges with colour at half the depth resolution."""
import dataclasses
import os

import numpy as np
import pytest

from badslam_b200 import scene as S
from oracle import cpu_oracle
from oracle import odometry_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RIGS = ["rig_half", "rig_same", "rig_half1"]


def d2c(sc):
    """DepthToColorPixelCorner's affine map (surfel_projection.h) of a scene's two cameras."""
    (fx, fy, cx, cy), (cfx, cfy, ccx, ccy) = [np.asarray(k, np.float32) for k in (sc.depth_K, sc.color_K)]
    return cfx / fx, -cfx * cx / fx + ccx, cfy / fy, -cfy * cy / fy + ccy


@pytest.mark.parametrize("name", RIGS)
def test_rig_scenes_are_deterministic_and_sized_by_their_cameras(name):
    cfg = S.config_by_name(name)
    a, b = S.make_scene(cfg), S.make_scene(cfg)
    for f in ("depth", "normals", "radius", "color", "poses_true", "poses_init", "surfels", "cfactor", "depth_K", "color_K"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    depth_K, color_K, cw, ch = S.camera_rig(cfg)
    K = cfg.num_keyframes
    assert a.depth.shape == (K, cfg.height, cfg.width) and a.color.shape == (K, ch, cw, 4)
    assert np.array_equal(a.depth_K, depth_K) and np.array_equal(a.color_K, color_K)
    fx, fy, cx, cy = a.depth_K
    assert fx != fy and cx != 0.5 * cfg.width - 0.5 and cy != 0.5 * cfg.height - 0.5
    # partial sparse cells: the last cfactor column and row cover fewer pixels than a cell
    assert cfg.width % cfg.cell or cfg.height % cfg.cell or cfg.cell == 1
    assert a.cfactor.shape == ((cfg.height - 1) // cfg.cell + 1, (cfg.width - 1) // cfg.cell + 1)
    assert a.num_surfels > 4000
    # the colour images show the scene (luma of invalid pixels is 0)
    assert (a.color[..., 3] > 0).mean() > 0.5
    # a rendered frame and a raw frame come with colour at the colour camera
    d, n, r, c = S.render_frame(a, a.poses_true[1])
    assert d.shape == (cfg.height, cfg.width) and c.shape == (ch, cw, 4)
    assert np.array_equal(c, a.color[1]) and np.array_equal(n, a.normals[1])
    raw, rgb = S.raw_frame(a, 1)
    assert raw.shape == (cfg.height, cfg.width) and rgb.shape == (ch, cw, 3)
    assert S.raw_frame(a, 1, scale=2)[1].shape == (2 * ch, 2 * cw, 3)


def test_rig_cameras():
    half, same = S.make_scene(S.config_by_name("rig_half")), S.make_scene(S.config_by_name("rig_same"))
    fx, cx, fy, cy = d2c(half)
    assert abs(fx - 0.52) < 1e-6 and abs(fy - 0.52) < 1e-6
    # strips along the depth image's borders map outside the colour image
    ch, cw = half.color.shape[1:3]
    xs = fx * (np.arange(half.cfg.width) + 0.5) + cx
    ys = fy * (np.arange(half.cfg.height) + 0.5) + cy
    assert (xs < 0).any() and (xs.astype(int) >= cw).any() and (ys < 0).any() and (ys.astype(int) >= ch).any()
    assert half.cfactor.shape == (31, 41)
    fx, cx, fy, cy = d2c(same)
    assert abs(fx - 1.06) < 1e-5 and abs(cx) > 1 and same.cfg.cell == 3 and same.cfactor.shape == (37, 51)


@pytest.mark.parametrize("name", ["cfg1", "tiny", "small", "many"])
def test_default_scenes_have_one_symmetric_camera(name):
    cfg = S.config_by_name(name)
    sc = S.make_scene(cfg)
    h, w = cfg.height, cfg.width
    assert np.array_equal(sc.depth_K, np.array([0.5 * h, 0.5 * h, 0.5 * w - 0.5, 0.5 * h - 0.5], np.float32))
    assert np.array_equal(sc.color_K, sc.depth_K) and sc.color.shape[1:3] == (h, w)
    assert S.render_frame(sc, sc.poses_true[0])[3].shape == (h, w, 4) and S.raw_frame(sc, 0)[1].shape == (h, w, 3)
    # the colour camera of a distorted copy (tests/gpu_checks.py::distorted_scene) does not re-render frames
    sc2 = dataclasses.replace(sc, color_K=(sc.color_K * np.float32(1.01)).astype(np.float32))
    assert np.array_equal(S.render_frame(sc2, sc.poses_true[1])[3], S.render_frame(sc, sc.poses_true[1])[3])
    if name == "cfg1":
        g = np.load(os.path.join(GOLDEN, "cfg1.npz"))
        assert abs(float(np.sum(sc.surfels[:3, :sc.num_surfels].astype(np.float64))) - float(g["surfel_checksum"])) < 1e-6


def test_oracle_drops_descriptor_residuals_outside_the_colour_image():
    for name in ("rig_half", "rig_same"):
        sc = S.make_scene(S.config_by_name(name))
        orc = cpu_oracle.Oracle(sc)
        st = [orc.pose_coeffs(k) for k in range(sc.cfg.num_keyframes)]
        assert all(s.n_assoc >= s.n_photo for s in st)
        assert sum(s.n_assoc > s.n_photo for s in st) >= sc.cfg.num_keyframes // 2, name
        # without descriptor residuals the association does not change
        orc_d = cpu_oracle.Oracle(sc, use_descriptor=False)
        assert [s.n_assoc for s in st] == [orc_d.pose_coeffs(k).n_assoc for k in range(sc.cfg.num_keyframes)]
    sc = S.make_scene(S.config_by_name("tiny"))
    orc = cpu_oracle.Oracle(sc)
    assert all(s.n_assoc == s.n_photo for s in (orc.pose_coeffs(k) for k in range(sc.cfg.num_keyframes)))


@pytest.mark.parametrize("use_pyramid_level_0", [True, False])
def test_oracle_odometry_converges_with_half_resolution_colour(use_pyramid_level_0):
    sc = S.make_scene(S.config_by_name("rig_half"))
    true_rel = S.se3_exp([0.02, -0.01, 0.015, 0.01, -0.008, 0.012])
    depth, normals, _, color = S.render_frame(sc, S.se3_mul(sc.poses_true[0], true_rel))
    od = odometry_oracle.Odometry(sc.depth_K, sc.color_K, sc.cfg.raw_to_float_depth, sc.cfg.baseline_fx, sc.cfg.cell, sc.depth_a,
                                  sc.cfactor)
    levels = od.build((sc.depth[0], sc.normals[0], sc.color[0]), (depth, normals, color), num_scales=3,
                      use_pyramid_level_0=use_pyramid_level_0)
    # the level cameras scale the colour camera by 2 / 2^scale (pairwise_frame_tracking.cc:417): level 0 sees the colour camera of
    # the depth resolution
    cam = levels[0]["cam"]
    assert (cam.cw, cam.ch) == (162, 122) and abs(cam.d2c_fx - 1.04) < 1e-6
    assert (levels[1]["cam"].cw, levels[1]["cam"].ch) == (81, 61)
    first = 0 if use_pyramid_level_0 else 1
    assert levels[first]["tracked"][2].shape == levels[first]["base"][2].shape
    ident = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
    est = od.track(ident)[0]
    # With level 0 the tracked frame's colour is read at depth pixel coordinates from the half-resolution image, as in the
    # reference (pairwise_frame_tracking.cc:298, "should be pyramid_level_for_color"): the descriptor residuals of that level
    # compare mismatched images, and the estimate improves less than with one camera.
    assert S.pose_error(est, true_rel)[0] < (0.9 if use_pyramid_level_0 else 0.5) * S.pose_error(ident, true_rel)[0]
