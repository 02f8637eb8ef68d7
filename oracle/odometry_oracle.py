"""CPU restatement (numpy, fp32 arithmetic) of the reference's image-pair odometry path.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/make_golden.py.  Nothing under badslam_b200/ may import this.

Follows, function by function:
  BadSlam::RunOdometry                          applications/badslam/src/badslam/bad_slam.cc:829-950
  ComputeBrightnessKernel (texture -> u8)       cuda_image_processing.cu:196-206
  ComputeSobelGradientMagnitudeKernel (texture) cuda_image_processing.cu:103-146
  CalibrateDepthAndTransformColorToDepthCUDA    kernel_downsample.cu:345-372
  CalibrateDepthCUDA                            kernel_downsample.cu:404-426
  CUDABuffer::SetToReadModeNormalized           libvis/src/libvis/cuda/cuda_buffer.cu:82-102
  CalibrateAndDownsampleImagesCUDAKernel        kernel_downsample.cu:40-105
  DownsampleImagesCUDAKernel                    kernel_downsample.cu:107-156
  AccumulatePoseEstimationCoeffsFromImages..._GradientXY / _GradMag   kernel_opt_pose.cu:422-885
  ComputeCostAndResidualCountFromImages...      kernel_opt_pose.cu:939-1296
  TrackFramePairwise                            pairwise_frame_tracking.cc:153-678
  IsScaleNPoseEstimationConverged               convergence_analysis.h:56-63
  PinholeCamera4f::Scaled                       libvis/src/libvis/camera.h:1086-1097,1696-1705
The texture unit is the bit-exact model of badslam_b200.scene.tex_luma (measured, tools/tex_probe.cu).  Pinned by
tests/golden/tiny_odometry.npz (outputs of the reference's own kernels on a B200, tools/make_golden.py --odometry-only).
"""
from __future__ import annotations

import numpy as np

from badslam_b200 import scene as S

f32 = np.float32
INF = f32(np.inf)


def _tex(img_u8, x, y):
    return S.tex_luma(img_u8, x, y)


def brightness(luma_u8, use_gradmag=False):
    """The intensity / gradient-magnitude image RunOdometry derives from a frame's colour texture (.w = luma)."""
    h, w = luma_u8.shape
    xs, ys = np.meshgrid(np.arange(w, dtype=f32), np.arange(h, dtype=f32))
    if not use_gradmag:
        return (f32(255.0) * _tex(luma_u8, xs + f32(0.5), ys + f32(0.5))).astype(np.uint8)   # truncation
    i = {}
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            i[dy, dx] = f32(255.0) * _tex(luma_u8, xs + f32(dx) + f32(0.5), ys + f32(dy) + f32(0.5))
    gx = i[-1, 1] - i[-1, -1] + f32(2) * i[0, 1] - f32(2) * i[0, -1] + i[1, 1] - i[1, -1]
    gy = i[1, -1] - i[-1, -1] + f32(2) * i[1, 0] - f32(2) * i[-1, 0] + i[1, 1] - i[-1, 1]
    norm = f32(255.99) / (f32(np.sqrt(f32(2.0))) * f32(4) * f32(255.0))
    return (norm * np.sqrt(gx * gx + gy * gy, dtype=f32)).astype(np.uint8)


class Camera:
    """One pyramid level's camera pair (surfel_projection.h:42-124 on PinholeCamera4f::Scaled cameras)."""

    def __init__(self, depth_K, color_K, depth_w, color_w, color_h, scale):
        sf = f32(2.0 ** scale)
        df = f32(f32(1.0) / sf)
        cf = f32(f32(1.0) / sf) if depth_w == color_w else f32(f32(2.0) / sf)
        dK = np.asarray(depth_K, f32) * df
        cK = np.asarray(color_K, f32) * cf
        self.fx, self.fy, self.cx, self.cy = [f32(v) for v in dK]
        self.fx_inv, self.fy_inv = f32(1.0) / self.fx, f32(1.0) / self.fy
        self.cx_inv = -(self.cx - f32(0.5)) * self.fx_inv
        self.cy_inv = -(self.cy - f32(0.5)) * self.fy_inv
        self.d2c_fx = cK[0] / dK[0]
        self.d2c_cx = f32(-1) * cK[0] * dK[2] / dK[0] + cK[2]
        self.d2c_fy = cK[1] / dK[1]
        self.d2c_cy = f32(-1) * cK[1] * dK[3] / dK[1] + cK[3]
        self.cw = int(float(cf) * color_w + 0.5)
        self.ch = int(float(cf) * color_h + 0.5)
        self.cfx, self.cfy = f32(cK[0]), f32(cK[1])

    def depth_to_color(self, px, py):
        cx = self.d2c_fx * px + self.d2c_cx
        cy = self.d2c_fy * py + self.d2c_cy
        with np.errstate(invalid="ignore"):
            ok = (cx >= 0) & (cy >= 0) & (cx.astype(np.int64) < self.cw) & (cy.astype(np.int64) < self.ch)
        return cx, cy, ok


def _closest_to_average(depths):
    """depths [4, h, w] with +inf for invalid -> (chosen depth or 0, index or -1)."""
    valid = np.isfinite(depths)
    count = valid.sum(0)
    dsum = np.where(valid, depths, f32(0)).astype(f32)
    total = dsum[0]
    for i in range(1, 4):   # the kernel adds in index order, skipping invalid entries
        total = (total + dsum[i]).astype(f32)
    with np.errstate(invalid="ignore", divide="ignore"):
        avg = (total / count.astype(f32)).astype(f32)
        dist = np.abs(depths - avg[None]).astype(f32)
    closest = np.zeros(count.shape, np.int64)
    best = np.full(count.shape, INF, f32)
    for i in range(4):
        with np.errstate(invalid="ignore"):
            better = dist[i] < best
        closest = np.where(better, i, closest)
        best = np.where(better, dist[i], best)
    chosen = np.take_along_axis(depths, closest[None], 0)[0]
    return np.where(count > 0, chosen, f32(0)).astype(f32), np.where(count > 0, closest, -1)


_OFFSETS = ((0, 0), (0, 1), (1, 0), (1, 1))   # (dy, dx), kernel_downsample.cu:53


def downsample(depth, normals, color):
    """DownsampleImagesCUDAKernel: one pyramid level."""
    h, w = depth.shape[0] // 2, depth.shape[1] // 2
    d4 = np.stack([depth[dy:2 * h:2, dx:2 * w:2] for dy, dx in _OFFSETS]).astype(f32)
    d4 = np.where(d4 > 0, d4, INF)
    out_d, idx = _closest_to_average(d4)
    n4 = np.stack([normals[dy:2 * h:2, dx:2 * w:2] for dy, dx in _OFFSETS])
    out_n = np.take_along_axis(n4, np.maximum(idx, 0)[None], 0)[0]
    out_n = np.where(idx >= 0, out_n, 0).astype(np.uint16)   # (left untouched by the kernel where the depth is invalid)
    xs, ys = np.meshgrid(np.arange(w, dtype=f32), np.arange(h, dtype=f32))
    out_c = (f32(255.0) * _tex(color, f32(2) * xs + f32(1.0), f32(2) * ys + f32(1.0)) + f32(0.5)).astype(np.uint8)
    return out_d, out_n, out_c


class Odometry:
    """RunOdometry + TrackFramePairwise for one (base keyframe, tracked frame) pair."""

    def __init__(self, depth_K, color_K, raw_to_float, baseline_fx, cell, a=0.0, cfactor=None, use_depth=True, use_desc=True):
        self.depth_K, self.color_K = np.asarray(depth_K, f32), np.asarray(color_K, f32)
        self.raw_to_float, self.baseline_fx, self.cell, self.a = f32(raw_to_float), f32(baseline_fx), int(cell), f32(a)
        self.cfactor = cfactor
        self.use_depth, self.use_desc = bool(use_depth), bool(use_desc)

    # ---- inputs ----------------------------------------------------------------------------------------------------------
    def _calibrate(self, raw, cell_y=None, cell_x=None):
        h, w = raw.shape
        ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        cy = (ys if cell_y is None else cell_y) // self.cell
        cx = (xs if cell_x is None else cell_x) // self.cell
        cf = self.cfactor[cy, cx] if self.cfactor is not None else f32(0)
        valid = (raw & 0x8000) == 0
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            d = S.raw_to_calibrated_depth(self.a, cf, self.raw_to_float, np.where(valid, raw, 1))
        return np.where(valid, d, f32(0)).astype(f32), valid

    def build(self, base, tracked, num_scales=5, use_pyramid_level_0=True, use_gradmag=False):
        """base / tracked = (depth u16, normals u16, colour uchar4).  Fills self.levels[scale] = dict(cam, base, tracked) with
        (depth f32, normals u16, colour u8) images."""
        bd, bn, bc = base
        td, tn, tc = tracked
        h, w = bd.shape
        ch, cw = bc.shape[:2]
        self.num_scales, self.first_scale, self.use_gradmag = num_scales, 0 if use_pyramid_level_0 else 1, use_gradmag
        base_gm = brightness(bc[..., 3], use_gradmag)
        trk_gm = brightness(tc[..., 3], use_gradmag)
        # CalibrateDepthAndTransformColorToDepthCUDAKernel (the unscaled DepthToColorPixelCorner of the two cameras)
        depth0, _ = self._calibrate(bd)
        xs, ys = np.meshgrid(np.arange(w, dtype=f32), np.arange(h, dtype=f32))
        d2c_fx = self.color_K[0] / self.depth_K[0]
        d2c_cx = f32(-1) * self.color_K[0] * self.depth_K[2] / self.depth_K[0] + self.color_K[2]
        d2c_fy = self.color_K[1] / self.depth_K[1]
        d2c_cy = f32(-1) * self.color_K[1] * self.depth_K[3] / self.depth_K[1] + self.color_K[3]
        cpx = d2c_fx * (xs + f32(0.5)) + d2c_cx
        cpy = d2c_fy * (ys + f32(0.5)) + d2c_cy
        inb = (cpx >= 0) & (cpy >= 0) & (cpx.astype(np.int64) < cw) & (cpy.astype(np.int64) < ch)
        base0 = (np.where(inb, depth0, f32(0)).astype(f32), bn.copy(), (f32(255.0) * _tex(base_gm, cpx, cpy) + f32(0.5)).astype(np.uint8))
        levels = [dict(cam=Camera(self.depth_K, self.color_K, w, cw, ch, s)) for s in range(num_scales)]
        levels[0]["base"] = base0
        if use_pyramid_level_0:
            d0, _ = self._calibrate(td)
            levels[0]["tracked"] = (d0, tn.copy(), (f32(255.0) * _tex(trk_gm, xs + f32(0.5), ys + f32(0.5))).astype(np.uint8))
        else:
            # CalibrateAndDownsampleImagesCUDAKernel: the cfactor cell is looked up with the DOWNSAMPLED pixel coordinates (:63-65)
            h1, w1 = int(h / 2.0), int(w / 2.0)
            ys1, xs1 = np.meshgrid(np.arange(h1), np.arange(w1), indexing="ij")
            d4 = []
            for dy, dx in _OFFSETS:
                d, valid = self._calibrate(td[dy:2 * h1:2, dx:2 * w1:2], ys1, xs1)
                d4.append(np.where(valid, d, INF))
            out_d, idx = _closest_to_average(np.stack(d4).astype(f32))
            n4 = np.stack([tn[dy:2 * h1:2, dx:2 * w1:2] for dy, dx in _OFFSETS])
            out_n = np.where(idx >= 0, np.take_along_axis(n4, np.maximum(idx, 0)[None], 0)[0], 0).astype(np.uint16)
            x1, y1 = xs1.astype(f32), ys1.astype(f32)
            if w == cw:
                col = _tex(trk_gm, f32(2) * x1 + f32(1.0), f32(2) * y1 + f32(1.0))
            else:
                col = _tex(trk_gm, x1 + f32(0.5), y1 + f32(0.5))
            levels[1]["tracked"] = (out_d, out_n, (f32(255.0) * col + f32(0.5)).astype(np.uint8))
        for s in range(1, num_scales):
            if s >= 2 or use_pyramid_level_0:
                levels[s]["tracked"] = downsample(*levels[s - 1]["tracked"])
            levels[s]["base"] = downsample(*levels[s - 1]["base"])
        self.levels = levels
        return levels

    # ---- per-pixel evaluation ----------------------------------------------------------------------------------------------
    def _eval(self, scale, base_T_frame, jac):
        """All base pixels of a level at one pose: dict(visible, raw_depth, raw1, raw2, Jd, J1, J2) (kernel_opt_pose.cu:442-576)."""
        L = self.levels[scale]
        c = L["cam"]
        bd, bn, bc = L["base"]
        td, tn, tc = L["tracked"]
        h, w = bd.shape
        T = S.se3_matrix(S.se3_inverse(np.asarray(base_T_frame, f32)))[:3].astype(f32)
        tf = f32(2.0 ** scale)
        ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        xf, yf = xs.astype(f32), ys.astype(f32)
        with np.errstate(all="ignore"):
            sd = bd
            ok = sd > 0
            nx0, ny0 = c.fx_inv * xf + c.cx_inv, c.fy_inv * yf + c.cy_inv
            P = np.stack([sd * nx0, sd * ny0, sd])
            lp = (T[:, :3] @ P.reshape(3, -1)).reshape(3, h, w).astype(f32) + T[:, 3, None, None]
            lp = lp.astype(f32)
            ok &= lp[2] > 0
            pxf = c.fx * (lp[0] / lp[2]) + c.cx
            pyf = c.fy * (lp[1] / lp[2]) + c.cy
            px = np.nan_to_num(pxf, nan=-1, posinf=-1, neginf=-1).astype(np.int64)
            py = np.nan_to_num(pyf, nan=-1, posinf=-1, neginf=-1).astype(np.int64)
            ok &= (pxf >= 0) & (pyf >= 0) & (px < w) & (py < h)
            pxc, pyc = np.clip(px, 0, w - 1), np.clip(py, 0, h - 1)
            pd = td[pyc, pxc]
            ok &= pd > 0
            sn = S.u16_to_image_space_normal(bn).astype(f32)           # [h, w, 3]
            ln = np.einsum("ij,hwj->ihw", T[:, :3], sn).astype(f32)
            nx, ny = c.fx_inv * pxc.astype(f32) + c.cx_inv, c.fy_inv * pyc.astype(f32) + c.cy_inv
            proj = np.abs(ln[0] * nx + ln[1] * ny + ln[2])
            stddev = (f32(0.1) * proj * (pd * pd)) / self.baseline_fx
            ok &= ~(np.abs(lp[2] - pd) > (tf * f32(10.0)) * stddev)
            dist = np.sqrt(lp[0] * lp[0] + lp[1] * lp[1] + lp[2] * lp[2])
            ok &= ~((f32(1.0) / dist) * (lp[0] * ln[0] + lp[1] * ln[1] + lp[2] * ln[2]) > 0)
            tnn = S.u16_to_image_space_normal(tn[pyc, pxc]).astype(f32)
            ok &= ~((ln[0] * tnn[..., 0] + ln[1] * tnn[..., 1] + ln[2] * tnn[..., 2]) < f32(0.76604))
            visible = ok.copy()
            out = {}
            if self.use_depth:
                inv_std = self.baseline_fx / (f32(0.1) * proj * (pd * pd))
                up = np.stack([pd * nx, pd * ny, pd])
                out["raw_depth"] = inv_std * (ln[0] * (up[0] - lp[0]) + ln[1] * (up[1] - lp[1]) + ln[2] * (up[2] - lp[2]))
                if jac:
                    out["Jd"] = np.stack([inv_std * ln[0], inv_std * ln[1], inv_std * ln[2],
                                          inv_std * (-ln[1] * up[2] + ln[2] * up[1]),
                                          inv_std * (ln[0] * up[2] - ln[2] * up[0]),
                                          inv_std * (-ln[0] * up[1] + ln[1] * up[0])])
            if self.use_desc:
                def photo_jac(gx, gy):
                    iz = f32(1.0) / lp[2]
                    zz = lp[2] * lp[2]
                    iz2 = iz * iz
                    xy = lp[0] * lp[1]
                    return np.stack([-gx * iz, -gy * iz, (lp[0] * gx + lp[1] * gy) * iz2,
                                     ((lp[1] * lp[1] + zz) * gy + xy * gx) * iz2,
                                     -((lp[0] * lp[0] + zz) * gx + xy * gy) * iz2,
                                     -(lp[0] * gy - lp[1] * gx) * iz])

                def grad(x, y, scale_):
                    ix = np.maximum(f32(0), x - f32(0.5)).astype(np.int64)
                    iy = np.maximum(f32(0), y - f32(0.5)).astype(np.int64)
                    tx = np.clip(x - f32(0.5) - ix.astype(f32), f32(0), f32(1))
                    ty = np.clip(y - f32(0.5) - iy.astype(f32), f32(0), f32(1))
                    fx_, fy_ = ix.astype(f32), iy.astype(f32)
                    tl = scale_ * _tex(tc, fx_ + f32(0.5), fy_ + f32(0.5))
                    tr = scale_ * _tex(tc, fx_ + f32(1.5), fy_ + f32(0.5))
                    bl = scale_ * _tex(tc, fx_ + f32(0.5), fy_ + f32(1.5))
                    br = scale_ * _tex(tc, fx_ + f32(1.5), fy_ + f32(1.5))
                    return ((br - bl) * ty + (tr - tl) * (f32(1) - ty)).astype(f32), ((br - tr) * tx + (bl - tl) * (f32(1) - tx)).astype(f32)

                def safe(v):
                    return np.nan_to_num(v, nan=0.0, posinf=0.0, neginf=0.0).astype(f32)

                if self.use_gradmag:
                    cx, cy, okc = c.depth_to_color(pxf, pyf)
                    visible &= okc
                    cxs, cys = safe(cx), safe(cy)
                    out["raw1"] = f32(255.0) * _tex(tc, cxs, cys) - bc.astype(f32)
                    if jac:
                        gx, gy = grad(cxs, cys, f32(255.0))
                        out["J1"] = photo_jac(gx * c.cfx, gy * c.cfy)
                else:
                    inner = (xs < w - 1) & (ys < h - 1)
                    visible &= inner
                    k255 = f32(1) / f32(255.0)
                    inten = k255 * bc.astype(f32)
                    t1 = k255 * np.roll(bc, -1, axis=1).astype(f32)
                    t2 = k255 * np.roll(bc, -1, axis=0).astype(f32)
                    desc1 = f32(180.0) * (t1 - inten)
                    desc2 = f32(180.0) * (t2 - inten)
                    plane_d = (nx0 * sd) * sn[..., 0] + (ny0 * sd) * sn[..., 1] + sd * sn[..., 2]
                    nx1 = c.fx_inv * (xf + f32(1)) + c.cx_inv
                    ny1 = c.fy_inv * (yf + f32(1)) + c.cy_inv
                    d1 = plane_d / (nx1 * sn[..., 0] + ny0 * sn[..., 1] + sn[..., 2])
                    d2 = plane_d / (nx0 * sn[..., 0] + ny1 * sn[..., 1] + sn[..., 2])

                    def transform(p):
                        return ((T[:, :3] @ p.reshape(3, -1)).reshape(3, h, w) + T[:, 3, None, None]).astype(f32)

                    q1 = transform(np.stack([d1 * nx1, d1 * ny0, d1]).astype(f32))
                    q2 = transform(np.stack([d2 * nx0, d2 * ny1, d2]).astype(f32))
                    t1x, t1y = c.fx * (q1[0] / q1[2]) + c.cx, c.fy * (q1[1] / q1[2]) + c.cy
                    t2x, t2y = c.fx * (q2[0] / q2[2]) + c.cx, c.fy * (q2[1] / q2[2]) + c.cy

                    def inside(x, y):
                        xi = np.nan_to_num(x, nan=-1, posinf=1e9, neginf=-1).astype(np.int64)
                        yi = np.nan_to_num(y, nan=-1, posinf=1e9, neginf=-1).astype(np.int64)
                        return ~((x < 0) | (y < 0) | (xi >= w) | (yi >= h))

                    visible &= inside(t1x, t1y) & inside(t2x, t2y)
                    cx, cy, okc = c.depth_to_color(pxf, pyf)
                    c1x, c1y, ok1 = c.depth_to_color(t1x, t1y)
                    c2x, c2y, ok2 = c.depth_to_color(t2x, t2y)
                    visible &= (q1[2] > 0) & (q2[2] > 0) & okc & ok1 & ok2
                    cx, cy, c1x, c1y, c2x, c2y = [safe(v) for v in (cx, cy, c1x, c1y, c2x, c2y)]
                    ci, i1, i2 = _tex(tc, cx, cy), _tex(tc, c1x, c1y), _tex(tc, c2x, c2y)
                    out["raw1"] = (f32(180.0) * (i1 - ci)) - desc1
                    out["raw2"] = (f32(180.0) * (i2 - ci)) - desc2
                    if jac:
                        cdx, cdy = grad(cx, cy, f32(1))
                        g1x, g1y = grad(c1x, c1y, f32(1))
                        g2x, g2y = grad(c2x, c2y, f32(1))
                        out["J1"] = photo_jac((f32(180.0) * (g1x - cdx)) * c.cfx, (f32(180.0) * (g1y - cdy)) * c.cfy)
                        out["J2"] = photo_jac((f32(180.0) * (g2x - cdx)) * c.cfx, (f32(180.0) * (g2y - cdy)) * c.cfy)
        out["visible"] = visible
        return out

    # robust_weighting.cuh:39-86 with the multi-resolution scaling of cost_function.cuh:91-98,177-185
    @staticmethod
    def _tukey_w(r, p):
        q = r / p
        t = f32(1) - q * q
        return np.where(np.abs(r) < p, t * t, f32(0)).astype(f32)

    @staticmethod
    def _tukey_c(r, p):
        q = r / p
        t = f32(1) - q * q
        return np.where(np.abs(r) < p, (f32(1) / f32(6)) * p * p * (f32(1) - t * t * t), (f32(1) / f32(6)) * p * p).astype(f32)

    @staticmethod
    def _huber_w(r, p):
        a = np.abs(r)
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(a < p, f32(1), p / a).astype(f32)

    @staticmethod
    def _huber_c(r, p):
        a = np.abs(r)
        return np.where(a < p, f32(0.5) * r * r, p * (a - f32(0.5) * p)).astype(f32)

    def coeffs(self, scale, base_T_frame):
        """AccumulatePoseEstimationCoeffsFromImagesCUDA with debug = true: (H[21], b[6], residual_count, residual_sum) in fp64 sums."""
        e = self._eval(scale, base_T_frame, True)
        v = e["visible"]
        tf = f32(2.0 ** scale)
        H, b = np.zeros((6, 6)), np.zeros(6)
        count, total = 0, 0.0
        terms = []
        if self.use_depth:
            r = e["raw_depth"][v]
            terms.append((e["Jd"][:, v], r, self._tukey_w(r, tf * f32(10))))
            count += int(v.sum())
            total += float(self._tukey_c(r, tf * f32(10)).astype(np.float64).sum())
        if self.use_desc:
            r1 = e["raw1"][v]
            terms.append((e["J1"][:, v], r1, tf * f32(1e-2) * self._huber_w(r1, f32(10))))
            if not self.use_gradmag:
                r2 = e["raw2"][v]
                terms.append((e["J2"][:, v], r2, tf * f32(1e-2) * self._huber_w(r2, f32(10))))
            count += int(v.sum())
            total += float((tf * f32(1e-2) * self._huber_c(r1, f32(10))).astype(np.float64).sum())
        for J, r, wgt in terms:
            J64, w64, r64 = J.astype(np.float64), wgt.astype(np.float64), r.astype(np.float64)
            H += (J64 * w64) @ J64.T
            b += J64 @ (w64 * r64)
        return H[np.triu_indices(6)], b, count, total

    def cost(self, scale, base_T_frame):
        """ComputeCostAndResidualCountFromImagesCUDA: (residual_count, cost)."""
        e = self._eval(scale, base_T_frame, False)
        v = e["visible"]
        tf = f32(2.0 ** scale)
        count, total = 0, 0.0
        if self.use_depth:
            count += int(v.sum())
            total += float(self._tukey_c(e["raw_depth"][v], tf * f32(10)).astype(np.float64).sum())
        if self.use_desc:
            n = 1 if self.use_gradmag else 2
            count += n * int(v.sum())
            total += float((tf * f32(1e-2) * self._huber_c(e["raw1"][v], f32(10))).astype(np.float64).sum())
            if not self.use_gradmag:
                total += float((tf * f32(1e-2) * self._huber_c(e["raw2"][v], f32(10))).astype(np.float64).sum())
        return count, total

    def track(self, init1, init2=None, test_different_initial_estimates=True, max_iterations=30):
        """TrackFramePairwise on the built pyramids: (base_T_frame_estimate, iterations per scale, chose_initial per scale)."""
        S_ = self.num_scales
        init1 = np.asarray(init1, f32)
        init2 = init1 if init2 is None else np.asarray(init2, f32)
        est, chosen = init1.copy(), init1.copy()
        iterations, chose = [0] * S_, [-1] * S_
        for scale in range(S_ - 1, self.first_scale - 1, -1):
            sf = f32(2.0 ** scale)
            if scale != S_ - 1 or test_different_initial_estimates:
                last = est if scale != S_ - 1 else init1
                initial = chosen if scale != S_ - 1 else init2
                cl, costl = self.cost(scale, last)
                ci, costi = self.cost(scale, initial)
                if cl > 2 * ci:
                    take_last = True
                elif ci > 2 * cl:
                    take_last = False
                else:
                    take_last = f32(costl) < f32(costi)
                est = (last if take_last else initial).copy()
                chose[scale] = 0 if take_last else 1
                if scale == S_ - 1:
                    chosen = est.copy()
            it = 0
            while it < max_iterations:
                Hu, b, _, _ = self.coeffs(scale, est)
                H = np.zeros((6, 6))
                H[np.triu_indices(6)] = Hu.astype(f32).astype(np.float64)
                H = H + H.T - np.diag(H.diagonal())
                try:
                    x = np.linalg.solve(H, b.astype(f32).astype(np.float64)).astype(f32)
                except np.linalg.LinAlgError:
                    x = np.zeros(6, f32)
                damping = f32(1)
                if scale == S_ - 2:
                    damping = f32(0.5)
                elif scale == S_ - 1:
                    damping = f32(0.25)
                est = S.se3_mul(est, S.se3_exp(-damping * x))
                it += 1
                if f32((x * x).sum()) < sf * sf * f32(1e-08):
                    break
            iterations[scale] = it
        return est, iterations, chose
