"""numpy restatement of the frame overlap measurement (bba_measure_frame_overlap, DESIGN.md §3.20).  Not in the reference; this
oracle is pinned by its own properties (tests/test_oracle_frame_overlap.py) and checks the CUDA kernels
(tests/test_gpu_frame_overlap.py).

A surfel is associated with the frame when stage 3 of the association test (covisibility_oracle.association, the test of surfel
creation's support pass) passes at the query pose, and covers the sparse cell of the pixel it projects to.  A cell is valid when
it holds a valid depth pixel inside the one-pixel border (the rule of scene._create_surfels_for_keyframe and of SeedKernel); its seed
is the valid pixel with the smallest SurfelArrivalKey of its raster index.  An uncovered cell's seed survives the filter
(FilterSeedsKernel) when, counting itself, it is observed by at least min_observation_count keyframes and violates the free space of
no more keyframes than observe it, over the keyframes whose frusta intersect the query's.

The kernels use fast maths, so a decision within rounding of a threshold may go the other way there: near_* bound how far each count
can move by such flips (every surfel within NEAR of a threshold can flip one cell and one association, every seed within NEAR of a
filter threshold one survival).
"""
from __future__ import annotations

import numpy as np

import covisibility_oracle as CO
import surfel_deform_oracle as D

f32 = np.float32
NEAR = CO.NEAR


def arrival_key(index):
    """SurfelArrivalKey: index * 0x9E3779B1 mod 2^32."""
    return (np.asarray(index, np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xffffffff)


def _project(cam, T, p):
    """ProjectIntoImage for the columns of p: (in image [N] bool, px, py)."""
    with np.errstate(all="ignore"):
        lz = T[8] * p[0] + T[9] * p[1] + T[10] * p[2] + T[11]
        lx = T[0] * p[0] + T[1] * p[1] + T[2] * p[2] + T[3]
        ly = T[4] * p[0] + T[5] * p[1] + T[6] * p[2] + T[7]
        inv_z = f32(1) / lz
        pxf = cam.fx * (lx * inv_z) + cam.cx
        pyf = cam.fy * (ly * inv_z) + cam.cy
        ok = (lz > 0) & (pxf >= 0) & (pyf >= 0) & (pxf < cam.w) & (pyf < cam.h)
        return ok, np.where(ok, pxf, 0).astype(np.int64), np.where(ok, pyf, 0).astype(np.int64), lx, ly, lz, pxf, pyf


def seeds(cam, depth):
    """(cell ids [V] of the valid cells, seed x [V], seed y [V])."""
    h, w = depth.shape
    ok = (depth & 0x8000) == 0
    ok[0, :] = ok[-1, :] = False
    ok[:, 0] = ok[:, -1] = False
    ys, xs = np.nonzero(ok)
    cf_w = (w - 1) // cam.cell + 1
    cell = (ys // cam.cell) * cf_w + xs // cam.cell
    key = arrival_key(ys * w + xs)
    order = np.lexsort((key, cell))
    cell, xs, ys = cell[order], xs[order], ys[order]
    first = np.r_[True, cell[1:] != cell[:-1]]
    return cell[first], xs[first], ys[first]


def seed_filter(cam, depth, normals, sx, sy, covis, min_observation_count):
    """(survives [S] bool, margin [S]) of the seed pixels (sx, sy) against covis, a list of (covis_T_frame [12] fp32, depth,
    normals) of the co-visible keyframes (AssociateFreeSpace, device_math.cuh)."""
    cell = (sy // cam.cell) * cam.cfactor.shape[1] + sx // cam.cell
    cf = cam.cfactor.reshape(-1)[cell]
    with np.errstate(all="ignore"):
        inv = f32(1) / (cam.raw_to_float * depth[sy, sx].astype(f32))
        d = f32(1) / (inv + cf * np.exp(-cam.a * inv))
    p_in = np.stack([d * (cam.fx_inv * sx.astype(f32) + cam.cx_inv), d * (cam.fy_inv * sy.astype(f32) + cam.cy_inv), d]).astype(f32)
    nv = normals[sy, sx]
    nx = (nv & 0xff).astype(np.uint8).view(np.int8).astype(f32) * f32(1.0 / 127)
    ny = (nv >> 8).astype(np.uint8).view(np.int8).astype(f32) * f32(1.0 / 127)
    n_in = np.stack([nx, ny, -np.sqrt(np.maximum(f32(1) - nx * nx - ny * ny, f32(0)))])
    S = len(sx)
    obs = np.ones(S, np.int64)
    viol = np.zeros(S, np.int64)
    margin = np.full(S, np.inf)
    frac = lambda v: np.abs(v - np.round(v))
    for R, kd, kn in covis:
        ok, px, py, lx, ly, lz, pxf, pyf = _project(cam, R, p_in)
        margin = np.where(lz > 0, np.minimum(margin, np.minimum(frac(pxf), frac(pyf))), margin)
        with np.errstate(all="ignore"):
            measured = kd[py, px]
            kfn = kn[py, px]
            kcf = cam.cfactor[py // cam.cell, px // cam.cell]
            valid = ok & ((measured & 0x8000) == 0)
            inv_depth = f32(1) / (cam.raw_to_float * measured.astype(f32))
            dk = f32(1) / (inv_depth + kcf * np.exp(-cam.a * inv_depth))
            ln = D._rotate(R, n_in)
            rx = cam.fx_inv * px.astype(f32) + cam.cx_inv
            ry = cam.fy_inv * py.astype(f32) + cam.cy_inv
            thr = D.K_DEPTH_TUKEY * ((D.K_DEPTH_UNCERTAINTY * np.abs(ln[0] * rx + ln[1] * ry + ln[2]) * (dk * dk)) / cam.baseline_fx)
            diff = dk - lz
            facing = lx * ln[0] + ly * ln[1] + lz * ln[2]
            kx = (kfn & 0xff).astype(np.uint8).view(np.int8).astype(f32) * f32(1.0 / 127)
            ky = (kfn >> 8).astype(np.uint8).view(np.int8).astype(f32) * f32(1.0 / 127)
            kz = -np.sqrt(np.maximum(f32(1) - kx * kx - ky * ky, f32(0)))
            compat = ln[0] * kx + ln[1] * ky + ln[2] * kz
            violation = valid & (diff > thr)
            assoc = valid & ~(diff > thr) & ~(diff < -thr) & ~(facing > 0) & ~(compat < D.K_COS_NORMAL)
            lp = np.sqrt(lx * lx + ly * ly + lz * lz)
            m = np.minimum(np.minimum(np.abs(np.abs(diff) - thr) / thr, np.abs(facing) / lp), np.abs(compat - D.K_COS_NORMAL) / D.K_COS_NORMAL)
        margin = np.where(valid, np.minimum(margin, np.where(np.isnan(m), 0.0, m)), margin)
        obs += assoc
        viol += violation
    return (obs >= min_observation_count) & ~(viol > obs), margin


def frame_overlap(cam, depth, normals, frame_T_global, surfels, n, covis, min_observation_count, keyframes=None):
    """The measurement of one query: depth / normals [h, w] u16 of the frame, frame_T_global [7] the inverse of the query pose, covis
    as seed_filter takes it; keyframes (depth list, normals list, frame_T_global [K, 7]) or None for shared.  Returns a dict with
    observed, valid, uncovered, new, shared ([K] int64 or None) and near_observed, near_uncovered, near_new, near_shared ([K])."""
    A, margin = CO.association(cam, [depth], [normals], surfels, n, np.asarray(frame_T_global, f32)[None])
    a, m = A[:, 0], margin[:, 0]
    near = m <= NEAR
    p = np.asarray(surfels, f32)[0:3, :n]
    _, px, py, *_ = _project(cam, D.quat_to_matrix_f32(frame_T_global), p)
    cf_w = (cam.w - 1) // cam.cell + 1
    covered = np.unique(((py // cam.cell) * cf_w + px // cam.cell)[a])
    cells, sx, sy = seeds(cam, depth)
    unc = ~np.isin(cells, covered)
    survives, fmargin = seed_filter(cam, depth, normals, sx[unc], sy[unc], covis, min_observation_count)
    out = dict(observed=int(a.sum()), valid=len(cells), uncovered=int(unc.sum()), new=int(survives.sum()),
               near_observed=int(near.sum()), near_uncovered=int(near.sum()),
               near_new=int(near.sum()) + int((fmargin <= NEAR).sum()), shared=None, near_shared=None)
    if keyframes is not None:
        kd, kn, kT = keyframes
        B, bm = CO.association(cam, kd, kn, surfels, n, np.asarray(kT, f32))
        out["shared"] = (B & a[:, None]).sum(axis=0).astype(np.int64)
        out["near_shared"] = ((bm <= NEAR) | near[:, None]).sum(axis=0).astype(np.int64)
    return out
