"""ctypes binding of the CPU oracle (oracle/badba_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  Nothing under badslam_b200/ may import this.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libbadba_oracle.so")


def build(force: bool = False) -> str:
    if force or not os.path.exists(_LIB_PATH) or any(
            os.path.getmtime(os.path.join(_HERE, f)) > os.path.getmtime(_LIB_PATH)
            for f in ("badba_oracle.c", "preprocess_oracle.c", "badba_oracle.h", "host_math.h")):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB_PATH


class Model(C.Structure):
    _fields_ = [("depth_w", C.c_int), ("depth_h", C.c_int), ("color_w", C.c_int), ("color_h", C.c_int),
                ("depth_K", C.c_float * 4), ("color_K", C.c_float * 4),
                ("raw_to_float_depth", C.c_float), ("baseline_fx", C.c_float), ("a", C.c_float),
                ("cell", C.c_int), ("cf_w", C.c_int), ("cf_h", C.c_int),
                ("cfactor", C.POINTER(C.c_float)),
                ("use_depth_residuals", C.c_int), ("use_descriptor_residuals", C.c_int)]


class Keyframes(C.Structure):
    _fields_ = [("K", C.c_int),
                ("depth", C.POINTER(C.c_uint16)), ("normals", C.POINTER(C.c_uint16)),
                ("radius", C.POINTER(C.c_uint16)), ("color", C.POINTER(C.c_uint8)),
                ("global_T_frame", C.POINTER(C.c_float)), ("activation", C.POINTER(C.c_int32)),
                ("min_depth", C.POINTER(C.c_float)), ("max_depth", C.POINTER(C.c_float)),
                ("covis", C.POINTER(C.c_uint8))]


class PoseStats(C.Structure):
    _fields_ = [("H", C.c_double * 21), ("b", C.c_double * 6),
                ("n_pair", C.c_uint64), ("n_inimg", C.c_uint64), ("n_depthok", C.c_uint64),
                ("n_assoc", C.c_uint64), ("n_photo", C.c_uint64),
                ("cost_depth", C.c_double), ("cost_desc1", C.c_double), ("cost_desc2", C.c_double)]


class BAOptions(C.Structure):
    _fields_ = [("optimize_depth_intrinsics", C.c_int), ("optimize_color_intrinsics", C.c_int),
                ("do_surfel_updates", C.c_int), ("optimize_poses", C.c_int), ("optimize_geometry", C.c_int),
                ("min_iterations", C.c_int), ("max_iterations", C.c_int),
                ("active_keyframe_window_start", C.c_int), ("active_keyframe_window_end", C.c_int),
                ("max_pose_iterations", C.c_int),
                ("ba_iteration_count", C.c_int), ("last_active_in_ba_iteration", C.POINTER(C.c_int32)),
                ("last_covis_in_ba_iteration", C.POINTER(C.c_int32)), ("surfel_merge_dist_factor", C.c_float),
                ("min_observation_count", C.c_int), ("max_surfels", C.c_uint32)]


class BAResult(C.Structure):
    _fields_ = [("iterations_done", C.c_int), ("converged", C.c_int),
                ("n_assoc", C.c_uint64), ("n_photo", C.c_uint64), ("cost", C.c_double),
                ("pose_iterations_total", C.c_int),
                ("surfels_size", C.c_uint32), ("surfels_created", C.c_uint32), ("surfels_merged", C.c_uint32)]


class PCGOptions(C.Structure):
    _fields_ = [("optimize_poses", C.c_int), ("optimize_geometry", C.c_int), ("optimize_depth_intrinsics", C.c_int),
                ("optimize_color_intrinsics", C.c_int), ("min_iterations", C.c_int), ("max_iterations", C.c_int),
                ("max_inner_iterations", C.c_int), ("gauge_keyframe", C.c_int),
                ("do_surfel_updates", C.c_int), ("increase_ba_iteration_count", C.c_int), ("ba_iteration_count", C.c_int),
                ("last_active_in_ba_iteration", C.POINTER(C.c_int32)), ("last_covis_in_ba_iteration", C.POINTER(C.c_int32)),
                ("surfel_merge_dist_factor", C.c_float), ("min_observation_count", C.c_int), ("max_surfels", C.c_uint32)]


class PCGResult(C.Structure):
    _fields_ = [("iterations_done", C.c_int), ("converged", C.c_int), ("inner_iterations_total", C.c_int),
                ("last_r_norm", C.c_float),
                ("surfels_size", C.c_uint32), ("surfels_created", C.c_uint32), ("surfels_merged", C.c_uint32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_tex_luma.restype = C.c_float
        _lib.orc_tex_luma.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_float]
        _lib.orc_estimate_frame_pose.restype = C.c_int
        _lib.orc_pair_residuals.restype = C.c_int
        _lib.orc_pair_residuals_debug.restype = C.c_int
        _lib.orc_get_max_threads.restype = C.c_int
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class Oracle:
    """Owns host copies of a scene and exposes the oracle's entry points on them."""

    def __init__(self, scene, use_depth=True, use_descriptor=True, poses=None):
        self.lib = lib()
        cfg = scene.cfg
        self.K = cfg.num_keyframes
        self.n = scene.num_surfels
        self.pitch = scene.pitch
        self.cfactor = np.ascontiguousarray(scene.cfactor, np.float32).copy()
        self.depth = np.ascontiguousarray(scene.depth)
        self.normals = np.ascontiguousarray(scene.normals)
        self.radius = np.ascontiguousarray(scene.radius)
        self.color = np.ascontiguousarray(scene.color)
        self.poses = np.ascontiguousarray(scene.poses_init if poses is None else poses, np.float32).copy()
        self.activation = np.zeros(self.K, np.int32)
        self.min_depth = np.ascontiguousarray(scene.min_depth, np.float32)
        self.max_depth = np.ascontiguousarray(scene.max_depth, np.float32)
        self.covis = np.zeros((self.K, self.K), np.uint8)
        self.surfels = np.ascontiguousarray(scene.surfels, np.float32).copy()
        self.active = np.zeros(max(self.surfels.shape[1], 1), np.uint8)   # capacity (surfel creation grows n)
        m = Model()
        m.depth_w, m.depth_h = cfg.width, cfg.height
        m.color_h, m.color_w = scene.color.shape[1:3]
        m.depth_K[:] = [float(v) for v in scene.depth_K]
        m.color_K[:] = [float(v) for v in scene.color_K]
        m.raw_to_float_depth = cfg.raw_to_float_depth
        m.baseline_fx = cfg.baseline_fx
        m.a = scene.depth_a
        m.cell = cfg.cell
        m.cf_h, m.cf_w = self.cfactor.shape
        m.cfactor = _p(self.cfactor, C.c_float)
        m.use_depth_residuals = int(use_depth)
        m.use_descriptor_residuals = int(use_descriptor)
        self.model = m
        k = Keyframes()
        k.K = self.K
        k.depth = _p(self.depth, C.c_uint16)
        k.normals = _p(self.normals, C.c_uint16)
        k.radius = _p(self.radius, C.c_uint16)
        k.color = _p(self.color, C.c_uint8)
        k.global_T_frame = _p(self.poses, C.c_float)
        k.activation = _p(self.activation, C.c_int32)
        k.min_depth = _p(self.min_depth, C.c_float)
        k.max_depth = _p(self.max_depth, C.c_float)
        k.covis = _p(self.covis, C.c_uint8)
        self.kfs = k
        self.lib.orc_compute_covisibility(C.byref(self.model), C.byref(self.kfs))

    # -- helpers
    def frame_T_global(self, pose):
        out = np.zeros(12, np.float32)
        pose = np.ascontiguousarray(pose, np.float32)
        self.lib.orc_frame_T_global(_p(pose, C.c_float), _p(out, C.c_float))
        return out

    def pose_coeffs(self, k, pose=None):
        T = self.frame_T_global(self.poses[k] if pose is None else pose)
        st = PoseStats()
        self.lib.orc_pose_coeffs(C.byref(self.model), C.byref(self.kfs), C.c_int(k), _p(T, C.c_float),
                                 _p(self.surfels, C.c_float), C.c_int(self.pitch), C.c_uint32(self.n), C.byref(st))
        return st

    def estimate_frame_pose(self, k, init=None, max_iterations=30):
        init = np.ascontiguousarray(self.poses[k] if init is None else init, np.float32)
        out = np.zeros(7, np.float32)
        conv = C.c_int(0)
        its = self.lib.orc_estimate_frame_pose(C.byref(self.model), C.byref(self.kfs), C.c_int(k), _p(init, C.c_float),
                                               _p(self.surfels, C.c_float), C.c_int(self.pitch), C.c_uint32(self.n),
                                               _p(out, C.c_float), C.byref(conv), C.c_int(max_iterations))
        return out, its, bool(conv.value)

    def update_activation(self):
        self.lib.orc_update_activation(C.byref(self.model), C.byref(self.kfs), _p(self.surfels, C.c_float),
                                       C.c_int(self.pitch), C.c_uint32(self.n), _p(self.active, C.c_uint8))

    def optimize_geometry_iteration(self):
        self.lib.orc_optimize_geometry_iteration(C.byref(self.model), C.byref(self.kfs), _p(self.surfels, C.c_float),
                                                 C.c_int(self.pitch), C.c_uint32(self.n), _p(self.active, C.c_uint8))

    def optimize_intrinsics(self, depth=True, color=True):
        self.lib.orc_optimize_intrinsics(C.byref(self.model), C.byref(self.kfs), _p(self.surfels, C.c_float),
                                         C.c_int(self.pitch), C.c_uint32(self.n), C.c_int(depth), C.c_int(color))

    min_observation_counts = (1, 2, 3)   # bad_slam_config.h:146,151,158

    def end_tasks(self):
        """PerformBASchemeEndTasks (direct_ba.cc:566-653): delete + radius update + compaction.  Returns the deleted count."""
        K = self.K
        b1, b2, mo = self.min_observation_counts
        min_obs = (b1 if K < 5 else b2) if K < 10 else mo     # direct_ba.h:220-226
        n = C.c_uint32(self.n)
        self.lib.orc_end_tasks.restype = C.c_uint32
        deleted = self.lib.orc_end_tasks(C.byref(self.model), C.byref(self.kfs), _p(self.surfels, C.c_float), C.c_int(self.pitch),
                                         C.byref(n), C.c_int(min_obs))
        self.n = int(n.value)
        return int(deleted)

    def min_observation_count(self):
        K = self.K
        b1, b2, mo = self.min_observation_counts
        return (b1 if K < 5 else b2) if K < 10 else mo     # direct_ba.h:220-226

    def create_surfels_for_keyframe(self, k, filter_new_surfels=True):
        """DirectBA::CreateSurfelsForKeyframe (direct_ba.cc:340-405); returns the number of new surfels."""
        n = C.c_uint32(self.n)
        self.lib.orc_create_surfels_for_keyframe.restype = C.c_uint32
        new = self.lib.orc_create_surfels_for_keyframe(C.byref(self.model), C.byref(self.kfs), C.c_int(k), C.c_int(filter_new_surfels),
                                                       C.c_int(self.min_observation_count()), _p(self.surfels, C.c_float),
                                                       C.c_int(self.pitch), C.byref(n), C.c_uint32(self.pitch))
        self.n = int(n.value)
        return int(new)

    def merge_surfels_for_keyframe(self, k, merge_dist_factor=0.8):
        """DetermineSupportingSurfelsAndMergeSurfelsCUDA (kernel_supporting_surfels.cc:40-118); returns the deleted count."""
        self.lib.orc_merge_surfels_for_keyframe.restype = C.c_uint32
        return int(self.lib.orc_merge_surfels_for_keyframe(C.byref(self.model), C.byref(self.kfs), C.c_int(k), C.c_float(merge_dist_factor),
                                                           _p(self.surfels, C.c_float), C.c_int(self.pitch), C.c_uint32(self.n)))

    def compact_surfels(self, with_active=True):
        self.lib.orc_compact_surfels.restype = C.c_uint32
        self.n = int(self.lib.orc_compact_surfels(_p(self.surfels, C.c_float), C.c_int(self.pitch), C.c_uint32(self.n),
                                                  _p(self.active, C.c_uint8) if with_active else None))
        return self.n

    # -- keyframe preprocessing (preprocess_oracle.c) --------------------------------------------------------------------
    def preprocess_frame(self, raw_depth, rgb, sigma_xy=1.5, sigma_inv_depth=0.005, radius_factor=2.0, max_depth=3.0):
        """BadSlam::PreprocessFrame + min / max depth: (depth, normals, radius, rgba, min_depth, max_depth)."""
        m = self.model
        raw = np.ascontiguousarray(raw_depth, np.uint16)
        assert raw.shape == (m.depth_h, m.depth_w)
        depth, normals, radius = (np.zeros_like(raw) for _ in range(3))
        rgba = None
        if rgb is not None:
            rgb = np.ascontiguousarray(rgb, np.uint8)
            assert rgb.shape == (m.color_h, m.color_w, 3)
            rgba = np.zeros((m.color_h, m.color_w, 4), np.uint8)
        mn, mx = C.c_float(), C.c_float()
        self.lib.orc_preprocess_frame(C.byref(m), C.c_float(sigma_xy), C.c_float(sigma_inv_depth), C.c_float(radius_factor),
                                      C.c_float(max_depth), _p(raw, C.c_uint16), None if rgb is None else _p(rgb, C.c_uint8),
                                      _p(depth, C.c_uint16), _p(normals, C.c_uint16), _p(radius, C.c_uint16),
                                      None if rgba is None else _p(rgba, C.c_uint8), C.byref(mn), C.byref(mx))
        return depth, normals, radius, rgba, mn.value, mx.value

    def bilateral_filter(self, raw_depth, sigma_xy=1.5, sigma_inv_depth=0.005, radius_factor=2.0, max_depth_raw=15000):
        raw = np.ascontiguousarray(raw_depth, np.uint16)
        out = np.zeros_like(raw)
        self.lib.orc_bilateral_filter_and_depth_cutoff(C.c_int(raw.shape[1]), C.c_int(raw.shape[0]), C.c_float(sigma_xy),
                                                       C.c_float(sigma_inv_depth), C.c_float(radius_factor),
                                                       C.c_uint16(max_depth_raw), C.c_float(self.model.raw_to_float_depth),
                                                       _p(raw, C.c_uint16), _p(out, C.c_uint16))
        return out

    def compute_normals(self, depth):
        d = np.ascontiguousarray(depth, np.uint16)
        out_d, out_n = np.zeros_like(d), np.zeros_like(d)
        self.lib.orc_compute_normals(C.byref(self.model), _p(d, C.c_uint16), _p(out_d, C.c_uint16), _p(out_n, C.c_uint16))
        return out_d, out_n

    def compute_radii(self, depth):
        d = np.ascontiguousarray(depth, np.uint16)
        rad, out_d = np.zeros_like(d), np.zeros_like(d)
        self.lib.orc_compute_point_radii_and_remove_isolated_pixels(C.byref(self.model), _p(d, C.c_uint16), _p(rad, C.c_uint16),
                                                                    _p(out_d, C.c_uint16))
        return rad, out_d

    def bundle_adjust(self, optimize_poses=True, optimize_geometry=True, min_iterations=1, max_iterations=10,
                      optimize_depth_intrinsics=False, optimize_color_intrinsics=False,
                      window_start=0, window_end=None, max_pose_iterations=30, end_tasks=True, do_surfel_updates=False,
                      surfel_merge_dist_factor=0.8):
        if not hasattr(self, "last_active_in_ba_iteration"):
            self.last_active_in_ba_iteration = np.full(self.K, -1, np.int32)   # keyframe.cc:47-48
            self.last_covis_in_ba_iteration = np.full(self.K, -1, np.int32)
            self.ba_iteration_count = 0
        o = BAOptions(int(optimize_depth_intrinsics), int(optimize_color_intrinsics), int(do_surfel_updates), int(optimize_poses),
                      int(optimize_geometry), min_iterations, max_iterations, window_start,
                      self.K - 1 if window_end is None else window_end, max_pose_iterations,
                      self.ba_iteration_count, _p(self.last_active_in_ba_iteration, C.c_int32),
                      _p(self.last_covis_in_ba_iteration, C.c_int32), float(surfel_merge_dist_factor),
                      self.min_observation_count(), self.pitch)
        r = BAResult()
        self.lib.orc_bundle_adjust(C.byref(self.model), C.byref(self.kfs), _p(self.surfels, C.c_float),
                                   C.c_int(self.pitch), C.c_uint32(self.n), _p(self.active, C.c_uint8),
                                   C.byref(o), C.byref(r))
        self.n = int(r.surfels_size)
        if end_tasks:     # increase_ba_iteration_count = true (direct_ba_alternating.cc:725-735)
            if do_surfel_updates:
                n = C.c_uint32(self.n)
                self.lib.orc_end_tasks_with_merge.restype = C.c_uint32
                self.surfels_deleted = int(self.lib.orc_end_tasks_with_merge(
                    C.byref(self.model), C.byref(self.kfs), _p(self.surfels, C.c_float), C.c_int(self.pitch), C.byref(n),
                    C.c_int(self.min_observation_count()), _p(self.last_active_in_ba_iteration, C.c_int32),
                    C.c_int(self.ba_iteration_count), C.c_float(surfel_merge_dist_factor)))
                self.n = int(n.value)
            else:
                self.surfels_deleted = self.end_tasks()
            self.ba_iteration_count += 1
        return r

    def _lifecycle_state(self):
        if not hasattr(self, "last_active_in_ba_iteration"):
            self.last_active_in_ba_iteration = np.full(self.K, -1, np.int32)   # keyframe.cc:47-48
            self.last_covis_in_ba_iteration = np.full(self.K, -1, np.int32)
            self.ba_iteration_count = 0

    def _pcg_options(self, optimize_poses, optimize_geometry, optimize_depth_intrinsics, optimize_color_intrinsics, min_iterations,
                     max_iterations, max_inner_iterations, gauge_keyframe, do_surfel_updates=False, increase=True,
                     surfel_merge_dist_factor=0.8):
        self._lifecycle_state()
        return PCGOptions(int(optimize_poses), int(optimize_geometry), int(optimize_depth_intrinsics),
                          int(optimize_color_intrinsics), min_iterations, max_iterations, max_inner_iterations, gauge_keyframe,
                          int(do_surfel_updates), int(increase), self.ba_iteration_count,
                          _p(self.last_active_in_ba_iteration, C.c_int32), _p(self.last_covis_in_ba_iteration, C.c_int32),
                          float(surfel_merge_dist_factor), self.min_observation_count(), self.pitch)

    def bundle_adjust_pcg(self, optimize_poses=True, optimize_geometry=True, optimize_depth_intrinsics=False,
                          optimize_color_intrinsics=False, min_iterations=1, max_iterations=1, max_inner_iterations=30,
                          gauge_keyframe=0, end_tasks=True, do_surfel_updates=False, surfel_merge_dist_factor=0.8):
        """DirectBA::BundleAdjustmentPCG; end_tasks = increase_ba_iteration_count (direct_ba_pcg.cc:763-776)."""
        o = self._pcg_options(optimize_poses, optimize_geometry, optimize_depth_intrinsics, optimize_color_intrinsics,
                              min_iterations, max_iterations, max_inner_iterations, gauge_keyframe, do_surfel_updates, end_tasks,
                              surfel_merge_dist_factor)
        r = PCGResult()
        self.lib.orc_bundle_adjust_pcg(C.byref(self.model), C.byref(self.kfs), _p(self.surfels, C.c_float),
                                       C.c_int(self.pitch), C.c_uint32(self.n), _p(self.active, C.c_uint8),
                                       C.byref(o), C.byref(r))
        self.n = int(r.surfels_size)
        if end_tasks:
            if do_surfel_updates:
                n = C.c_uint32(self.n)
                self.lib.orc_end_tasks_with_merge.restype = C.c_uint32
                self.surfels_deleted = int(self.lib.orc_end_tasks_with_merge(
                    C.byref(self.model), C.byref(self.kfs), _p(self.surfels, C.c_float), C.c_int(self.pitch), C.byref(n),
                    C.c_int(self.min_observation_count()), _p(self.last_active_in_ba_iteration, C.c_int32),
                    C.c_int(self.ba_iteration_count), C.c_float(surfel_merge_dist_factor)))
                self.n = int(n.value)
            else:
                self.surfels_deleted = self.end_tasks()
            self.ba_iteration_count += 1
        return r

    def pcg_debug(self, optimize_poses=True, optimize_geometry=True, optimize_depth_intrinsics=False,
                  optimize_color_intrinsics=False, gauge_keyframe=0):
        o = self._pcg_options(optimize_poses, optimize_geometry, optimize_depth_intrinsics, optimize_color_intrinsics, 1, 1, 30,
                              gauge_keyframe)
        self.lib.orc_pcg_debug.restype = C.c_uint32
        args = (C.byref(self.model), C.byref(self.kfs), _p(self.surfels, C.c_float), C.c_int(self.pitch), C.c_uint32(self.n),
                C.byref(o))
        n = self.lib.orc_pcg_debug(*args, None, None, None, None, None)
        r, M, p, g = (np.zeros(n, np.float32) for _ in range(4))
        sc = np.zeros(2, np.float64)
        self.lib.orc_pcg_debug(*args, _p(r, C.c_float), _p(M, C.c_float), _p(p, C.c_float), _p(g, C.c_float), _p(sc, C.c_double))
        return r, M, p, g, sc

    def pair_residuals(self, k, surfel8, pose=None):
        T = self.frame_T_global(self.poses[k] if pose is None else pose)
        s = np.ascontiguousarray(surfel8, np.float32)
        r = np.zeros(3, np.float32)
        Jp = np.zeros(18, np.float32)
        Jg = np.zeros(9, np.float32)
        dbg = np.zeros(16, np.float32)
        flags = self.lib.orc_pair_residuals_debug(C.byref(self.model), C.byref(self.kfs), C.c_int(k), _p(T, C.c_float),
                                                  _p(s, C.c_float), _p(r, C.c_float), _p(Jp, C.c_float), _p(Jg, C.c_float),
                                                  _p(dbg, C.c_float))
        self.last_debug = dbg
        return flags, r, Jp.reshape(3, 6), Jg.reshape(3, 3)

    def tex_luma(self, k, x, y):
        return self.lib.orc_tex_luma(C.byref(self.model), C.byref(self.kfs), C.c_int(k), C.c_float(x), C.c_float(y))


def se3_exp(a):
    a = np.ascontiguousarray(a, np.float32)
    out = np.zeros(7, np.float32)
    lib().orc_se3_exp(_p(a, C.c_float), _p(out, C.c_float))
    return out


def se3_log(T):
    T = np.ascontiguousarray(T, np.float32)
    out = np.zeros(6, np.float32)
    lib().orc_se3_log(_p(T, C.c_float), _p(out, C.c_float))
    return out


def se3_mul(A, B):
    A = np.ascontiguousarray(A, np.float32)
    B = np.ascontiguousarray(B, np.float32)
    out = np.zeros(7, np.float32)
    lib().orc_se3_mul(_p(A, C.c_float), _p(B, C.c_float), _p(out, C.c_float))
    return out


def se3_inverse(A):
    A = np.ascontiguousarray(A, np.float32)
    out = np.zeros(7, np.float32)
    lib().orc_se3_inverse(_p(A, C.c_float), _p(out, C.c_float))
    return out
