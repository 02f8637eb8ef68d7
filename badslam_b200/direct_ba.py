"""Host-side mirror of the reference's `DirectBA` / `Keyframe` interface on top of the C ABI.

Same names, argument meaning and error behaviour as
applications/badslam/src/badslam/direct_ba.h:65-550 and keyframe.h:50-237, so the parity tests
read like the reference's own tests (test/test_*_optimization_*.cc).  PyTorch is used only for
device memory and streams; every computation happens inside libbadba_b200.so.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch

from . import _lib
from ._lib import BadBAError


@dataclass
class PinholeCamera4f:
    """libvis PinholeCamera4f (libvis/src/libvis/camera.h:1005-1056): fx, fy, cx, cy in pixel-corner convention."""
    width: int
    height: int
    parameters: np.ndarray

    def __post_init__(self):
        self.parameters = np.asarray(self.parameters, dtype=np.float32).copy()

    def Scaled(self, factor: float) -> "PinholeCamera4f":
        """Camera::Scaled (camera.h:1696-1704, ScaleParameters :1086-1096): the camera of the image resized by `factor`, e.g.
        0.5 ** pyramid_level from a full-resolution calibration (main.cc:457-460).  Size int(factor * size + 0.5); fx, fy, cx,
        cy (pixel-corner convention) times factor in fp32."""
        factor = float(factor)
        return PinholeCamera4f(int(factor * self.width + 0.5), int(factor * self.height + 0.5),
                               self.parameters * np.float32(factor))


def _as_u16(t: torch.Tensor) -> torch.Tensor:
    assert t.dtype in (torch.uint16, torch.int16), t.dtype
    return t


def _frame_buffers(frames):
    """The bba_frame_buffers table of a sequence of (depth, normals, colour) device tensors."""
    bufs = (_lib.FrameBuffers * len(frames))()
    for b, (depth, normals, color) in zip(bufs, frames):
        b.depth, b.depth_pitch = depth.data_ptr(), depth.stride(0) * 2
        b.normals, b.normals_pitch = normals.data_ptr(), normals.stride(0) * 2
        b.color_rgba, b.color_pitch = color.data_ptr(), color.stride(0)
    return bufs


@dataclass
class FrameOverlap:
    """DirectBA.MeasureFrameOverlap's result: per query, the surfels associated with the frame, the sparse cells with a valid
    depth pixel, those no associated surfel falls into, and those whose new surfel would survive the filter (uint32 [n]);
    shared [n, K] uint32 (surfels shared with each keyframe) or None."""
    observed_surfels: np.ndarray
    valid_cells: np.ndarray
    uncovered_cells: np.ndarray
    new_surfels: np.ndarray
    shared: Optional[np.ndarray]


def _odometry_options(num_scales, use_pyramid_level_0, use_gradmag, test_different_initial_estimates, max_iterations_per_scale):
    return _lib.OdometryOptions(int(num_scales), int(use_pyramid_level_0), int(use_gradmag), int(test_different_initial_estimates),
                                int(max_iterations_per_scale))


class Keyframe:
    """Mirror of vis::Keyframe's buffer-taking constructor (keyframe.cc:41-79): owns the device buffers."""

    def __init__(self, frame_index: int, min_depth: float, max_depth: float,
                 depth_buffer: torch.Tensor, normals_buffer: torch.Tensor, radius_buffer: torch.Tensor,
                 color_buffer: torch.Tensor, global_T_frame):
        self.frame_index = frame_index
        self.min_depth = float(min_depth)
        self.max_depth = float(max_depth)
        self.depth_buffer = _as_u16(depth_buffer)          # [h, w] u16
        self.normals_buffer = _as_u16(normals_buffer)      # [h, w] u16
        self.radius_buffer = _as_u16(radius_buffer)        # [h, w] u16
        self.color_buffer = color_buffer                   # [h, w, 4] u8
        self._global_T_frame = np.asarray(global_T_frame, dtype=np.float32).copy()
        self.id = -1
        self._ba: Optional["DirectBA"] = None

    @classmethod
    def from_host(cls, frame_index, depth, normals, radius, color, global_T_frame, min_depth, max_depth, device):
        def up(a, dt):
            return torch.from_numpy(np.ascontiguousarray(a).view(dt)).to(device)
        return cls(frame_index, min_depth, max_depth, up(depth, np.int16).view(torch.uint16),
                   up(normals, np.int16).view(torch.uint16), up(radius, np.int16).view(torch.uint16),
                   torch.from_numpy(np.ascontiguousarray(color)).to(device), global_T_frame)

    def global_T_frame(self) -> np.ndarray:
        if self._ba is not None:
            return self._ba._get_pose(self.id)
        return self._global_T_frame.copy()

    def set_global_T_frame(self, pose):
        self._global_T_frame = np.asarray(pose, dtype=np.float32).copy()
        if self._ba is not None:
            self._ba._set_pose(self.id, self._global_T_frame)

    def activation(self) -> int:
        return self._ba._get_activation(self.id) if self._ba is not None else 0

    def SetActivation(self, activation: int):
        self._ba._set_activation(self.id, activation)


@dataclass
class BAResult:
    iterations_done: int
    converged: bool
    depth_residual_count: int
    descriptor_residual_count: int
    cost: float
    pose_iterations_total: int
    ms_surfel_activation: float
    ms_geometry_optimization: float
    ms_pose_optimization: float
    ms_intrinsics_optimization: float
    kernel_launches: int
    pcg_inner_iterations_total: int = 0
    pcg_last_r_norm: float = 0.0
    ms_pcg: float = 0.0
    surfels_deleted: int = 0
    surfels_size: int = 0
    surfels_created: int = 0
    surfels_merged: int = 0

    @property
    def residual_count(self):
        return self.depth_residual_count + self.descriptor_residual_count


class MotionModel:
    """The constant-motion model BadSlam keeps in front of TrackFramePairwise (base_kf_tr_frame_ / frame_tr_base_kf_,
    bad_slam.cc:542-565, 767-827, 949-954, 1057-1068), on the library's host functions.  One tracked frame of RunOdometry:

        e1, e2 = mm.PredictFramePose()
        estimate, _ = ba.TrackFramePairwise(stream, base_kf_id, depth, normals, color, e1, e2)
        mm.Push(estimate)

    and mm.Rebase() after a keyframe was created from the frame tracked last."""

    def __init__(self, use_motion_model: bool = True):
        self._lib = _lib.load()
        self._m = _lib.MotionModelRecord()
        self.use_motion_model = bool(use_motion_model)
        self.Clear()

    def Clear(self, last_kf_frame_T_global=None, global_T_frame=None):
        """BadSlam::ClearMotionModel: restart from the frame's pose relative to the last keyframe (identity without arguments)."""
        a = None if last_kf_frame_T_global is None else np.ascontiguousarray(last_kf_frame_T_global, np.float32)
        b = None if global_T_frame is None else np.ascontiguousarray(global_T_frame, np.float32)
        self._lib.bba_host_motion_model_clear(C.byref(self._m), None if a is None else a.ctypes.data, None if b is None else b.ctypes.data)

    def PredictFramePose(self):
        """BadSlam::PredictFramePose -> (base_kf_tr_frame_initial_estimate, base_kf_tr_frame_initial_estimate_2)."""
        e1, e2 = np.zeros(7, np.float32), np.zeros(7, np.float32)
        if not self._lib.bba_host_motion_model_predict(C.byref(self._m), int(self.use_motion_model), e1.ctypes.data, e2.ctypes.data):
            raise BadBAError(1, "motion model holds no estimate")
        return e1, e2

    def Push(self, base_T_frame_estimate):
        e = np.ascontiguousarray(base_T_frame_estimate, np.float32)
        self._lib.bba_host_motion_model_push(C.byref(self._m), e.ctypes.data)

    def Rebase(self):
        self._lib.bba_host_motion_model_rebase(C.byref(self._m))

    @property
    def base_kf_tr_frame(self):
        return np.array([list(self._m.base_kf_tr_frame[i]) for i in range(self._m.count)], np.float32).reshape(-1, 7)

    @property
    def frame_tr_base_kf(self):
        return np.array([list(self._m.frame_tr_base_kf[i]) for i in range(self._m.count)], np.float32).reshape(-1, 7)


def deform_trajectory(start_frame: int, end_frame: int, keyframe_frame_indices, original_keyframe_T_global,
                      keyframe_global_T_frame, frame_poses):
    """ExtrapolateAndInterpolateKeyframePoseChanges (trajectory_deformation.cc:45-130) on explicit keyframe poses
    (bba_host_deform_trajectory): the non-keyframe frames in [start_frame, min(end_frame, len(frame_poses) - 1)] of
    frame_poses ([N, 7] global_T_frame) follow the change from original_keyframe_T_global ([K, 7] frame_T_global before the BA
    call) to keyframe_global_T_frame ([K, 7] after it).  frame_poses is updated in place and returned."""
    idx = np.ascontiguousarray(keyframe_frame_indices, np.int32)
    original = np.ascontiguousarray(original_keyframe_T_global, np.float32).reshape(-1, 7)
    current = np.ascontiguousarray(keyframe_global_T_frame, np.float32).reshape(-1, 7)
    if not (len(idx) == len(original) == len(current)):
        raise BadBAError(_lib.ERR_INVALID_ARGUMENT, "one frame index, original and current pose per keyframe")
    if frame_poses.dtype != np.float32 or frame_poses.ndim != 2 or frame_poses.shape[1] != 7 or not frame_poses.flags.c_contiguous:
        raise BadBAError(_lib.ERR_INVALID_ARGUMENT, "frame_poses must be a C-contiguous float32 [N, 7] array (updated in place)")
    end_frame = min(int(end_frame), frame_poses.shape[0] - 1)   # trajectory_deformation.cc:51
    st = _lib.load().bba_host_deform_trajectory(len(idx), idx.ctypes.data, original.ctypes.data, current.ctypes.data,
                                                int(start_frame), end_frame, frame_poses.ctypes.data)
    if st != _lib.OK:
        raise BadBAError(st, "bba_host_deform_trajectory: invalid arguments")
    return frame_poses



def exact_sum(values) -> float:
    """The exact sum of fp32 values rounded once to fp64 (bba_host_exact_sum, the accumulator of the deterministic mode): the
    result does not depend on the order of the values."""
    v = np.ascontiguousarray(values, np.float32).ravel()
    out = C.c_double()
    _lib.load().bba_host_exact_sum(v.ctypes.data, v.size, C.byref(out))
    return out.value

class DirectBA:
    """Drop-in for vis::DirectBA (direct_ba.h:65-550) backed by the sm_90a library."""

    def __init__(self, max_surfel_count: int, raw_to_float_depth: float, baseline_fx: float,
                 sparse_surfel_cell_size: int, surfel_merge_dist_factor: float = 0.8,
                 min_observation_count_while_bootstrapping_1: int = 1,
                 min_observation_count_while_bootstrapping_2: int = 2, min_observation_count: int = 3,
                 color_camera_initial_estimate: PinholeCamera4f = None,
                 depth_camera_initial_estimate: PinholeCamera4f = None, pyramid_level_for_color: int = 0,
                 use_depth_residuals: bool = True, use_descriptor_residuals: bool = True,
                 render_window=None, global_T_anchor_frame=None, *, device=None, max_keyframes: int = 1024,
                 rank: int = 0, world_size: int = 1):
        if not torch.cuda.is_available():
            raise BadBAError(_lib.ERR_NO_DEVICE, "no CUDA device: libbadba_b200 has no CPU fallback")
        self._lib = _lib.load()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.surfel_merge_dist_factor = surfel_merge_dist_factor
        self.min_observation_counts = (min_observation_count_while_bootstrapping_1,
                                       min_observation_count_while_bootstrapping_2, min_observation_count)
        cc, dc = color_camera_initial_estimate, depth_camera_initial_estimate
        cfg = _lib.Config()
        cfg.depth_width, cfg.depth_height = dc.width, dc.height
        cfg.color_width, cfg.color_height = cc.width, cc.height
        cfg.depth_intrinsics[:] = [float(v) for v in dc.parameters]
        cfg.color_intrinsics[:] = [float(v) for v in cc.parameters]
        cfg.raw_to_float_depth = raw_to_float_depth
        cfg.baseline_fx = baseline_fx
        cfg.sparse_surfel_cell_size = int(sparse_surfel_cell_size)
        cfg.max_surfel_count = int(max_surfel_count)
        cfg.max_keyframes = int(max_keyframes)
        cfg.use_depth_residuals = int(use_depth_residuals)
        cfg.use_descriptor_residuals = int(use_descriptor_residuals)
        cfg.device = self.device.index if self.device.index is not None else torch.cuda.current_device()
        cfg.rank, cfg.world_size = rank, world_size
        (cfg.min_observation_count_while_bootstrapping_1, cfg.min_observation_count_while_bootstrapping_2,
         cfg.min_observation_count) = self.min_observation_counts
        cfg.surfel_merge_dist_factor = surfel_merge_dist_factor
        self._cfg = cfg
        self._h = C.c_void_p()
        st = self._lib.bba_create(C.byref(cfg), C.byref(self._h))
        if st != _lib.OK:
            raise BadBAError(st, "bba_create failed")
        self._keyframes: List[Keyframe] = []
        self._surfels: Optional[torch.Tensor] = None
        self._active: Optional[torch.Tensor] = None
        self._allgather_cb = None
        self.depth_width, self.depth_height = dc.width, dc.height
        self.color_width, self.color_height = cc.width, cc.height

    # -- plumbing -------------------------------------------------------------------------------
    def __del__(self):
        try:
            if getattr(self, "_h", None) is not None and self._h.value:
                self._lib.bba_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    def close(self):
        self.__del__()

    def _check(self, st):
        if st != _lib.OK:
            raise BadBAError(st, self._lib.bba_last_error(self._h).decode())

    @staticmethod
    def _stream_ptr(stream):
        if stream is None:
            stream = torch.cuda.current_stream()
        if isinstance(stream, torch.cuda.Stream):
            return C.c_void_p(stream.cuda_stream)
        return C.c_void_p(int(stream))

    def _get_pose(self, kf_id):
        p = np.zeros(7, np.float32)
        self._check(self._lib.bba_get_keyframe_pose(self._h, kf_id, p.ctypes.data_as(C.POINTER(C.c_float))))
        return p

    def _set_pose(self, kf_id, pose):
        p = np.ascontiguousarray(pose, np.float32)
        self._check(self._lib.bba_set_keyframe_pose(self._h, kf_id, p.ctypes.data_as(C.POINTER(C.c_float))))

    def _get_activation(self, kf_id):
        a = C.c_int()
        self._check(self._lib.bba_get_keyframe_activation(self._h, kf_id, C.byref(a)))
        return a.value

    def _set_activation(self, kf_id, a):
        self._check(self._lib.bba_set_keyframe_activation(self._h, kf_id, int(a)))

    # -- scene model (direct_ba.h:95-121, 243-377) ------------------------------------------------
    def AddKeyframe(self, keyframe: Keyframe, stream=None) -> int:
        kf = keyframe
        out = C.c_int(-1)
        pose = np.ascontiguousarray(kf._global_T_frame, np.float32)
        self._check(self._lib.bba_add_keyframe(
            self._h,
            kf.depth_buffer.data_ptr(), kf.depth_buffer.stride(0) * 2,
            kf.normals_buffer.data_ptr(), kf.normals_buffer.stride(0) * 2,
            kf.radius_buffer.data_ptr(), kf.radius_buffer.stride(0) * 2,
            kf.color_buffer.data_ptr(), kf.color_buffer.stride(0),
            pose.ctypes.data_as(C.POINTER(C.c_float)), kf.min_depth, kf.max_depth,
            self._stream_ptr(stream), C.byref(out)))
        kf.id = out.value
        kf._ba = self
        self._keyframes.append(kf)
        return kf.id

    # -- keyframe preprocessing (SURVEY.md 8(f3)) ------------------------------------------------------
    def PreprocessFrame(self, raw_depth: torch.Tensor, rgb: Optional[torch.Tensor] = None, *,
                        bilateral_filter_sigma_xy: float = 1.5, bilateral_filter_sigma_inv_depth: float = 0.005,
                        bilateral_filter_radius_factor: float = 2.0, max_depth: float = 3.0,
                        median_filter_and_densify_iterations: int = 0, pyramid_level_for_depth: int = 0,
                        pyramid_level_for_color: int = 0, want_min_max: bool = True, stream=None):
        """BadSlam::PreprocessFrame (bad_slam.cc:649-765) + ComputeMinMaxDepthCUDA (bad_slam.cc:978) in one kernel launch:
        raw u16 depth (0 = no measurement) and uchar3 colour [.., .., 3] on the device -> (depth, normals, radius, rgba,
        min_depth, max_depth), the buffers Keyframe() / AddKeyframe take.  Defaults: bad_slam_config.h:74-122.
        With every option 0 the images are used as they are (bba_preprocess_frame).  Otherwise (bba_preprocess_raw_frame) the
        depth is median filtered and densified n times, or downscaled from Camera::Scaled(2^L) of the depth camera's size, and
        the colour is level L of the pyramid of an image 2^L times the colour camera's size; the outputs have the cameras' sizes."""
        assert raw_depth.is_cuda and raw_depth.dim() == 2 and raw_depth.element_size() == 2 and raw_depth.stride(1) == 1
        dev = raw_depth.device
        raw_stage = (median_filter_and_densify_iterations, pyramid_level_for_depth, pyramid_level_for_color) != (0, 0, 0)
        h, w = (self.depth_height, self.depth_width) if raw_stage else raw_depth.shape
        depth = torch.empty((h, w), dtype=torch.int16, device=dev)
        normals = torch.empty((h, w), dtype=torch.int16, device=dev)
        radius = torch.empty((h, w), dtype=torch.int16, device=dev)
        rgba = None
        rgb_ptr, rgb_pitch, rgba_ptr, rgba_pitch = None, 0, None, 0
        if rgb is not None:
            assert rgb.is_cuda and rgb.dtype == torch.uint8 and rgb.dim() == 3 and rgb.shape[2] == 3 and rgb.stride(2) == 1 \
                and rgb.stride(1) == 3
            ch, cw = (self.color_height, self.color_width) if raw_stage else rgb.shape[:2]
            rgba = torch.empty((ch, cw, 4), dtype=torch.uint8, device=dev)
            rgb_ptr, rgb_pitch, rgba_ptr, rgba_pitch = rgb.data_ptr(), rgb.stride(0), rgba.data_ptr(), rgba.stride(0)
        opt = _lib.PreprocessOptions(bilateral_filter_sigma_xy, bilateral_filter_sigma_inv_depth,
                                     bilateral_filter_radius_factor, max_depth)
        mn, mx = C.c_float(float("inf")), C.c_float(0.0)
        outputs = (depth.data_ptr(), depth.stride(0) * 2, normals.data_ptr(), normals.stride(0) * 2,
                   radius.data_ptr(), radius.stride(0) * 2, rgba_ptr, rgba_pitch,
                   C.byref(mn) if want_min_max else None, C.byref(mx) if want_min_max else None, self._stream_ptr(stream))
        if raw_stage:
            ropt = _lib.RawFrameOptions(opt, int(median_filter_and_densify_iterations), int(pyramid_level_for_depth),
                                        int(pyramid_level_for_color))
            rgb_h, rgb_w = rgb.shape[:2] if rgb is not None else (0, 0)
            self._check(self._lib.bba_preprocess_raw_frame(
                self._h, C.byref(ropt), raw_depth.data_ptr(), raw_depth.stride(0) * 2, raw_depth.shape[1], raw_depth.shape[0],
                rgb_ptr, rgb_pitch, rgb_w, rgb_h, *outputs))
        else:
            self._check(self._lib.bba_preprocess_frame(
                self._h, C.byref(opt), raw_depth.data_ptr(), raw_depth.stride(0) * 2, rgb_ptr, rgb_pitch, *outputs))
        u16 = lambda a: a.view(torch.uint16)
        return u16(depth), u16(normals), u16(radius), rgba, mn.value, mx.value

    def CreateKeyframeFromFrame(self, frame_index: int, raw_depth: torch.Tensor, rgb: torch.Tensor, global_T_frame,
                                stream=None, **preprocess_options) -> "Keyframe":
        """Preprocesses a raw frame and adds it as a keyframe (BadSlam::CreateKeyframe, bad_slam.cc:957-1010: min / max depth,
        Keyframe(), DirectBA::AddKeyframe)."""
        depth, normals, radius, rgba, mn, mx = self.PreprocessFrame(raw_depth, rgb, stream=stream, **preprocess_options)
        if not (mn > 0.0 and mx >= mn):
            raise BadBAError(_lib.ERR_STATE, "CreateKeyframeFromFrame: the frame has no valid depth (keyframe.cc:57-59 requires min_depth > 0)")
        kf = Keyframe(frame_index, mn, mx, depth, normals, radius, rgba, global_T_frame)
        self.AddKeyframe(kf, stream=stream)
        return kf

    def keyframes(self) -> List[Keyframe]:
        return self._keyframes

    def SetSurfels(self, surfels: torch.Tensor, surfels_size: int, active: Optional[torch.Tensor] = None):
        """surfels_: [17, pitch] float32 CUDA tensor (kernels.cuh:69-93), used in place."""
        assert surfels.is_cuda and surfels.dtype == torch.float32 and surfels.shape[0] == 17
        if active is None:
            active = torch.zeros(max(int(surfels.shape[1]), 1), dtype=torch.uint8, device=surfels.device)
        self._surfels, self._active = surfels, active
        self._check(self._lib.bba_set_surfels(self._h, surfels.data_ptr(), surfels.stride(0) * 4, int(surfels_size)))
        self._check(self._lib.bba_set_active_flags(self._h, active.data_ptr()))

    def SetSurfelsHost(self, surfels: np.ndarray, surfels_size: int, stream=None):
        s = np.ascontiguousarray(surfels, np.float32)
        self._check(self._lib.bba_set_surfels_host(self._h, s.ctypes.data, s.strides[0], int(surfels_size),
                                                   self._stream_ptr(stream)))

    def surfels(self) -> torch.Tensor:
        return self._surfels

    def active_surfels(self) -> torch.Tensor:
        return self._active

    def surfels_size(self) -> int:
        n = C.c_uint32()
        self._check(self._lib.bba_get_surfels_device(self._h, None, None, C.byref(n)))
        return n.value

    def GetSurfelsHost(self, rows: int = 8, stream=None) -> np.ndarray:
        n = self.surfels_size()
        out = np.zeros((rows, max(n, 1)), np.float32)
        self._check(self._lib.bba_get_surfels_host(self._h, out.ctypes.data, out.strides[0], rows, self._stream_ptr(stream)))
        return out[:, :n]

    def GetActiveHost(self, stream=None) -> np.ndarray:
        n = self.surfels_size()
        out = np.zeros(max(n, 1), np.uint8)
        self._check(self._lib.bba_get_active_flags_host(self._h, out.ctypes.data, self._stream_ptr(stream)))
        return out[:n]

    def _intrinsics(self):
        d = (C.c_float * 4)()
        c = (C.c_float * 4)()
        a = C.c_float()
        self._check(self._lib.bba_get_intrinsics(self._h, d, c, C.byref(a)))
        return np.array(d[:], np.float32), np.array(c[:], np.float32), a.value

    def depth_camera(self) -> PinholeCamera4f:
        return PinholeCamera4f(self.depth_width, self.depth_height, self._intrinsics()[0])

    def color_camera(self) -> PinholeCamera4f:
        return PinholeCamera4f(self.color_width, self.color_height, self._intrinsics()[1])

    def a(self) -> float:
        return self._intrinsics()[2]

    def SetColorCamera(self, camera: PinholeCamera4f):
        d, _, a = self._intrinsics()
        self._set_intrinsics(d, camera.parameters, a)

    def SetDepthCamera(self, camera: PinholeCamera4f):
        _, c, a = self._intrinsics()
        self._set_intrinsics(camera.parameters, c, a)

    # direct_ba.h:317-328
    def use_depth_residuals(self) -> bool:
        d, c = C.c_int(), C.c_int()
        self._check(self._lib.bba_get_residual_types(self._h, C.byref(d), C.byref(c)))
        return bool(d.value)

    def use_descriptor_residuals(self) -> bool:
        d, c = C.c_int(), C.c_int()
        self._check(self._lib.bba_get_residual_types(self._h, C.byref(d), C.byref(c)))
        return bool(c.value)

    def SetUseDepthResiduals(self, use_depth_residuals: bool):
        self._check(self._lib.bba_set_residual_types(self._h, int(use_depth_residuals), int(self.use_descriptor_residuals())))

    def SetUseDescriptorResiduals(self, use_descriptor_residuals: bool):
        self._check(self._lib.bba_set_residual_types(self._h, int(self.use_depth_residuals()), int(use_descriptor_residuals)))

    def deterministic(self) -> bool:
        """Whether the deterministic mode is on (the published mode, bba_get_deterministic)."""
        on = C.c_int()
        self._check(self._lib.bba_get_deterministic(self._h, C.byref(on)))
        return bool(on.value)

    def SetDeterministic(self, on: bool):
        """The deterministic mode (bba_set_deterministic): bitwise reproducible bundle adjustment, frame pose estimation and
        odometry on one GPU, from the next call on.  Off by default."""
        self._check(self._lib.bba_set_deterministic(self._h, int(on)))

    def DebugExactSum(self, values: torch.Tensor, stream=None) -> float:
        """Parity hook (bba_debug_exact_sum): the exact sum of a contiguous fp32 device tensor, deposited by many CTAs in a scrambled
        order and rounded to fp64."""
        assert values.dtype == torch.float32 and values.is_cuda and values.is_contiguous()
        out = C.c_double()
        self._check(self._lib.bba_debug_exact_sum(self._h, values.data_ptr(), values.numel(), C.byref(out), self._stream_ptr(stream)))
        return out.value

    def SetA(self, a: float):
        d, c, _ = self._intrinsics()
        self._set_intrinsics(d, c, a)

    def _set_intrinsics(self, d, c, a):
        d = np.ascontiguousarray(d, np.float32)
        c = np.ascontiguousarray(c, np.float32)
        self._check(self._lib.bba_set_intrinsics(self._h, d.ctypes.data_as(C.POINTER(C.c_float)),
                                                 c.ctypes.data_as(C.POINTER(C.c_float)), float(a)))

    def cfactor_buffer(self, stream=None) -> np.ndarray:
        w, h = C.c_int(), C.c_int()
        self._check(self._lib.bba_cfactor_size(self._h, C.byref(w), C.byref(h)))
        out = np.zeros((h.value, w.value), np.float32)
        self._check(self._lib.bba_get_cfactor_host(self._h, out.ctypes.data, self._stream_ptr(stream)))
        return out

    def SetCFactorBuffer(self, cfactor: np.ndarray, stream=None):
        c = np.ascontiguousarray(cfactor, np.float32)
        self._check(self._lib.bba_set_cfactor_host(self._h, c.ctypes.data, self._stream_ptr(stream)))

    def SetKeyframeStates(self, poses=None, activations=None):
        K = len(self._keyframes)
        p = None if poses is None else np.ascontiguousarray(poses, np.float32)
        a = None if activations is None else np.ascontiguousarray(activations, np.int32)
        self._check(self._lib.bba_set_keyframe_states(self._h, K, None if p is None else p.ctypes.data,
                                                      None if a is None else a.ctypes.data))

    def GetKeyframeStates(self):
        K = len(self._keyframes)
        p = np.zeros((K, 7), np.float32)
        a = np.zeros(K, np.int32)
        self._check(self._lib.bba_get_keyframe_states(self._h, K, p.ctypes.data, a.ctypes.data))
        return p, a

    # -- soft pose priors (not in the reference; include/badba.h "Soft pose priors") ----------------------------------------
    def SetKeyframePosePriors(self, ids, poses, information):
        """Anchors keyframes `ids` to prior global_T_frame poses ([n, 7]) with the cost 1/2 r^T L r, r = log(prior^-1 *
        global_T_frame) (translation, then rotation).  information: [n, 21] upper triangles of L, or [n, 6, 6] / [6, 6]
        matrices (one matrix for all).  Refused as a whole (nothing changes) for an unknown id, a non-finite value or an L that
        is not positive semi-definite."""
        ids = np.ascontiguousarray(np.atleast_1d(ids), np.int32)
        n = len(ids)
        p = np.ascontiguousarray(np.asarray(poses, np.float32).reshape(n, 7))
        L = np.asarray(information, np.float32)
        if L.shape[-2:] == (6, 6):
            L = np.broadcast_to(L, (n, 6, 6))[:, np.triu_indices(6)[0], np.triu_indices(6)[1]]
        L = np.ascontiguousarray(np.broadcast_to(L.reshape(-1, 21), (n, 21)), np.float32)
        self._check(self._lib.bba_set_keyframe_pose_priors(self._h, n, ids.ctypes.data, p.ctypes.data, L.ctypes.data))

    def ClearKeyframePosePriors(self, ids=None):
        """Removes the priors of keyframes `ids`, or every prior with ids=None."""
        if ids is None:
            self._check(self._lib.bba_clear_keyframe_pose_priors(self._h, -1, None))
            return
        ids = np.ascontiguousarray(np.atleast_1d(ids), np.int32)
        self._check(self._lib.bba_clear_keyframe_pose_priors(self._h, len(ids), ids.ctypes.data))

    def KeyframePosePrior(self, keyframe_id: int):
        """(prior global_T_frame [7], L upper triangle [21]) of a keyframe as last published, or None without a prior."""
        p, L, has = np.zeros(7, np.float32), np.zeros(21, np.float32), C.c_int()
        self._check(self._lib.bba_get_keyframe_pose_prior(self._h, keyframe_id, p.ctypes.data, L.ctypes.data, C.byref(has)))
        return (p, L) if has.value else None

    # -- soft relative pose constraints (not in the reference; include/badba.h "Soft relative pose constraints") -------------
    def AddKeyframePoseConstraints(self, a_ids, b_ids, a_T_b, information) -> np.ndarray:
        """Adds constraints (a, b, Z = a_T_b, L) with the cost 1/2 r^T L r, r = log(Z^-1 global_T_a^-1 global_T_b) (translation,
        then rotation), and returns their ids ([n] int32).  a_T_b: [n, 7]; information: [n, 21] upper triangles of L, or
        [n, 6, 6] / [6, 6] matrices (one matrix for all).  Refused as a whole (nothing changes) for an unknown keyframe, a == b,
        a non-finite value, a zero quaternion or an L that is not positive semi-definite."""
        a = np.atleast_1d(np.asarray(a_ids, np.int64))
        b = np.atleast_1d(np.asarray(b_ids, np.int64))
        n = len(a)
        if len(b) != n:
            raise ValueError("a_ids and b_ids differ in length")
        Z = np.asarray(a_T_b, np.float32).reshape(n, 7)
        L = np.asarray(information, np.float32)
        if L.shape[-2:] == (6, 6):
            L = np.broadcast_to(L, (n, 6, 6))[:, np.triu_indices(6)[0], np.triu_indices(6)[1]]
        L = np.broadcast_to(L.reshape(-1, 21), (n, 21))
        recs = (_lib.PoseConstraint * max(n, 1))()
        for i in range(n):
            recs[i].keyframe_a, recs[i].keyframe_b = int(a[i]), int(b[i])
            recs[i].a_T_b[:] = [float(v) for v in Z[i]]
            recs[i].information[:] = [float(v) for v in L[i]]
        ids = np.zeros(max(n, 1), np.int32)
        self._check(self._lib.bba_add_keyframe_pose_constraints(self._h, n, recs, ids.ctypes.data))
        return ids[:n]

    def RemoveKeyframePoseConstraints(self, ids=None):
        """Removes the constraints `ids`, or every constraint with ids=None."""
        if ids is None:
            self._check(self._lib.bba_remove_keyframe_pose_constraints(self._h, -1, None))
            return
        ids = np.ascontiguousarray(np.atleast_1d(ids), np.int32)
        self._check(self._lib.bba_remove_keyframe_pose_constraints(self._h, len(ids), ids.ctypes.data))

    def KeyframePoseConstraints(self):
        """The constraints as last published, in id order: (ids [n], a [n], b [n], a_T_b [n, 7], L upper triangles [n, 21])."""
        count = C.c_int()
        self._check(self._lib.bba_get_keyframe_pose_constraints(self._h, 0, None, None, C.byref(count)))
        n = count.value
        ids = np.zeros(max(n, 1), np.int32)
        recs = (_lib.PoseConstraint * max(n, 1))()
        self._check(self._lib.bba_get_keyframe_pose_constraints(self._h, n, ids.ctypes.data, recs, C.byref(count)))
        n = min(n, count.value)
        a = np.array([recs[i].keyframe_a for i in range(n)], np.int32)
        b = np.array([recs[i].keyframe_b for i in range(n)], np.int32)
        Z = np.array([list(recs[i].a_T_b) for i in range(n)], np.float32).reshape(n, 7)
        L = np.array([list(recs[i].information) for i in range(n)], np.float32).reshape(n, 21)
        return ids[:n], a, b, Z, L

    # -- robust losses on the priors and constraints (not in the reference; include/badba.h "Robust losses") ----------------
    LOSS_TYPES = {"trivial": 0, "huber": 1, "cauchy": 2}

    @classmethod
    def _losses(cls, n, loss, scale):
        """n bba_robust_loss records from a type name or number (one for all, or [n]) and scale(s)."""
        types = [cls.LOSS_TYPES.get(t, t) if isinstance(t, str) else t for t in (loss if isinstance(loss, (list, tuple, np.ndarray)) else [loss] * n)]
        scales = np.broadcast_to(np.asarray(scale, np.float32), (n,))
        if len(types) != n:
            raise ValueError("one loss per id")
        recs = (_lib.RobustLoss * max(n, 1))()
        for i in range(n):
            recs[i].type, recs[i].scale = int(types[i]), float(scales[i])
        return recs

    def SetKeyframePosePriorLosses(self, ids, loss, scale=1.0):
        """Gives the priors of keyframes `ids` a robust loss: "trivial", "huber" or "cauchy" (or BBA_LOSS_* numbers; one for all,
        or one per id) with scale delta in units of sqrt(r^T L r).  Refused as a whole (nothing changes) for an unknown type, a
        scale that is not finite and > 0, or a keyframe without a prior."""
        ids = np.ascontiguousarray(np.atleast_1d(ids), np.int32)
        self._check(self._lib.bba_set_keyframe_pose_prior_losses(self._h, len(ids), ids.ctypes.data, self._losses(len(ids), loss, scale)))

    def KeyframePosePriorLoss(self, keyframe_id: int):
        """(type, scale) of a keyframe's prior loss as last published."""
        r = _lib.RobustLoss()
        self._check(self._lib.bba_get_keyframe_pose_prior_loss(self._h, keyframe_id, C.byref(r)))
        return r.type, r.scale

    def SetKeyframePoseConstraintLosses(self, ids, loss, scale=1.0):
        """Gives the constraints `ids` a robust loss (as SetKeyframePosePriorLosses); refused as a whole for an unknown id."""
        ids = np.ascontiguousarray(np.atleast_1d(ids), np.int32)
        self._check(self._lib.bba_set_keyframe_pose_constraint_losses(self._h, len(ids), ids.ctypes.data,
                                                                      self._losses(len(ids), loss, scale)))

    def GetKeyframePoseConstraintLosses(self):
        """The constraints' losses as last published, in id order: (ids [n], types [n] int32, scales [n] float32)."""
        count = C.c_int()
        self._check(self._lib.bba_get_keyframe_pose_constraint_losses(self._h, 0, None, None, C.byref(count)))
        n = count.value
        ids = np.zeros(max(n, 1), np.int32)
        recs = (_lib.RobustLoss * max(n, 1))()
        self._check(self._lib.bba_get_keyframe_pose_constraint_losses(self._h, n, ids.ctypes.data, recs, C.byref(count)))
        n = min(n, count.value)
        return ids[:n], np.array([recs[i].type for i in range(n)], np.int32), np.array([recs[i].scale for i in range(n)], np.float32)

    def EvaluateKeyframePoseTerms(self, stream=None) -> dict:
        """s = r^T L r and the robust weight w of every term at the current poses, evaluated on the device: prior_s /
        prior_weight [keyframes] (NaN without a prior), constraint_ids / constraint_s / constraint_weight [constraints] in id
        order.  A constraint that a robust pose graph rejected has w near 0.  Synchronises the stream."""
        K = self._lib.bba_keyframe_count(self._h)
        ids = self.GetKeyframePoseConstraintLosses()[0]
        n = len(ids)
        ps, pw = np.zeros(max(K, 1)), np.zeros(max(K, 1))
        cs, cw = np.zeros(max(n, 1)), np.zeros(max(n, 1))
        self._check(self._lib.bba_evaluate_keyframe_pose_terms(self._h, K, ps.ctypes.data, pw.ctypes.data, n, cs.ctypes.data,
                                                               cw.ctypes.data, self._stream_ptr(stream)))
        return {"prior_s": ps[:K], "prior_weight": pw[:K], "constraint_ids": ids, "constraint_s": cs[:n], "constraint_weight": cw[:n]}

    # -- attitude priors (not in the reference; include/badba.h "Attitude priors") ----------------------------------------------
    def SetKeyframeAttitudePriors(self, ids, reference_directions, measured_directions, information, loss="trivial", scale=1.0):
        """Gives keyframes `ids` an attitude prior: the angle theta between R^-1 d_ref (R: the rotation of global_T_frame) and
        d_meas costs 1/2 rho(L theta^2).  reference_directions: d_ref in the map frame ([n, 3] or one [3] for all, e.g. gravity);
        measured_directions: d_meas in each keyframe's camera frame ([n, 3]); information: L in rad^-2 (one for all, or [n]);
        loss / scale as SetKeyframePosePriorLosses.  The directions are normalised.  Refused as a whole (nothing changes) for an
        unknown id, a non-finite value, a direction of norm < 1e-6, L not finite and > 0, or a bad loss."""
        ids = np.ascontiguousarray(np.atleast_1d(ids), np.int32)
        n = len(ids)
        d_ref = np.broadcast_to(np.asarray(reference_directions, np.float32).reshape(-1, 3), (n, 3))
        d_meas = np.broadcast_to(np.asarray(measured_directions, np.float32).reshape(-1, 3), (n, 3))
        L = np.broadcast_to(np.asarray(information, np.float32).reshape(-1), (n,))
        losses = self._losses(n, loss, scale)
        recs = (_lib.AttitudePrior * max(n, 1))()
        for i in range(n):
            recs[i].reference_direction[:] = [float(v) for v in d_ref[i]]
            recs[i].measured_direction[:] = [float(v) for v in d_meas[i]]
            recs[i].information = float(L[i])
            recs[i].loss = losses[i]
        self._check(self._lib.bba_set_keyframe_attitude_priors(self._h, n, ids.ctypes.data, recs))

    def ClearKeyframeAttitudePriors(self, ids=None):
        """Removes the attitude priors of keyframes `ids`, or every one with ids=None."""
        if ids is None:
            self._check(self._lib.bba_clear_keyframe_attitude_priors(self._h, -1, None))
            return
        ids = np.ascontiguousarray(np.atleast_1d(ids), np.int32)
        self._check(self._lib.bba_clear_keyframe_attitude_priors(self._h, len(ids), ids.ctypes.data))

    def GetKeyframeAttitudePrior(self, keyframe_id: int):
        """A keyframe's attitude prior as last published, as a dict (reference_direction [3], measured_direction [3],
        information, loss_type, loss_scale), or None without one."""
        r, has = _lib.AttitudePrior(), C.c_int()
        self._check(self._lib.bba_get_keyframe_attitude_prior(self._h, keyframe_id, C.byref(r), C.byref(has)))
        if not has.value:
            return None
        return {"reference_direction": np.array(r.reference_direction[:], np.float32),
                "measured_direction": np.array(r.measured_direction[:], np.float32), "information": r.information,
                "loss_type": r.loss.type, "loss_scale": r.loss.scale}

    def EvaluateKeyframeAttitudePriors(self, stream=None):
        """(s = L theta^2 [keyframes], w [keyframes]) of every attitude prior at the current poses, evaluated on the device (NaN
        where a keyframe has none).  Synchronises the stream."""
        K = self._lib.bba_keyframe_count(self._h)
        s, w = np.zeros(max(K, 1)), np.zeros(max(K, 1))
        self._check(self._lib.bba_evaluate_keyframe_attitude_priors(self._h, K, s.ctypes.data, w.ctypes.data, self._stream_ptr(stream)))
        return s[:K], w[:K]

    def OptimizePoseGraph(self, add_current_state_odometry_constraints=True, gauge_keyframe=0, max_iterations=20,
                          odometry_information=None, stream=None) -> dict:
        """bba_optimize_pose_graph (the reference's PoseGraphOptimizer, here on the device): Gauss-Newton over the keyframe poses
        with the priors, the constraints and -- with add_current_state_odometry_constraints -- one edge per consecutive pair of
        keyframes at their current relative pose, information odometry_information ([21] upper triangle or [6, 6]; None:
        identity).  gauge_keyframe (-1: none) keeps its pose, as do untouched keyframes and the lowest id of every component
        without the gauge or a prior.  Returns the result as a dict (iterations, converged, linear_iterations, held_keyframes,
        initial_cost, final_cost).  Synchronises the stream."""
        o = _lib.PoseGraphOptions()
        o.gauge_keyframe = int(gauge_keyframe)
        o.max_iterations = int(max_iterations)
        o.use_odometry_chain = int(bool(add_current_state_odometry_constraints))
        L = np.eye(6, dtype=np.float32) if odometry_information is None else np.asarray(odometry_information, np.float32)
        if L.shape == (6, 6):
            L = L[np.triu_indices(6)]
        o.odometry_information[:] = [float(v) for v in L.reshape(21)]
        r = _lib.PoseGraphResult()
        self._check(self._lib.bba_optimize_pose_graph(self._h, C.byref(o), C.byref(r), self._stream_ptr(stream)))
        return {name: getattr(r, name) for name, _ in _lib.PoseGraphResult._fields_}

    # -- trajectory deformation around a BA call (trajectory_deformation.h:43-58) ----------------------------------------
    def RememberKeyframePoses(self) -> np.ndarray:
        """RememberKeyframePoses (trajectory_deformation.cc:33-42): frame_T_global of every keyframe, [K, 7], all from one
        publication of the poses (bba_get_keyframe_states), so the front-end thread may call it while a BA call runs."""
        K = self._lib.bba_keyframe_count(self._h)
        p = np.zeros((K, 7), np.float32)
        self._check(self._lib.bba_get_keyframe_states(self._h, K, p.ctypes.data, None))
        out = np.empty_like(p)
        for k in range(K):
            self._lib.bba_host_se3_inverse(p[k].ctypes.data, out[k].ctypes.data)
        return out

    def ExtrapolateAndInterpolateKeyframePoseChanges(self, start_frame: int, end_frame: int, original_keyframe_T_global,
                                                     keyframe_frame_indices, frame_poses: np.ndarray) -> np.ndarray:
        """ExtrapolateAndInterpolateKeyframePoseChanges (trajectory_deformation.cc:45-130): moves the frames that are not
        keyframes with the keyframes' pose change since RememberKeyframePoses.  original_keyframe_T_global: what
        RememberKeyframePoses returned ([K, 7]); keyframe_frame_indices: the frame index of each of those K keyframes
        (Keyframe.frame_index); frame_poses: global_T_frame of every frame, a C-contiguous float32 [N, 7] array, updated in place
        and returned.  The keyframes' own rows are not touched."""
        K = len(original_keyframe_T_global)
        current = np.zeros((K, 7), np.float32)
        self._check(self._lib.bba_get_keyframe_states(self._h, K, current.ctypes.data, None))
        return deform_trajectory(start_frame, end_frame, keyframe_frame_indices, original_keyframe_T_global, current, frame_poses)

    def DeformSurfelsWithKeyframePoseChanges(self, original_keyframe_T_global, stream=None):
        """bba_deform_surfels (not in the reference): after an outside correction of the keyframe poses, moves every surfel
        with the keyframes it is associated with at the remembered poses.  original_keyframe_T_global: what RememberKeyframePoses
        returned ([count, 7], keyframes 0 .. count-1).  Returns (moved, unobserved): surfels whose rows changed, and surfels that
        no keyframe observed (they follow the keyframe with the nearest original camera centre).  Synchronises the stream."""
        original = np.ascontiguousarray(original_keyframe_T_global, np.float32).reshape(-1, 7)
        moved, unobserved = C.c_uint32(), C.c_uint32()
        self._check(self._lib.bba_deform_surfels(self._h, len(original), original.ctypes.data, C.byref(moved), C.byref(unobserved),
                                                 self._stream_ptr(stream)))
        return moved.value, unobserved.value

    def MeasureKeyframeCovisibility(self, ids=None, stream=None) -> np.ndarray:
        """bba_measure_keyframe_covisibility (not in the reference): uint32 [len(ids), K], entry [i, b] the number of surfels
        associated with both keyframe ids[i] and keyframe b at their current poses ([i, ids[i]]: the surfels ids[i] observes).
        ids=None: every keyframe in id order.  Synchronises the stream."""
        K = self.KeyframeCount()
        if ids is None:
            out = np.zeros((K, K), np.uint32)
            self._check(self._lib.bba_measure_keyframe_covisibility(self._h, -1, None, K, out.ctypes.data, self._stream_ptr(stream)))
            return out
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        out = np.zeros((len(ids), K), np.uint32)
        self._check(self._lib.bba_measure_keyframe_covisibility(self._h, len(ids), ids.ctypes.data if len(ids) else None, K,
                                                                out.ctypes.data, self._stream_ptr(stream)))
        return out

    def _exposure_ids(self, ids):
        if ids is None:
            ids = np.arange(self.KeyframeCount(), dtype=np.int32)
        return np.ascontiguousarray(ids, np.int32).reshape(-1)

    def EstimateKeyframeExposures(self, ids=None, gauge_keyframe: int = -1, min_luma: int = 0, max_luma: int = 0,
                                  inlier_threshold: float = 0.0, outer_iterations: int = 0, stream=None):
        """bba_estimate_keyframe_exposures (not in the reference, DESIGN §3.21): (gains float32, observations uint32, inliers
        uint32), each [len(ids)], the gains relative to the gauge keyframe (NaN outside its component).  ids=None: every keyframe
        in id order.  Changes nothing on the handle; synchronises the stream."""
        ids = self._exposure_ids(ids)
        o = _lib.ExposureOptions(int(gauge_keyframe), int(min_luma), int(max_luma), float(inlier_threshold), int(outer_iterations))
        n = len(ids)
        gains = np.zeros(n, np.float32)
        obs = np.zeros(n, np.uint32)
        inl = np.zeros(n, np.uint32)
        self._check(self._lib.bba_estimate_keyframe_exposures(self._h, C.byref(o), n, ids.ctypes.data if n else None,
                                                              gains.ctypes.data if n else None, obs.ctypes.data if n else None,
                                                              inl.ctypes.data if n else None, self._stream_ptr(stream)))
        return gains, obs, inl

    def SetKeyframeExposures(self, gains, ids=None, stream=None):
        """bba_set_keyframe_exposures: keyframe ids[i] gets gain gains[i] (ids=None: every keyframe in id order) and its luma is
        re-extracted from its colour image."""
        ids = self._exposure_ids(ids)
        g = np.ascontiguousarray(gains, np.float32).reshape(-1)
        if len(g) != len(ids):
            raise ValueError("one gain per keyframe id")
        self._check(self._lib.bba_set_keyframe_exposures(self._h, len(ids), ids.ctypes.data if len(ids) else None,
                                                         g.ctypes.data if len(g) else None, self._stream_ptr(stream)))

    def GetKeyframeExposures(self, ids=None) -> np.ndarray:
        """bba_get_keyframe_exposures: the published gains of ids (ids=None: every keyframe), float32."""
        ids = self._exposure_ids(ids)
        out = np.zeros(len(ids), np.float32)
        self._check(self._lib.bba_get_keyframe_exposures(self._h, len(ids), ids.ctypes.data if len(ids) else None,
                                                         out.ctypes.data if len(ids) else None))
        return out

    def DebugExposureSystem(self, count: int):
        """bba_debug_get_exposure_system: (C uint32 [count, count], r int64 [count]) of the last round of the last estimate."""
        Cm = np.zeros((count, count), np.uint32)
        r = np.zeros(count, np.int64)
        self._check(self._lib.bba_debug_get_exposure_system(self._h, int(count), Cm.ctypes.data, r.ctypes.data))
        return Cm, r

    def MeasureFrameOverlap(self, frames, queries, with_shared: bool = True, stream=None) -> FrameOverlap:
        """bba_measure_frame_overlap (not in the reference, DESIGN §3.20): what the surfel map already explains of frames that are
        not keyframes.  frames: a sequence of (depth, normals[, colour]) [h, w] u16 device tensors (colour is not read); queries: a
        sequence of (frame index, global_T_frame [7], min_depth, max_depth).  With the same buffers, pose and depth range,
        AddKeyframe + CreateSurfelsForKeyframe would create uncovered_cells surfels unfiltered and new_surfels filtered.
        with_shared=False skips the keyframes' side (shared is None then, as it is without keyframes).  Synchronises the stream."""
        bufs = (_lib.FrameBuffers * len(frames))()
        for b, fr in zip(bufs, frames):
            depth, normals = fr[0], fr[1]
            b.depth, b.depth_pitch = depth.data_ptr(), depth.stride(0) * 2
            b.normals, b.normals_pitch = normals.data_ptr(), normals.stride(0) * 2
        qs = (_lib.FrameOverlapQuery * max(1, len(queries)))()
        for q, (f, pose, lo, hi) in zip(qs, queries):
            q.frame = int(f)
            q.global_T_frame[:] = np.ascontiguousarray(pose, np.float32).reshape(7).tolist()
            q.min_depth, q.max_depth = float(lo), float(hi)
        n, K = len(queries), self.KeyframeCount()
        out = (_lib.FrameOverlap * max(1, n))()
        shared = np.zeros((n, K), np.uint32) if with_shared and K > 0 else None
        self._check(self._lib.bba_measure_frame_overlap(self._h, len(frames), bufs if len(frames) else None, n, qs if n else None, K,
                                                        None if shared is None else shared.ctypes.data, out if n else None,
                                                        self._stream_ptr(stream)))
        col = lambda name: np.array([getattr(o, name) for o in list(out)[:n]], np.uint32)
        return FrameOverlap(col("observed_surfels"), col("valid_cells"), col("uncovered_cells"), col("new_surfels"), shared)

    def DebugSetCovisibilityChunk(self, surfels: int):
        """bba_debug_set_covisibility_chunk: surfels per chunk of MeasureKeyframeCovisibility (0: the 128 MiB budget rule)."""
        self._check(self._lib.bba_debug_set_covisibility_chunk(self._h, int(surfels)))

    def SurfelsDeviceView(self) -> torch.Tensor:
        """The 17-row surfel buffer as a torch tensor, whoever owns it (zero-copy)."""
        if self._surfels is not None:
            return self._surfels
        ptr, pitch, n = C.c_void_p(), C.c_size_t(), C.c_uint32()
        self._check(self._lib.bba_get_surfels_device(self._h, C.byref(ptr), C.byref(pitch), C.byref(n)))

        class _Raw:
            pass
        raw = _Raw()
        raw.__cuda_array_interface__ = {"shape": (17, pitch.value // 4), "typestr": "<f4", "data": (ptr.value, False),
                                        "version": 2, "strides": None}
        self._raw_keepalive = raw
        return torch.as_tensor(raw, device=self.device)

    def covisibility(self) -> np.ndarray:
        K = len(self._keyframes)
        out = np.zeros((K, K), np.uint8)
        for k in range(K):
            self._check(self._lib.bba_get_covisibility(self._h, k, out[k].ctypes.data))
        return out

    # -- hot path ---------------------------------------------------------------------------------
    def AccumulatePoseEstimationCoeffs(self, keyframe_id: int, global_T_frame_estimate, stream=None):
        """kernels.h:156-174 AccumulatePoseEstimationCoeffsCUDA (debug = true)."""
        p = np.ascontiguousarray(global_T_frame_estimate, np.float32)
        out = _lib.PoseCoeffs()
        self._check(self._lib.bba_accumulate_pose_coeffs(self._h, keyframe_id, p.ctypes.data_as(C.POINTER(C.c_float)),
                                                         C.byref(out), self._stream_ptr(stream)))
        return out

    def PoseCoeffsBatch(self, keyframe_ids, global_T_frame_estimates, variant: int = _lib.POSE_VARIANT_AUTO, with_stats: bool = True,
                        stream=None):
        """Parity hook (bba_debug_pose_coeffs_batch): the pose kernel over a work list of keyframes, each at its own pose
        ([count, 7]), in the instantiation the BA pose step runs (or a forced one, _lib.POSE_VARIANT_*).  Returns
        (H [K, 21], b [K, 6], counts [K, 4] = in image / depth ok / associated / photometric, costs [K, 3]) indexed by keyframe
        id over all K keyframes; rows of keyframes outside the list are what the launch left in their records (zeros)."""
        ids = np.ascontiguousarray(keyframe_ids, np.int32)
        poses = np.ascontiguousarray(global_T_frame_estimates, np.float32).reshape(len(ids), 7)
        K = len(self._keyframes)
        H, b, costs = np.zeros((K, 21)), np.zeros((K, 6)), np.zeros((K, 3))
        counts = np.zeros((K, 4), np.uint64)
        self._check(self._lib.bba_debug_pose_coeffs_batch(self._h, len(ids), ids.ctypes.data, poses.ctypes.data, int(variant),
                                                          int(with_stats), H.ctypes.data, b.ctypes.data, counts.ctypes.data,
                                                          costs.ctypes.data, self._stream_ptr(stream)))
        return H, b, counts, costs

    def DebugSetPoseGroup(self, keyframes: int):
        """bba_debug_set_pose_group: keyframes per staged surfel tile in every later pose-kernel launch (0: the library's choice)."""
        self._check(self._lib.bba_debug_set_pose_group(self._h, int(keyframes)))

    def DebugSetGeometryPass(self, pass_: int, tile_shift: int = 0):
        """bba_debug_set_geometry_pass: 0 (auto) / 2 (one tile-major launch when the keyframes fit) or 1 (the two group-major launches)
        for the normal and position / descriptor updates of every later geometry step; tile_shift 5..8 (0: the library's choice)."""
        self._check(self._lib.bba_debug_set_geometry_pass(self._h, int(pass_), int(tile_shift)))

    def EstimateFramePose(self, stream, global_T_frame_initial_estimate, keyframe_id: int):
        """direct_ba.h:122-129; returns (global_T_frame_estimate, iterations, converged)."""
        p = np.ascontiguousarray(global_T_frame_initial_estimate, np.float32)
        out = np.zeros(7, np.float32)
        it, conv = C.c_int(), C.c_int()
        self._check(self._lib.bba_estimate_frame_pose(self._h, keyframe_id, p.ctypes.data_as(C.POINTER(C.c_float)),
                                                      out.ctypes.data_as(C.POINTER(C.c_float)), C.byref(it), C.byref(conv),
                                                      self._stream_ptr(stream)))
        return out, it.value, bool(conv.value)

    def EstimateFramePoseFromBuffers(self, stream, global_T_frame_initial_estimate, depth_buffer: torch.Tensor,
                                     normals_buffer: torch.Tensor, color_buffer: torch.Tensor):
        """The buffer-taking form of DirectBA::EstimateFramePose (direct_ba.h:122-129) for a frame that is not a keyframe:
        depth / normals [h, w] u16 and colour [ch, cw, 4] u8 (.w = luma) device tensors.  Returns
        (global_T_frame_estimate, iterations, converged)."""
        p = np.ascontiguousarray(global_T_frame_initial_estimate, np.float32)
        out = np.zeros(7, np.float32)
        it, conv = C.c_int(), C.c_int()
        self._check(self._lib.bba_estimate_frame_pose_for_frame(
            self._h, depth_buffer.data_ptr(), depth_buffer.stride(0) * 2, normals_buffer.data_ptr(), normals_buffer.stride(0) * 2,
            color_buffer.data_ptr(), color_buffer.stride(0), p.ctypes.data_as(C.POINTER(C.c_float)),
            out.ctypes.data_as(C.POINTER(C.c_float)), C.byref(it), C.byref(conv), self._stream_ptr(stream)))
        return out, it.value, bool(conv.value)

    def EstimateFramePosesFromBuffers(self, stream, frames, initial_poses, frame_of_entry=None, with_coeffs: bool = False):
        """EstimateFramePoseFromBuffers for many entries in one call (bba_estimate_frame_poses_for_frames).  frames: a sequence of
        (depth, normals, colour) device tensors as EstimateFramePoseFromBuffers takes them; initial_poses: [count, 7]
        global_T_frame starts, entry i tracking frames[frame_of_entry[i]] (frames[i] without frame_of_entry).  Returns
        (global_T_frame_estimates [count, 7], iterations [count], converged [count] bool) and, with with_coeffs, a list of the
        count PoseCoeffs at the returned poses as a fourth element.  The entries run in chunks of as many as there are free
        keyframe slots."""
        bufs = _frame_buffers(frames)
        init = np.ascontiguousarray(initial_poses, np.float32).reshape(-1, 7)
        count = len(init)
        fmap = None if frame_of_entry is None else np.ascontiguousarray(frame_of_entry, np.int32)
        out = np.zeros((count, 7), np.float32)
        it, conv = np.zeros(count, np.int32), np.zeros(count, np.int32)
        coeffs = (_lib.PoseCoeffs * count)() if with_coeffs else None
        self._check(self._lib.bba_estimate_frame_poses_for_frames(
            self._h, len(frames), bufs, count, None if fmap is None else fmap.ctypes.data, init.ctypes.data, out.ctypes.data,
            it.ctypes.data, conv.ctypes.data, coeffs, self._stream_ptr(stream)))
        if with_coeffs:
            return out, it, conv.astype(bool), list(coeffs)
        return out, it, conv.astype(bool)

    def TrackFramePairwise(self, stream, base_keyframe_id: int, depth_buffer: torch.Tensor, normals_buffer: torch.Tensor,
                           color_buffer: torch.Tensor, base_T_frame_initial_estimate_1, base_T_frame_initial_estimate_2=None,
                           num_scales: int = 5, use_pyramid_level_0: bool = True, use_gradmag: bool = False,
                           test_different_initial_estimates: bool = True, max_iterations_per_scale: int = 30):
        """BadSlam::RunOdometry -> TrackFramePairwise (bad_slam.cc:829-950, pairwise_frame_tracking.cc:153-678): the frame given by
        depth / normals [h, w] u16 and colour [ch, cw, 4] u8 (.w = luma) device tensors is tracked against keyframe
        `base_keyframe_id`.  Defaults = what RunOdometry passes.  Returns (base_T_frame_estimate, OdometryResult)."""
        p1 = np.ascontiguousarray(base_T_frame_initial_estimate_1, np.float32)
        p2 = p1 if base_T_frame_initial_estimate_2 is None else np.ascontiguousarray(base_T_frame_initial_estimate_2, np.float32)
        out = np.zeros(7, np.float32)
        o = _odometry_options(num_scales, use_pyramid_level_0, use_gradmag, test_different_initial_estimates, max_iterations_per_scale)
        res = _lib.OdometryResult()
        F = C.POINTER(C.c_float)
        self._check(self._lib.bba_track_frame_pairwise(
            self._h, C.byref(o), int(base_keyframe_id), depth_buffer.data_ptr(), depth_buffer.stride(0) * 2, normals_buffer.data_ptr(),
            normals_buffer.stride(0) * 2, color_buffer.data_ptr(), color_buffer.stride(0), p1.ctypes.data_as(F), p2.ctypes.data_as(F),
            out.ctypes.data_as(F), C.byref(res), self._stream_ptr(stream)))
        return out, res

    def TrackFramePairwiseToFrame(self, stream, base_depth_buffer: torch.Tensor, base_normals_buffer: torch.Tensor,
                                  base_color_buffer: torch.Tensor, depth_buffer: torch.Tensor, normals_buffer: torch.Tensor,
                                  color_buffer: torch.Tensor, base_T_frame_initial_estimate_1, base_T_frame_initial_estimate_2=None,
                                  num_scales: int = 5, use_pyramid_level_0: bool = True, use_gradmag: bool = False,
                                  test_different_initial_estimates: bool = True, max_iterations_per_scale: int = 30):
        """TrackFramePairwise against a base frame that is not a keyframe (yet), given by the buffers AddKeyframe would take
        (depth / normals [h, w] u16, colour [ch, cw, 4] u8): what the odometry thread does with the keyframe the BA thread has not
        added yet.  Same result as TrackFramePairwise against those buffers as a keyframe.  Returns (base_T_frame_estimate,
        OdometryResult)."""
        p1 = np.ascontiguousarray(base_T_frame_initial_estimate_1, np.float32)
        p2 = p1 if base_T_frame_initial_estimate_2 is None else np.ascontiguousarray(base_T_frame_initial_estimate_2, np.float32)
        out = np.zeros(7, np.float32)
        o = _odometry_options(num_scales, use_pyramid_level_0, use_gradmag, test_different_initial_estimates, max_iterations_per_scale)
        res = _lib.OdometryResult()
        F = C.POINTER(C.c_float)
        self._check(self._lib.bba_track_frame_pairwise_to_frame(
            self._h, C.byref(o), base_depth_buffer.data_ptr(), base_depth_buffer.stride(0) * 2, base_normals_buffer.data_ptr(),
            base_normals_buffer.stride(0) * 2, base_color_buffer.data_ptr(), base_color_buffer.stride(0),
            depth_buffer.data_ptr(), depth_buffer.stride(0) * 2, normals_buffer.data_ptr(), normals_buffer.stride(0) * 2,
            color_buffer.data_ptr(), color_buffer.stride(0), p1.ctypes.data_as(F), p2.ctypes.data_as(F), out.ctypes.data_as(F),
            C.byref(res), self._stream_ptr(stream)))
        return out, res

    def TrackFramesPairwise(self, stream, frames, entries, num_scales: int = 5, use_pyramid_level_0: bool = True,
                            use_gradmag: bool = False, test_different_initial_estimates: bool = True, max_iterations_per_scale: int = 30):
        """TrackFramePairwise / TrackFramePairwiseToFrame for many independent pairs in one call (bba_track_frames_pairwise), all
        with the same options.  frames: a sequence of (depth, normals, colour) device tensors as TrackFramePairwise takes them;
        entries: a sequence of (base_keyframe_id, base_frame, tracked_frame, base_T_frame_initial_1[, base_T_frame_initial_2]),
        base_keyframe_id -1 meaning frames[base_frame] is the base.  Returns (base_T_frame_estimates [count, 7], a list of the count
        OdometryResult, the kernel launches of the whole call).  The entries run in chunks of _lib.ODOMETRY_CHUNK_ENTRIES."""
        bufs = _frame_buffers(frames)
        ents = (_lib.OdometryEntry * len(entries))()
        for e, spec in zip(ents, entries):
            e.base_keyframe_id, e.base_frame, e.tracked_frame = int(spec[0]), int(spec[1]), int(spec[2])
            p1 = np.ascontiguousarray(spec[3], np.float32).reshape(7)
            p2 = p1 if len(spec) < 5 or spec[4] is None else np.ascontiguousarray(spec[4], np.float32).reshape(7)
            e.base_T_frame_initial_1[:] = p1.tolist()
            e.base_T_frame_initial_2[:] = p2.tolist()
        count = len(entries)
        out = np.zeros((count, 7), np.float32)
        results = (_lib.OdometryResult * count)()
        launches = C.c_uint32()
        o = _odometry_options(num_scales, use_pyramid_level_0, use_gradmag, test_different_initial_estimates, max_iterations_per_scale)
        self._check(self._lib.bba_track_frames_pairwise(self._h, C.byref(o), len(frames), bufs, count, ents, out.ctypes.data, results,
                                                        C.byref(launches), self._stream_ptr(stream)))
        return out, list(results), launches.value

    def VerifyLoopClosures(self, stream, candidates, num_scales: int = 5, use_pyramid_level_0: bool = True,
                           use_gradmag: bool = False, max_iterations_per_scale: int = 30, max_angle_difference: float = 0.0,
                           max_translation_difference: float = 0.0, max_pixel_distance: float = 0.0):
        """LoopDetector's verification of loop-closure candidates (loop_detector.cc:436-668, bba_verify_loop_closures): each
        (current_keyframe_id, matched_keyframe_id, old_T_cur_initial[7]) is refined against the matched keyframe and its two
        neighbours, the three estimates are tested for agreement and averaged, and the correction is tested for necessity.
        Thresholds <= 0 select the reference's (10 deg, 0.02 m, 1 px).  Returns a list of the count LoopVerification records;
        `status` is one of _lib.LOOP_*, and cur_T_old is the loop edge a_T_b for AddKeyframePoseConstraints(current, matched)."""
        cands = (_lib.LoopCandidate * len(candidates))()
        for c, spec in zip(cands, candidates):
            c.current_keyframe_id, c.matched_keyframe_id = int(spec[0]), int(spec[1])
            c.old_T_cur_initial[:] = np.ascontiguousarray(spec[2], np.float32).reshape(7).tolist()
        o = _lib.LoopVerificationOptions(_odometry_options(num_scales, use_pyramid_level_0, use_gradmag, False, max_iterations_per_scale),
                                         float(max_angle_difference), float(max_translation_difference), float(max_pixel_distance))
        out = (_lib.LoopVerification * max(1, len(candidates)))()
        self._check(self._lib.bba_verify_loop_closures(self._h, C.byref(o), len(candidates), cands, out, self._stream_ptr(stream)))
        return list(out)[:len(candidates)]

    def IndexKeyframes(self, ids=None, num_ferns: int = 512, min_depth: float = 0.5, max_depth: float = 3.0, stream=None):
        """Encodes keyframes into the randomized-fern place index (bba_index_keyframes, DESIGN §3.18) from their current images;
        ids None: every keyframe.  Options that differ from the current ones reset the index first.  Index a keyframe again
        after changing its images."""
        ids = np.arange(self.KeyframeCount(), dtype=np.int32) if ids is None else np.ascontiguousarray(ids, np.int32).reshape(-1)
        o = _lib.PlaceIndexOptions(int(num_ferns), float(min_depth), float(max_depth))
        self._check(self._lib.bba_index_keyframes(self._h, C.byref(o), len(ids), ids.ctypes.data if len(ids) else None,
                                                  self._stream_ptr(stream)))

    def KeyframeCount(self) -> int:
        """The published keyframe count (bba_keyframe_count)."""
        return int(self._lib.bba_keyframe_count(self._h))

    def PlaceIndexOptions(self):
        """The published place index's (num_ferns, min_raw, max_raw) (bba_get_place_index_options); zeros before the first index."""
        v = [C.c_int(), C.c_int(), C.c_int()]
        self._check(self._lib.bba_get_place_index_options(self._h, *(C.byref(x) for x in v)))
        return tuple(x.value for x in v)

    def QueryPlaceIndex(self, queries, frames=(), max_matches: int = 8, stream=None):
        """Place-index queries in one call (bba_query_place_index).  queries: a sequence of (keyframe_id, frame, first_keyframe,
        last_keyframe), keyframe_id -1 meaning the frame frames[frame] (a (depth, normals or None, colour) tuple of device
        tensors) is encoded in this call.  Returns per query (ids, differences): the indexed keyframes of the range, the query
        keyframe excluded, ordered by (difference, id), at most max_matches of them."""
        bufs = (_lib.FrameBuffers * max(1, len(frames)))()
        for b, (depth, normals, color) in zip(bufs, frames):
            b.depth, b.depth_pitch = depth.data_ptr(), depth.stride(0) * 2
            if normals is not None:
                b.normals, b.normals_pitch = normals.data_ptr(), normals.stride(0) * 2
            b.color_rgba, b.color_pitch = color.data_ptr(), color.stride(0)
        qs = (_lib.PlaceQuery * max(1, len(queries)))()
        for q, spec in zip(qs, queries):
            q.keyframe_id, q.frame, q.first_keyframe, q.last_keyframe = (int(v) for v in spec)
        n = len(queries)
        ids = np.zeros((max(1, n), max_matches), np.int32)
        diffs = np.zeros((max(1, n), max_matches), np.int32)
        counts = np.zeros(max(1, n), np.int32)
        self._check(self._lib.bba_query_place_index(self._h, len(frames), bufs if frames else None, n, qs, int(max_matches),
                                                    ids.ctypes.data, diffs.ctypes.data, counts.ctypes.data, self._stream_ptr(stream)))
        return [(ids[i, :counts[i]].copy(), diffs[i, :counts[i]].copy()) for i in range(n)]

    def PlaceIndexCodes(self, ids, stream=None):
        """The published place-index codes of indexed keyframes (bba_get_place_index_codes): uint32 [len(ids), num_ferns / 8]."""
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        words = self.PlaceIndexOptions()[0] // 8
        out = np.zeros((len(ids), max(1, words)), np.uint32)
        self._check(self._lib.bba_get_place_index_codes(self._h, len(ids), ids.ctypes.data if len(ids) else None, words,
                                                        out.ctypes.data, self._stream_ptr(stream)))
        return out

    def OdometryLevel(self, which: int, scale: int, stream=None):
        """Parity hook: (depth f32, normals u16, colour u8) of one pyramid level of the last TrackFramePairwise call
        (which: 0 = base keyframe, 1 = tracked frame)."""
        w, h = C.c_int(), C.c_int()
        self._check(self._lib.bba_odometry_get_level(self._h, which, scale, None, None, None, C.byref(w), C.byref(h), self._stream_ptr(stream)))
        d = np.zeros((h.value, w.value), np.float32)
        n = np.zeros((h.value, w.value), np.uint16)
        c = np.zeros((h.value, w.value), np.uint8)
        self._check(self._lib.bba_odometry_get_level(self._h, which, scale, d.ctypes.data, n.ctypes.data, c.ctypes.data, C.byref(w),
                                                     C.byref(h), self._stream_ptr(stream)))
        return d, n, c

    def OdometryCoeffs(self, scale: int, base_T_frame_a, base_T_frame_b=None, use_gradmag: bool = False, stream=None):
        """Parity hook on the pyramids of the last TrackFramePairwise call: AccumulatePoseEstimationCoeffsFromImagesCUDA at pose a
        -> (H[21], b[6], residual_count, residual_sum) and ComputeCostAndResidualCountFromImagesCUDA at a and b -> (counts[2], costs[2])."""
        pa = np.ascontiguousarray(base_T_frame_a, np.float32)
        pb = pa if base_T_frame_b is None else np.ascontiguousarray(base_T_frame_b, np.float32)
        H, b = np.zeros(21, np.float32), np.zeros(6, np.float32)
        cnt, rs = C.c_uint32(), C.c_float()
        counts, costs = np.zeros(2, np.uint32), np.zeros(2, np.float32)
        F = C.POINTER(C.c_float)
        self._check(self._lib.bba_odometry_debug_coeffs(self._h, scale, int(use_gradmag), pa.ctypes.data_as(F), pb.ctypes.data_as(F),
                                                        H.ctypes.data, b.ctypes.data, C.byref(cnt), C.byref(rs), counts.ctypes.data,
                                                        costs.ctypes.data, self._stream_ptr(stream)))
        return H, b, cnt.value, rs.value, counts, costs

    def UpdateSurfelActivation(self, stream=None):
        self._check(self._lib.bba_update_surfel_activation(self._h, self._stream_ptr(stream)))

    def OptimizeGeometryIteration(self, stream=None):
        self._check(self._lib.bba_optimize_geometry_iteration(self._h, self._stream_ptr(stream)))

    def OptimizeIntrinsics(self, optimize_depth_intrinsics: bool, optimize_color_intrinsics: bool, stream=None):
        self._check(self._lib.bba_optimize_intrinsics(self._h, int(optimize_depth_intrinsics),
                                                      int(optimize_color_intrinsics), self._stream_ptr(stream)))

    def IntrinsicsCoeffs(self, optimize_depth_intrinsics: bool, optimize_color_intrinsics: bool, stream=None):
        """Parity hook (bba_debug_intrinsics_coeffs): the normal equations of the intrinsics step before the Schur complement.
        Returns (sums [34] fp64: A upper triangle, b1, colour H upper triangle, colour b; cells [8, cf_h * cf_w] fp32: the five
        rows of B, D, b2 and the observation count per sparse cell).  The handle's state does not change."""
        w, h = C.c_int(), C.c_int()
        self._check(self._lib.bba_cfactor_size(self._h, C.byref(w), C.byref(h)))
        sums, cells = np.zeros(34), np.zeros((8, w.value * h.value), np.float32)
        self._check(self._lib.bba_debug_intrinsics_coeffs(self._h, int(optimize_depth_intrinsics), int(optimize_color_intrinsics),
                                                          sums.ctypes.data, cells.ctypes.data, self._stream_ptr(stream)))
        return sums, cells

    def BundleAdjustment(self, stream, optimize_depth_intrinsics: bool, optimize_color_intrinsics: bool,
                         do_surfel_updates: bool, optimize_poses: bool, optimize_geometry: bool,
                         min_iterations: int, max_iterations: int, use_pcg: bool = False,
                         active_keyframe_window_start: int = 0, active_keyframe_window_end: int = -1,
                         increase_ba_iteration_count: bool = True, time_limit: float = 0.0,
                         pcg_max_inner_iterations: int = 30, pcg_max_keyframes: int = 2500,
                         pcg_gauge_keyframe: int = -1, progress_function=None) -> BAResult:
        """direct_ba.h:143-162.  pcg_gauge_keyframe >= 0 pins the keyframe the PCG solver holds fixed (the reference draws
        rand() % K in every iteration, direct_ba_pcg.cc:324).  progress_function(iteration) -> bool is called at the top of
        every iteration; False stops the optimisation (direct_ba_alternating.cc:346-348)."""
        if active_keyframe_window_end < 0:
            active_keyframe_window_end = len(self._keyframes) - 1
        o = _lib.BAOptions(int(optimize_depth_intrinsics), int(optimize_color_intrinsics), int(do_surfel_updates),
                           int(optimize_poses), int(optimize_geometry), int(min_iterations), int(max_iterations),
                           int(use_pcg), int(active_keyframe_window_start), int(active_keyframe_window_end),
                           int(increase_ba_iteration_count), float(time_limit), int(pcg_max_inner_iterations),
                           int(pcg_max_keyframes), int(pcg_gauge_keyframe))
        if progress_function is not None:
            cb = _lib.PROGRESS_FN(lambda _user, iteration: 1 if progress_function(int(iteration)) else 0)
            o.progress_function = cb   # `cb` stays referenced until the call returns
        r = _lib.BAResult()
        self._check(self._lib.bba_bundle_adjust(self._h, C.byref(o), C.byref(r), self._stream_ptr(stream)))
        return BAResult(r.iterations_done, bool(r.converged), r.depth_residual_count, r.descriptor_residual_count,
                        r.cost, r.pose_iterations_total, r.ms_surfel_activation, r.ms_geometry_optimization,
                        r.ms_pose_optimization, r.ms_intrinsics_optimization, r.kernel_launches,
                        r.pcg_inner_iterations_total, r.pcg_last_r_norm, r.ms_pcg, r.surfels_deleted, r.surfels_size,
                        r.surfels_created, r.surfels_merged)

    def ba_iteration_count(self) -> int:
        a, b = C.c_int(), C.c_int()
        self._check(self._lib.bba_get_ba_iteration_counts(self._h, C.byref(a), C.byref(b)))
        return a.value

    def last_ba_iteration_count(self) -> int:
        a, b = C.c_int(), C.c_int()
        self._check(self._lib.bba_get_ba_iteration_counts(self._h, C.byref(a), C.byref(b)))
        return b.value

    def SetLastBAIterationCount(self, count: int):
        """direct_ba.h:377."""
        self._check(self._lib.bba_set_ba_iteration_counts(self._h, self.ba_iteration_count(), int(count)))

    def CreateSurfelsForKeyframe(self, stream, filter_new_surfels: bool, keyframe_id: int) -> int:
        """direct_ba.h:114-117; returns the number of surfels created."""
        c = C.c_uint32()
        self._check(self._lib.bba_create_surfels_for_keyframe(self._h, int(keyframe_id), int(filter_new_surfels), C.byref(c),
                                                              self._stream_ptr(stream)))
        return c.value

    def MergeSurfelsForKeyframe(self, keyframe_id: int, stream=None) -> int:
        """DetermineSupportingSurfelsAndMergeSurfelsCUDA for one keyframe; returns the number of surfels marked deleted."""
        d = C.c_uint32()
        self._check(self._lib.bba_merge_surfels_for_keyframe(self._h, int(keyframe_id), C.byref(d), self._stream_ptr(stream)))
        return d.value

    def CompactSurfels(self, free_count: int, with_active_flags: bool = True, stream=None) -> int:
        n = C.c_uint32()
        self._check(self._lib.bba_compact_surfels(self._h, int(free_count), int(with_active_flags), C.byref(n), self._stream_ptr(stream)))
        return n.value

    def PerformBASchemeEndTasks(self, stream=None, do_surfel_updates: bool = False):
        """direct_ba.cc:566-653 (with do_surfel_updates: merge similar surfels of the keyframes active in this BA block; then
        delete badly observed surfels, update radii, compact).  Returns (deleted, surfels_size)."""
        d, n = C.c_uint32(), C.c_uint32()
        self._check(self._lib.bba_perform_end_tasks(self._h, int(bool(do_surfel_updates)), C.byref(d), C.byref(n),
                                                    self._stream_ptr(stream)))
        return d.value, n.value

    def PCGDebug(self, optimize_poses=True, optimize_geometry=True, optimize_depth_intrinsics=False,
                 optimize_color_intrinsics=False, gauge_keyframe=0, stream=None):
        """Parity hook (bba_pcg_debug at step 0): r, M, p0, g = J^T W J p0 and (alpha_n, alpha_d) of the PCG solver's first step."""
        s = self.PCGProbe(0, False, optimize_poses, optimize_geometry, optimize_depth_intrinsics, optimize_color_intrinsics,
                          gauge_keyframe, stream)
        return s["r"], s["M"], s["p"], s["g"], np.array([s["alpha_n"], s["alpha_d"]])

    def PCGProbe(self, step, apply=False, optimize_poses=True, optimize_geometry=True, optimize_depth_intrinsics=False,
                 optimize_color_intrinsics=False, gauge_keyframe=0, stream=None) -> dict:
        """bba_pcg_debug: the PCG solver's init pass, `step` complete inner steps, then inner step `step` observed before
        PCGStep2 (r, M, p, g, delta, alpha_n, alpha_d), after it (r_step2, delta_step2, z, beta_n) and after PCGStep3 (p_step3,
        g_step3, alpha_d_step3).  apply=True then applies delta to the surfels, cfactors, poses and intrinsics."""
        o = _lib.BAOptions(int(optimize_depth_intrinsics), int(optimize_color_intrinsics), 0, int(optimize_poses),
                           int(optimize_geometry), 1, 1, 1, 0, len(self._keyframes) - 1, 0, 0.0, 30, 2500, int(gauge_keyframe))
        n = C.c_uint32()
        self._check(self._lib.bba_pcg_debug(self._h, C.byref(o), int(step), 0, C.byref(n), None, self._stream_ptr(stream)))
        vectors = ("r", "M", "p", "g", "delta", "r_step2", "delta_step2", "z", "p_step3", "g_step3")
        out = {k: np.zeros(n.value, np.float32) for k in vectors}
        probe = _lib.PcgProbe(**{k: out[k].ctypes.data for k in vectors})
        self._check(self._lib.bba_pcg_debug(self._h, C.byref(o), int(step), int(bool(apply)), C.byref(n), C.byref(probe),
                                            self._stream_ptr(stream)))
        for k in ("alpha_n", "alpha_d", "beta_n", "alpha_d_step3"):
            out[k] = getattr(probe, k)
        return out

    def EnablePeerExchange(self, group=None) -> int:
        """Maps the surfel replicas of the other ranks into this process (CUDA IPC over NVLink, bba_peer_export /
        bba_peer_import): the geometry kernels then store updated surfels straight into every replica and the exchange
        step is a barrier.  Collective call.  All ranks end up in the same mode: if the mapping fails anywhere (IPC not
        permitted, ...) every rank unmaps and 0 is returned, otherwise the number of mapped peers."""
        import torch
        import torch.distributed as dist
        world = dist.get_world_size(group)
        ok = 1
        ph = _lib.PeerHandle()
        if self._lib.bba_peer_export(self._h, C.byref(ph)) != 0:
            ok = 0
        blobs = [None] * world
        dist.all_gather_object(blobs, bytes(ph) if ok else None, group=group)
        if ok and all(b is not None for b in blobs):
            arr = (_lib.PeerHandle * world)()
            for r, b in enumerate(blobs):
                C.memmove(C.byref(arr[r]), b, C.sizeof(_lib.PeerHandle))
            if self._lib.bba_peer_import(self._h, arr, world) != 0:
                ok = 0
        else:
            ok = 0
        flag = torch.tensor([ok], dtype=torch.int32, device=self._surfels.device if self._surfels is not None else "cuda")
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
        if int(flag.item()) == 0:
            self._lib.bba_peer_unmap(self._h)
            return 0
        return int(self._lib.bba_peer_count(self._h))

    # -- multi-GPU (one process per GPU) ---------------------------------------------------------------
    def MarkReplicaRewritten(self):
        """bba_mark_replica_rewritten: call on every rank after rewriting the surfel replica outside the library (e.g. restoring a
        snapshot) while peers are mapped."""
        self._check(self._lib.bba_mark_replica_rewritten(self._h))

    def SetCollective(self, group=None):
        """Registers the exchange step (bba_set_collective) on top of torch.distributed (NCCL over NVLink): in-place
        all-gather of the updated surfel shards, sum all-reduce of the pose slots."""
        import torch.distributed as dist
        lib_defs = _lib
        rank, world = self._cfg.rank, self._cfg.world_size
        views = {}

        def view(ptr, nbytes, dtype):
            key = (ptr, nbytes, dtype)
            t = views.get(key)
            if t is None:
                class _Raw:
                    pass
                raw = _Raw()
                n = nbytes // (4 if dtype == torch.float32 else 1)
                raw.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4" if dtype == torch.float32 else "|u1",
                                                "data": (ptr, False), "version": 2, "strides": None}
                t = torch.as_tensor(raw, device=self.device)
                views[key] = (t, raw)
                return t
            return t[0]

        def cb(user, op, ptr, count, stream):
            st = torch.cuda.ExternalStream(stream or 0, device=self.device) if stream else torch.cuda.default_stream(self.device)
            with torch.cuda.stream(st):
                if op == lib_defs.COLLECTIVE_ALLGATHER:
                    out = view(ptr, count * world, torch.uint8)
                    dist.all_gather_into_tensor(out, out[rank * count:(rank + 1) * count], group=group)
                else:
                    dist.all_reduce(view(ptr, count * 4, torch.float32), group=group)

        self._collective_cb = lib_defs.COLLECTIVE_FN(cb)   # keep alive
        self._check(self._lib.bba_set_collective(self._h, self._collective_cb, None))

    def DebugCollective(self, op: int, buffer: torch.Tensor, count: int, stream=None):
        """bba_debug_collective: runs the registered exchange (a LocalGroup's or SetCollective's) once on `buffer`, as the BA
        code does (op _lib.COLLECTIVE_ALLREDUCE_SUM: `count` fp32 values; _lib.COLLECTIVE_ALLGATHER: world slices of `count`
        bytes).  Every rank makes the same call."""
        self._check(self._lib.bba_debug_collective(self._h, int(op), C.c_void_p(buffer.data_ptr()), int(count),
                                                   self._stream_ptr(stream)))

    @classmethod
    def create_local_ranks(cls, scene, world: int, devices=None, **kw) -> List["DirectBA"]:
        """The `world` ranks of a multi-GPU job on `scene` as handles of this process (rank r on devices[r], default cuda:0),
        ready for LocalGroup.  Keyword arguments go to from_scene."""
        devices = devices or ["cuda:0"] * world
        if len(devices) != world:
            raise ValueError("one device per rank")
        return [cls.from_scene(scene, device=devices[r], rank=r, world_size=world, **kw) for r in range(world)]

    def kernel_launch_count(self) -> int:
        return int(self._lib.bba_kernel_launch_count(self._h))

    def SetProfiling(self, level: int):
        """0 off, 1 per-launch event timing, 2 timing + byte-model counters in every Gauss-Newton iteration."""
        self._check(self._lib.bba_set_profiling(self._h, int(level)))

    def GetProfile(self, reset: bool = False) -> dict:
        p = _lib.Profile()
        self._check(self._lib.bba_get_profile(self._h, C.byref(p), int(reset)))
        return {name: getattr(p, name) for name, _ in p._fields_}

    def AddKeyframeHost(self, depth, normals, radius, color, global_T_frame, min_depth, max_depth, stream=None) -> int:
        """Keyframe whose device buffers are owned by the library (uploaded from host arrays)."""
        out = C.c_int(-1)
        pose = np.ascontiguousarray(global_T_frame, np.float32)
        arrs = [np.ascontiguousarray(a) for a in (depth, normals, radius, color)]
        self._check(self._lib.bba_add_keyframe_host(self._h, arrs[0].ctypes.data, arrs[1].ctypes.data, arrs[2].ctypes.data,
                                                    arrs[3].ctypes.data, pose.ctypes.data_as(C.POINTER(C.c_float)),
                                                    float(min_depth), float(max_depth), self._stream_ptr(stream), C.byref(out)))
        kf = Keyframe.__new__(Keyframe)
        kf.frame_index, kf.min_depth, kf.max_depth = out.value, float(min_depth), float(max_depth)
        kf.depth_buffer = kf.normals_buffer = kf.radius_buffer = kf.color_buffer = None
        kf._global_T_frame = pose.copy()
        kf.id, kf._ba = out.value, self
        self._keyframes.append(kf)
        return out.value

    def UpdateKeyframeHost(self, keyframe_id: int, depth=None, normals=None, radius=None, color=None, stream=None):
        """bba_update_keyframe_host: re-uploads keyframe images from (pinned) host memory."""
        def ptr(a):
            if a is None:
                return None
            if isinstance(a, torch.Tensor):
                return a.data_ptr()
            return a.ctypes.data
        self._check(self._lib.bba_update_keyframe_host(self._h, keyframe_id, ptr(depth), ptr(normals), ptr(radius), ptr(color),
                                                       self._stream_ptr(stream)))

    # -- convenience: build from a synthetic scene ---------------------------------------------------
    @classmethod
    def from_scene(cls, scene, poses=None, use_depth_residuals=True, use_descriptor_residuals=True,
                   device=None, max_keyframes=None, host_owned=False, **kw):
        """Builds a DirectBA from a synthetic scene.  host_owned=True uploads everything through the `_host`
        entry points (library-owned device memory) -- the e2e path of bench.py."""
        kw_host_owned = host_owned
        cfg = scene.cfg
        cam_d = PinholeCamera4f(cfg.width, cfg.height, scene.depth_K)
        cam_c = PinholeCamera4f(scene.color.shape[2], scene.color.shape[1], scene.color_K)
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        ba = cls(max_surfel_count=scene.pitch, raw_to_float_depth=cfg.raw_to_float_depth, baseline_fx=cfg.baseline_fx,
                 sparse_surfel_cell_size=cfg.cell, color_camera_initial_estimate=cam_c,
                 depth_camera_initial_estimate=cam_d, use_depth_residuals=use_depth_residuals,
                 use_descriptor_residuals=use_descriptor_residuals, device=device,
                 max_keyframes=max_keyframes or max(cfg.num_keyframes, 1), **kw)
        poses = scene.poses_init if poses is None else poses
        if kw_host_owned:
            for k in range(cfg.num_keyframes):
                ba.AddKeyframeHost(scene.depth[k], scene.normals[k], scene.radius[k], scene.color[k], poses[k],
                                   scene.min_depth[k], scene.max_depth[k])
            ba.SetSurfelsHost(scene.surfels, scene.num_surfels)
            if scene.depth_a != 0.0:
                ba.SetA(scene.depth_a)
            if np.any(scene.cfactor != 0):
                ba.SetCFactorBuffer(scene.cfactor)
            return ba
        for k in range(cfg.num_keyframes):
            kf = Keyframe.from_host(k, scene.depth[k], scene.normals[k], scene.radius[k], scene.color[k], poses[k],
                                    scene.min_depth[k], scene.max_depth[k], device)
            ba.AddKeyframe(kf)
        surf = torch.from_numpy(scene.surfels).to(device)
        ba.SetSurfels(surf, scene.num_surfels)
        if scene.depth_a != 0.0:
            ba.SetA(scene.depth_a)
        if np.any(scene.cfactor != 0):
            ba.SetCFactorBuffer(scene.cfactor)
        return ba


class LocalGroup:
    """The ranks of a multi-GPU job as DirectBA handles of this process (bba_local_group_create): the library exchanges between
    them itself, through device memory and CUDA events, without a host collective.  handles[r] must have been created with
    rank r and world_size len(handles) (DirectBA.create_local_ranks); peer_stores maps every surfel replica into every rank.

        with LocalGroup(DirectBA.create_local_ranks(scene, 2)) as group:
            results = group.run(lambda rank, ba: ba.BundleAdjustment(None, False, False, False, True, True, 3, 3))

    run() is the way to drive the members: every BA-side call of a member belongs on its own thread, and all members make the
    same calls.  Close the group (or leave the with-block) before closing its members."""

    def __init__(self, handles, peer_stores: bool = False):
        self._lib = _lib.load()
        self.handles = list(handles)
        self._g = C.c_void_p()
        arr = (C.c_void_p * len(self.handles))(*[ba._h.value for ba in self.handles])
        st = self._lib.bba_local_group_create(arr, len(self.handles), int(peer_stores), C.byref(self._g))
        if st != _lib.OK:
            msg = self._lib.bba_last_error(self.handles[0]._h).decode() if self.handles else ""
            for ba in self.handles:   # (the message is on the handle the check refused)
                m = self._lib.bba_last_error(ba._h).decode()
                if m.startswith("bba_local_group_create"):
                    msg = m
            raise BadBAError(st, msg)
        # one stream per rank: two ranks on one device then queue their work side by side
        self._streams = [torch.cuda.Stream(device=ba.device) for ba in self.handles]

    def run(self, fn):
        """Calls fn(rank, ba) on one thread per rank, inside torch.cuda.device(ba.device) and on a stream of the rank's own,
        joins the threads and returns the list of their results.  Re-raises the first error.  Any error on a rank's thread
        poisons the group, also one that fn raises outside the library, so that the other ranks' exchanges return instead of
        waiting for that rank; reset() restores service."""
        import threading
        n = len(self.handles)
        results, errors = [None] * n, []
        lock = threading.Lock()

        def body(rank):
            ba = self.handles[rank]
            try:
                with torch.cuda.device(ba.device), torch.cuda.stream(self._streams[rank]):
                    results[rank] = fn(rank, ba)
                    self._streams[rank].synchronize()
            except BaseException as e:  # noqa: B036 -- handed to the calling thread
                self._lib.bba_local_group_poison(self._g)
                with lock:
                    errors.append(e)

        threads = [threading.Thread(target=body, args=(r,), name=f"bba-rank-{r}") for r in range(n)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise errors[0]
        return results

    def reset(self):
        """bba_local_group_reset: clears the poisoned state after a failed run."""
        st = self._lib.bba_local_group_reset(self._g)
        if st != _lib.OK:
            raise BadBAError(st, "bba_local_group_reset")

    def close(self):
        if getattr(self, "_g", None) is not None and self._g.value:
            self._lib.bba_local_group_destroy(self._g)
            self._g = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
