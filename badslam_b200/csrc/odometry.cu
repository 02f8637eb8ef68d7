// odometry.cu -- image-pair odometry (frame-to-keyframe direct tracking) for sm_90a, SURVEY.md 8(f4).
//
// What is computed follows the reference (BadSlam::RunOdometry bad_slam.cc:829-950, TrackFramePairwise
// pairwise_frame_tracking.cc:153-678, kernel_downsample.cu, cuda_image_processing.cu:103-206, kernel_opt_pose.cu:422-1340);
// how it is scheduled is our own:
//   * the reference runs, per Gauss-Newton iteration, 2 buffer clears + one 2-D kernel with 27-54 block-wide CUB reductions and
//     atomics + 2 device-to-host copies + a stream synchronisation, then solves the 6x6 system on the CPU -- up to 30
//     iterations on each of 5 pyramid levels, plus two cost evaluations per level (kernel_opt_pose.cc:99-260);
//   * here the WHOLE coarse-to-fine optimisation is ONE persistent launch (OdomTrackKernel): one CTA per SM walks 32x8 pixel
//     tiles, every lane keeps H (21) / b (6) / count / cost in registers over all its pixels, a warp reduces them with the
//     31-shuffle transposed butterfly, CTAs meet at a grid-wide barrier, and every CTA then solves the same 6x6 system in fp64
//     and applies the same SE3 update (replicated, deterministic control flow: no host round trip until the pose is final);
//   * the image pyramids of both frames are built by one launch per level for BOTH images.
//
// Built with -use_fast_math like the reference's kernels; the fp64 solve and the double-evaluated trigonometry of
// host_math.hpp are not affected by it.
#include "odometry.cuh"

#include <math_constants.h>

#include "device_math.cuh"
#include "host_math.hpp"

namespace bba {
namespace odom {

// ------------------------------------------------------------------------------------------------
// Stage 1: intensity / Sobel gradient magnitude of a luma texture (colour-sized).

__global__ void __launch_bounds__(256) BrightnessKernel(const __grid_constant__ BrightnessArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int f = blockIdx.z;
  if (x >= a.w || y >= a.h) return;
  const cudaTextureObject_t tex = a.luma_tex[f];
  uint8_t v;
  if (!a.use_gradmag) {
    // ComputeBrightnessKernel(texture), cuda_image_processing.cu:196-206 (truncation, no rounding offset)
    v = static_cast<uint8_t>(255.f * tex2D<float>(tex, x + 0.5f, y + 0.5f));
  } else {
    // ComputeSobelGradientMagnitudeKernel(texture), cuda_image_processing.cu:103-146; the block's halo reads of the reference
    // go through the same clamped texture
    float i[3][3];
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) i[dy + 1][dx + 1] = 255.f * tex2D<float>(tex, x + dx + 0.5f, y + dy + 0.5f);
    const float gx = 1 * i[0][2] - 1 * i[0][0] + 2 * i[1][2] - 2 * i[1][0] + 1 * i[2][2] - 1 * i[2][0];
    const float gy = 1 * i[2][0] - 1 * i[0][0] + 2 * i[2][1] - 2 * i[0][1] + 1 * i[2][2] - 1 * i[0][2];
    constexpr float kNormalizer = 255.99f / (CUDART_SQRT_TWO_F * 4 * 255.f);
    v = static_cast<uint8_t>(kNormalizer * sqrtf(gx * gx + gy * gy));
  }
  a.out[f][static_cast<size_t>(y) * a.out_pitch[f] + x] = v;
}

void LaunchBrightness(const BrightnessArgs& a, cudaStream_t stream) {
  dim3 grid((a.w + 31) / 32, (a.h + 7) / 8, 2);
  BrightnessKernel<<<grid, 256, 0, stream>>>(a);
}

// ------------------------------------------------------------------------------------------------
// Stage 2: level 0 of both images.

__device__ __forceinline__ uint16_t LoadU16(const uint16_t* base, uint32_t pitch_bytes, int x, int y) {
  return *(reinterpret_cast<const uint16_t*>(reinterpret_cast<const char*>(base) + static_cast<size_t>(y) * pitch_bytes) + x);
}
__device__ __forceinline__ void StoreU16(uint16_t* base, uint32_t pitch_bytes, int x, int y, uint16_t v) {
  *(reinterpret_cast<uint16_t*>(reinterpret_cast<char*>(base) + static_cast<size_t>(y) * pitch_bytes) + x) = v;
}

// depths[4] of a 2x2 block -> the one closest to their mean (kernel_downsample.cu:72-90, 129-150).  Returns the index or -1.
__device__ __forceinline__ int ClosestToAverage(const float (&depths)[4], float depth_sum, int depth_count) {
  if (depth_count == 0) return -1;
  const float average_depth = depth_sum / depth_count;
  int closest_index = 0;
  float closest_distance = CUDART_INF_F;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float distance = fabsf(depths[i] - average_depth);
    if (distance < closest_distance) {
      closest_index = i;
      closest_distance = distance;
    }
  }
  return closest_index;
}

__global__ void __launch_bounds__(256) Level0Kernel(const __grid_constant__ Level0Args a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int f = blockIdx.z;   // 0 base, 1 tracked
  const Image& o = a.out[f];
  if (f == 1 && a.skip_level0) {
    // CalibrateAndDownsampleImagesCUDAKernel, kernel_downsample.cu:40-105 (the cfactor cell is indexed with the DOWNSAMPLED
    // pixel coordinates there, :63-65 -- kept)
    if (x >= a.out_w || y >= a.out_h) return;
    constexpr int kOffsets[4][2] = {{0, 0}, {0, 1}, {1, 0}, {1, 1}};
    float depths[4];
    float depth_sum = 0;
    int depth_count = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint16_t raw = LoadU16(a.raw_depth[1], a.raw_depth_pitch[1], 2 * x + kOffsets[i][1], 2 * y + kOffsets[i][0]);
      if (!(raw & kInvalidDepthBit)) {
        depths[i] = RawToCalibratedDepth(a.a, a.cfactor[(y / a.cell) * a.cf_w + (x / a.cell)], a.raw_to_float, raw);
        depth_sum += depths[i];
        depth_count += 1;
      } else {
        depths[i] = CUDART_INF_F;
      }
    }
    const int c = ClosestToAverage(depths, depth_sum, depth_count);
    if (c < 0) {
      o.depth[static_cast<size_t>(y) * o.depth_pitch + x] = 0;
    } else {
      o.depth[static_cast<size_t>(y) * o.depth_pitch + x] = depths[c];
      StoreU16(o.normals, o.normals_pitch, x, y, LoadU16(a.raw_normals, a.raw_normals_pitch, 2 * x + kOffsets[c][1], 2 * y + kOffsets[c][0]));
    }
    const float color = a.downsample_color ? tex2D<float>(a.gradmag_tex[1], 2 * x + 1.0f, 2 * y + 1.0f)
                                           : tex2D<float>(a.gradmag_tex[1], x + 0.5f, y + 0.5f);
    o.color[static_cast<size_t>(y) * o.color_pitch + x] = static_cast<uint8_t>(255.f * color + 0.5f);
    return;
  }
  if (x >= a.w || y >= a.h) return;
  const uint16_t raw = LoadU16(a.raw_depth[f], a.raw_depth_pitch[f], x, y);
  float depth = 0;
  if (!(raw & kInvalidDepthBit)) depth = RawToCalibratedDepth(a.a, a.cfactor[(y / a.cell) * a.cf_w + (x / a.cell)], a.raw_to_float, raw);
  if (f == 0) {
    // CalibrateDepthAndTransformColorToDepthCUDAKernel, kernel_downsample.cu:345-372
    const float cpx = a.d2c_fx * (x + 0.5f) + a.d2c_cx;
    const float cpy = a.d2c_fy * (y + 0.5f) + a.d2c_cy;
    const bool in_bounds = cpx >= 0 && cpy >= 0 && static_cast<int>(cpx) < a.cw && static_cast<int>(cpy) < a.ch;
    o.depth[static_cast<size_t>(y) * o.depth_pitch + x] = in_bounds ? depth : 0;
    const float color = tex2D<float>(a.gradmag_tex[0], cpx, cpy);
    o.color[static_cast<size_t>(y) * o.color_pitch + x] = static_cast<uint8_t>(255.f * color + 0.5f);
  } else {
    // CalibrateDepthCUDAKernel (:404-426) + SetToReadModeNormalized (cuda_buffer.cu:82-91: factor 255, truncation)
    o.depth[static_cast<size_t>(y) * o.depth_pitch + x] = depth;
    o.color[static_cast<size_t>(y) * o.color_pitch + x] = static_cast<uint8_t>(255.f * tex2D<float>(a.gradmag_tex[1], x + 0.5f, y + 0.5f));
  }
}

void LaunchLevel0(const Level0Args& a, cudaStream_t stream) {
  dim3 grid((a.w + 31) / 32, (a.h + 7) / 8, 2);
  Level0Kernel<<<grid, 256, 0, stream>>>(a);
}

// ------------------------------------------------------------------------------------------------
// Stage 3: one pyramid level of (up to) both images.

__global__ void __launch_bounds__(256) DownsampleKernel(const __grid_constant__ DownsampleArgs a) {
  const int x = blockIdx.x * 32 + (threadIdx.x & 31);
  const int y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= a.w || y >= a.h) return;
  const Image& in = a.in[blockIdx.z];
  const Image& o = a.out[blockIdx.z];
  // DownsampleImagesCUDAKernel, kernel_downsample.cu:107-156 (block order {0,0}, {0,1}, {1,0}, {1,1} as (row, column) offsets)
  float depths[4];
  float depth_sum = 0;
  int depth_count = 0;
  // (With image sizes that are not multiples of 2^levels a coarse level can be one pixel wider than half the finer one rounded
  //  down allows -- 37 -> 18 needs column 37 -- and the reference then reads the row padding.  Clamped here: defined, and
  //  identical to the reference whenever the reference's result is defined.)
  const int x1 = min(2 * x + 1, a.in_w - 1), y1 = min(2 * y + 1, a.in_h - 1);
  const int xs[4] = {2 * x, x1, 2 * x, x1}, ys[4] = {2 * y, 2 * y, y1, y1};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    depths[i] = in.depth[static_cast<size_t>(ys[i]) * in.depth_pitch + xs[i]];
    if (depths[i] > 0) {
      depth_sum += depths[i];
      depth_count += 1;
    } else {
      depths[i] = CUDART_INF_F;
    }
  }
  const int c = ClosestToAverage(depths, depth_sum, depth_count);
  if (c < 0) {
    o.depth[static_cast<size_t>(y) * o.depth_pitch + x] = 0;
  } else {
    o.depth[static_cast<size_t>(y) * o.depth_pitch + x] = depths[c];
    StoreU16(o.normals, o.normals_pitch, x, y, LoadU16(in.normals, in.normals_pitch, xs[c], ys[c]));
  }
  const float color = tex2D<float>(in.color_tex, 2 * x + 1.0f, 2 * y + 1.0f);
  o.color[static_cast<size_t>(y) * o.color_pitch + x] = static_cast<uint8_t>(255.f * color + 0.5f);
}

void LaunchDownsample(const DownsampleArgs& a, cudaStream_t stream) {
  if (a.count <= 0) return;
  dim3 grid((a.w + 31) / 32, (a.h + 7) / 8, a.count);
  DownsampleKernel<<<grid, 256, 0, stream>>>(a);
}

// ------------------------------------------------------------------------------------------------
// Stage 4: coarse-to-fine Gauss-Newton.

// Everything one base pixel contributes at one pose estimate (the body shared by
// AccumulatePoseEstimationCoeffsFromImagesCUDAKernel_{GradientXY,GradMag} kernel_opt_pose.cu:422-885 and
// ComputeCostAndResidualCountFromImagesCUDAKernel_* :939-1296).
struct PixelEval {
  float raw_depth;        // raw depth residual
  float raw_desc1, raw_desc2;
  float Jd[6], J1[6], J2[6];
};

// Finite-difference gradient at a sample point from the four texels around it, read as point samples of the filtered texture
// exactly like DescriptorJacobianWrtProjectedPositionWithFloatTexture / ColorJacobianWrtProjectedPosition
// (cost_function.cuh:256-317, 335-352).  scale = 1 (intensities in [0, 1]) or 255.
__device__ __forceinline__ void TexelGradient(cudaTextureObject_t tex, float x, float y, float scale, float* dx, float* dy) {
  const int ix = static_cast<int>(::max(0.f, x - 0.5f));
  const int iy = static_cast<int>(::max(0.f, y - 0.5f));
  const float tx = ::max(0.f, ::min(1.f, x - 0.5f - ix));
  const float ty = ::max(0.f, ::min(1.f, y - 0.5f - iy));
  const float top_left = scale * tex2D<float>(tex, ix + 0.5f, iy + 0.5f);
  const float top_right = scale * tex2D<float>(tex, ix + 1.5f, iy + 0.5f);
  const float bottom_left = scale * tex2D<float>(tex, ix + 0.5f, iy + 1.5f);
  const float bottom_right = scale * tex2D<float>(tex, ix + 1.5f, iy + 1.5f);
  *dx = (bottom_right - bottom_left) * ty + (top_right - top_left) * (1 - ty);
  *dy = (bottom_right - top_right) * tx + (bottom_left - top_left) * (1 - tx);
}

// kernel_opt_pose.cu:170-189 / 209-221: Jacobian of a photometric residual wrt the pose from its image gradient
__device__ __forceinline__ void PhotoPoseJacobian(float gx_fx, float gy_fy, const Vec3& ls, float (&J)[6]) {
  const float inv_ls_z = 1.f / ls.z;
  const float ls_z_sq = ls.z * ls.z;
  const float inv_ls_z_sq = inv_ls_z * inv_ls_z;
  J[0] = -gx_fx * inv_ls_z;
  J[1] = -gy_fy * inv_ls_z;
  J[2] = (ls.x * gx_fx + ls.y * gy_fy) * inv_ls_z_sq;
  const float ls_x_y = ls.x * ls.y;
  J[3] = ((ls.y * ls.y + ls_z_sq) * gy_fy + ls_x_y * gx_fx) * inv_ls_z_sq;
  J[4] = -((ls.x * ls.x + ls_z_sq) * gx_fx + ls_x_y * gy_fy) * inv_ls_z_sq;
  J[5] = -(ls.x * gy_fy - ls.y * gx_fx) * inv_ls_z;
}

__device__ __forceinline__ bool DepthToColorLevel(const LevelCamera& c, float px, float py, float* cx, float* cy) {   // surfel_projection.cuh:196-207
  *cx = c.d2c_fx * px + c.d2c_cx;
  *cy = c.d2c_fy * py + c.d2c_cy;
  return *cx >= 0 && *cy >= 0 && static_cast<int>(*cx) < c.cw && static_cast<int>(*cy) < c.ch;
}

template <bool GRADMAG, bool JAC>
__device__ __forceinline__ bool EvalPixel(const Level& L, const float* __restrict__ T, float threshold_factor, float baseline_fx,
                                          bool use_depth, bool use_desc, int x, int y, PixelEval* e) {
  const LevelCamera& c = L.cam;
  const float sd = L.base.depth[static_cast<size_t>(y) * L.base.depth_pitch + x];
  if (!(sd > 0)) return false;
  // estimate_frame_T_surfel_frame.MultiplyIfResultZIsPositive(UnprojectPoint(x, y, sd)), cuda_matrix.cuh:115-124
  const Vec3 P = V3(sd * (c.fx_inv * x + c.cx_inv), sd * (c.fy_inv * y + c.cy_inv), sd);
  Vec3 lp;
  lp.z = T[8] * P.x + T[9] * P.y + T[10] * P.z + T[11];
  if (lp.z <= 0.f) return false;
  lp.x = T[0] * P.x + T[1] * P.y + T[2] * P.z + T[3];
  lp.y = T[4] * P.x + T[5] * P.y + T[6] * P.z + T[7];
  // ProjectSurfelToImage, util.cuh:98-114
  const float pxf = c.fx * (lp.x / lp.z) + c.cx;
  const float pyf = c.fy * (lp.y / lp.z) + c.cy;
  const int px = static_cast<int>(pxf), py = static_cast<int>(pyf);
  if (pxf < 0 || pyf < 0 || px >= c.w || py >= c.h) return false;
  const float pd = L.tracked.depth[static_cast<size_t>(py) * L.tracked.depth_pitch + px];
  if (!(pd > 0)) return false;
  // IsAssociatedWithPixel<false> for a surfel that is a pixel, surfel_projection_nvcc_only.cuh:178-237
  const uint16_t base_n = LoadU16(L.base.normals, L.base.normals_pitch, x, y);
  const Vec3 ln = Rotate(T, U16ToImageSpaceNormal(base_n));
  const float nx = c.fx_inv * px + c.cx_inv, ny = c.fy_inv * py + c.cy_inv;
  const float stddev = (kDepthUncertaintyFactor * fabsf(ln.x * nx + ln.y * ny + ln.z) * (pd * pd)) / baseline_fx;
  if (fabsf(lp.z - pd) > (threshold_factor * kDepthTukey) * stddev) return false;
  const float surfel_distance = sqrtf(Dot(lp, lp));
  if ((1.0f / surfel_distance) * Dot(lp, ln) > 0) return false;
  const Vec3 tn = U16ToImageSpaceNormal(LoadU16(L.tracked.normals, L.tracked.normals_pitch, px, py));
  if (Dot(ln, tn) < kCosNormalCompat) return false;
  bool visible = true;

  if (use_depth) {
    // ComputeDepthResidualInvStddevEstimate + ComputeRawDepthResidual(AndJacobian), cost_function.cuh:56-88, kernel_opt_pose.cu:45-94
    const float inv_stddev = baseline_fx / (kDepthUncertaintyFactor * fabsf(ln.x * nx + ln.y * ny + ln.z) * (pd * pd));
    const Vec3 up = V3(pd * nx, pd * ny, pd);
    e->raw_depth = inv_stddev * Dot(ln, up - lp);
    if (JAC) {
      e->Jd[0] = inv_stddev * ln.x;
      e->Jd[1] = inv_stddev * ln.y;
      e->Jd[2] = inv_stddev * ln.z;
      e->Jd[3] = inv_stddev * (-ln.y * up.z + ln.z * up.y);
      e->Jd[4] = inv_stddev * (ln.x * up.z - ln.z * up.x);
      e->Jd[5] = inv_stddev * (-ln.x * up.y + ln.y * up.x);
    }
  }

  if (use_desc) {
    const cudaTextureObject_t tex = L.tracked.color_tex;
    if (GRADMAG) {
      // kernel_opt_pose.cu:791-805, ComputeRawColorResidualAndJacobian :192-222
      float cx, cy;
      if (DepthToColorLevel(c, pxf, pyf, &cx, &cy)) {
        const float surfel_gradmag = L.base.color[static_cast<size_t>(y) * L.base.color_pitch + x];
        e->raw_desc1 = 255.f * tex2D<float>(tex, cx, cy) - surfel_gradmag;
        if (JAC) {
          float gx, gy;
          TexelGradient(tex, cx, cy, 255.f, &gx, &gy);
          PhotoPoseJacobian(gx * c.cfx, gy * c.cfy, lp, e->J1);
        }
      } else {
        visible = false;
      }
    } else if (x < c.w - 1 && y < c.h - 1) {
      // kernel_opt_pose.cu:502-566: the descriptor of the base pixel from its right / lower neighbours, the two offset points
      // placed on the pixel's tangent plane and projected into the tracked frame
      const uint8_t* row = L.base.color + static_cast<size_t>(y) * L.base.color_pitch;
      const float intensity = 1 / 255.f * row[x];
      const float t1_intensity = 1 / 255.f * row[x + 1];
      const float t2_intensity = 1 / 255.f * row[L.base.color_pitch + x];
      const float surfel_descriptor_1 = (180.f * (t1_intensity - intensity));
      const float surfel_descriptor_2 = (180.f * (t2_intensity - intensity));
      const Vec3 sn = U16ToImageSpaceNormal(base_n);
      const float nx0 = c.fx_inv * x + c.cx_inv, ny0 = c.fy_inv * y + c.cy_inv;
      const float plane_d = (nx0 * sd) * sn.x + (ny0 * sd) * sn.y + sd * sn.z;
      const float nx1 = c.fx_inv * (x + 1) + c.cx_inv, ny1 = c.fy_inv * (y + 1) + c.cy_inv;
      const float x_plus_1_depth = plane_d / (nx1 * sn.x + ny0 * sn.y + sn.z);
      const Vec3 q1 = Transform(T, V3(x_plus_1_depth * nx1, x_plus_1_depth * ny0, x_plus_1_depth));
      const float t1x = c.fx * (q1.x / q1.z) + c.cx, t1y = c.fy * (q1.y / q1.z) + c.cy;
      if (t1x < 0 || t1y < 0 || static_cast<int>(t1x) >= c.w || static_cast<int>(t1y) >= c.h) visible = false;
      const float y_plus_1_depth = plane_d / (nx0 * sn.x + ny1 * sn.y + sn.z);
      const Vec3 q2 = Transform(T, V3(y_plus_1_depth * nx0, y_plus_1_depth * ny1, y_plus_1_depth));
      const float t2x = c.fx * (q2.x / q2.z) + c.cx, t2y = c.fy * (q2.y / q2.z) + c.cy;
      if (t2x < 0 || t2y < 0 || static_cast<int>(t2x) >= c.w || static_cast<int>(t2y) >= c.h) visible = false;
      float cx, cy, c1x, c1y, c2x, c2y;
      if (visible && q1.z > 0 && q2.z > 0 && DepthToColorLevel(c, pxf, pyf, &cx, &cy) && DepthToColorLevel(c, t1x, t1y, &c1x, &c1y) &&
          DepthToColorLevel(c, t2x, t2y, &c2x, &c2y)) {
        // ComputeRawDescriptorResidual(AndJacobian)WithFloatTexture, cost_function.cuh:158-173, kernel_opt_pose.cu:144-190
        const float ci = tex2D<float>(tex, cx, cy);
        const float i1 = tex2D<float>(tex, c1x, c1y);
        const float i2 = tex2D<float>(tex, c2x, c2y);
        e->raw_desc1 = (180.f * (i1 - ci)) - surfel_descriptor_1;
        e->raw_desc2 = (180.f * (i2 - ci)) - surfel_descriptor_2;
        if (JAC) {
          float cdx, cdy, d1x, d1y, d2x, d2y;
          TexelGradient(tex, cx, cy, 1.f, &cdx, &cdy);
          TexelGradient(tex, c1x, c1y, 1.f, &d1x, &d1y);
          TexelGradient(tex, c2x, c2y, 1.f, &d2x, &d2y);
          PhotoPoseJacobian((180.f * (d1x - cdx)) * c.cfx, (180.f * (d1y - cdy)) * c.cfy, lp, e->J1);
          PhotoPoseJacobian((180.f * (d2x - cdx)) * c.cfx, (180.f * (d2y - cdy)) * c.cfy, lp, e->J2);
        }
      } else {
        visible = false;
      }
    } else {
      visible = false;
    }
  }
  return visible;
}

// cost_function.cuh:91-98, 177-185 with the multi-resolution scaling
__device__ __forceinline__ float DepthWeightScaled(float r, float s) { return TukeyWeight(r, s * kDepthTukey); }
__device__ __forceinline__ float DepthCostScaled(float r, float s) { return TukeyResidual(r, s * kDepthTukey); }
__device__ __forceinline__ float DescWeightScaled(float r, float s) { return s * kDescWeight * HuberWeight(r, kDescHuber); }
__device__ __forceinline__ float DescCostScaled(float r, float s) { return s * kDescWeight * HuberResidual(r, kDescHuber); }

// H += w J^T J (upper triangle, row-major), b += w r J   (gauss_newton.cuh:59-92, per thread)
__device__ __forceinline__ void AccumulateHb(float (&acc)[32], const float (&J)[6], float raw, float w) {
  int idx = 0;
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    const float wj = w * J[r];
#pragma unroll
    for (int c = r; c < 6; ++c) acc[idx++] += wj * J[c];
  }
  const float wr = w * raw;
#pragma unroll
  for (int i = 0; i < 6; ++i) acc[21 + i] += wr * J[i];
}

__device__ __forceinline__ unsigned int LoadAcquireU32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Grid-wide barrier of a persistent kernel whose CTAs are all resident (one per SM).  bar[0] = arrival count, bar[1] = generation.
// A CTA that waits longer than ~2^22 polls (seconds; a pass takes microseconds) gives up and raises *timeout: the launch is
// cooperative, so this can only happen after a device fault elsewhere -- the kernel must still terminate.
__device__ __forceinline__ void GridBarrier(unsigned int* bar, unsigned int* timeout) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int gen = LoadAcquireU32(bar + 1);
    __threadfence();
    if (atomicAdd(bar, 1u) == gridDim.x - 1) {
      bar[0] = 0u;
      __threadfence();
      atomicAdd(bar + 1, 1u);
    } else {
      unsigned int polls = 0;
      while (LoadAcquireU32(bar + 1) == gen) {
        __nanosleep(64);
        if (++polls > (1u << 22)) {
          *timeout = 1u;
          break;
        }
      }
    }
    __threadfence();
  }
  __syncthreads();
}

constexpr int kTrackThreads = 256;

// One pass over the base image of a level: MODE 0 accumulates H, b, residual count and cost at pose T; MODE 1 evaluates residual
// count and cost at the two poses TA and TB (ComputeCostAndResidualCountFromImagesCUDA twice, pairwise_frame_tracking.cc:433-475).
// Slots: MODE 0: 0..20 H, 21..26 b, 27 count, 28 cost.  MODE 1: 0 count A, 1 cost A, 2 count B, 3 cost B.
template <bool GRADMAG, int MODE>
__device__ __forceinline__ void LevelPass(const TrackArgs& a, const Level& L, const float* TA, const float* TB, float threshold_factor,
                                          double* s_acc, double* g_acc) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  const int tiles_x = (L.cam.w + 31) / 32, tiles_y = (L.cam.h + 7) / 8;
  bool any = false;
  for (int t = blockIdx.x; t < tiles_x * tiles_y; t += gridDim.x) {
    const int x = (t % tiles_x) * 32 + lane, y = (t / tiles_x) * 8 + warp;
    if (x >= L.cam.w || y >= L.cam.h) continue;
    PixelEval e;
    if (MODE == 0) {
      if (!EvalPixel<GRADMAG, true>(L, TA, threshold_factor, a.baseline_fx, a.use_depth, a.use_desc, x, y, &e)) continue;
      any = true;
      if (a.use_depth) {
        AccumulateHb(acc, e.Jd, e.raw_depth, DepthWeightScaled(e.raw_depth, threshold_factor));
        acc[27] += 1.f;
        acc[28] += DepthCostScaled(e.raw_depth, threshold_factor);
      }
      if (a.use_desc) {
        AccumulateHb(acc, e.J1, e.raw_desc1, DescWeightScaled(e.raw_desc1, threshold_factor));
        if (!GRADMAG) AccumulateHb(acc, e.J2, e.raw_desc2, DescWeightScaled(e.raw_desc2, threshold_factor));
        acc[27] += 1.f;   // (the reference's debug counters take the first descriptor residual only, kernel_opt_pose.cu:649-657)
        acc[28] += DescCostScaled(e.raw_desc1, threshold_factor);
      }
    } else {
#pragma unroll
      for (int arm = 0; arm < 2; ++arm) {
        if (!EvalPixel<GRADMAG, false>(L, arm ? TB : TA, threshold_factor, a.baseline_fx, a.use_depth, a.use_desc, x, y, &e)) continue;
        any = true;
        if (a.use_depth) {
          acc[2 * arm] += 1.f;
          acc[2 * arm + 1] += DepthCostScaled(e.raw_depth, threshold_factor);
        }
        if (a.use_desc) {
          acc[2 * arm] += GRADMAG ? 1.f : 2.f;
          acc[2 * arm + 1] += DescCostScaled(e.raw_desc1, threshold_factor);
          if (!GRADMAG) acc[2 * arm + 1] += DescCostScaled(e.raw_desc2, threshold_factor);
        }
      }
    }
  }
  // warp -> CTA -> grid
  if (threadIdx.x < 32) s_acc[threadIdx.x] = 0.0;
  __syncthreads();
  if (__any_sync(0xffffffffu, any)) {
    const float total = WarpTransposeReduce(acc, lane);
    if (total != 0.f) atomicAdd(&s_acc[lane], static_cast<double>(total));
  }
  __syncthreads();
  if (threadIdx.x < 32 && s_acc[threadIdx.x] != 0.0) atomicAdd(g_acc + threadIdx.x, s_acc[threadIdx.x]);
}

template <bool GRADMAG>
__global__ void __launch_bounds__(kTrackThreads, 1) OdomTrackKernel(const __grid_constant__ TrackArgs a) {
  __shared__ double s_acc[32];
  __shared__ float s_T[2][12];   // frame_T_base of the current estimate (and of the second arm of a cost comparison)
  __shared__ int s_flag;
  // replicated per-CTA state, touched by thread 0 only
  Pose est, chosen_initial;
  unsigned int pass = 0;

  auto set_matrix = [&](int slot, const Pose& base_T_frame) { ToMatrix3x4(Inverse(base_T_frame), s_T[slot]); };
  auto load_pose = [&](const float* p) {
    Pose r;
    r.q[0] = p[0]; r.q[1] = p[1]; r.q[2] = p[2]; r.q[3] = p[3];
    r.t[0] = p[4]; r.t[1] = p[5]; r.t[2] = p[6];
    return r;
  };
  // rotating accumulators: pass p sums into buffer p % 3; block 0 clears buffer (p + 1) % 3 before it arrives at the barrier of
  // pass p (its last readers left it before the barrier of pass p - 1)
  auto next_buffer_clear = [&]() {
    if (blockIdx.x == 0 && threadIdx.x < 32) a.acc[((pass + 1) % 3) * 32 + threadIdx.x] = 0.0;
  };

  if (threadIdx.x == 0) {
    est = load_pose(a.init1);
    chosen_initial = est;
  }

  if (a.debug_scale >= 0) {
    // parity hook: AccumulatePoseEstimationCoeffsFromImagesCUDA at init1, ComputeCostAndResidualCountFromImagesCUDA at init1 / init2
    const Level& L = a.level[a.debug_scale];
    const float threshold_factor = static_cast<float>(1 << a.debug_scale);
    if (threadIdx.x == 0) {
      set_matrix(0, load_pose(a.init1));
      set_matrix(1, load_pose(a.init2));
    }
    __syncthreads();
    LevelPass<GRADMAG, 0>(a, L, s_T[0], s_T[0], threshold_factor, s_acc, a.acc);
    LevelPass<GRADMAG, 1>(a, L, s_T[0], s_T[1], threshold_factor, s_acc, a.acc + 32);
    GridBarrier(a.barrier, &a.result->barrier_timeout);
    if (blockIdx.x == 0 && threadIdx.x < 36) a.result->debug[threadIdx.x] = __ldcg(a.acc + threadIdx.x);
    return;
  }

  for (int scale = a.num_scales - 1; scale >= a.first_scale; --scale) {
    const Level& L = a.level[scale];
    const float scaling_factor = static_cast<float>(1 << scale);
    const float threshold_factor = scaling_factor;   // pairwise_frame_tracking.cc:419

    if (scale != a.num_scales - 1 || a.test_different_initial_estimates) {
      // pairwise_frame_tracking.cc:427-508: continue from the better of (last scale's result | initial estimate), resp. of the
      // two initial estimates on the coarsest scale
      Pose arm_a, arm_b;
      if (threadIdx.x == 0) {
        arm_a = (scale != a.num_scales - 1) ? est : load_pose(a.init1);
        arm_b = (scale != a.num_scales - 1) ? chosen_initial : load_pose(a.init2);
        set_matrix(0, arm_a);
        set_matrix(1, arm_b);
      }
      __syncthreads();
      double* g = a.acc + (pass % 3) * 32;
      LevelPass<GRADMAG, 1>(a, L, s_T[0], s_T[1], threshold_factor, s_acc, g);
      next_buffer_clear();
      GridBarrier(a.barrier, &a.result->barrier_timeout);
      if (threadIdx.x == 0) {
        const unsigned int count_a = static_cast<unsigned int>(__ldcg(g + 0) + 0.5), count_b = static_cast<unsigned int>(__ldcg(g + 2) + 0.5);
        const float cost_a = static_cast<float>(__ldcg(g + 1)), cost_b = static_cast<float>(__ldcg(g + 3));
        bool take_a;
        if (count_a > 2 * count_b) take_a = true;
        else if (count_b > 2 * count_a) take_a = false;
        else take_a = cost_a < cost_b;
        est = take_a ? arm_a : arm_b;
        if (scale == a.num_scales - 1) chosen_initial = est;
        if (blockIdx.x == 0) a.result->chose_initial[scale] = take_a ? 0 : 1;
      }
      ++pass;
    } else if (blockIdx.x == 0 && threadIdx.x == 0) {
      a.result->chose_initial[scale] = -1;
    }

    int iteration = 0;
    for (; iteration < a.max_iterations;) {
      if (threadIdx.x == 0) set_matrix(0, est);
      __syncthreads();
      double* g = a.acc + (pass % 3) * 32;
      LevelPass<GRADMAG, 0>(a, L, s_T[0], s_T[0], threshold_factor, s_acc, g);
      next_buffer_clear();
      GridBarrier(a.barrier, &a.result->barrier_timeout);
      if (threadIdx.x == 0) {
        // the reference's buffers are fp32 and are cast to double for the solve (pairwise_frame_tracking.cc:557-566)
        double H[21], b[6], xd[6];
        for (int j = 0; j < 21; ++j) H[j] = static_cast<double>(static_cast<float>(__ldcg(g + j)));
        for (int j = 0; j < 6; ++j) b[j] = static_cast<double>(static_cast<float>(__ldcg(g + 21 + j)));
        SolveLDLT<6>(H, b, xd);
        float x[6], step[6];
        // damping, pairwise_frame_tracking.cc:581-590
        float damping = 1.f;
        if (scale == a.num_scales - 2) damping = 0.5f;
        else if (scale == a.num_scales - 1) damping = 0.25f;
        for (int j = 0; j < 6; ++j) {
          x[j] = static_cast<float>(xd[j]);
          step[j] = -damping * x[j];
        }
        est = Compose(est, Exp(step));
        // IsScaleNPoseEstimationConverged, convergence_analysis.h:56-63 (both thresholds 1e-8: no rotation rescaling)
        const float sq = x[0] * x[0] + x[1] * x[1] + x[2] * x[2] + x[3] * x[3] + x[4] * x[4] + x[5] * x[5];
        s_flag = (sq < scaling_factor * scaling_factor * 1e-08f) ? 1 : 0;
        if (blockIdx.x == 0) {
          a.result->residual_count = static_cast<unsigned int>(__ldcg(g + 27) + 0.5);
          a.result->residual_sum = static_cast<float>(__ldcg(g + 28));
        }
      }
      ++pass;
      ++iteration;
      __syncthreads();
      if (s_flag) break;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) a.result->iterations[scale] = iteration;
    __syncthreads();
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (int j = 0; j < 4; ++j) a.result->base_T_frame[j] = est.q[j];
    for (int j = 0; j < 3; ++j) a.result->base_T_frame[4 + j] = est.t[j];
    a.result->passes = pass;
  }
}

void LaunchTrack(const TrackArgs& a, int sm_count, cudaStream_t stream) {
  // one CTA per SM (all co-resident: the grid barrier needs it), never more CTAs than the finest level has tiles
  const Level& L0 = a.level[a.first_scale];
  const int tiles = ((L0.cam.w + 31) / 32) * ((L0.cam.h + 7) / 8);
  const int grid = tiles < sm_count ? (tiles > 0 ? tiles : 1) : sm_count;
  // cooperative launch: the runtime guarantees that all CTAs are resident at the same time (or refuses the launch)
  void* params[] = {const_cast<TrackArgs*>(&a)};
  if (a.use_gradmag) cudaLaunchCooperativeKernel(reinterpret_cast<void*>(OdomTrackKernel<true>), dim3(grid), dim3(kTrackThreads), params, 0, stream);
  else cudaLaunchCooperativeKernel(reinterpret_cast<void*>(OdomTrackKernel<false>), dim3(grid), dim3(kTrackThreads), params, 0, stream);
}

}  // namespace odom
}  // namespace bba
