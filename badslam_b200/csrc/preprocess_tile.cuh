// Keyframe preprocessing: raw RGB-D frame -> the four keyframe buffers the BA path reads (SURVEY.md 8(f3)).
//
// The reference runs five kernels per frame, each a full pass over the image through HBM (BadSlam::PreprocessFrame,
// bad_slam.cc:692-765, and ComputeMinMaxDepthCUDA at keyframe creation, bad_slam.cc:978):
//   ComputeBrightnessCUDA                          cuda_image_processing.cu:165-193   rgb -> rgba with .w = luma
//   BilateralFilteringAndDepthCutoffCUDA           cuda_depth_processing.cu:42-128    raw depth -> filtered depth "A"
//   ComputeNormalsCUDA                             cuda_depth_processing.cu:134-276   A -> depth "B" + normals
//   ComputePointRadiiAndRemoveIsolatedPixelsCUDA   cuda_depth_processing.cu:295-383   B -> radius^2 (half) + final depth
//   ComputeMinMaxDepthCUDA                         cuda_depth_processing.cu:390-465   final depth -> min / max depth
// Here one CTA owns a 32x32 tile of the depth image, stages the raw depth of the tile plus its halo in shared memory once and
// runs the depth stages back to back on it (A on tile+2, B on tile+1, radius / final depth / min-max on the tile); the raw
// depth is read from HBM once and the intermediate images never exist in memory.
// For a raw frame (bba_preprocess_raw_frame) a stage 0 in front of them builds that raw depth from the sensor's image: n
// passes of the median densify filter on a halo grown by n pixels, or the median downscaling of the full-resolution depth; the
// colour chunks then read the 2^L x 2^L block of each output pixel and halve it L times in registers (DESIGN.md 3.6b).
//
// This header holds the tile program itself, written against a small "team" interface (thread index, thread count, barrier,
// min/max commit) so that the same code runs as a CUDA block (preprocess.cu) and, one thread at a time, on the host in the
// CPU test-suite (tests/test_oracle_preprocess.py compiles it with g++ and compares it with oracle/preprocess_oracle.c).
// The host instantiation is a test harness, not a fallback: the library only ever launches the CUDA kernel.
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#include <cuda_fp16.h>

#include "launch.hpp"
#define BBA_PRE_HD __host__ __device__ __forceinline__
#else
#define BBA_PRE_HD inline
#endif
#if defined(__CUDA_ARCH__)
#define BBA_PRE_UNROLL _Pragma("unroll")   // register arrays: every index must be a constant
#else
#define BBA_PRE_UNROLL
#endif

namespace bba {
namespace pre {

constexpr uint16_t kUnknownDepth = 65535;      // kernels.cuh:41
constexpr uint16_t kInvalidDepthBit = 0x8000;  // kernels.cuh:38
constexpr int kTile = 32;                      // output tile edge
constexpr int kHaloA = 2;                      // filtered depth is needed on tile +- 2 (normals of the 4-neighbours' neighbours)
constexpr int kMaxFilterRadius = 16;

struct FrameArgs {
  // depth camera / deformation model (DirectBA members, direct_ba.h:420-470)
  int w, h;
  float fx_inv, fy_inv, cx_inv, cy_inv;        // PixelCenterUnprojector (surfel_projection.cuh:92-99)
  float raw_to_float, a;
  int cell, cf_w;
  const float* cfactor;                        // dense [cf_h][cf_w]
  // bilateral filter (cuda_depth_processing.cu:100-128)
  float denom_xy, denom_value;                 // 2 sigma_xy^2, 2 sigma_value^2
  int radius, radius_squared;
  uint16_t max_depth;                          // raw units
  // images (pitches in bytes)
  const uint16_t* raw_depth; uint32_t raw_pitch;
  uint16_t* out_depth; uint32_t out_depth_pitch;
  uint16_t* out_normals; uint32_t out_normals_pitch;
  uint16_t* out_radius; uint32_t out_radius_pitch;
  float* min_max;                              // [2], initialised to {+inf, 0} (cuda_depth_processing.cc:41)
  // colour image
  int cw, ch;
  const uint8_t* rgb; uint32_t rgb_pitch;      // uchar3
  uint8_t* rgba; uint32_t rgba_pitch;          // uchar4, .w = luma
  int tiles_x, tiles_y;                        // depth tiles; CTAs behind them convert colour rows
  // stage 0 of a raw frame (bba_preprocess_raw_frame); all 0 for bba_preprocess_frame
  int median_iterations;                       // MedianFilterAndDensifyDepthMap passes, 0..kMaxMedianIterations
  int depth_level;                             // pyramid_level_for_depth: raw_depth (raw_w x raw_h) is downscaled to w x h
  int raw_w, raw_h;
  int color_level;                             // pyramid_level_for_color: rgb is (cw << color_level) x (ch << color_level)
};

// Stage 0: how the raw depth of a tile (the input of the bilateral filter) is produced.
enum class Stage0 { kCopy, kMedian, kDownscale };
constexpr int kMaxMedianIterations = 8;        // halo growth: 2 px of shared memory edge per iteration
constexpr int kMaxPyramidLevel = 3;            // boxes of up to 8 x 8 raw pixels, median selected in registers

BBA_PRE_HD int RawEdge(int radius) { return kTile + 2 * (kHaloA + radius); }
BBA_PRE_HD int SharedWords(int radius) {   // u16 elements: raw | A | B
  const int e = RawEdge(radius);
  return e * e + (kTile + 4) * (kTile + 4) + (kTile + 2) * (kTile + 2);
}
// With n median iterations the raw depth is staged n pixels further out and filtered ping-pong between two buffers, each pass
// on a region one pixel smaller: S0 (edge + 2n)^2 | S1 (edge + 2n - 2)^2 | A | B.  n = 8, radius 16: 32.5 KB.
BBA_PRE_HD int SharedWordsRaw(int radius, int median_iterations) {
  if (median_iterations <= 0) return SharedWords(radius);
  const int e0 = RawEdge(radius) + 2 * median_iterations;
  return e0 * e0 + (e0 - 2) * (e0 - 2) + (kTile + 4) * (kTile + 4) + (kTile + 2) * (kTile + 2);
}

template <typename T>
BBA_PRE_HD T* RowPtr(T* base, uint32_t pitch, int y) {
  return reinterpret_cast<T*>(reinterpret_cast<char*>(base) + static_cast<size_t>(y) * pitch);
}
template <typename T>
BBA_PRE_HD const T* RowPtr(const T* base, uint32_t pitch, int y) {
  return reinterpret_cast<const T*>(reinterpret_cast<const char*>(base) + static_cast<size_t>(y) * pitch);
}

// __float2half_rn as bits (cuda_depth_processing.cu:355).
BBA_PRE_HD uint16_t FloatToHalfBits(float f) {
#if defined(__CUDA_ARCH__)
  return __half_as_ushort(__float2half_rn(f));
#else
  union { float f; uint32_t u; } v; v.f = f;
  const uint32_t sign = (v.u >> 16) & 0x8000u;
  const uint32_t mag = v.u & 0x7fffffffu;
  if (mag >= 0x7f800000u) return static_cast<uint16_t>(sign | (mag > 0x7f800000u ? 0x7e00u : 0x7c00u));
  if (mag >= 0x477ff000u) return static_cast<uint16_t>(sign | 0x7c00u);            // rounds to >= 65520 -> inf
  if (mag < 0x33000001u) return static_cast<uint16_t>(sign);                        // <= 2^-25 -> 0 (ties to even)
  const int exp = static_cast<int>(mag >> 23) - 127;
  uint32_t man = (mag & 0x7fffffu) | 0x800000u;
  int shift = (exp < -14) ? (13 + (-14 - exp)) : 13;                                // subnormal halves lose more bits
  const uint32_t halfway = 1u << (shift - 1);
  const uint32_t rem = man & ((1u << shift) - 1);
  uint32_t q = man >> shift;
  if (rem > halfway || (rem == halfway && (q & 1u))) ++q;
  const uint32_t bits = (exp < -14) ? q : ((static_cast<uint32_t>(exp + 15 - 1) << 10) + q);   // carry of q propagates into the exponent
  return static_cast<uint16_t>(sign | bits);
#endif
}

// static_cast<u16>(float) as nvcc compiles it (F2I.U32.TRUNC, low 16 bits stored).  The filtered depth is a weighted mean of
// u16 samples, so it never reaches 65536; the host build only has to agree below that.
BBA_PRE_HD uint16_t TruncToU16(float f) {
#if defined(__CUDA_ARCH__)
  return static_cast<uint16_t>(f);
#else
  if (!(f > 0.f)) return 0;
  return f >= 65535.f ? static_cast<uint16_t>(65535) : static_cast<uint16_t>(f);
#endif
}

// util.cuh:121-136
BBA_PRE_HD uint16_t ImageSpaceNormalToU16(float x, float y) {
  const int8_t qx = static_cast<int8_t>(x * 127 + ((x > 0) ? 0.5f : -0.5f));
  const int8_t qy = static_cast<int8_t>(y * 127 + ((y > 0) ? 0.5f : -0.5f));
  return static_cast<uint16_t>(static_cast<uint8_t>(qx)) | static_cast<uint16_t>(static_cast<uint16_t>(static_cast<uint8_t>(qy)) << 8);
}

// util.cuh:62-69
BBA_PRE_HD float CalibratedDepth(const FrameArgs& f, int x, int y, uint16_t raw) {
  const float cfactor = f.cfactor[static_cast<size_t>(y / f.cell) * f.cf_w + (x / f.cell)];
  const float inv_depth = 1.0f / (f.raw_to_float * raw);
  return 1.f / (inv_depth + cfactor * expf(-f.a * inv_depth));
}

// BilateralFilteringAndDepthCutoffCUDAKernel (cuda_depth_processing.cu:42-98) for the pixel (x, y) of the image; `raw` is the
// shared-memory copy of the raw depth, origin (rx0, ry0), row length `edge`; pixels outside the image hold 0 there, which the
// filter skips exactly like the reference's clamped window does.
BBA_PRE_HD uint16_t BilateralPixel(const FrameArgs& f, const uint16_t* raw, int edge, int rx0, int ry0, int x, int y) {
  const uint16_t center_value = raw[(y - ry0) * edge + (x - rx0)];
  if (center_value == 0 || center_value > f.max_depth) return kUnknownDepth;
  const float inv_center_value = 1.0f / (f.raw_to_float * center_value);
  float sum = 0;
  float weight = 0;
  for (int dy = -f.radius; dy <= f.radius; ++dy) {
    const uint16_t* row = raw + (y + dy - ry0) * edge + (x - rx0);
    for (int dx = -f.radius; dx <= f.radius; ++dx) {
      const int grid_distance_squared = dx * dx + dy * dy;
      if (grid_distance_squared > f.radius_squared) continue;
      const uint16_t sample = row[dx];
      if (sample == 0) continue;
      const float inv_sample = 1.0f / (f.raw_to_float * sample);
      float value_distance_squared = inv_center_value - inv_sample;
      value_distance_squared *= value_distance_squared;
      const float w = expf(-grid_distance_squared / f.denom_xy + -value_distance_squared / f.denom_value);
      sum += w * inv_sample;
      weight += w;
    }
  }
  return (weight == 0) ? kUnknownDepth : TruncToU16(1.0f / (f.raw_to_float * sum / weight));
}

struct Float3 { float x, y, z; };
BBA_PRE_HD Float3 Sub(const Float3& a, const Float3& b) { return Float3{a.x - b.x, a.y - b.y, a.z - b.z}; }
BBA_PRE_HD float SquaredLength(const Float3& a) { return a.x * a.x + a.y * a.y + a.z * a.z; }
BBA_PRE_HD Float3 Unproject(const FrameArgs& f, int x, int y, float depth) {   // surfel_projection.cuh:108-112
  return Float3{depth * (f.fx_inv * x + f.cx_inv), depth * (f.fy_inv * y + f.cy_inv), depth};
}

// The normal of ComputeNormalsCUDAKernel (cuda_depth_processing.cu:170-250) from the five filtered raw depths.
BBA_PRE_HD uint16_t NormalPixel(const FrameArgs& f, int x, int y, uint16_t c, uint16_t l, uint16_t t, uint16_t r, uint16_t b) {
  const Float3 left_point = Unproject(f, x - 1, y, CalibratedDepth(f, x - 1, y, l));
  const Float3 top_point = Unproject(f, x, y - 1, CalibratedDepth(f, x, y - 1, t));
  const Float3 right_point = Unproject(f, x + 1, y, CalibratedDepth(f, x + 1, y, r));
  const Float3 bottom_point = Unproject(f, x, y + 1, CalibratedDepth(f, x, y + 1, b));
  const Float3 center_point = Unproject(f, x, y, CalibratedDepth(f, x, y, c));
  constexpr float kRatioThresholdSquared = 2.f * 2.f;

  const float left_dist_squared = SquaredLength(Sub(left_point, center_point));
  const float right_dist_squared = SquaredLength(Sub(right_point, center_point));
  const float left_right_ratio = left_dist_squared / right_dist_squared;
  Float3 left_to_right;
  if (left_right_ratio < kRatioThresholdSquared && left_right_ratio > 1.f / kRatioThresholdSquared) {
    left_to_right = Sub(right_point, left_point);
  } else if (left_dist_squared < right_dist_squared) {
    left_to_right = Sub(center_point, left_point);
  } else {
    left_to_right = Sub(right_point, center_point);
  }

  const float bottom_dist_squared = SquaredLength(Sub(bottom_point, center_point));
  const float top_dist_squared = SquaredLength(Sub(top_point, center_point));
  const float bottom_top_ratio = bottom_dist_squared / top_dist_squared;
  Float3 bottom_to_top;
  if (bottom_top_ratio < kRatioThresholdSquared && bottom_top_ratio > 1.f / kRatioThresholdSquared) {
    bottom_to_top = Sub(top_point, bottom_point);
  } else if (bottom_dist_squared < top_dist_squared) {
    bottom_to_top = Sub(center_point, bottom_point);
  } else {
    bottom_to_top = Sub(top_point, center_point);
  }

  // CrossProduct (cuda_util.cuh:76-80)
  float nx = left_to_right.y * bottom_to_top.z - bottom_to_top.y * left_to_right.z;
  float ny = bottom_to_top.x * left_to_right.z - left_to_right.x * bottom_to_top.z;
  const float nz = left_to_right.x * bottom_to_top.y - bottom_to_top.x * left_to_right.y;
  const float length = sqrtf(nx * nx + ny * ny + nz * nz);
  if (!(length > 1e-6f)) {
    nx = 0;
    ny = 0;
  } else {
    const float inv_length = ((f.fy_inv < 0) ? -1.0f : 1.0f) / length;
    nx *= inv_length;
    ny *= inv_length;
  }
  return ImageSpaceNormalToU16(nx, ny);
}

// ComputePointRadius (cuda_depth_processing.cu:295-328): squared distance to the closest of the valid 4-neighbours.
BBA_PRE_HD float PointRadius(const FrameArgs& f, int x, int y, uint16_t c, const uint16_t nb[4], int* neighbor_count) {
  const float depth = f.raw_to_float * c;
  const Float3 local{depth * (f.fx_inv * x + f.cx_inv), depth * (f.fy_inv * y + f.cy_inv), depth};
  const int ox[4] = {0, -1, 1, 0}, oy[4] = {-1, 0, 0, 1};   // the reference's 3x3 raster order without the diagonals
  float min_sq = INFINITY;
  int count = 0;
  for (int i = 0; i < 4; ++i) {
    if (nb[i] & kInvalidDepthBit) continue;
    ++count;
    const float dd = f.raw_to_float * nb[i];
    const Float3 other{dd * (f.fx_inv * (x + ox[i]) + f.cx_inv), dd * (f.fy_inv * (y + oy[i]) + f.cy_inv), dd};
    const float dist = SquaredLength(Sub(other, local));
    if (dist < min_sq) min_sq = dist;
  }
  *neighbor_count = count;
  return min_sq;
}

// ComputeBrightnessKernel (cuda_image_processing.cu:165-176)
BBA_PRE_HD uint8_t Luma(uint8_t r, uint8_t g, uint8_t b) {
  return static_cast<uint8_t>((0.299f * r + 0.587f * g + 0.114f * b) + 0.5f);
}

// ---- stage 0 of a raw frame: median densify filter / median downscaling (the reference runs both on the host) ----

// a / b rounded to nearest: -use_fast_math would otherwise turn the division into an approximate reciprocal product, and the
// reference computes these means on the CPU.
BBA_PRE_HD float DivRn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

constexpr uint32_t kExcluded = 0x10000u;   // a slot without a value: larger than every u16, so it sorts behind the valid ones

// The median of the `count` valid entries of v (the others hold kExcluded) as the reference's sort-based code picks it
// (preprocessing.cc:66-79, image.h:1036-1047): odd count -> the middle value; even count -> the lower middle value if it is
// strictly closer to the mean (fp32 sum / count; the sums of at most 64 u16 values are exact) than the upper one, else the
// upper one.  Counting selection: v[i] is the k-th smallest iff #{v < v[i]} <= k < #{v <= v[i]}; fully unrolled, so v stays
// in registers.
template <int N>
BBA_PRE_HD uint16_t SortedMedian(const uint32_t (&v)[N], int count, float sum) {
  const int k_lo = (count - 1) >> 1, k_hi = count >> 1;
  uint32_t lo = 0, hi = 0;
BBA_PRE_UNROLL
  for (int i = 0; i < N; ++i) {
    int less = 0, leq = 0;
BBA_PRE_UNROLL
    for (int j = 0; j < N; ++j) {
      less += v[j] < v[i] ? 1 : 0;
      leq += v[j] <= v[i] ? 1 : 0;
    }
    if (less <= k_lo && k_lo < leq) lo = v[i];
    if (less <= k_hi && k_hi < leq) hi = v[i];
  }
  if (count & 1) return static_cast<uint16_t>(hi);
  const float mean = DivRn(sum, static_cast<float>(count));
  return static_cast<uint16_t>(fabsf(static_cast<float>(lo) - mean) < fabsf(static_cast<float>(hi) - mean) ? lo : hi);
}

// MedianFilterAndDensifyDepthMap (preprocessing.cc:40-85) for one pixel: `src` holds the previous pass with row length `es`,
// (lx, ly) is the pixel there.  Pixels outside the image hold 0 in every pass, so skipping zeros reproduces the reference's
// window clamped to the image.  Fewer than 2 non-zero values in the 3x3 window: the pixel keeps its value.
BBA_PRE_HD uint16_t MedianDensifyPixel(const uint16_t* src, int es, int lx, int ly) {
  uint32_t v[9];
  int count = 0;
  float sum = 0;
BBA_PRE_UNROLL
  for (int k = 0; k < 9; ++k) {
    const uint16_t u = src[(ly + k / 3 - 1) * es + (lx + k % 3 - 1)];
    v[k] = u ? u : kExcluded;
    count += u ? 1 : 0;
    sum += static_cast<float>(u);
  }
  if (count < 2) return src[ly * es + lx];
  return SortedMedian(v, count, sum);
}

// Image::DownscaleUsingMedianWhileExcluding(0, w, h) (libvis image.h:1003-1053) for the output pixel (x, y): the median of
// the non-zero raw pixels of its box [W x / w, W (x + 1) / w) x [H y / h, H (y + 1) / h) (u32 arithmetic like the reference),
// 0 for a box without one.  The host checks W <= w 2^kLevel and H <= h 2^kLevel, so a box spans at most 2^kLevel pixels per axis.
template <int kLevel>
BBA_PRE_HD uint16_t DownscaledPixel(const FrameArgs& f, int x, int y) {
  constexpr int S = 1 << kLevel;
  const uint32_t W = static_cast<uint32_t>(f.raw_w), H = static_cast<uint32_t>(f.raw_h);
  const uint32_t w = static_cast<uint32_t>(f.w), h = static_cast<uint32_t>(f.h);
  const uint32_t sx0 = (W * static_cast<uint32_t>(x)) / w, sx1 = (W * static_cast<uint32_t>(x + 1)) / w;
  const uint32_t sy0 = (H * static_cast<uint32_t>(y)) / h, sy1 = (H * static_cast<uint32_t>(y + 1)) / h;
  uint32_t v[S * S];
  int count = 0;
  float sum = 0;
BBA_PRE_UNROLL
  for (int dy = 0; dy < S; ++dy) {
    const bool row_in = sy0 + dy < sy1;
    const uint16_t* row = RowPtr(f.raw_depth, f.raw_pitch, static_cast<int>(row_in ? sy0 + dy : sy0));
BBA_PRE_UNROLL
    for (int dx = 0; dx < S; ++dx) {
      const uint16_t u = (row_in && sx0 + dx < sx1) ? row[sx0 + dx] : static_cast<uint16_t>(0);
      v[dy * S + dx] = u ? u : kExcluded;
      count += u ? 1 : 0;
      sum += static_cast<float>(u);
    }
  }
  if (count == 0) return 0;
  return SortedMedian(v, count, sum);
}

// One depth tile.  `Team` provides: int tid(), int size(), void sync(), void commit_min_max(float mn, float mx, float* out).
// kS0 selects stage 0 (kLevel: the depth pyramid level of kDownscale); everything after it is the same for all of them.
template <class Team, Stage0 kS0 = Stage0::kCopy, int kLevel = 0>
BBA_PRE_HD void DepthTile(const FrameArgs& f, int tile_x, int tile_y, uint16_t* smem, Team team) {
  const int halo = kHaloA + f.radius;
  const int edge = RawEdge(f.radius);
  uint16_t* raw = smem;
  uint16_t* A = raw + edge * edge;                       // (kTile+4)^2, origin (x0-2, y0-2)
  uint16_t* B = A + (kTile + 4) * (kTile + 4);           // (kTile+2)^2, origin (x0-1, y0-1)
  const int x0 = tile_x * kTile, y0 = tile_y * kTile;
  const int rx0 = x0 - halo, ry0 = y0 - halo;

  if constexpr (kS0 == Stage0::kMedian) {
    // raw depth of the tile, its halo and n more pixels; then n passes, pass `it` on the region n - it pixels beyond the halo
    const int n = f.median_iterations;
    const int e0 = edge + 2 * n;
    uint16_t* src = smem;
    uint16_t* dst = smem + e0 * e0;
    A = dst + (e0 - 2) * (e0 - 2);
    B = A + (kTile + 4) * (kTile + 4);
    for (int i = team.tid(); i < e0 * e0; i += team.size()) {
      const int ly = i / e0, lx = i - ly * e0;
      const int x = rx0 - n + lx, y = ry0 - n + ly;
      uint16_t v = 0;
      if (x >= 0 && y >= 0 && x < f.w && y < f.h) v = RowPtr(f.raw_depth, f.raw_pitch, y)[x];
      src[i] = v;
    }
    team.sync();
    for (int it = 1; it <= n; ++it) {
      const int es = e0 - 2 * (it - 1), ed = es - 2, o = n - it;   // dst origin: (rx0 - o, ry0 - o)
      for (int i = team.tid(); i < ed * ed; i += team.size()) {
        const int ly = i / ed, lx = i - ly * ed;
        const int x = rx0 - o + lx, y = ry0 - o + ly;
        uint16_t v = 0;                                   // outside the image: stays "no measurement" in every pass
        if (x >= 0 && y >= 0 && x < f.w && y < f.h) v = MedianDensifyPixel(src, es, lx + 1, ly + 1);
        dst[i] = v;
      }
      team.sync();
      uint16_t* t = src; src = dst; dst = t;
    }
    raw = src;                                           // edge x edge, origin (rx0, ry0)
  } else {
    // raw depth of the tile and its halo (downscaled: the box medians of the full-resolution image); 0 (= no measurement)
    // outside the image
    for (int i = team.tid(); i < edge * edge; i += team.size()) {
      const int ly = i / edge, lx = i - ly * edge;
      const int x = rx0 + lx, y = ry0 + ly;
      uint16_t v = 0;
      if (x >= 0 && y >= 0 && x < f.w && y < f.h) {
        if constexpr (kS0 == Stage0::kDownscale) v = DownscaledPixel<kLevel>(f, x, y);
        else v = RowPtr(f.raw_depth, f.raw_pitch, y)[x];
      }
      raw[i] = v;
    }
    team.sync();
  }

  // A: bilateral filter + depth cut-off on tile +- 2
  constexpr int ea = kTile + 4;
  for (int i = team.tid(); i < ea * ea; i += team.size()) {
    const int ly = i / ea, lx = i - ly * ea;
    const int x = x0 - 2 + lx, y = y0 - 2 + ly;
    uint16_t v = kUnknownDepth;
    if (x >= 0 && y >= 0 && x < f.w && y < f.h) v = BilateralPixel(f, raw, edge, rx0, ry0, x, y);
    A[i] = v;
  }
  team.sync();

  // B: pixels without a complete 4-neighbourhood are dropped; normals for the tile itself
  constexpr int eb = kTile + 2;
  for (int i = team.tid(); i < eb * eb; i += team.size()) {
    const int ly = i / eb, lx = i - ly * eb;
    const int x = x0 - 1 + lx, y = y0 - 1 + ly;
    if (x < 0 || y < 0 || x >= f.w || y >= f.h) { B[i] = kUnknownDepth; continue; }
    const bool inner = lx >= 1 && ly >= 1 && lx <= kTile && ly <= kTile;
    uint16_t depth = kUnknownDepth, normal = 0;   // ImageSpaceNormalToU16(0, 0) == 0
    if (!(x < 1 || y < 1 || x >= f.w - 1 || y >= f.h - 1)) {
      const uint16_t* a = A + (ly + 1) * ea + (lx + 1);
      const uint16_t c = a[0], l = a[-1], r = a[1], t = a[-ea], b = a[ea];
      if (!((c | l | r | t | b) & kInvalidDepthBit)) {
        depth = c;
        if (inner) normal = NormalPixel(f, x, y, c, l, t, r, b);
      }
    }
    B[i] = depth;
    if (inner) RowPtr(f.out_normals, f.out_normals_pitch, y)[x] = normal;
  }
  team.sync();

  // radius^2, removal of pixels without four valid neighbours, min / max depth
  float mn = INFINITY, mx = 0;
  for (int i = team.tid(); i < kTile * kTile; i += team.size()) {
    const int ly = i / kTile, lx = i - ly * kTile;
    const int x = x0 + lx, y = y0 + ly;
    if (x >= f.w || y >= f.h) continue;
    const uint16_t* b = B + (ly + 1) * eb + (lx + 1);
    const uint16_t c = b[0];
    uint16_t depth = kUnknownDepth, radius = 0;
    if (!(c & kInvalidDepthBit)) {
      const uint16_t nb[4] = {b[-eb], b[-1], b[1], b[eb]};
      int count;
      const float r2 = PointRadius(f, x, y, c, nb, &count);
      if (count >= 4) {
        depth = c;
        radius = FloatToHalfBits(r2);
        const float d = f.raw_to_float * c;
        mn = fminf(mn, d);
        mx = fmaxf(mx, d);
      }
    }
    RowPtr(f.out_depth, f.out_depth_pitch, y)[x] = depth;
    RowPtr(f.out_radius, f.out_radius_pitch, y)[x] = radius;
  }
  team.commit_min_max(mn, mx, f.min_max);
}

struct Rgb8 { uint8_t r, g, b; };

// Pixel (x, y) of level kLevel of the colour pyramid of rgb: ImagePyramid (image_cache.h:205-231) applies
// Image::DownscaleToHalfSize (libvis image.h:929-948) once per level, a / 4 + b / 4 + c / 4 + d / 4 per channel with
// truncation -- level by level, which is not one average over the 2^kLevel x 2^kLevel block.
template <int kLevel>
BBA_PRE_HD Rgb8 PyramidColor(const FrameArgs& f, int x, int y) {
  if constexpr (kLevel == 0) {
    const uint8_t* s = RowPtr(f.rgb, f.rgb_pitch, y) + 3 * x;
    return Rgb8{s[0], s[1], s[2]};
  } else {
    const Rgb8 a = PyramidColor<kLevel - 1>(f, 2 * x, 2 * y), b = PyramidColor<kLevel - 1>(f, 2 * x + 1, 2 * y);
    const Rgb8 c = PyramidColor<kLevel - 1>(f, 2 * x, 2 * y + 1), d = PyramidColor<kLevel - 1>(f, 2 * x + 1, 2 * y + 1);
    return Rgb8{static_cast<uint8_t>(a.r / 4 + b.r / 4 + c.r / 4 + d.r / 4),
                static_cast<uint8_t>(a.g / 4 + b.g / 4 + c.g / 4 + d.g / 4),
                static_cast<uint8_t>(a.b / 4 + b.b / 4 + c.b / 4 + d.b / 4)};
  }
}

// One chunk of colour pixels (rows are split into chunks of kTile * kTile pixels); kLevel: pyramid level of the rgb input.
template <class Team, int kLevel = 0>
BBA_PRE_HD void ColorChunk(const FrameArgs& f, int chunk, Team team) {
  const long long total = static_cast<long long>(f.cw) * f.ch;
  const long long begin = static_cast<long long>(chunk) * (kTile * kTile);
  for (int i = team.tid(); i < kTile * kTile; i += team.size()) {
    const long long p = begin + i;
    if (p >= total) break;
    const int y = static_cast<int>(p / f.cw), x = static_cast<int>(p - static_cast<long long>(y) * f.cw);
    const Rgb8 src = PyramidColor<kLevel>(f, x, y);
    const uint8_t r = src.r, g = src.g, b = src.b;
    uint8_t* dst = RowPtr(f.rgba, f.rgba_pitch, y) + 4 * x;
#if defined(__CUDA_ARCH__)
    *reinterpret_cast<uchar4*>(dst) = make_uchar4(r, g, b, Luma(r, g, b));
#else
    dst[0] = r; dst[1] = g; dst[2] = b; dst[3] = Luma(r, g, b);
#endif
  }
}

inline int ColorChunks(int cw, int ch) {
  const long long total = static_cast<long long>(cw) * ch;
  return static_cast<int>((total + kTile * kTile - 1) / (kTile * kTile));
}

}  // namespace pre

#if defined(__CUDACC__)
LaunchResult LaunchPreprocessFrame(const pre::FrameArgs& f, cudaStream_t stream);      // preprocess.cu
LaunchResult LaunchPreprocessRawFrame(const pre::FrameArgs& f, cudaStream_t stream);   // preprocess.cu: stage 0 per f's raw-frame fields
#endif

}  // namespace bba
