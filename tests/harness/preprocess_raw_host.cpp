// TEST HARNESS (CPU suite only): runs the tile program of badslam_b200/csrc/preprocess_tile.cuh with a raw-frame stage 0 -- the
// code the CUDA kernel PreprocessRawFrameKernel executes -- one "thread" at a time on the host, so that the grown halo, the
// ping-pong median passes, the box reads of the full-resolution depth and the colour blocks can be checked against
// oracle/preprocess_raw_oracle.c without a GPU.  Built by tests/test_oracle_preprocess_raw.py with g++; it is not part of
// libbadba_b200.so and nothing in the product loads it.
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../badslam_b200/csrc/preprocess_tile.cuh"

namespace {

struct HostTeam {
  int threads;   // emulated team size: the loops are strided exactly like on the device
  int id;
  int tid() const { return id; }
  int size() const { return threads; }
  void sync() const {}
  void commit_min_max(float mn, float mx, float* out) const {
    if (mn < out[0]) out[0] = mn;
    if (mx > out[1]) out[1] = mx;
  }
};

// One host thread stands in for the whole team (size 1): every strided loop covers its full range before the next stage
// starts, which is the schedule the barriers give a CUDA block.
}  // namespace

extern "C" {

// The raw-frame variant (bba_preprocess_raw_frame): raw depth raw_w x raw_h, rgb (cw << color_level) x (ch << color_level), the
// outputs w x h / cw x ch; stage 0 per median_iterations / depth_level (the caller passes valid combinations).
int harness_preprocess_raw_frame(int w, int h, const float depth_K[4], float raw_to_float, float a, int cell, int cf_w,
                                 const float* cfactor, float sigma_xy, float sigma_inv_depth, float radius_factor, float max_depth_m,
                                 int median_iterations, int depth_level, int color_level, int raw_w, int raw_h,
                                 const uint16_t* raw_depth, uint16_t* out_depth, uint16_t* out_normals, uint16_t* out_radius,
                                 int cw, int ch, const uint8_t* rgb, uint8_t* rgba, float* min_max) {
  using namespace bba::pre;
  FrameArgs f{};
  f.w = w; f.h = h;
  f.fx_inv = 1.0f / depth_K[0]; f.fy_inv = 1.0f / depth_K[1];
  f.cx_inv = -(depth_K[2] - 0.5f) * f.fx_inv; f.cy_inv = -(depth_K[3] - 0.5f) * f.fy_inv;
  f.raw_to_float = raw_to_float; f.a = a; f.cell = cell; f.cf_w = cf_w; f.cfactor = cfactor;
  f.denom_xy = 2.0f * sigma_xy * sigma_xy;
  f.denom_value = 2.0f * sigma_inv_depth * sigma_inv_depth;
  f.radius = static_cast<int>(radius_factor * sigma_xy + 0.5f);
  f.radius_squared = f.radius * f.radius;
  const float max_raw = max_depth_m / raw_to_float;
  f.max_depth = max_raw >= 65535.f ? static_cast<uint16_t>(65535) : static_cast<uint16_t>(max_raw);
  f.raw_depth = raw_depth; f.raw_pitch = static_cast<uint32_t>(2 * raw_w);
  f.out_depth = out_depth; f.out_depth_pitch = static_cast<uint32_t>(2 * w);
  f.out_normals = out_normals; f.out_normals_pitch = static_cast<uint32_t>(2 * w);
  f.out_radius = out_radius; f.out_radius_pitch = static_cast<uint32_t>(2 * w);
  min_max[0] = INFINITY; min_max[1] = 0.f;
  f.min_max = min_max;
  f.cw = cw; f.ch = ch;
  f.rgb = rgb; f.rgb_pitch = static_cast<uint32_t>(3 * (cw << color_level));
  f.rgba = rgba; f.rgba_pitch = static_cast<uint32_t>(4 * cw);
  f.tiles_x = (w + kTile - 1) / kTile;
  f.tiles_y = (h + kTile - 1) / kTile;
  f.median_iterations = median_iterations;
  f.depth_level = depth_level;
  f.raw_w = raw_w; f.raw_h = raw_h;
  f.color_level = color_level;
  std::vector<uint16_t> smem(static_cast<size_t>(SharedWordsRaw(f.radius, median_iterations)));
  const HostTeam team{1, 0};
  for (int ty = 0; ty < f.tiles_y; ++ty) {
    for (int tx = 0; tx < f.tiles_x; ++tx) {
      if (median_iterations > 0) DepthTile<HostTeam, Stage0::kMedian>(f, tx, ty, smem.data(), team);
      else if (depth_level == 0) DepthTile<HostTeam, Stage0::kCopy>(f, tx, ty, smem.data(), team);
      else if (depth_level == 1) DepthTile<HostTeam, Stage0::kDownscale, 1>(f, tx, ty, smem.data(), team);
      else if (depth_level == 2) DepthTile<HostTeam, Stage0::kDownscale, 2>(f, tx, ty, smem.data(), team);
      else DepthTile<HostTeam, Stage0::kDownscale, 3>(f, tx, ty, smem.data(), team);
    }
  }
  if (rgb && rgba) {
    for (int c = 0; c < ColorChunks(cw, ch); ++c) {
      if (color_level == 0) ColorChunk<HostTeam, 0>(f, c, team);
      else if (color_level == 1) ColorChunk<HostTeam, 1>(f, c, team);
      else if (color_level == 2) ColorChunk<HostTeam, 2>(f, c, team);
      else ColorChunk<HostTeam, 3>(f, c, team);
    }
  }
  return f.tiles_x * f.tiles_y;
}

}  // extern "C"
