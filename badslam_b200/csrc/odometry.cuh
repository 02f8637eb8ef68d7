// odometry.cuh -- launch interface of the image-pair odometry (frame-to-keyframe direct tracking), SURVEY.md 8(f4).
//
// Reference: BadSlam::RunOdometry (bad_slam.cc:829-950) -> TrackFramePairwise (pairwise_frame_tracking.cc:153-678) with the
// kernels of kernel_downsample.cu, cuda_image_processing.cu:196-206 and kernel_opt_pose.cu:422-1340.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "launch.hpp"

namespace bba {
namespace odom {

constexpr int kMaxScales = 8;

// One image of one pyramid level (pitched device memory; the colour plane also as a texture with the reference's sampler
// state: clamp, linear filter, normalised float, unnormalised coordinates -- pairwise_frame_tracking.cc:55-79).
struct Image {
  float* depth;                 // calibrated depth in metres, 0 = invalid
  uint32_t depth_pitch;         // floats per row
  uint16_t* normals;            // 2 x s8 image-space normal (util.cuh:126-146)
  uint32_t normals_pitch;       // bytes per row
  uint8_t* color;               // intensity (or gradient magnitude)
  uint32_t color_pitch;         // bytes per row
  cudaTextureObject_t color_tex;
};

// Camera model of one pyramid level (PinholeCamera4f::Scaled of the depth / colour camera, pairwise_frame_tracking.cc:412-417,
// through the builders of surfel_projection.h:42-124).
struct LevelCamera {
  int w, h;                               // depth image size at this level
  float fx, fy, cx, cy;                   // depth PixelCornerProjector
  float fx_inv, fy_inv, cx_inv, cy_inv;   // depth PixelCenterUnprojector
  float d2c_fx, d2c_fy, d2c_cx, d2c_cy;   // DepthToColorPixelCorner
  int cw, ch;                             // its width / height (the scaled colour camera's)
  float cfx, cfy;                         // colour PixelCenterProjector fx, fy
};

struct Level {
  LevelCamera cam;
  Image base;      // the "surfel" image: every valid pixel is a point that is projected into the tracked frame
  Image tracked;   // the "frame" image
};

// One image of a chunk and its pyramid, as the stage kernels read it from a device table indexed by grid.z.  The table lists the
// base images first (role 0), then the tracked ones (role 1).
struct PyramidImage {
  cudaTextureObject_t luma_tex;      // stage 1 input: u8 luma, normalised float reads
  uint8_t* gradmag;                  // stage 1 output (colour-sized) ...
  uint32_t gradmag_pitch;
  cudaTextureObject_t gradmag_tex;   // ... and the same plane as stage 2 reads it
  const uint16_t* raw_depth;         // the preprocessed u16 depth and normals of the image
  uint32_t raw_depth_pitch;          // bytes
  const uint16_t* raw_normals;
  uint32_t raw_normals_pitch;
  int tracked;                       // role: 0 base, 1 tracked
  Image level[kMaxScales];           // level 0 normals are raw_normals
};

// Stage 1 (colour-sized): intensity (ComputeBrightnessKernel, cuda_image_processing.cu:196-206) or Sobel gradient magnitude
// (:103-146) of the luma textures of every image of a chunk, one launch for all (grid.z = image).
struct BrightnessArgs {
  const PyramidImage* images;
  int count;
  int w, h;
  int use_gradmag;
};
LaunchResult LaunchBrightness(const BrightnessArgs& a, cudaStream_t stream);

// Stage 2 (depth-sized, level 0): base = CalibrateDepthAndTransformColorToDepthCUDAKernel (kernel_downsample.cu:345-372);
// tracked = CalibrateDepthCUDAKernel (:404-426) + CUDABuffer::SetToReadModeNormalized (cuda_buffer.cu:82-102), or -- without
// pyramid level 0 -- CalibrateAndDownsampleImagesCUDAKernel (:40-105) straight into level 1.  One launch for every image.
struct Level0Args {
  const PyramidImage* images;
  int count;
  int w, h;                       // depth image size (level 0)
  int out_w, out_h;               // tracked output size when skip_level0
  float d2c_fx, d2c_fy, d2c_cx, d2c_cy;
  int cw, ch;
  float a, raw_to_float;
  const float* cfactor;
  int cf_w, cell;
  int skip_level0;                // !use_pyramid_level_0
  int downsample_color;           // depth width == colour width (pairwise_frame_tracking.cc:309)
};
LaunchResult LaunchLevel0(const Level0Args& a, cudaStream_t stream);

// Stage 3: DownsampleImagesCUDAKernel (kernel_downsample.cu:107-156), level s-1 -> s, for the first `count` images of the table
// in one launch (the base images only, or all).
struct DownsampleArgs {
  const PyramidImage* images;
  int count;
  int level;      // output level s >= 1
  int w, h;       // output size
  int in_w, in_h; // input size (>= 2 w, 2 h; one more when the finer level is odd-sized)
};
LaunchResult LaunchDownsample(const DownsampleArgs& a, cudaStream_t stream);

// Stage 4: the whole coarse-to-fine Gauss-Newton of TrackFramePairwise for a list of entries in ONE persistent launch: groups of
// CTAs run one entry at a time (group-wide barriers between passes, the 6x6 solve + SE3 update replicated in every CTA of the
// group).
struct TrackResult {           // written by the kernel (device memory, copied back by the host)
  float base_T_frame[7];
  int iterations[kMaxScales];  // Gauss-Newton iterations per scale
  int chose_initial[kMaxScales];   // the "initial estimate" arm won the cost comparison at this scale (-1: no comparison)
  unsigned int residual_count;     // last accumulation pass (debug counters of kernel_opt_pose.cu:619-657)
  float residual_sum;
  unsigned int passes;
  unsigned int barrier_timeout;    // a CTA gave up waiting at a grid barrier (device fault): the result is invalid
  double debug[36];                // debug_scale >= 0: [0..20] H, [21..26] b, [27] count, [28] cost at init1; [32..35] count / cost at init1, init2
};
// One (base, tracked) pair: images index the chunk's PyramidImage table.
struct TrackEntry {
  float init1[7], init2[7];    // base_T_frame initial estimates
  int base, tracked;
};
struct TrackArgs {
  LevelCamera cam[kMaxScales];
  const PyramidImage* images;
  const TrackEntry* entries;
  int count;                   // entries; group g starts with entry g and then takes the next one left until none are left
  int group_size;              // CTAs per group; the grid is a whole number of groups, at most `count` of them
  int virtual_grid;            // the one-entry grid TrackGrid: the tiles of a pass are split over this many virtual CTAs
  int num_scales;
  int first_scale;             // 0 with pyramid level 0, else 1
  int max_iterations;          // kMaxIterationsPerScale = 30
  int use_depth, use_desc, use_gradmag;
  int test_different_initial_estimates;
  int debug_scale;             // >= 0: parity hook on entry 0 -- one accumulation pass and one cost pass on this level at init1 / init2, no optimisation
  float baseline_fx;
  double* acc;                 // [groups][3][32] rotating accumulators, zero at launch
  double* partials;            // deterministic mode: [groups][3][virtual_grid][32] per-virtual-CTA totals, summed in order; else null
  unsigned int* control;       // [groups][2] barrier {arrival count, generation}, [1] entry queue, [groups][2] next entry; zero at launch
  TrackResult* result;         // [count]
};
// Words of TrackArgs::control for `groups` groups.
inline int TrackControlWords(int groups) { return 4 * groups + 1; }
// The grid of one entry: one CTA per SM, never more than the finest level has tiles.  With more entries the grid is split into
// groups of CTAs (TrackGroupSize); in the deterministic mode a group of any size sums what this grid's CTAs would.
int TrackGrid(const LevelCamera& finest, int sm_count);
// CTAs per group for `count` entries: the whole one-entry grid for one entry, one CTA each from sm_count entries on.
int TrackGroupSize(int count, int virtual_grid, int sm_count);
// The number of groups: one per entry, as many as fit on sm_count SMs.
int TrackGroups(int count, int group_size, int sm_count);
LaunchResult LaunchTrack(const TrackArgs& a, int groups, cudaStream_t stream);

}  // namespace odom
}  // namespace bba
