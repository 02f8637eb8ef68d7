// Fused keyframe preprocessing kernel (one launch per frame; the tile program lives in preprocess_tile.cuh).
//
// Grid: one CTA of 256 threads per 32x32 depth tile (300 CTAs at 640x480), followed by one CTA per 1024 colour pixels (300
// more): a single wave on the H100's 132 SMs (39 registers, 8.4 KB of shared memory per CTA: up to 8 resident CTAs per SM).  Algorithmic bytes per frame: 2 (raw
// depth) + 3 (rgb) read, 2 + 2 + 2 (depth, normals, radius) + 4 (rgba) written per pixel = 15 B/pixel, 4.6 MB at 640x480 --
// well under a microsecond of HBM time, so the kernel
// is bound by launch latency and by the ~30 exp / rcp per pixel of the bilateral filter; what the fusion buys is one launch
// instead of five and no intermediate images (the reference moves 2 + 4 + 4 + 6 + 2 = 18 B/pixel of depth traffic alone).
#include <cuda_runtime.h>

#include "preprocess_tile.cuh"

namespace bba {
namespace pre {

constexpr int kThreads = 256;

struct BlockTeam {
  __device__ __forceinline__ int tid() const { return static_cast<int>(threadIdx.x); }
  __device__ __forceinline__ int size() const { return kThreads; }
  __device__ __forceinline__ void sync() const { __syncthreads(); }
  // ComputeMinMaxDepthCUDAKernel (cuda_depth_processing.cu:390-424): block reduction, then atomicMin / atomicMax on the bit
  // patterns (monotonic for non-negative floats).
  __device__ __forceinline__ void commit_min_max(float mn, float mx, float* out) const {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if ((threadIdx.x & 31) == 0) {
      if (mn < INFINITY) atomicMin(reinterpret_cast<int*>(out), __float_as_int(mn));
      if (mx > 0.f) atomicMax(reinterpret_cast<int*>(out + 1), __float_as_int(mx));
    }
  }
};

__global__ void __launch_bounds__(kThreads) PreprocessFrameKernel(FrameArgs f) {
  extern __shared__ uint16_t smem[];
  const int depth_tiles = f.tiles_x * f.tiles_y;
  const int b = static_cast<int>(blockIdx.x);
  if (b < depth_tiles) {
    DepthTile(f, b % f.tiles_x, b / f.tiles_x, smem, BlockTeam());
  } else {
    ColorChunk(f, b - depth_tiles, BlockTeam());
  }
}

__global__ void InitMinMaxKernel(float* min_max) {
  min_max[0] = INFINITY;   // cuda_depth_processing.cc:41
  min_max[1] = 0.f;
}

}  // namespace pre

// Enqueues the initialisation of min_max and the fused kernel; returns the number of launches (2).
int LaunchPreprocessFrame(const pre::FrameArgs& f, cudaStream_t stream) {
  pre::InitMinMaxKernel<<<1, 1, 0, stream>>>(f.min_max);
  const int blocks = f.tiles_x * f.tiles_y + ((f.rgb && f.rgba) ? pre::ColorChunks(f.cw, f.ch) : 0);
  const size_t smem = sizeof(uint16_t) * static_cast<size_t>(pre::SharedWords(f.radius));
  pre::PreprocessFrameKernel<<<blocks, pre::kThreads, smem, stream>>>(f);
  return 2;
}

}  // namespace bba
