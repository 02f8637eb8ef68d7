// spatial_order.cu -- the surfels' spatial (Morton) order and the pose and geometry steps' surfel streams in that order.
//
// The pose kernel evaluates (keyframe, 256-surfel chunk) sub-items.  In the caller's order (creation order: raster order inside the
// keyframe that created them) a chunk is a band across a whole source image, partly inside and partly outside any other keyframe's
// view: most of its warp steps run the gather path with a few live lanes, and hardly any chunk can be skipped as a whole.  In Morton
// order a chunk is a compact cluster; its bounding box decides for whole chunks that they are outside a view, and the chunks that
// remain have nearly all lanes in the image.  Only the work changes: the kernel still evaluates every pair that projects into the
// image, and correctness needs nothing of the order but that it is a permutation.
//
// Built with -use_fast_math like kernels.cu: the stream's frame rows are computed with the same code as before.
#include "kernels.cuh"

#include <cub/device/device_radix_sort.cuh>

namespace bba {

namespace {

constexpr int kMortonBits = 10;   // per axis: 30-bit keys

// Spreads the low 10 bits of v to every third bit.
__device__ __forceinline__ uint32_t Spread3(uint32_t v) {
  v &= 0x3ffu;
  v = (v | (v << 16)) & 0x030000ffu;
  v = (v | (v << 8)) & 0x0300f00fu;
  v = (v | (v << 4)) & 0x030c30c3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}

// Bounding box of the finite positions: per-thread min / max, warp reduction, one atomic per warp and axis.  bounds[0..2] must
// start at 0xffffffff (min), bounds[3..5] at 0 (max).
__global__ void __launch_bounds__(256) SurfelBoundsKernel(const float* __restrict__ surfels, uint32_t pitch, uint32_t n,
                                                         unsigned int* __restrict__ bounds) {
  unsigned int lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float v = surfels[static_cast<size_t>(kRowX + a) * pitch + i];
      if (isfinite(v)) {
        lo[a] = min(lo[a], OrderedBits(v));
        hi[a] = max(hi[a], OrderedBits(v));
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = __reduce_min_sync(0xffffffffu, lo[a]);
    hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (lo[a] != 0xffffffffu) atomicMin(bounds + a, lo[a]);
      if (hi[a] != 0u) atomicMax(bounds + 3 + a, hi[a]);
    }
  }
}

// key[i] = Morton code of surfel i's position quantised to 10 bits per axis inside the bounding box; index[i] = i.  Non-finite
// coordinates quantise to 0: such a surfel never projects into an image, where it sorts to does not matter.
__global__ void __launch_bounds__(256) MortonKeysKernel(const float* __restrict__ surfels, uint32_t pitch, uint32_t n,
                                                       const unsigned int* __restrict__ bounds, uint32_t* __restrict__ keys,
                                                       uint32_t* __restrict__ index) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t key = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const unsigned int blo = __ldg(bounds + a), bhi = __ldg(bounds + 3 + a);
    uint32_t q = 0;
    if (blo != 0xffffffffu) {   // some finite coordinate on this axis
      const float lo = FromOrderedBits(blo), hi = FromOrderedBits(bhi);
      const float scale = hi > lo ? static_cast<float>(1 << kMortonBits) / (hi - lo) : 0.f;
      const float t = (surfels[static_cast<size_t>(kRowX + a) * pitch + i] - lo) * scale;
      q = static_cast<uint32_t>(fminf(fmaxf(t, 0.f), static_cast<float>((1 << kMortonBits) - 1)));   // fmaxf: NaN -> 0
    }
    key |= Spread3(q) << a;
  }
  keys[i] = key;
  index[i] = i;
}

// One block per 256-column chunk: gather surfel perm[s] into stream column s, and the chunk's bounding box.
__global__ void __launch_bounds__(kSpatialChunk) PoseStreamKernel(const float* __restrict__ surfels, uint32_t pitch, uint32_t n,
                                                                 const uint32_t* __restrict__ perm, float* __restrict__ stream,
                                                                 uint32_t stream_pitch, float* __restrict__ boxes) {
  const uint32_t s = blockIdx.x * kSpatialChunk + threadIdx.x;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  if (s < n) {
    const size_t P = pitch, i = perm ? __ldg(perm + s) : s;
    const Vec3 gp = V3(surfels[kRowX * P + i], surfels[kRowY * P + i], surfels[kRowZ * P + i]);
    const Vec3 nrm = UnpackNormal(__float_as_uint(surfels[kRowNormal * P + i]));
    Vec3 q1, q2;
    TangentPoints(gp, nrm, surfels[kRowRadiusSq * P + i], &q1, &q2);
    const size_t F = stream_pitch;
    stream[0 * F + s] = gp.x;  stream[1 * F + s] = gp.y;  stream[2 * F + s] = gp.z;
    stream[3 * F + s] = surfels[kRowD1 * P + i];
    stream[4 * F + s] = surfels[kRowD2 * P + i];
    stream[5 * F + s] = nrm.x; stream[6 * F + s] = nrm.y; stream[7 * F + s] = nrm.z;
    stream[8 * F + s] = q1.x;  stream[9 * F + s] = q1.y;  stream[10 * F + s] = q1.z;
    stream[11 * F + s] = q2.x; stream[12 * F + s] = q2.y; stream[13 * F + s] = q2.z;
    const float c[3] = {gp.x, gp.y, gp.z};
#pragma unroll
    for (int a = 0; a < 3; ++a)
      if (isfinite(c[a])) lo[a] = hi[a] = c[a];
  }
  __shared__ float s_red[kSpatialChunk / 32][6];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      s_red[warp][a] = lo[a];
      s_red[warp][3 + a] = hi[a];
    }
  }
  __syncthreads();
  if (threadIdx.x < 8) {
    const int f = threadIdx.x;   // 0-2 min, 4-6 max, 3 / 7 padding
    float v = 0.f;
    if (f != 3 && f != 7) {
      const int k = f < 3 ? f : f - 1;
      v = s_red[0][k];
      for (int w = 1; w < kSpatialChunk / 32; ++w) v = f < 3 ? fminf(v, s_red[w][k]) : fmaxf(v, s_red[w][k]);
    }
    boxes[static_cast<size_t>(blockIdx.x) * 8 + f] = v;
  }
}

// One thread per local index of the launch: gather surfel perm[s] into geometry-stream column s (GeometryArgs).  Without desc_rows
// the rows radius^2, d1, d2 are left alone: only the position / descriptor kernel with descriptors reads them.
__global__ void __launch_bounds__(256) GeometryStreamKernel(const __grid_constant__ GeometryArgs a, bool desc_rows) {
  const uint32_t li = a.begin + blockIdx.x * blockDim.x + threadIdx.x;
  if (li >= a.end) return;
  const uint32_t s = SurfelShardToGlobal(li, a.shard_rank, a.shard_world);
  if (s >= a.n) return;
  const size_t P = a.pitch, F = a.stream_pitch, i = a.perm ? __ldg(a.perm + s) : s;
  constexpr int kRows[kGeoStreamRows - 1] = {kRowX, kRowY, kRowZ, kRowNormal, kRowRadiusSq, kRowD1, kRowD2};
#pragma unroll
  for (int r = 0; r < 4; ++r) a.stream[r * F + s] = a.surfels[kRows[r] * P + i];
  if (desc_rows) {
#pragma unroll
    for (int r = 4; r < kGeoStreamRows - 1; ++r) a.stream[r * F + s] = a.surfels[kRows[r] * P + i];
  }
  a.stream[(kGeoStreamRows - 1) * F + s] = __uint_as_float(a.active[i]);
}

}  // namespace

LaunchResult LaunchGeometryStream(const GeometryArgs& a, bool desc_rows, cudaStream_t stream) {
  if (a.end <= a.begin) return {};
  GeometryStreamKernel<<<(a.end - a.begin + 255) / 256, 256, 0, stream>>>(a, desc_rows);
  return {1};
}

size_t SpatialOrderTempBytes(uint32_t capacity) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, static_cast<const uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                  static_cast<const uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr), static_cast<int>(capacity), 0,
                                  3 * kMortonBits);
  return bytes;
}

// The sort reports some errors (a temp buffer that is too small) only through its return value, never through the last error.
LaunchResult LaunchSpatialOrder(const float* surfels, uint32_t pitch, uint32_t n, const SpatialOrderBuffers& b, cudaStream_t stream) {
  if (n == 0) return {};
  LaunchResult r{3};   // bounds, keys, the sort
  r += cudaMemsetAsync(b.bounds, 0xff, 3 * sizeof(unsigned int), stream);
  r += cudaMemsetAsync(b.bounds + 3, 0, 3 * sizeof(unsigned int), stream);
  const uint32_t blocks = min((n + 255u) / 256u, 1024u);
  SurfelBoundsKernel<<<blocks, 256, 0, stream>>>(surfels, pitch, n, b.bounds);
  MortonKeysKernel<<<(n + 255) / 256, 256, 0, stream>>>(surfels, pitch, n, b.bounds, b.keys_in, b.index_in);
  size_t temp_bytes = b.temp_bytes;
  r += cub::DeviceRadixSort::SortPairs(b.temp, temp_bytes, b.keys_in, b.keys_out, b.index_in, b.perm, static_cast<int>(n), 0,
                                       3 * kMortonBits, stream);
  return r;
}

LaunchResult LaunchPoseStream(const float* surfels, uint32_t pitch, uint32_t n, const uint32_t* perm, float* stream, uint32_t stream_pitch,
                              float* boxes, cudaStream_t cuda_stream) {
  if (n == 0) return {};
  PoseStreamKernel<<<(n + kSpatialChunk - 1) / kSpatialChunk, kSpatialChunk, 0, cuda_stream>>>(surfels, pitch, n, perm, stream,
                                                                                             stream_pitch, boxes);
  return {1};
}

}  // namespace bba
