// persistent.cuh -- the machinery the persistent kernels share: warp and block reductions and the block scan, the (keyframe
// group x surfel tile) work-item loop with its per-tile epochs, the stores into the surfel replicas, the keyframe record loaders
// and the launch sizing.
#pragma once

#include <algorithm>
#include <type_traits>

#include "kernels.cuh"

namespace bba {

__device__ __forceinline__ unsigned int LoadAcquire(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void StoreRelease(unsigned int* p, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

template <typename T>
__device__ __forceinline__ T WarpSum(T v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum of v over the block: a butterfly within each warp, one partial per warp in shared memory, then a butterfly over the
// partials in warp 0.  The total is valid in warp 0 only.  A second call in the same kernel needs a __syncthreads() in between:
// warp 0 may still be reading the partials.
template <typename T>
__device__ __forceinline__ T BlockSum(T v) {
  __shared__ T partial[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = WarpSum(v);
  if (lane == 0) partial[warp] = v;
  __syncthreads();
  if (warp == 0) v = WarpSum(lane < static_cast<int>(blockDim.x >> 5) ? partial[lane] : T(0));
  return v;
}

// Exclusive scan of one count per thread over a block of 1024 threads: a shuffle-up scan within each warp, then warp 0 scans the
// 32 warp totals.  Returns the thread's exclusive offset; *total receives the block total.  A second call in the same kernel
// needs a __syncthreads() in between: slow threads may still be reading the warp offsets.
__device__ __forceinline__ unsigned int BlockExclusiveScan(unsigned int v, unsigned int* total) {
  __shared__ unsigned int warp_offset[32];
  __shared__ unsigned int block_total;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_offset[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const unsigned int w = warp_offset[lane];
    unsigned int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    warp_offset[lane] = winc - w;
    if (lane == 31) block_total = winc;
  }
  __syncthreads();
  *total = block_total;
  return warp_offset[warp] + inc - v;
}

// Sums v[i] over the warp for all N i at once (N = 8, 16, 32): afterwards lane L holds the total of v[L % N].  For N = 32 that
// is 16+8+4+2+1 = 31 shuffles instead of 32 x 5.  One template level per butterfly stage: written as a loop over the stages,
// the outer loop is not unrolled and v lives in a stack frame (128 bytes for N = 32).
template <int HALF, int N>
__device__ __forceinline__ void WarpTransposeStage(float (&v)[N], int lane) {
  const bool upper = (lane & HALF) != 0;
#pragma unroll
  for (int i = 0; i < HALF; ++i) {
    const float lo = v[i], hi = v[i + HALF];
    const float send = upper ? lo : hi;
    const float keep = upper ? hi : lo;
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, HALF);
  }
  if constexpr (HALF > 1) WarpTransposeStage<HALF / 2>(v, lane);
}
template <int N>
__device__ __forceinline__ float WarpTransposeReduce(float (&v)[N], int lane) {
  static_assert(N == 8 || N == 16 || N == 32, "WarpTransposeReduce: N = 8, 16 or 32");
  WarpTransposeStage<N / 2>(v, lane);
  float r = v[0];
#pragma unroll
  for (int o = N; o < 32; o <<= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  return r;
}

// Work items (keyframe group, surfel tile) are owned by WARPS and handed out group-major through the global counter *queue, so
// that all resident warps gather from the images of the same few keyframes at a time (L2-resident).  With tile_epoch (kernels
// that park partial sums between groups), item (g, t) is handed over only once (g - 1, t) has been retired (RetireItem); every
// launched CTA must then be resident (EpochOrderedGrid).  Kernels without epochs pass a literal nullptr, which removes the wait at
// compile time.  Must be called by all 32 lanes.
template <typename Epochs>   // a pointer to the per-tile epoch words, or decltype(nullptr)
__device__ __forceinline__ bool ClaimItem(unsigned int* queue, uint32_t n_tiles, uint32_t n_items, Epochs tile_epoch, uint32_t* group,
                                          uint32_t* tile) {
  unsigned int item = 0;
  if ((threadIdx.x & 31) == 0) {
    item = atomicAdd(queue, 1u);
    if constexpr (!std::is_same<Epochs, decltype(nullptr)>::value) {
      if (item < n_items) {
        const uint32_t g = item / n_tiles, t = item - g * n_tiles;
        while (LoadAcquire(tile_epoch + t) < g) __nanosleep(64);
      }
    }
  }
  item = __shfl_sync(0xffffffffu, item, 0);
  if (item >= n_items) return false;
  *group = item / n_tiles;
  *tile = item - *group * n_tiles;
  return true;
}
__device__ __forceinline__ void RetireItem(unsigned int* tile_epoch, uint32_t group, uint32_t tile) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) {
    __threadfence();
    StoreRelease(tile_epoch + tile, group + 1);
  }
}

// A result store into the local replica (element o of local) and, when peers are mapped, into every other rank's (NVLink).
template <typename T>
__device__ __forceinline__ void StoreReplicas(T* local, T* const (&peers)[kMaxPeers], int peer_count, size_t o, T v) {
  local[o] = v;
#pragma unroll
  for (int p = 0; p < kMaxPeers; ++p)
    if (p < peer_count) peers[p][o] = v;
}

// A keyframe record from shared memory (staged by the TMA engine together with the surfel tile).  Returns the keyframe id (pad).
__device__ __forceinline__ int LoadKfShared(const KfDevice* rec, KfRegs* r) {
  const float4* p = reinterpret_cast<const float4*>(rec);
  const float4 a = p[0], b = p[1], c = p[2];
  r->T[0] = a.x; r->T[1] = a.y; r->T[2] = a.z; r->T[3] = a.w;
  r->T[4] = b.x; r->T[5] = b.y; r->T[6] = b.z; r->T[7] = b.w;
  r->T[8] = c.x; r->T[9] = c.y; r->T[10] = c.z; r->T[11] = c.w;
  const ulonglong2 q = *reinterpret_cast<const ulonglong2*>(p + 3);
  r->depth = reinterpret_cast<const uint16_t*>(q.x);
  r->normals = reinterpret_cast<const uint16_t*>(q.y);
  const ulonglong2 q2 = *reinterpret_cast<const ulonglong2*>(p + 4);
  r->tex = static_cast<cudaTextureObject_t>(q2.x);
  r->depth_pitch = static_cast<uint32_t>(q2.y & 0xffffffffu);
  r->normals_pitch = static_cast<uint32_t>(q2.y >> 32);
  const int2 tail = *reinterpret_cast<const int2*>(p + 5);
  r->activation = tail.x;
  return tail.y;
}

// Keyframe kf's record from global memory, without the activation.
__device__ __forceinline__ void LoadKfGlobal(const KfDevice* __restrict__ kfs, int kf, KfRegs* r) {
  const KfDevice& k = kfs[kf];
#pragma unroll
  for (int i = 0; i < 12; ++i) r->T[i] = __ldg(&k.T[i]);
  r->depth = k.depth;
  r->normals = k.normals;
  r->tex = k.tex;
  r->depth_pitch = k.depth_pitch;
  r->normals_pitch = k.normals_pitch;
}

// Launch sizing.  per_sm is the occupancy query's result for the caller's kernel, threads and shared memory.
//
// Epoch-ordered kernels: as many CTAs as can be co-resident (the epoch wait relies on every launched CTA being scheduled), and no
// more than one item per warp.  The tile (the unit one warp walks through, 32..256 surfels, log2 in *tile_shift) is chosen so that
// every keyframe group offers several items per resident warp: with too few tiles the per-tile epoch chain serialises the groups
// (seen at 2+ ranks).  n: surfels of the launch.
inline uint32_t EpochOrderedGrid(int per_sm, int sm_count, int threads, uint32_t n, uint32_t n_groups, int* tile_shift) {
  const uint64_t resident_ctas = static_cast<uint64_t>(std::max(per_sm, 1)) * sm_count;
  const uint64_t resident_warps = resident_ctas * (threads / 32);
  int shift = 8;
  while (shift > 5 && 2 * static_cast<uint64_t>((n + (1u << shift) - 1) >> shift) < 3 * resident_warps) --shift;
  *tile_shift = shift;
  const uint64_t n_items = static_cast<uint64_t>((n + (1u << shift) - 1) >> shift) * n_groups;
  return static_cast<uint32_t>(std::min<uint64_t>((n_items + threads / 32 - 1) / (threads / 32), resident_ctas));
}
// Kernels without epochs: 8 items per CTA, at most the resident CTAs.
inline uint32_t ItemGrid(int per_sm, int sm_count, uint64_t n_items) {
  return static_cast<uint32_t>(std::min<uint64_t>((n_items + 7) / 8, static_cast<uint64_t>(std::max(per_sm, 1)) * sm_count));
}
// Tile-major kernels (one item per tile, every keyframe inside it): 32-surfel tiles, one warp sub-step each, unless a tile of
// 2^forced_shift surfels (5..8) is asked for; the shift goes to *tile_shift.  The cost of a tile varies with how many keyframes
// see it, and the smallest tiles even that out best in the tail: on cfg3 GeometryPassKernel took 5.22 ms at 32 surfels, 5.47 at
// 64, 6.24 at 128 and 7.45 at 256 (DESIGN §7.1).
constexpr int kTileMajorShift = 5;
inline uint32_t TileGrid(int per_sm, int sm_count, uint32_t n, int forced_shift, int* tile_shift) {
  const int shift = forced_shift >= 5 && forced_shift <= 8 ? forced_shift : kTileMajorShift;
  *tile_shift = shift;
  return ItemGrid(per_sm, sm_count, (static_cast<uint64_t>(n) + (1u << shift) - 1) >> shift);
}

}  // namespace bba
