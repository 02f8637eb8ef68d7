// lifecycle.cu -- end-of-BA surfel maintenance (DirectBA::PerformBASchemeEndTasks, direct_ba.cc:566-653):
//  * ObservationStatsKernel: DeleteSurfelsAndUpdateRadiiCUDA (kernel_delete_surfels.cc:40-98, kernel_delete_surfels.cu:42-164).
//    Per surfel, over EVERY keyframe: observation count, free-space violations (the pixel's surface lies behind the surfel
//    by more than the association threshold) and the smallest measured radius^2; then delete (x = NaN pattern) surfels
//    with too few observations or more violations than observations, and store the new radius^2 otherwise.
//    The reference launches one kernel per keyframe that read-modify-writes three accumulator rows; here one persistent
//    launch walks (keyframe group, surfel tile) items group-major like the geometry kernels (kernels.cu).
//  * Compact*: CompactSurfelsCUDA (kernel_compact_surfels.cu:159-279): the r-th valid surfel counted from the END moves into
//    the r-th free spot counted from the front when that spot lies in front of it -- the same permutation as the reference
//    (two cub::DeviceScan passes there; one three-kernel exclusive scan here).
#include <cuda.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "kernels.cuh"

namespace bba {

namespace {

constexpr int kThreads = 256;
constexpr int kGroup = 16;
constexpr uint32_t kDeletedPattern = 0x7fffffffu;   // CUDART_NAN_F

__device__ __forceinline__ unsigned int LoadAcquire(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void StoreRelease(unsigned int* p, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

}  // namespace

__global__ void __launch_bounds__(kThreads) ObservationStatsKernel(const __grid_constant__ SurfelStatsArgs a) {
  const uint32_t tile_len = 1u << a.tile_shift;
  const uint32_t n_tiles = (a.local_count + tile_len - 1) >> a.tile_shift;
  const uint32_t n_groups = (a.kf_count + kGroup - 1) / kGroup;
  const uint32_t n_items = n_groups * n_tiles;
  const size_t P = a.pitch;
  const int lane = threadIdx.x & 31;
  const CameraParams& cam = a.cam;
  // result rows of this rank's surfels go to the local replica and -- with mapped peers -- to every other rank's (NVLink)
  auto store_row = [&](int row, uint32_t i, float v) {
    const size_t o = static_cast<size_t>(row) * P + i;
    a.surfels[o] = v;
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p)
      if (p < a.peers.count) a.peers.surfels[p][o] = v;
  };
  for (;;) {
    // warp-owned item (group, tile); (g, t) runs after (g - 1, t) has been retired
    unsigned int item = 0;
    if (lane == 0) {
      item = atomicAdd(a.queue, 1u);
      if (item < n_items) {
        const uint32_t g = item / n_tiles, t = item - g * n_tiles;
        while (LoadAcquire(a.tile_epoch + t) < g) __nanosleep(64);
      }
    }
    item = __shfl_sync(0xffffffffu, item, 0);
    if (item >= n_items) break;
    const uint32_t group = item / n_tiles, tile = item - group * n_tiles;
    const bool first = group == 0, last = group + 1 == n_groups;
    const int j_begin = group * kGroup, j_end = min(a.kf_count, static_cast<int>(group + 1) * kGroup);
    unsigned int deleted_here = 0;
    for (uint32_t sub = 0; sub < tile_len / 32; ++sub) {
      const uint32_t li = (tile << a.tile_shift) + sub * 32 + lane;   // local index of the granule sharding (identity on one GPU)
      const uint32_t i = SurfelShardToGlobal(li, a.shard_rank, a.shard_world);
      bool deleted = false;
      if (li < a.local_count && i < a.n) {
        float obs = 0.f, viol = 0.f, min_r2 = __int_as_float(0x7f800000);   // +inf (kernel_delete_surfels.cu:50)
        if (!first) {
          obs = __ldcg(a.surfels + (kRowAccum0 + 0) * P + i);
          viol = __ldcg(a.surfels + (kRowAccum0 + 1) * P + i);
          min_r2 = __ldcg(a.surfels + (kRowAccum0 + 2) * P + i);
        }
        const float x = a.surfels[kRowX * P + i];
        const Vec3 gp = V3(x, a.surfels[kRowY * P + i], a.surfels[kRowZ * P + i]);
        const Vec3 nrm = UnpackNormal(__float_as_uint(a.surfels[kRowNormal * P + i]));
        for (int kf = j_begin; kf < j_end; ++kf) {
          const KfDevice& K = a.kfs[kf];
          float T[12];
#pragma unroll
          for (int c = 0; c < 12; ++c) T[c] = __ldg(&K.T[c]);
          Assoc r;
          if (!ProjectIntoImage(cam, T, gp, &r)) continue;
          const PixelLoads l = LoadPixel(cam, K.depth, K.depth_pitch, K.normals, K.normals_pitch, r);
          // IsAssociatedWithPixel<return_free_space_violations = true> (surfel_projection_nvcc_only.cuh:48-127)
          if (l.measured & kInvalidDepthBit) continue;
          const float d = RawToCalibratedDepth(cam.a, l.cf, cam.raw_to_float, l.measured);
          const Vec3 ln = Rotate(T, nrm);
          const float nx = cam.fx_inv * r.px + cam.cx_inv, ny = cam.fy_inv * r.py + cam.cy_inv;
          const float thr = kDepthTukey * ((kDepthUncertaintyFactor * fabsf(ln.x * nx + ln.y * ny + ln.z) * (d * d)) / cam.baseline_fx);
          const float diff = d - r.lp.z;
          if (diff > thr) {
            viol += 1.f;
            continue;
          }
          if (diff < -thr) continue;
          if (Dot(r.lp, ln) > 0) continue;
          if (Dot(ln, U16ToImageSpaceNormal(l.kf_normal)) < kCosNormalCompat) continue;
          obs += 1.f;
          const KfRadius& R = a.radius[kf];
          const uint16_t h = __ldg(reinterpret_cast<const uint16_t*>(reinterpret_cast<const char*>(R.ptr) + static_cast<size_t>(r.py) * R.pitch) + r.px);
          min_r2 = fminf(min_r2, __half2float(__ushort_as_half(h)));
        }
        if (!last) {
          __stcg(a.surfels + (kRowAccum0 + 0) * P + i, obs);
          __stcg(a.surfels + (kRowAccum0 + 1) * P + i, viol);
          __stcg(a.surfels + (kRowAccum0 + 2) * P + i, min_r2);
        } else {
          // MarkDeletedSurfelsCUDAKernel (kernel_delete_surfels.cu:129-164)
          if (obs < static_cast<float>(a.min_observation_count) || viol > obs) {
            if (__float_as_uint(x) != kDeletedPattern) {
              store_row(kRowX, i, __uint_as_float(kDeletedPattern));
              deleted = true;
            }
          } else {
            store_row(kRowRadiusSq, i, min_r2);
          }
        }
      }
      deleted_here += __popc(__ballot_sync(0xffffffffu, deleted));
    }
    __syncwarp();
    if (lane == 0) {
      if (deleted_here) atomicAdd(a.deleted_count, deleted_here);
      __threadfence();
      StoreRelease(a.tile_epoch + tile, group + 1);
    }
  }
}

// ---- compaction ---------------------------------------------------------------------------------------------------------
constexpr int kScanItems = 4;                               // surfels per thread
constexpr int kScanBlock = 1024 * kScanItems;               // surfels per block

// flags (1 = deleted) -> scratch row Accum2; per-block number of deleted surfels -> block_sums
__global__ void __launch_bounds__(1024) CompactFlagKernel(float* __restrict__ surfels, uint32_t pitch, uint32_t n, unsigned int* __restrict__ block_sums) {
  __shared__ unsigned int warp_sums[32];
  const size_t P = pitch;
  const uint32_t base = blockIdx.x * kScanBlock + threadIdx.x * kScanItems;
  unsigned int cnt = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const uint32_t i = base + k;
    if (i < n) {
      const unsigned int f = __float_as_uint(surfels[kRowX * P + i]) == kDeletedPattern ? 1u : 0u;
      reinterpret_cast<unsigned int*>(surfels + (kRowAccum0 + 2) * P)[i] = f;
      cnt += f;
    }
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x < 32) {
    unsigned int s = warp_sums[threadIdx.x];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = s;
  }
}

// exclusive scan of the block sums in place (one block); block_sums[n_blocks] receives the total
__global__ void __launch_bounds__(1024) CompactScanBlocksKernel(unsigned int* __restrict__ block_sums, uint32_t n_blocks) {
  __shared__ unsigned int warp_tot[32];
  __shared__ unsigned int chunk_total;
  unsigned int carry = 0;   // identical in every thread
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t base = 0; base < n_blocks; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const unsigned int v = i < n_blocks ? block_sums[i] : 0u;
    unsigned int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      const unsigned int w = warp_tot[lane];
      unsigned int winc = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned int t = __shfl_up_sync(0xffffffffu, winc, o);
        if (lane >= o) winc += t;
      }
      warp_tot[lane] = winc - w;   // exclusive offset of each warp
      if (lane == 31) chunk_total = winc;
    }
    __syncthreads();
    if (i < n_blocks) block_sums[i] = carry + warp_tot[warp] + inc - v;
    carry += chunk_total;
    __syncthreads();   // warp_tot / chunk_total are rewritten by the next chunk
  }
  if (threadIdx.x == 0) block_sums[n_blocks] = carry;
}

// exclusive count of deleted surfels in front of every surfel -> scratch row Accum0; list of free spots -> row Accum3
__global__ void __launch_bounds__(1024) CompactListKernel(float* __restrict__ surfels, uint32_t pitch, uint32_t n,
                                                          const unsigned int* __restrict__ block_offsets) {
  __shared__ unsigned int warp_tot[32];
  const size_t P = pitch;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t base = blockIdx.x * kScanBlock + threadIdx.x * kScanItems;
  const unsigned int* flags = reinterpret_cast<const unsigned int*>(surfels + (kRowAccum0 + 2) * P);
  unsigned int* before = reinterpret_cast<unsigned int*>(surfels + (kRowAccum0 + 0) * P);
  unsigned int* free_list = reinterpret_cast<unsigned int*>(surfels + (kRowAccum0 + 3) * P);
  unsigned int f[kScanItems], mine = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    f[k] = (base + k < n) ? flags[base + k] : 0u;
    mine += f[k];
  }
  unsigned int inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const unsigned int w = warp_tot[lane];
    unsigned int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    warp_tot[lane] = winc - w;
  }
  __syncthreads();
  unsigned int run = block_offsets[blockIdx.x] + warp_tot[warp] + inc - mine;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const uint32_t i = base + k;
    if (i < n) {
      before[i] = run;
      if (f[k]) free_list[run] = i;
      run += f[k];
    }
  }
}

// CompactSurfelsCUDAKernel (kernel_compact_surfels.cu:126-157) with adapt_active_surfels = false (direct_ba.cc:618)
__global__ void __launch_bounds__(256) CompactMoveKernel(float* __restrict__ surfels, uint32_t pitch, uint32_t n, uint32_t free_count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t P = pitch;
  const unsigned int* flags = reinterpret_cast<const unsigned int*>(surfels + (kRowAccum0 + 2) * P);
  if (flags[i]) return;
  const unsigned int* before = reinterpret_cast<const unsigned int*>(surfels + (kRowAccum0 + 0) * P);
  const unsigned int* free_list = reinterpret_cast<const unsigned int*>(surfels + (kRowAccum0 + 3) * P);
  // number of valid surfels behind i = (valid total) - (valid up to and including i)
  const uint32_t valid_total = n - free_count;
  const uint32_t reverse_index = valid_total - (i + 1 - before[i]);
  if (reverse_index >= free_count) return;
  const uint32_t spot = free_list[reverse_index];
  if (spot >= i) return;
#pragma unroll
  for (int row = 0; row < kRowAccum0; ++row) surfels[row * P + spot] = surfels[row * P + i];
}


// =============================================================================================================================
// In-loop surfel lifecycle: CreateSurfelsForKeyframe (direct_ba.cc:340-405, kernel_create_surfels.cc:40-183,
// kernel_create_surfels.cu:40-405) and DetermineSupportingSurfelsAndMergeSurfels (kernel_supporting_surfels.cc:40-118,
// kernel_supporting_surfels.cu:44-101).
//
// The reference resolves two races with atomicCAS "first come": which pixel of an unoccupied sparse cell seeds the new surfel
// and which (up to 3) surfels become the supporting surfels of a cell.  Here both are the outcome of executing the reference's
// threads in a FIXED order: the seed is the valid pixel of its cell with the smallest hashed raster index; the surfels "arrive" in
// the order of a bijective hash of their index (SurfelArrivalKey; a pseudo-random order like the hardware's, whereas plain
// index order would always favour the oldest surfels), so the supporting surfels of a cell are its associated surfels with
// the three smallest keys (three atomicMin passes).  The result is reproducible (bit-identical to oracle/badba_oracle.c) and,
// with sparse_surfel_cell_size = 1, the creation is identical to the reference's.
constexpr unsigned int kInvalidIndex = 0xffffffffu;
constexpr int kMergeBuffers = 3;   // kernels.cuh:51
// arrival order of the surfels in the merge: multiplication by an odd constant is a bijection on 32-bit integers
__host__ __device__ inline unsigned int SurfelArrivalKey(unsigned int index) { return index * 0x9E3779B1u; }
__host__ __device__ inline unsigned int SurfelOfArrivalKey(unsigned int key) { return key * 0x0E8B2F51u; }   // modular inverse
static_assert(0x9E3779B1u * 0x0E8B2F51u == 1u, "inverse of the arrival hash");

namespace {

__device__ __forceinline__ unsigned int* CellCache(const LifecycleArgs& a) {   // scratch row Accum0: cell of every surfel
  return reinterpret_cast<unsigned int*>(a.surfels + static_cast<size_t>(kRowAccum0) * a.pitch);
}

// kernel_supporting_surfels.cu:66-85
__device__ __forceinline__ bool MergeTest(const LifecycleArgs& a, uint32_t sup, uint32_t self) {
  const size_t P = a.pitch;
  const Vec3 sn = UnpackNormal(__float_as_uint(a.surfels[kRowNormal * P + sup]));
  const Vec3 tn = UnpackNormal(__float_as_uint(a.surfels[kRowNormal * P + self]));
  if (!(Dot(sn, tn) > kCosNormalCompat)) return false;
  const Vec3 d = V3(a.surfels[kRowX * P + sup], a.surfels[kRowY * P + sup], a.surfels[kRowZ * P + sup]) -
                 V3(a.surfels[kRowX * P + self], a.surfels[kRowY * P + self], a.surfels[kRowZ * P + self]);
  const float min_r2 = fminf(a.surfels[kRowRadiusSq * P + sup], a.surfels[kRowRadiusSq * P + self]);
  return Dot(d, d) < min_r2 * a.cell_merge_dist_squared;
}

// tex2D<float4>(color_texture, x, y) channel c of the caller's uchar4 image, with the measured hardware bilinear filter
// (1.8 fixed-point fractions, far weight (a*b+128)>>8, unorm16 texels, one rounding; oracle/badba_oracle.c tex_w_hw)
__device__ __forceinline__ float SampleRgbaChannel(const LifecycleArgs& a, float x, float y, int c) {
  const float xb = x - 0.5f, yb = y - 0.5f;
  const float fi = floorf(xb), fj = floorf(yb);
  const int i = static_cast<int>(fi), j = static_cast<int>(fj);
  const int fa = static_cast<int>(floorf((xb - fi) * 256.f + 0.5f)), fb = static_cast<int>(floorf((yb - fj) * 256.f + 0.5f));
  const int w11 = (fa * fb + 128) >> 8, w10 = fa - w11, w01 = fb - w11, w00 = 256 - w11 - w10 - w01;
  int t[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int ii = min(max(i + (q & 1), 0), a.cam.cw - 1), jj = min(max(j + (q >> 1), 0), a.cam.ch - 1);
    t[q] = a.rgba[static_cast<size_t>(jj) * a.rgba_pitch + 4 * ii + c] * 257;
  }
  const long long sum = static_cast<long long>(w00) * t[0] + static_cast<long long>(w10) * t[1] + static_cast<long long>(w01) * t[2] +
                        static_cast<long long>(w11) * t[3];
  return __fdiv_rn(static_cast<float>((sum + 128) >> 8), 65535.f);   // IEEE division: the texture unit's value, also under -use_fast_math
}

__device__ __forceinline__ unsigned int CellOf(const CameraParams& cam, int px, int py) {
  const unsigned int cx = (cam.cell == 1) ? static_cast<unsigned int>(px) : __umulhi(static_cast<unsigned int>(px), cam.cell_magic);
  const unsigned int cy = (cam.cell == 1) ? static_cast<unsigned int>(py) : __umulhi(static_cast<unsigned int>(py), cam.cell_magic);
  return cy * cam.cf_w + cx;
}

}  // namespace

// pass 0: the cell every surfel is associated with (cached) + smallest surfel index per cell
__global__ void __launch_bounds__(256) SupportLevel0Kernel(const __grid_constant__ LifecycleArgs a) {
  unsigned int* cache = CellCache(a);
  const size_t P = a.pitch;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const Vec3 gp = V3(a.surfels[kRowX * P + i], a.surfels[kRowY * P + i], a.surfels[kRowZ * P + i]);
    const Vec3 nrm = UnpackNormal(__float_as_uint(a.surfels[kRowNormal * P + i]));
    Assoc r;
    unsigned int cell = kInvalidIndex;
    if (ProjectAssociate(a.cam, a.T, a.depth, a.depth_pitch, a.normals, a.normals_pitch, gp, nrm, &r) == 3) {
      cell = CellOf(a.cam, r.px, r.py);
      atomicMin(a.sup + cell, SurfelArrivalKey(i));   // (0xffffffff is the key of one index < 2^32 only in theory: n < 2^31)
    }
    cache[i] = cell;
  }
}

// pass `level` (1, 2): the next smallest index per cell
__global__ void __launch_bounds__(256) SupportNextKernel(const __grid_constant__ LifecycleArgs a, int level) {
  const unsigned int* cache = CellCache(a);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const unsigned int cell = cache[i];
    if (cell == kInvalidIndex) continue;
    const unsigned int key = SurfelArrivalKey(i);
    if (a.sup[cell] == key) continue;
    if (level == 2 && a.sup[a.cells + cell] == key) continue;
    atomicMin(a.sup + static_cast<size_t>(level) * a.cells + cell, key);
  }
}

// per cell: are supporting surfels 1 and 2 themselves merged away (bit 0 / bit 1)?
__global__ void __launch_bounds__(256) MergeDecideKernel(const __grid_constant__ LifecycleArgs a) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.cells) return;
  const unsigned int k1 = a.sup[a.cells + c], k2 = a.sup[2 * static_cast<size_t>(a.cells) + c];
  const unsigned int s0 = SurfelOfArrivalKey(a.sup[c]), s1 = SurfelOfArrivalKey(k1), s2 = SurfelOfArrivalKey(k2);
  unsigned int bits = 0;
  if (k1 != kInvalidIndex && MergeTest(a, s0, s1)) bits |= 1u;
  if (k2 != kInvalidIndex && (MergeTest(a, s0, s2) || (!(bits & 1u) && MergeTest(a, s1, s2)))) bits |= 2u;
  a.cell_bits[c] = bits;
}

__global__ void __launch_bounds__(256) MergeApplyKernel(const __grid_constant__ LifecycleArgs a) {
  const unsigned int* cache = CellCache(a);
  const size_t P = a.pitch;
  unsigned int deleted_here = 0;
  for (uint32_t base = blockIdx.x * blockDim.x; base < a.n; base += gridDim.x * blockDim.x) {
    const uint32_t i = base + threadIdx.x;
    bool del = false;
    if (i < a.n) {
      const unsigned int cell = cache[i];
      if (cell != kInvalidIndex) {
        const unsigned int k0 = a.sup[cell], k1 = a.sup[a.cells + cell], k2 = a.sup[2 * static_cast<size_t>(a.cells) + cell];
        const unsigned int key = SurfelArrivalKey(i);
        const unsigned int bits = a.cell_bits[cell];
        if (key == k0) del = false;
        else if (key == k1) del = bits & 1u;
        else if (key == k2) del = bits & 2u;
        else   // (a cell with a 4th surfel has three supporting surfels)
          del = MergeTest(a, SurfelOfArrivalKey(k0), i) || (!(bits & 1u) && MergeTest(a, SurfelOfArrivalKey(k1), i)) ||
                (!(bits & 2u) && MergeTest(a, SurfelOfArrivalKey(k2), i));
      }
    }
    deleted_here += __popc(__ballot_sync(0xffffffffu, del));
    if (del) a.surfels[kRowX * P + i] = __uint_as_float(kDeletedPattern);
  }
  if ((threadIdx.x & 31) == 0 && deleted_here) atomicAdd(a.counter, deleted_here);
}

// one seed pixel per unsupported cell (kernel_create_surfels.cu:40-73); flags are pre-zeroed.  The reference takes whichever
// valid pixel of the cell wins an atomicCAS; here it is the valid pixel with the smallest hashed raster index (a fixed
// pseudo-random choice: always taking the first pixel would put the seeds on a regular lattice).
__global__ void __launch_bounds__(256) SeedKernel(const __grid_constant__ LifecycleArgs a) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.cells || a.sup[c] != kInvalidIndex) return;
  const int cy = c / a.cam.cf_w, cx = c - cy * a.cam.cf_w;
  unsigned int best_key = kInvalidIndex, best = kInvalidIndex;
  for (int y = cy * a.cam.cell; y < min((cy + 1) * a.cam.cell, a.cam.h); ++y) {
    for (int x = cx * a.cam.cell; x < min((cx + 1) * a.cam.cell, a.cam.w); ++x) {
      if (x < 1 || y < 1 || x >= a.cam.w - 1 || y >= a.cam.h - 1) continue;
      if (LoadPixelU16(a.depth, a.depth_pitch, x, y) & kInvalidDepthBit) continue;
      const unsigned int seq = static_cast<unsigned int>(y) * a.cam.w + x;
      const unsigned int key = SurfelArrivalKey(seq);
      if (best == kInvalidIndex || key < best_key) {
        best_key = key;
        best = seq;
      }
    }
  }
  if (best != kInvalidIndex) a.flags[best] = 1u;
}

// CountObservationsForNewSurfels over the co-visible keyframes + FilterNewSurfels (kernel_create_surfels.cu:211-334)
__global__ void __launch_bounds__(128) FilterSeedsKernel(const __grid_constant__ LifecycleArgs a) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.cells || a.sup[c] != kInvalidIndex) return;
  const CameraParams& cam = a.cam;
  const int cy = c / cam.cf_w, cx = c - cy * cam.cf_w;
  int sx = -1, sy = -1;
  for (int y = cy * cam.cell; y < min((cy + 1) * cam.cell, cam.h) && sx < 0; ++y)
    for (int x = cx * cam.cell; x < min((cx + 1) * cam.cell, cam.w); ++x)
      if (a.flags[static_cast<size_t>(y) * cam.w + x]) { sx = x; sy = y; break; }
  if (sx < 0) return;
  const float d = RawToCalibratedDepth(cam.a, __ldg(cam.cfactor + c), cam.raw_to_float, LoadPixelU16(a.depth, a.depth_pitch, sx, sy));
  const Vec3 p_in = V3(d * (cam.fx_inv * sx + cam.cx_inv), d * (cam.fy_inv * sy + cam.cy_inv), d);
  const Vec3 n_in = U16ToImageSpaceNormal(LoadPixelU16(a.normals, a.normals_pitch, sx, sy));
  unsigned int obs = 1, viol = 0;
  for (int k = 0; k < a.covis_count; ++k) {
    const CovisEntry& ce = a.covis[k];
    Assoc r;
    if (!ProjectIntoImage(cam, ce.R, p_in, &r)) continue;
    // IsAssociatedWithPixel<true> for a pixel-defined surfel (surfel_projection_nvcc_only.cuh:130-236)
    const uint16_t measured = LoadPixelU16(ce.depth, ce.depth_pitch, r.px, r.py);
    if (measured & kInvalidDepthBit) continue;
    const float pd = RawToCalibratedDepth(cam.a, __ldg(cam.cfactor + CellOf(cam, r.px, r.py)), cam.raw_to_float, measured);
    const Vec3 ln = Rotate(ce.R, n_in);
    const float nx = cam.fx_inv * r.px + cam.cx_inv, ny = cam.fy_inv * r.py + cam.cy_inv;
    const float thr = kDepthTukey * ((kDepthUncertaintyFactor * fabsf(ln.x * nx + ln.y * ny + ln.z) * (pd * pd)) / cam.baseline_fx);
    const float diff = pd - r.lp.z;
    if (diff > thr) {
      ++viol;
      continue;
    }
    if (diff < -thr) continue;
    if (Dot(r.lp, ln) > 0) continue;
    if (Dot(ln, U16ToImageSpaceNormal(LoadPixelU16(ce.normals, ce.normals_pitch, r.px, r.py))) < kCosNormalCompat) continue;
    ++obs;
  }
  if (obs < static_cast<unsigned int>(a.min_observation_count) || viol > obs) a.flags[static_cast<size_t>(sy) * cam.w + sx] = 0u;
}

// CreateNewSurfel (kernel_create_surfels.cu:97-165) for every flagged pixel, appended in raster order
__global__ void __launch_bounds__(256) CreateSurfelsKernel(const __grid_constant__ LifecycleArgs a, const unsigned int* __restrict__ index) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  const CameraParams& cam = a.cam;
  if (s >= static_cast<uint32_t>(cam.w) * cam.h || !a.flags[s]) return;
  const int y = s / cam.w, x = s - y * cam.w;
  const uint32_t out = a.n + index[s];
  const size_t P = a.pitch;
  const float d = RawToCalibratedDepth(cam.a, __ldg(cam.cfactor + CellOf(cam, x, y)), cam.raw_to_float, LoadPixelU16(a.depth, a.depth_pitch, x, y));
  const Vec3 gp = Transform(a.G, V3(d * (cam.fx_inv * x + cam.cx_inv), d * (cam.fy_inv * y + cam.cy_inv), d));
  const Vec3 gn = Rotate(a.G, U16ToImageSpaceNormal(LoadPixelU16(a.normals, a.normals_pitch, x, y)));
  const float r2 = __half2float(__ushort_as_half(LoadPixelU16(a.radius, a.radius_pitch, x, y)));
  a.surfels[kRowX * P + out] = gp.x;
  a.surfels[kRowY * P + out] = gp.y;
  a.surfels[kRowZ * P + out] = gp.z;
  a.surfels[kRowNormal * P + out] = __uint_as_float(PackNormal(gn));
  a.surfels[kRowRadiusSq * P + out] = r2;
  float ccx, ccy;
  DepthToColor(cam, x + 0.5f, y + 0.5f, &ccx, &ccy);
  unsigned int col = 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) col |= static_cast<unsigned int>(static_cast<unsigned char>(255.f * SampleRgbaChannel(a, ccx, ccy, c))) << (8 * c);
  a.surfels[kRowColor * P + out] = __uint_as_float(col);
  float t1x, t1y, t2x, t2y;
  TangentProjections(cam, a.T, gp, gn, r2, &t1x, &t1y, &t2x, &t2y);
  DescEval e;
  EvalDescriptor(a.tex, ccx, ccy, t1x, t1y, t2x, t2y, 0.f, 0.f, &e);
  a.surfels[kRowD1 * P + out] = e.r1;
  a.surfels[kRowD2 * P + out] = e.r2;
}

// ---- generic exclusive scan of a u32 array (block sums -> CompactScanBlocksKernel -> apply) -----------------------------------
__global__ void __launch_bounds__(1024) ScanBlockSumsKernel(const unsigned int* __restrict__ in, uint32_t n, unsigned int* __restrict__ block_sums) {
  __shared__ unsigned int warp_sums[32];
  const uint32_t base = blockIdx.x * kScanBlock + threadIdx.x * kScanItems;
  unsigned int cnt = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k)
    if (base + k < n) cnt += in[base + k];
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x < 32) {
    unsigned int v = warp_sums[threadIdx.x];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = v;
  }
}

__global__ void __launch_bounds__(1024) ScanApplyKernel(const unsigned int* __restrict__ in, uint32_t n, const unsigned int* __restrict__ block_offsets,
                                                        unsigned int* __restrict__ out) {
  __shared__ unsigned int warp_tot[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t base = blockIdx.x * kScanBlock + threadIdx.x * kScanItems;
  unsigned int f[kScanItems], mine = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    f[k] = (base + k < n) ? in[base + k] : 0u;
    mine += f[k];
  }
  unsigned int inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const unsigned int w = warp_tot[lane];
    unsigned int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    warp_tot[lane] = winc - w;
  }
  __syncthreads();
  unsigned int run = block_offsets[blockIdx.x] + warp_tot[warp] + inc - mine;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < n) out[base + k] = run;
    run += f[k];
  }
}

// CompactSurfelsCUDAKernel with adapt_active_surfels = true (direct_ba_alternating.cc:530)
__global__ void __launch_bounds__(256) CompactMoveActiveKernel(float* __restrict__ surfels, uint32_t pitch, uint32_t n, uint32_t free_count,
                                                               uint8_t* __restrict__ active) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t P = pitch;
  const unsigned int* flags = reinterpret_cast<const unsigned int*>(surfels + (kRowAccum0 + 2) * P);
  if (flags[i]) return;
  const unsigned int* before = reinterpret_cast<const unsigned int*>(surfels + (kRowAccum0 + 0) * P);
  const unsigned int* free_list = reinterpret_cast<const unsigned int*>(surfels + (kRowAccum0 + 3) * P);
  const uint32_t valid_total = n - free_count;
  const uint32_t reverse_index = valid_total - (i + 1 - before[i]);
  if (reverse_index >= free_count) return;
  const uint32_t spot = free_list[reverse_index];
  if (spot >= i) return;
#pragma unroll
  for (int row = 0; row < kRowAccum0; ++row) surfels[row * P + spot] = surfels[row * P + i];
  active[spot] = active[i];
}

static uint32_t GridFor(uint32_t n, int sm_count) {
  return static_cast<uint32_t>(std::min<uint64_t>((static_cast<uint64_t>(n) + 255) / 256, static_cast<uint64_t>(sm_count) * 16));
}

void LaunchSupportSurfels(const LifecycleArgs& a, int sm_count, cudaStream_t stream) {
  cudaMemsetAsync(a.sup, 0xff, sizeof(unsigned int) * kMergeBuffers * a.cells, stream);   // kernel_supporting_surfels.cc:61-63
  if (a.n == 0) return;
  SupportLevel0Kernel<<<GridFor(a.n, sm_count), 256, 0, stream>>>(a);
}

void LaunchMergeSurfels(const LifecycleArgs& a, int sm_count, cudaStream_t stream) {
  LaunchSupportSurfels(a, sm_count, stream);
  if (a.n == 0) return;
  SupportNextKernel<<<GridFor(a.n, sm_count), 256, 0, stream>>>(a, 1);
  SupportNextKernel<<<GridFor(a.n, sm_count), 256, 0, stream>>>(a, 2);
  MergeDecideKernel<<<(a.cells + 255) / 256, 256, 0, stream>>>(a);
  MergeApplyKernel<<<GridFor(a.n, sm_count), 256, 0, stream>>>(a);
}

void LaunchSeedNewSurfels(const LifecycleArgs& a, bool filter, cudaStream_t stream) {
  const uint32_t pixels = static_cast<uint32_t>(a.cam.w) * a.cam.h;
  cudaMemsetAsync(a.flags, 0, sizeof(unsigned int) * pixels, stream);
  SeedKernel<<<(a.cells + 255) / 256, 256, 0, stream>>>(a);
  if (filter) FilterSeedsKernel<<<(a.cells + 127) / 128, 128, 0, stream>>>(a);
}

uint32_t ScanScratchWords(uint32_t n) { return (n + kScanBlock - 1) / kScanBlock + 2; }

// out[i] = sum of in[0 .. i-1]; block_sums[ceil(n / 4096)] receives the total
void LaunchExclusiveScan(const unsigned int* in, uint32_t n, unsigned int* out, unsigned int* block_sums, cudaStream_t stream) {
  const uint32_t n_blocks = (n + kScanBlock - 1) / kScanBlock;
  ScanBlockSumsKernel<<<n_blocks, 1024, 0, stream>>>(in, n, block_sums);
  CompactScanBlocksKernel<<<1, 1024, 0, stream>>>(block_sums, n_blocks);
  ScanApplyKernel<<<n_blocks, 1024, 0, stream>>>(in, n, block_sums, out);
}

void LaunchCreateSurfels(const LifecycleArgs& a, const unsigned int* index, cudaStream_t stream) {
  const uint32_t pixels = static_cast<uint32_t>(a.cam.w) * a.cam.h;
  CreateSurfelsKernel<<<(pixels + 255) / 256, 256, 0, stream>>>(a, index);
}

// rows x (deletion marker) and radius^2 of this rank's shard, in local index order
__global__ void __launch_bounds__(256) PackStatsShardKernel(const float* __restrict__ surfels, uint32_t pitch, uint32_t n, uint32_t rank,
                                                            uint32_t world, uint32_t shard_len, float* __restrict__ slice) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= shard_len) return;
  const uint32_t i = SurfelShardToGlobal(c, rank, world);
  const bool in = i < n;
  slice[c] = in ? surfels[static_cast<size_t>(kRowX) * pitch + i] : 0.f;
  slice[static_cast<size_t>(shard_len) + c] = in ? surfels[static_cast<size_t>(kRowRadiusSq) * pitch + i] : 0.f;
}
__global__ void __launch_bounds__(256) UnpackStatsShardsKernel(float* __restrict__ surfels, uint32_t pitch, uint32_t n, uint32_t shard_len,
                                                               uint32_t world, int skip_rank, const float* __restrict__ buffer) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t granule = i >> kShardGranuleShift;
  const uint32_t rank = granule % world;
  if (static_cast<int>(rank) == skip_rank) return;
  const uint32_t c = ((granule / world) << kShardGranuleShift) | (i & ((1u << kShardGranuleShift) - 1u));
  const float* slice = buffer + static_cast<size_t>(rank) * 2 * shard_len;
  surfels[static_cast<size_t>(kRowX) * pitch + i] = slice[c];
  surfels[static_cast<size_t>(kRowRadiusSq) * pitch + i] = slice[static_cast<size_t>(shard_len) + c];
}
void LaunchPackStatsShard(const float* surfels, uint32_t pitch, uint32_t n, uint32_t rank, uint32_t world, uint32_t shard_len, float* slice,
                          cudaStream_t stream) {
  if (shard_len == 0) return;
  PackStatsShardKernel<<<(shard_len + 255) / 256, 256, 0, stream>>>(surfels, pitch, n, rank, world, shard_len, slice);
}
void LaunchUnpackStatsShards(float* surfels, uint32_t pitch, uint32_t n, uint32_t shard_len, int world, int skip_rank, const float* buffer,
                             cudaStream_t stream) {
  if (n == 0) return;
  UnpackStatsShardsKernel<<<(n + 255) / 256, 256, 0, stream>>>(surfels, pitch, n, shard_len, static_cast<uint32_t>(world), skip_rank, buffer);
}

void LaunchObservationStats(SurfelStatsArgs a, int sm_count, cudaStream_t stream) {
  if (a.local_count == 0 || a.kf_count <= 0) return;
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ObservationStatsKernel, kThreads, 0);
  if (per_sm < 1) per_sm = 1;
  const uint64_t resident_warps = static_cast<uint64_t>(per_sm) * sm_count * (kThreads / 32);
  int shift = 8;
  while (shift > 5 && 2 * static_cast<uint64_t>((a.local_count + (1u << shift) - 1) >> shift) < 3 * resident_warps) --shift;
  a.tile_shift = shift;
  const uint32_t n_tiles = (a.local_count + (1u << shift) - 1) >> shift;
  const uint64_t n_items = static_cast<uint64_t>(n_tiles) * ((a.kf_count + kGroup - 1) / kGroup);
  cudaMemsetAsync(a.queue, 0, sizeof(unsigned int), stream);
  cudaMemsetAsync(a.tile_epoch, 0, sizeof(unsigned int) * n_tiles, stream);
  const uint64_t ctas = std::min<uint64_t>((n_items + kThreads / 32 - 1) / (kThreads / 32), static_cast<uint64_t>(per_sm) * sm_count);
  ObservationStatsKernel<<<static_cast<uint32_t>(ctas), kThreads, 0, stream>>>(a);
}

uint32_t CompactScratchWords(uint32_t n) { return (n + kScanBlock - 1) / kScanBlock + 2; }

void LaunchCompactSurfels(float* surfels, uint32_t pitch, uint32_t n, uint32_t free_count, unsigned int* block_sums, uint8_t* active,
                          cudaStream_t stream) {
  if (n == 0 || free_count == 0) return;
  const uint32_t n_blocks = (n + kScanBlock - 1) / kScanBlock;
  CompactFlagKernel<<<n_blocks, 1024, 0, stream>>>(surfels, pitch, n, block_sums);
  CompactScanBlocksKernel<<<1, 1024, 0, stream>>>(block_sums, n_blocks);
  CompactListKernel<<<n_blocks, 1024, 0, stream>>>(surfels, pitch, n, block_sums);
  if (active) CompactMoveActiveKernel<<<(n + 255) / 256, 256, 0, stream>>>(surfels, pitch, n, free_count, active);
  else CompactMoveKernel<<<(n + 255) / 256, 256, 0, stream>>>(surfels, pitch, n, free_count);
}

}  // namespace bba
