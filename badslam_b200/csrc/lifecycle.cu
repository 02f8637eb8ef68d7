// lifecycle.cu -- end-of-BA surfel maintenance (DirectBA::PerformBASchemeEndTasks, direct_ba.cc:566-653):
//  * ObservationStatsKernel: DeleteSurfelsAndUpdateRadiiCUDA (kernel_delete_surfels.cc:40-98, kernel_delete_surfels.cu:42-164).
//    Per surfel, over EVERY keyframe: observation count, free-space violations (the pixel's surface lies behind the surfel
//    by more than the association threshold) and the smallest measured radius^2; then delete (x = NaN pattern) surfels
//    with too few observations or more violations than observations, and store the new radius^2 otherwise.
//    The reference launches one kernel per keyframe that read-modify-writes three accumulator rows; here one persistent
//    launch walks (keyframe group, surfel tile) items group-major like the geometry kernels (kernels.cu).
//  * Compaction: CompactSurfelsCUDA (kernel_compact_surfels.cu:159-279): the r-th valid surfel counted from the END moves into
//    the r-th free spot counted from the front when that spot lies in front of it -- the same permutation as the reference
//    (two cub::DeviceScan passes there; here one three-kernel exclusive scan, then CompactMoveKernel).  The surfel creation
//    below finds its append positions with the same scan; a policy (CompactionScan / CreationScan) says what it reads and writes.
#include <cuda.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "persistent.cuh"

namespace bba {

namespace {

constexpr int kThreads = 256;
constexpr int kGroup = 16;
constexpr uint32_t kDeletedPattern = 0x7fffffffu;   // CUDART_NAN_F

}  // namespace

__global__ void __launch_bounds__(kThreads) ObservationStatsKernel(const __grid_constant__ SurfelStatsArgs a) {
  const uint32_t tile_len = 1u << a.tile_shift;
  const uint32_t n_tiles = (a.local_count + tile_len - 1) >> a.tile_shift;
  const uint32_t n_groups = (a.kf_count + kGroup - 1) / kGroup;
  const uint32_t n_items = n_groups * n_tiles;
  const size_t P = a.pitch;
  const int lane = threadIdx.x & 31;
  const CameraParams& cam = a.cam;
  uint32_t group, tile;
  while (ClaimItem(a.queue, n_tiles, n_items, a.tile_epoch, &group, &tile)) {
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
          KfRegs K;
          LoadKfGlobal(a.kfs, kf, &K);
          Assoc r;
          if (!ProjectIntoImage(cam, K.T, gp, &r)) continue;
          const PixelLoads l = LoadPixel(cam, K.depth, K.depth_pitch, K.normals, K.normals_pitch, r);
          const FreeSpaceTest t = AssociateFreeSpace(cam, K.T, nrm, l, &r);
          if (t == kFreeSpaceViolation) viol += 1.f;
          if (t != kFreeSpaceAssociated) continue;
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
              StoreReplicas(a.surfels, a.peers.surfels, a.peers.count, kRowX * P + i, __uint_as_float(kDeletedPattern));
              deleted = true;
            }
          } else {
            StoreReplicas(a.surfels, a.peers.surfels, a.peers.count, kRowRadiusSq * P + i, min_r2);
          }
        }
      }
      deleted_here += __popc(__ballot_sync(0xffffffffu, deleted));
    }
    if (lane == 0 && deleted_here) atomicAdd(a.deleted_count, deleted_here);
    RetireItem(a.tile_epoch, group, tile);
  }
}

// ---- exclusive scan of u32 counts (compaction, surfel creation) -----------------------------------------------------------
// ScanCountKernel sums the counts of every block, CompactScanBlocksKernel scans the block sums, ScanApplyKernel scans within
// each block and hands every element its exclusive offset.  A policy says where the counts come from and what is written at the
// offsets: Count(i) is element i's count in the counting pass, Load(i) the same count in the apply pass, Store(i, offset, count)
// the apply pass's output.
constexpr int kScanItems = 4;                               // elements per thread
constexpr int kScanBlock = 1024 * kScanItems;               // elements per block

namespace {

// compaction: flag (1 = deleted) -> scratch row Accum2; exclusive count of deleted surfels in front of every surfel -> row
// Accum0; list of free spots -> row Accum3
struct CompactionScan {
  float* surfels;
  size_t P;
  __device__ unsigned int* Row(int k) const { return reinterpret_cast<unsigned int*>(surfels + (kRowAccum0 + k) * P); }
  __device__ unsigned int Count(uint32_t i) const {
    const unsigned int f = __float_as_uint(surfels[kRowX * P + i]) == kDeletedPattern ? 1u : 0u;
    Row(2)[i] = f;
    return f;
  }
  __device__ unsigned int Load(uint32_t i) const { return Row(2)[i]; }
  __device__ void Store(uint32_t i, unsigned int before, unsigned int f) const {
    Row(0)[i] = before;
    if (f) Row(3)[before] = i;
  }
};

// surfel creation: out[i] = in[0] + ... + in[i - 1]
struct CreationScan {
  const unsigned int* in;
  unsigned int* out;
  __device__ unsigned int Count(uint32_t i) const { return in[i]; }
  __device__ unsigned int Load(uint32_t i) const { return in[i]; }
  __device__ void Store(uint32_t i, unsigned int offset, unsigned int) const { out[i] = offset; }
};

}  // namespace

// per-block sum of the counts -> block_sums
template <class Scan>
__global__ void __launch_bounds__(1024) ScanCountKernel(const Scan s, uint32_t n, unsigned int* __restrict__ block_sums) {
  const uint32_t base = blockIdx.x * kScanBlock + threadIdx.x * kScanItems;
  unsigned int cnt = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k)
    if (base + k < n) cnt += s.Count(base + k);
  cnt = BlockSum(cnt);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = cnt;
}

// exclusive scan of the block sums in place (one block); block_sums[n_blocks] receives the total
__global__ void __launch_bounds__(1024) CompactScanBlocksKernel(unsigned int* __restrict__ block_sums, uint32_t n_blocks) {
  unsigned int carry = 0;   // identical in every thread
  for (uint32_t base = 0; base < n_blocks; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    unsigned int chunk_total;
    const unsigned int offset = BlockExclusiveScan(i < n_blocks ? block_sums[i] : 0u, &chunk_total);
    if (i < n_blocks) block_sums[i] = carry + offset;
    carry += chunk_total;
    __syncthreads();   // the next chunk's scan rewrites the warp offsets and the total
  }
  if (threadIdx.x == 0) block_sums[n_blocks] = carry;
}

template <class Scan>
__global__ void __launch_bounds__(1024) ScanApplyKernel(const Scan s, uint32_t n, const unsigned int* __restrict__ block_offsets) {
  const uint32_t base = blockIdx.x * kScanBlock + threadIdx.x * kScanItems;
  unsigned int c[kScanItems], mine = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    c[k] = (base + k < n) ? s.Load(base + k) : 0u;
    mine += c[k];
  }
  unsigned int block_total;
  unsigned int run = block_offsets[blockIdx.x] + BlockExclusiveScan(mine, &block_total);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < n) s.Store(base + k, run, c[k]);
    run += c[k];
  }
}

// CompactSurfelsCUDAKernel (kernel_compact_surfels.cu:126-157); ACTIVE = adapt_active_surfels (direct_ba_alternating.cc:530;
// not at the end of a BA call, direct_ba.cc:618): the active flags move with the surfels
template <bool ACTIVE>
__global__ void __launch_bounds__(256) CompactMoveKernel(float* __restrict__ surfels, uint32_t pitch, uint32_t n, uint32_t free_count,
                                                         uint8_t* __restrict__ active) {
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
  if constexpr (ACTIVE) active[spot] = active[i];
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
      cell = SparseCell(a.cam, r.px, r.py);
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

// The seed pixel of sparse cell c (kernel_create_surfels.cu:40-73): the reference takes whichever valid pixel of the cell wins an
// atomicCAS; here it is the valid pixel inside the one-pixel border with the smallest hashed raster index (a fixed pseudo-random
// choice: always taking the first pixel would put the seeds on a regular lattice).  Its raster index, or kInvalidIndex when the
// cell holds no valid pixel.  SeedKernel and FrameSeedCountKernel.
__device__ __forceinline__ unsigned int CellSeedPixel(const CameraParams& cam, const uint16_t* depth, uint32_t depth_pitch, uint32_t c) {
  const int cy = c / cam.cf_w, cx = c - cy * cam.cf_w;
  unsigned int best_key = kInvalidIndex, best = kInvalidIndex;
  for (int y = cy * cam.cell; y < min((cy + 1) * cam.cell, cam.h); ++y) {
    for (int x = cx * cam.cell; x < min((cx + 1) * cam.cell, cam.w); ++x) {
      if (x < 1 || y < 1 || x >= cam.w - 1 || y >= cam.h - 1) continue;
      if (LoadPixelU16(depth, depth_pitch, x, y) & kInvalidDepthBit) continue;
      const unsigned int seq = static_cast<unsigned int>(y) * cam.w + x;
      const unsigned int key = SurfelArrivalKey(seq);
      if (best == kInvalidIndex || key < best_key) {
        best_key = key;
        best = seq;
      }
    }
  }
  return best;
}

// CountObservationsForNewSurfels over the co-visible keyframes + FilterNewSurfels (kernel_create_surfels.cu:211-334) for the seed
// pixel (sx, sy) of cell c: does it keep its new surfel?  FilterSeedsKernel and FrameSeedCountKernel.
__device__ __forceinline__ bool SeedSurvives(const CameraParams& cam, const uint16_t* depth, uint32_t depth_pitch, const uint16_t* normals,
                                             uint32_t normals_pitch, const CovisEntry* covis, int covis_count, int min_observation_count,
                                             uint32_t c, int sx, int sy) {
  const float d = RawToCalibratedDepth(cam.a, __ldg(cam.cfactor + c), cam.raw_to_float, LoadPixelU16(depth, depth_pitch, sx, sy));
  const Vec3 p_in = V3(d * (cam.fx_inv * sx + cam.cx_inv), d * (cam.fy_inv * sy + cam.cy_inv), d);
  const Vec3 n_in = U16ToImageSpaceNormal(LoadPixelU16(normals, normals_pitch, sx, sy));
  unsigned int obs = 1, viol = 0;
  for (int k = 0; k < covis_count; ++k) {
    const CovisEntry& ce = covis[k];
    Assoc r;
    if (!ProjectIntoImage(cam, ce.R, p_in, &r)) continue;
    // IsAssociatedWithPixel<true> for a pixel-defined surfel (surfel_projection_nvcc_only.cuh:130-236)
    const PixelLoads l{LoadPixelU16(ce.depth, ce.depth_pitch, r.px, r.py), LoadPixelU16(ce.normals, ce.normals_pitch, r.px, r.py),
                       __ldg(cam.cfactor + SparseCell(cam, r.px, r.py))};
    const FreeSpaceTest t = AssociateFreeSpace(cam, ce.R, n_in, l, &r);
    if (t == kFreeSpaceViolation) ++viol;
    if (t != kFreeSpaceAssociated) continue;
    ++obs;
  }
  return !(obs < static_cast<unsigned int>(min_observation_count) || viol > obs);
}

// one seed pixel per unsupported cell; flags are pre-zeroed
__global__ void __launch_bounds__(256) SeedKernel(const __grid_constant__ LifecycleArgs a) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.cells || a.sup[c] != kInvalidIndex) return;
  const unsigned int best = CellSeedPixel(a.cam, a.depth, a.depth_pitch, c);
  if (best != kInvalidIndex) a.flags[best] = 1u;
}

// the filter of every seed pixel (the flagged pixel of an unsupported cell)
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
  if (!SeedSurvives(cam, a.depth, a.depth_pitch, a.normals, a.normals_pitch, a.covis, a.covis_count, a.min_observation_count, c, sx, sy))
    a.flags[static_cast<size_t>(sy) * cam.w + sx] = 0u;
}

// bba_measure_frame_overlap's seed count (DESIGN §3.20): thread (cell c, frame blockIdx.y) decides what SeedKernel and
// FilterSeedsKernel would decide for c if the frame were a keyframe whose supported cells are its covered bits -- valid (c has a
// seed pixel), uncovered (valid, and no associated surfel in c: creation seeds it) and surviving (uncovered, and the seed passes
// the filter against the frame's co-visible keyframes).  Warp ballots, one integer atomic per warp and count.
__global__ void __launch_bounds__(256) FrameSeedCountKernel(const __grid_constant__ FrameSeedArgs a) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  const int f = blockIdx.y;
  const KfDevice& fr = a.frames[f];
  const uint16_t* depth = fr.depth;
  const uint32_t depth_pitch = fr.depth_pitch;
  bool valid = false, uncovered = false, survives = false;
  if (c < a.cells) {
    const unsigned int seed = CellSeedPixel(a.cam, depth, depth_pitch, c);
    valid = seed != kInvalidIndex;
    uncovered = valid && !((__ldg(a.covered + static_cast<size_t>(f) * a.cell_words + (c >> 5)) >> (c & 31u)) & 1u);
    if (uncovered) {
      const int sy = seed / a.cam.w, sx = seed - sy * a.cam.w;
      const int begin = __ldg(a.covis_offsets + f), end = __ldg(a.covis_offsets + f + 1);
      survives = SeedSurvives(a.cam, depth, depth_pitch, fr.normals, fr.normals_pitch, a.covis + begin, end - begin, a.min_observation_count,
                              c, sx, sy);
    }
  }
  const unsigned v = __ballot_sync(0xffffffffu, valid), u = __ballot_sync(0xffffffffu, uncovered),
                 s = __ballot_sync(0xffffffffu, survives);
  if ((threadIdx.x & 31) == 0) {
    uint32_t* out = a.counts + 3 * static_cast<size_t>(f);
    if (v) atomicAdd(out + 0, static_cast<uint32_t>(__popc(v)));
    if (u) atomicAdd(out + 1, static_cast<uint32_t>(__popc(u)));
    if (s) atomicAdd(out + 2, static_cast<uint32_t>(__popc(s)));
  }
}

// CreateNewSurfel (kernel_create_surfels.cu:97-165) for every flagged pixel, appended in raster order
__global__ void __launch_bounds__(256) CreateSurfelsKernel(const __grid_constant__ LifecycleArgs a, const unsigned int* __restrict__ index) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  const CameraParams& cam = a.cam;
  if (s >= static_cast<uint32_t>(cam.w) * cam.h || !a.flags[s]) return;
  const int y = s / cam.w, x = s - y * cam.w;
  const uint32_t out = a.n + index[s];
  const size_t P = a.pitch;
  const float d = RawToCalibratedDepth(cam.a, __ldg(cam.cfactor + SparseCell(cam, x, y)), cam.raw_to_float, LoadPixelU16(a.depth, a.depth_pitch, x, y));
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

static uint32_t GridFor(uint32_t n, int sm_count) {
  return static_cast<uint32_t>(std::min<uint64_t>((static_cast<uint64_t>(n) + 255) / 256, static_cast<uint64_t>(sm_count) * 16));
}

LaunchResult LaunchSupportSurfels(const LifecycleArgs& a, int sm_count, cudaStream_t stream) {
  // kernel_supporting_surfels.cc:61-63
  const cudaError_t e = cudaMemsetAsync(a.sup, 0xff, sizeof(unsigned int) * kMergeBuffers * a.cells, stream);
  if (a.n == 0) return {0, e};
  SupportLevel0Kernel<<<GridFor(a.n, sm_count), 256, 0, stream>>>(a);
  return {1, e};
}

LaunchResult LaunchMergeSurfels(const LifecycleArgs& a, int sm_count, cudaStream_t stream) {
  LaunchResult r = LaunchSupportSurfels(a, sm_count, stream);
  if (a.n == 0) return r;
  SupportNextKernel<<<GridFor(a.n, sm_count), 256, 0, stream>>>(a, 1);
  SupportNextKernel<<<GridFor(a.n, sm_count), 256, 0, stream>>>(a, 2);
  MergeDecideKernel<<<(a.cells + 255) / 256, 256, 0, stream>>>(a);
  MergeApplyKernel<<<GridFor(a.n, sm_count), 256, 0, stream>>>(a);
  r.kernels += 4;
  return r;
}

LaunchResult LaunchSeedNewSurfels(const LifecycleArgs& a, bool filter, cudaStream_t stream) {
  const uint32_t pixels = static_cast<uint32_t>(a.cam.w) * a.cam.h;
  const cudaError_t e = cudaMemsetAsync(a.flags, 0, sizeof(unsigned int) * pixels, stream);
  SeedKernel<<<(a.cells + 255) / 256, 256, 0, stream>>>(a);
  if (filter) FilterSeedsKernel<<<(a.cells + 127) / 128, 128, 0, stream>>>(a);
  return {filter ? 2 : 1, e};
}

// block_sums holds one offset per block of kScanBlock elements and the total behind them
uint32_t ScanTotalIndex(uint32_t n) { return (n + kScanBlock - 1) / kScanBlock; }
uint32_t ScanScratchWords(uint32_t n) { return ScanTotalIndex(n) + 2; }

template <class Scan>
static LaunchResult LaunchScan(const Scan& s, uint32_t n, unsigned int* block_sums, cudaStream_t stream) {
  const uint32_t n_blocks = ScanTotalIndex(n);
  ScanCountKernel<<<n_blocks, 1024, 0, stream>>>(s, n, block_sums);
  CompactScanBlocksKernel<<<1, 1024, 0, stream>>>(block_sums, n_blocks);
  ScanApplyKernel<<<n_blocks, 1024, 0, stream>>>(s, n, block_sums);
  return {3};
}

LaunchResult LaunchExclusiveScan(const unsigned int* in, uint32_t n, unsigned int* out, unsigned int* block_sums, cudaStream_t stream) {
  return LaunchScan(CreationScan{in, out}, n, block_sums, stream);
}

LaunchResult LaunchFrameSeedCount(const FrameSeedArgs& a, cudaStream_t stream) {
  if (a.frame_count <= 0 || a.cells == 0) return {};
  if (a.frame_count > 65535) return {0, cudaErrorInvalidValue};
  FrameSeedCountKernel<<<dim3((a.cells + 255) / 256, a.frame_count), 256, 0, stream>>>(a);
  return {1};
}

LaunchResult LaunchCreateSurfels(const LifecycleArgs& a, const unsigned int* index, cudaStream_t stream) {
  const uint32_t pixels = static_cast<uint32_t>(a.cam.w) * a.cam.h;
  CreateSurfelsKernel<<<(pixels + 255) / 256, 256, 0, stream>>>(a, index);
  return {1};
}

LaunchResult LaunchObservationStats(SurfelStatsArgs a, int sm_count, cudaStream_t stream) {
  if (a.local_count == 0 || a.kf_count <= 0) return {};
  int per_sm = 0;
  LaunchResult r{1, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ObservationStatsKernel, kThreads, 0)};
  const uint32_t ctas = EpochOrderedGrid(per_sm, sm_count, kThreads, a.local_count, (a.kf_count + kGroup - 1) / kGroup, &a.tile_shift);
  const uint32_t n_tiles = (a.local_count + (1u << a.tile_shift) - 1) >> a.tile_shift;
  r += cudaMemsetAsync(a.queue, 0, sizeof(unsigned int), stream);
  r += cudaMemsetAsync(a.tile_epoch, 0, sizeof(unsigned int) * n_tiles, stream);
  ObservationStatsKernel<<<ctas, kThreads, 0, stream>>>(a);
  return r;
}

LaunchResult LaunchCompactSurfels(float* surfels, uint32_t pitch, uint32_t n, uint32_t free_count, unsigned int* block_sums,
                                  uint8_t* active, cudaStream_t stream) {
  if (n == 0 || free_count == 0) return {};
  LaunchResult r = LaunchScan(CompactionScan{surfels, pitch}, n, block_sums, stream);
  if (active) CompactMoveKernel<true><<<(n + 255) / 256, 256, 0, stream>>>(surfels, pitch, n, free_count, active);
  else CompactMoveKernel<false><<<(n + 255) / 256, 256, 0, stream>>>(surfels, pitch, n, free_count, nullptr);
  r.kernels += 1;
  return r;
}

}  // namespace bba
