// intrinsics.cu -- camera-intrinsics + depth-deformation step of the alternating BA (OptimizeIntrinsicsCUDA,
// applications/badslam/src/badslam/kernel_opt_intrinsics.cc:39-281).
//
// Unknowns: (fx^-1, fy^-1, cx^-1, cy^-1, a) of the depth camera + one cfactor per sparse cell (arrow-shaped normal
// equations: A 5x5, B 5xP, D diagonal P) and the four pinhole parameters of the colour camera.
//  * IntrinsicsAccumulateKernel: the reference launches AccumulateIntrinsicsCoefficientsCUDAKernel once per keyframe
//    (kernel_opt_intrinsics.cu:46-217) with 20 block-wide CUB reductions + atomics per block; here ONE persistent
//    launch walks (keyframe group, surfel tile) items group-major (images L2-resident), each lane keeps the 34 global
//    sums in registers, one transposed warp reduction + fp64 REDs per item; the per-cell terms go out as fp32 REDs.
//  * IntrinsicsSchurKernel: A -= B D^-1 B^T, b1 -= B D^-1 b2 (kernel_opt_intrinsics.cu:265-347).
//  * IntrinsicsCellUpdateKernel: cfactor -= D^-1 b2 - D^-1 B^T x1 (kernel_opt_intrinsics.cu:374-424).
// The 5x5 / 4x4 solves stay on the host in fp64 like the reference (kernel_opt_intrinsics.cc:171,272).
#include <cuda.h>

#include "persistent.cuh"

namespace bba {

namespace {

constexpr int kThreads = 256;
constexpr int kGroup = 16;
constexpr int kTile = 256;

}  // namespace

// sums layout: [0..14] A upper triangle (5x5), [15..19] b1, [20..29] colour H upper triangle (4x4), [30..33] colour b
// DET (the deterministic mode): every fp32 atomic below except the observation count (an integer below 2^24, exact in any order)
// becomes a deposit into an exact sum.  A cell's sums receive one deposit per associated pair that falls into it, a few per keyframe
// and cell size squared (tens of thousands at cfg3), a global sum one per work item, at most ceil(n / 256) x ceil(K / 16): both far
// below the 2^31 deposits an ExactSum holds.
template <bool OPT_COLOR, bool OPT_DEPTH, bool DET>
__global__ void __launch_bounds__(kThreads) IntrinsicsAccumulateKernel(const __grid_constant__ IntrinsicsArgs a) {
  const uint32_t n_tiles = (a.end - a.begin + kTile - 1) / kTile;
  const uint32_t n_groups = (a.kf_count + kGroup - 1) / kGroup;
  const uint32_t n_items = n_groups * n_tiles;
  const size_t P = a.pitch;
  const int lane = threadIdx.x & 31;
  const CameraParams& cam = a.cam;
  uint32_t group, tile;
  while (ClaimItem(a.queue, n_tiles, n_items, nullptr, &group, &tile)) {
    const int j_begin = group * kGroup, j_end = min(a.kf_count, static_cast<int>(group + 1) * kGroup);
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    float extra0 = 0.f, extra1 = 0.f;   // sums 32, 33
    for (uint32_t sub = 0; sub < kTile / 32; ++sub) {
      const uint32_t li = a.begin + tile * kTile + sub * 32 + lane;
      const uint32_t i = SurfelShardToGlobal(li, a.shard_rank, a.shard_world);
      if (li >= a.end || i >= a.n) continue;
      const Vec3 gp = V3(a.surfels[kRowX * P + i], a.surfels[kRowY * P + i], a.surfels[kRowZ * P + i]);
      const Vec3 nrm = UnpackNormal(__float_as_uint(a.surfels[kRowNormal * P + i]));
      float radius_sq = 0.f, d1 = 0.f, d2 = 0.f;
      if (OPT_COLOR) {
        radius_sq = a.surfels[kRowRadiusSq * P + i];
        d1 = a.surfels[kRowD1 * P + i];
        d2 = a.surfels[kRowD2 * P + i];
      }
      for (int j = j_begin; j < j_end; ++j) {
        KfRegs K;
        LoadKfGlobal(a.kfs, __ldg(a.kf_list + j), &K);
        Assoc r;
        PixelLoads l;
        DescEval e;
        bool photo = false;
        if (!ProjectIntoImage(cam, K.T, gp, &r)) continue;
        if (EvalPair(cam, K, gp, nrm, radius_sq, d1, d2, OPT_COLOR, &r, &l, &e, &photo) != 3) continue;
        if (OPT_DEPTH) {
          float J[6];
          if (fabsf(DepthIntrinsicsJacobian(cam, r, l, J)) > 1e-4f) {
            float inv_stddev;
            Vec3 up;
            const float raw = DepthResidual(cam, r, &inv_stddev, &up);
            const float w = DepthWeight(raw);
            int idx = 0;
#pragma unroll
            for (int rr = 0; rr < 5; ++rr) {
              const float wj = w * J[rr];
#pragma unroll
              for (int c = rr; c < 5; ++c) acc[idx++] += wj * J[c];
            }
            const float wr = w * raw;
#pragma unroll
            for (int rr = 0; rr < 5; ++rr) acc[15 + rr] += wr * J[rr];
            // per-cell terms (kernel_opt_intrinsics.cu:173-190)
            const unsigned int sp = SparseCell(cam, r.px, r.py);
            if constexpr (DET) {
#pragma unroll
              for (int rr = 0; rr < 5; ++rr) ExactDeposit(a.exact_cells + static_cast<size_t>(rr) * a.cell_count + sp, w * J[rr] * J[5]);
              ExactDeposit(a.exact_cells + static_cast<size_t>(5) * a.cell_count + sp, w * J[5] * J[5]);
              ExactDeposit(a.exact_cells + static_cast<size_t>(6) * a.cell_count + sp, w * raw * J[5]);
            } else {
#pragma unroll
              for (int rr = 0; rr < 5; ++rr) atomicAdd(a.cell_B + static_cast<size_t>(rr) * a.cell_count + sp, w * J[rr] * J[5]);
              atomicAdd(a.cell_D + sp, w * J[5] * J[5]);
              atomicAdd(a.cell_b2 + sp, w * raw * J[5]);
            }
            atomicAdd(a.cell_obs + sp, 1.0f);   // fp32 count: exact to 2^24, only tested against 0
          }
        }
        if (OPT_COLOR && photo) {
          // kernel_opt_intrinsics.cu:139-160,193-211: residuals that are exactly 0 are skipped
          float J1[4], J2[4];
          ColorIntrinsicsJacobians(r, e, J1, J2);
          const float w1 = (e.r1 != 0) ? DescWeight(e.r1) : 0.f;
          const float w2 = (e.r2 != 0) ? DescWeight(e.r2) : 0.f;
          int idx = 20;
#pragma unroll
          for (int rr = 0; rr < 4; ++rr) {
#pragma unroll
            for (int c = rr; c < 4; ++c) acc[idx++] += w1 * J1[rr] * J1[c] + w2 * J2[rr] * J2[c];
          }
          acc[30] += w1 * e.r1 * J1[0] + w2 * e.r2 * J2[0];
          acc[31] += w1 * e.r1 * J1[1] + w2 * e.r2 * J2[1];
          extra0 += w1 * e.r1 * J1[2] + w2 * e.r2 * J2[2];
          extra1 += w1 * e.r1 * J1[3] + w2 * e.r2 * J2[3];
        }
      }
    }
    __syncwarp();
    const float total = WarpTransposeReduce(acc, lane);
    auto store = [&](int slot, float v) {
      if constexpr (DET) ExactDeposit(a.exact_sums + slot, v);
      else atomicAdd(a.sums + slot, static_cast<double>(v));
    };
    if (total != 0.f) store(lane, total);
    if (OPT_COLOR) {
      extra0 = WarpSum(extra0);
      extra1 = WarpSum(extra1);
      if (lane == 0 && (extra0 != 0.f || extra1 != 0.f)) {
        store(32, extra0);
        store(33, extra1);
      }
    }
  }
}

// Schur complement over the sparse cells (kernel_opt_intrinsics.cu:265-347): A -= B D^-1 B^T, b1 -= B D^-1 b2, and
// B <- D^-1 B^T, D <- D^-1 b2 in place.  ONE block walks all cells in a fixed order and reduces in a fixed tree, so the
// result is bit-reproducible: with several ranks every replica computes exactly the same intrinsics update.
__global__ void __launch_bounds__(1024) IntrinsicsSchurKernel(uint32_t cell_count, float* __restrict__ B, float* __restrict__ D,
                                                              const float* __restrict__ b2, double* __restrict__ sums) {
  __shared__ double partial[32][20];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double v[20];
#pragma unroll
  for (int i = 0; i < 20; ++i) v[i] = 0.0;
  for (uint32_t p = threadIdx.x; p < cell_count; p += blockDim.x) {
    const float D_inverse = 1.0f / D[p];
    if (!(D_inverse < 1e12f)) {
      D[p] = __int_as_float(0x7fffffff);   // NaN marks cells without constraint
      continue;
    }
    const float D_inv_b2 = D_inverse * b2[p];
    D[p] = D_inv_b2;
    float Bp[5];
#pragma unroll
    for (int r = 0; r < 5; ++r) Bp[r] = B[static_cast<size_t>(r) * cell_count + p];
    int idx = 0;
#pragma unroll
    for (int r = 0; r < 5; ++r) {
#pragma unroll
      for (int c = r; c < 5; ++c) v[idx++] -= static_cast<double>(Bp[r] * D_inverse * Bp[c]);
    }
#pragma unroll
    for (int r = 0; r < 5; ++r) v[15 + r] -= static_cast<double>(Bp[r] * D_inv_b2);
#pragma unroll
    for (int r = 0; r < 5; ++r) B[static_cast<size_t>(r) * cell_count + p] = D_inverse * Bp[r];
  }
#pragma unroll
  for (int i = 0; i < 20; ++i) {
    double s = v[i];
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) partial[warp][i] = s;
  }
  __syncthreads();
  if (threadIdx.x < 20) {
    double s = 0.0;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) s += partial[w][threadIdx.x];
    sums[threadIdx.x] += s;
  }
}

// kernel_opt_intrinsics.cu:374-424
__global__ void __launch_bounds__(256) IntrinsicsCellUpdateKernel(uint32_t cell_count, const float* __restrict__ obs,
                                                                  const float* __restrict__ B, const float* __restrict__ D,
                                                                  const float* __restrict__ x1, float* __restrict__ cfactor) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= cell_count) return;
  float offset = D[p];
  if (isnan(offset)) {
    offset = 0;
  } else {
#pragma unroll
    for (int r = 0; r < 5; ++r) offset -= B[static_cast<size_t>(r) * cell_count + p] * x1[r];
  }
  float cf = cfactor[p] - offset;
  if (obs[p] == 0.f) cf = 0;
  cfactor[p] = cf;
}

LaunchResult LaunchIntrinsicsAccumulate(const IntrinsicsArgs& a, int sm_count, bool optimize_color, bool optimize_depth,
                                        cudaStream_t stream) {
  if (a.end <= a.begin || a.kf_count <= 0) return {};
  LaunchResult r{0, cudaMemsetAsync(a.queue, 0, sizeof(unsigned int), stream)};
  const uint32_t n_tiles = (a.end - a.begin + kTile - 1) / kTile;
  const uint32_t n_groups = (a.kf_count + kGroup - 1) / kGroup;
  const uint64_t n_items = static_cast<uint64_t>(n_tiles) * n_groups;
  auto launch = [&](auto kernel) {
    int per_sm = 0;
    r += cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0);
    kernel<<<ItemGrid(per_sm, sm_count, n_items), kThreads, 0, stream>>>(a);
    r.kernels = 1;
  };
  const bool det = a.exact_cells != nullptr;
  if (optimize_color && optimize_depth) det ? launch(IntrinsicsAccumulateKernel<true, true, true>) : launch(IntrinsicsAccumulateKernel<true, true, false>);
  else if (optimize_color) det ? launch(IntrinsicsAccumulateKernel<true, false, true>) : launch(IntrinsicsAccumulateKernel<true, false, false>);
  else if (optimize_depth) det ? launch(IntrinsicsAccumulateKernel<false, true, true>) : launch(IntrinsicsAccumulateKernel<false, true, false>);
  return r;
}

// One thread per value: the 7 cell rows (cell_B's 5, then cell_D and cell_b2, which follow it in memory) as fp32 of the rounded
// exact sum, then the kIntrinsicsSums global sums in fp64.
__global__ void __launch_bounds__(256) IntrinsicsFinalizeKernel(uint32_t cell_count, const ExactSum* __restrict__ exact_cells,
                                                                float* __restrict__ cells, const ExactSum* __restrict__ exact_sums,
                                                                double* __restrict__ sums) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t n_cells = static_cast<size_t>(7) * cell_count;
  if (i < n_cells) cells[i] = static_cast<float>(ExactFinalize(exact_cells[i]));
  else if (i < n_cells + kIntrinsicsSums) sums[i - n_cells] = ExactFinalize(exact_sums[i - n_cells]);
}
LaunchResult LaunchIntrinsicsFinalize(uint32_t cell_count, const ExactSum* exact_cells, float* cell_B, const ExactSum* exact_sums, double* sums,
                                      cudaStream_t stream) {
  const size_t n = static_cast<size_t>(7) * cell_count + kIntrinsicsSums;
  IntrinsicsFinalizeKernel<<<static_cast<unsigned int>((n + 255) / 256), 256, 0, stream>>>(cell_count, exact_cells, cell_B, exact_sums, sums);
  return {1};
}

__global__ void IntrinsicsConvertSumsKernel(double* sums, float* head, int to_float) {
  const int i = threadIdx.x;
  if (i >= kIntrinsicsSums) return;
  if (to_float) head[i] = static_cast<float>(sums[i]);
  else sums[i] = static_cast<double>(head[i]);
}
LaunchResult LaunchIntrinsicsConvertSums(double* sums, float* head, bool to_float, cudaStream_t stream) {
  IntrinsicsConvertSumsKernel<<<1, 64, 0, stream>>>(sums, head, to_float ? 1 : 0);
  return {1};
}

LaunchResult LaunchIntrinsicsSchur(uint32_t cell_count, float* B, float* D, const float* b2, double* sums, cudaStream_t stream) {
  IntrinsicsSchurKernel<<<1, 1024, 0, stream>>>(cell_count, B, D, b2, sums);
  return {1};
}

LaunchResult LaunchIntrinsicsCellUpdate(uint32_t cell_count, const float* obs, const float* B, const float* D, const float* x1,
                                        float* cfactor, cudaStream_t stream) {
  IntrinsicsCellUpdateKernel<<<(cell_count + 255) / 256, 256, 0, stream>>>(cell_count, obs, B, D, x1, cfactor);
  return {1};
}

}  // namespace bba
