// pcg.cu -- matrix-free preconditioned-conjugate-gradient Gauss-Newton step over ALL unknowns at once
// (DirectBA::BundleAdjustmentPCG, applications/badslam/src/badslam/direct_ba_pcg.cc:43-819; kernels kernel_pcg.cu:179-1372).
//
// Unknown vector (direct_ba_pcg.cc:273-309): [6 per keyframe except the gauge keyframe] [1 or 3 per surfel: offset along the
// normal, descriptor 1, descriptor 2] [fx^-1 fy^-1 cx^-1 cy^-1 a + one cfactor per sparse cell] [colour fx fy cx cy].
//
// The reference launches PCGInitCUDAKernel / PCGStep1CUDAKernel once per keyframe (2K launches per inner step) and sums every
// pose / intrinsics entry with a block-wide CUB reduction + atomic.  Here ONE persistent launch per pass walks
// (group of 16 keyframes) x (32-surfel tile) items group-major (the images of a group stay in L2): a lane owns one surfel
// for the whole item, keeps its surfel-unknown sums in registers (one RED per unknown per item), pose sums leave through a
// transposed warp reduction per keyframe, intrinsics sums and the scalar p^T A p once per item.
// The dot products alpha_n / alpha_d / beta_n are accumulated in fp64 (the vectors stay fp32 = PCGScalar, kernels.cuh:62).
#include <cuda.h>

#include <algorithm>

#include "persistent.cuh"

namespace bba {

namespace {

constexpr int kThreads = 256;
constexpr int kGroup = 16;
constexpr float kDiagEpsilon = 1e-8f;   // kernel_pcg.cu:44
constexpr float kAPriorWeight = 10.f;   // kernel_pcg.cu:48

// Grid-wide fp64 sum in a FIXED order (for the vector kernels): every block parks its partial sum, the last block to arrive adds
// them up in block order and folds the total into *dst.  The result depends on the inputs only -- not on the order in which
// atomics land -- so the replicas of a multi-GPU job, which run these kernels on identical vectors, compute bit-identical
// alpha / beta (and with them identical step lengths and identical inner-loop decisions), and single-GPU runs are reproducible.
// partials: >= gridDim.x doubles; counter: zero before the launch, zero again after it.
__device__ __forceinline__ void GridOrderedAdd(double* dst, double v, double* partials, unsigned int* counter) {
  v = BlockSum(v);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = v;
    __threadfence();
    if (atomicAdd(counter, 1u) == gridDim.x - 1) {
      __threadfence();
      double total = 0.0;
      for (unsigned int b = 0; b < gridDim.x; ++b) total += __ldcg(partials + b);
      *dst += total;
      *counter = 0u;
    }
  }
  __syncthreads();   // (BlockSum's partials are reused by the next call)
}

__device__ __forceinline__ float DiagExtra(uint32_t i, uint32_t a_index) {   // lambda (+ the prior on `a`) on the diagonal
  return kDiagEpsilon + ((i == a_index) ? (kAPriorWeight * kAPriorWeight) : 0.f);
}

}  // namespace

// INIT = true : r -= J^T W F, M += diag(J^T W J)          (PCGInitCUDAKernel, kernel_pcg.cu:179-507)
// INIT = false: g += J^T W J p, alpha_d += p^T J^T W J p   (PCGStep1CUDAKernel, kernel_pcg.cu:644-1037)
template <bool INIT>
__global__ void __launch_bounds__(kThreads) PcgAccumulateKernel(const __grid_constant__ PcgArgs a) {
  const uint32_t n_tiles = (a.end - a.begin + 31u) / 32u;
  const uint32_t n_groups = (a.kf_count + kGroup - 1) / kGroup;
  const uint32_t n_items = n_groups * n_tiles;
  const size_t P = a.pitch;
  const int lane = threadIdx.x & 31;
  const CameraParams& cam = a.cam;
  const bool use_depth = cam.use_depth != 0, use_desc = cam.use_desc != 0;

  uint32_t group, tile;
  while (ClaimItem(a.queue, n_tiles, n_items, nullptr, &group, &tile)) {
    const int j_begin = group * kGroup, j_end = min(a.kf_count, static_cast<int>(group + 1) * kGroup);
    // this rank's surfels through the dense local index of the 256-surfel granule sharding (kernels.cuh; identity on one GPU)
    const uint32_t li = a.begin + tile * 32u + lane;
    const uint32_t i = SurfelShardToGlobal(li, a.shard_rank, a.shard_world);
    const bool valid = li < a.end && i < a.n;

    Vec3 gp = V3(0, 0, 0), nrm = V3(0, 0, 1);
    float radius_sq = 0.f, d1 = 0.f, d2 = 0.f;
    if (valid) {
      gp = V3(a.surfels[kRowX * P + i], a.surfels[kRowY * P + i], a.surfels[kRowZ * P + i]);
      nrm = UnpackNormal(__float_as_uint(a.surfels[kRowNormal * P + i]));
      if (use_desc) {
        radius_sq = a.surfels[kRowRadiusSq * P + i];
        d1 = a.surfels[kRowD1 * P + i];
        d2 = a.surfels[kRowD2 * P + i];
      }
    }
    const uint32_t su = a.surfel_start + a.surfel_stride * i;   // first unknown of this surfel
    float ps[3] = {0.f, 0.f, 0.f};   // p of the surfel unknowns (STEP1)
    if (!INIT && valid && a.opt_geometry) {
      ps[0] = __ldg(a.p + su);
      if (use_desc) {
        ps[1] = __ldg(a.p + su + 1);
        ps[2] = __ldg(a.p + su + 2);
      }
    }
    float pdi[5] = {0, 0, 0, 0, 0}, pci[4] = {0, 0, 0, 0};
    if (!INIT) {
      if (a.opt_depth_intr) {
#pragma unroll
        for (int c = 0; c < 5; ++c) pdi[c] = __ldg(a.p + a.depth_intr_start + c);
      }
      if (a.opt_color_intr) {
#pragma unroll
        for (int c = 0; c < 4; ++c) pci[c] = __ldg(a.p + a.color_intr_start + c);
      }
    }
    // surfel sums: INIT {r0 r1 r2 M0 M1 M2}, STEP1 {g0 g1 g2}
    float ss[INIT ? 6 : 3];
#pragma unroll
    for (int c = 0; c < (INIT ? 6 : 3); ++c) ss[c] = 0.f;
    // item sums: INIT {di_r 0-4, di_M 5-9, ci_r 10-13, ci_M 14-17}, STEP1 {di_g 0-4, ci_g 5-8, alpha_d 9}
    constexpr int kItemSlots = INIT ? 32 : 16;
    float is[kItemSlots];
#pragma unroll
    for (int c = 0; c < kItemSlots; ++c) is[c] = 0.f;

    for (int kf = j_begin; kf < j_end; ++kf) {
      KfRegs K;
      LoadKfGlobal(a.kfs, kf, &K);
      const bool do_pose = a.opt_poses && kf != a.gauge_kf;
      const uint32_t pose_u = 6u * static_cast<uint32_t>(kf < a.gauge_kf ? kf : kf - 1);   // direct_ba_pcg.cc:325-333
      int st = 0;
      Assoc r;
      PixelLoads l;
      DescEval e;
      bool photo = false;
      if (valid && ProjectIntoImage(cam, K.T, gp, &r)) st = EvalPair(cam, K, gp, nrm, radius_sq, d1, d2, use_desc, &r, &l, &e, &photo);
      bool visible = st == 3;
      if (__ballot_sync(0xffffffffu, visible) == 0) continue;

      // pose sums of this keyframe: INIT {r 0-5, M 6-11}, STEP1 {g 0-5}
      constexpr int kPoseSlots = INIT ? 16 : 8;
      float pa[kPoseSlots];
#pragma unroll
      for (int c = 0; c < kPoseSlots; ++c) pa[c] = 0.f;
      float pp[6] = {0, 0, 0, 0, 0, 0};
      if (!INIT && do_pose) {
#pragma unroll
        for (int c = 0; c < 6; ++c) pp[c] = __ldg(a.p + pose_u + c);
      }

      if (visible) {
        // --- depth residual (kernel_pcg.cu:204-322 / 670-808)
        if (use_depth) {
          float inv_stddev;
          Vec3 up;
          const float raw = DepthResidual(cam, r, &inv_stddev, &up);
          const float w = DepthWeight(raw);
          const float jg = -inv_stddev;
          float J[6];
          DepthPoseJacobian(r, inv_stddev, up, J);
          bool di_valid = false;
          float Jd[6] = {0, 0, 0, 0, 0, 0};   // Jd[5]: wrt the pixel's cfactor
          uint32_t cf_u = 0;
          if (a.opt_depth_intr) {
            di_valid = !(fabsf(DepthIntrinsicsJacobian(cam, r, l, Jd)) < 1e-4f);
            cf_u = a.depth_intr_start + 5u + SparseCell(cam, r.px, r.py);
          }
          if constexpr (INIT) {
            const float wr = w * raw;
            if (a.opt_geometry) {
              ss[0] -= jg * wr;
              ss[3] += jg * w * jg;
            }
            if (do_pose) {
#pragma unroll
              for (int c = 0; c < 6; ++c) {
                pa[c] -= J[c] * wr;
                pa[6 + c] += J[c] * w * J[c];
              }
            }
            if (a.opt_depth_intr) {
              // the reference clears `visible` for the rest of the pair here (kernel_pcg.cu:266-268)
              if (!di_valid) {
                visible = false;
              } else {
#pragma unroll
                for (int c = 0; c < 5; ++c) {
                  is[c] -= Jd[c] * wr;
                  is[5 + c] += Jd[c] * w * Jd[c];
                }
                atomicAdd(a.r + cf_u, -Jd[5] * wr);
                atomicAdd(a.M + cf_u, Jd[5] * w * Jd[5]);
              }
            }
          } else {
            float sum = 0.f;
            if (a.opt_geometry) sum += jg * ps[0];
            if (do_pose) {
#pragma unroll
              for (int c = 0; c < 6; ++c) sum += J[c] * pp[c];
            }
            if (a.opt_depth_intr && di_valid) {
#pragma unroll
              for (int c = 0; c < 5; ++c) sum += Jd[c] * pdi[c];
              sum += Jd[5] * __ldg(a.p + cf_u);
            }
            is[9] += sum * w * sum;
            sum *= w;
            if (a.opt_geometry) ss[0] += jg * sum;
            if (do_pose) {
#pragma unroll
              for (int c = 0; c < 6; ++c) pa[c] += J[c] * sum;
            }
            if (a.opt_depth_intr && di_valid) {
#pragma unroll
              for (int c = 0; c < 5; ++c) is[c] += Jd[c] * sum;
              atomicAdd(a.g + cf_u, Jd[5] * sum);
            }
          }
        }
        // --- descriptor residuals (kernel_pcg.cu:330-505 / 810-1036)
        if (use_desc && visible && photo) {
          const float gx1 = e.gx1 * cam.cfx, gy1 = e.gy1 * cam.cfy, gx2 = e.gx2 * cam.cfx, gy2 = e.gy2 * cam.cfy;
          const float w1 = DescWeight(e.r1), w2 = DescWeight(e.r2);
          float jg1 = 0.f, jg2 = 0.f;
          if (a.opt_geometry) {
            // PositionDescriptorKernel's copy applies cfx / cfy inside term1 / term2 instead; the two orders round differently
            const float term1 = -(r.ln.x * r.lp.z - r.ln.z * r.lp.x);
            const float term2 = -(r.ln.y * r.lp.z - r.ln.z * r.lp.y);
            const float term3 = 1.f / (r.lp.z * r.lp.z);
            jg1 = -(gx1 * term1 + gy1 * term2) * term3;
            jg2 = -(gx2 * term1 + gy2 * term2) * term3;
          }
          float J1[6], J2[6];
          DescPoseJacobian(cam, r.lp, e.gx1, e.gy1, J1);
          DescPoseJacobian(cam, r.lp, e.gx2, e.gy2, J2);
          float C1[4], C2[4];
          ColorIntrinsicsJacobians(r, e, C1, C2);
          if constexpr (INIT) {
            const float wr1 = w1 * e.r1, wr2 = w2 * e.r2;
            if (a.opt_geometry) {
              ss[0] -= jg1 * wr1 + jg2 * wr2;
              ss[3] += jg1 * w1 * jg1 + jg2 * w2 * jg2;
              ss[1] += wr1;   // Jacobian wrt descriptor 1 is -1 for residual 1, 0 for residual 2
              ss[4] += w1;
              ss[2] += wr2;
              ss[5] += w2;
            }
            if (do_pose) {
#pragma unroll
              for (int c = 0; c < 6; ++c) {
                pa[c] -= J1[c] * wr1 + J2[c] * wr2;
                pa[6 + c] += J1[c] * w1 * J1[c] + J2[c] * w2 * J2[c];
              }
            }
            if (a.opt_color_intr) {
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                is[10 + c] -= C1[c] * wr1 + C2[c] * wr2;
                is[14 + c] += C1[c] * w1 * C1[c] + C2[c] * w2 * C2[c];
              }
            }
          } else {
            float sum1 = 0.f, sum2 = 0.f;
            if (a.opt_geometry) {
              sum1 += jg1 * ps[0] - ps[1];
              sum2 += jg2 * ps[0] - ps[2];
            }
            if (do_pose) {
#pragma unroll
              for (int c = 0; c < 6; ++c) {
                sum1 += J1[c] * pp[c];
                sum2 += J2[c] * pp[c];
              }
            }
            if (a.opt_color_intr) {
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                sum1 += C1[c] * pci[c];
                sum2 += C2[c] * pci[c];
              }
            }
            is[9] += sum1 * w1 * sum1 + sum2 * w2 * sum2;
            sum1 *= w1;
            sum2 *= w2;
            if (a.opt_geometry) {
              ss[0] += jg1 * sum1 + jg2 * sum2;
              ss[1] -= sum1;
              ss[2] -= sum2;
            }
            if (do_pose) {
#pragma unroll
              for (int c = 0; c < 6; ++c) pa[c] += J1[c] * sum1 + J2[c] * sum2;
            }
            if (a.opt_color_intr) {
#pragma unroll
              for (int c = 0; c < 4; ++c) is[5 + c] += C1[c] * sum1 + C2[c] * sum2;
            }
          }
        }
      }
      if (do_pose) {
        const float total = WarpTransposeReduce(pa, lane);
        if constexpr (INIT) {
          if (lane < 6) atomicAdd(a.r + pose_u + lane, total);
          else if (lane < 12) atomicAdd(a.M + pose_u + (lane - 6), total);
        } else if (lane < 6) {
          atomicAdd(a.g + pose_u + lane, total);
        }
      }
    }

    // surfel unknowns: one RED per unknown and item (other keyframe groups add to the same entries)
    if (valid && a.opt_geometry) {
      const int n_u = use_desc ? 3 : 1;
      for (int c = 0; c < n_u; ++c) {
        if constexpr (INIT) {
          if (ss[c] != 0.f) atomicAdd(a.r + su + c, ss[c]);
          if (ss[3 + c] != 0.f) atomicAdd(a.M + su + c, ss[3 + c]);
        } else if (ss[c] != 0.f) {
          atomicAdd(a.g + su + c, ss[c]);
        }
      }
    }
    // intrinsics sums (+ alpha_d)
    if constexpr (INIT) {
      if (a.opt_depth_intr || a.opt_color_intr) {
        const float total = WarpTransposeReduce(is, lane);
        if (total != 0.f) {
          if (lane < 5) atomicAdd(a.r + a.depth_intr_start + lane, total);
          else if (lane < 10) atomicAdd(a.M + a.depth_intr_start + (lane - 5), total);
          else if (lane < 14) atomicAdd(a.r + a.color_intr_start + (lane - 10), total);
          else if (lane < 18) atomicAdd(a.M + a.color_intr_start + (lane - 14), total);
        }
      }
    } else {
      const float total = WarpTransposeReduce(is, lane);
      if (total != 0.f) {
        if (lane < 5) { if (a.opt_depth_intr) atomicAdd(a.g + a.depth_intr_start + lane, total); }
        else if (lane < 9) { if (a.opt_color_intr) atomicAdd(a.g + a.color_intr_start + (lane - 5), total); }
        else if (lane == 9) atomicAdd(a.scalars + a.alpha_d_slot, static_cast<double>(total));
      }
    }
  }
}

// PCGInit2CUDAKernel (kernel_pcg.cu:569-605): p0 = M^-1 r0 (prior on `a` and lambda added here), delta = 0, g = 0,
// alpha_n = r0^T p0.  Also pre-loads alpha_d with the lambda/prior term the reference adds after every per-keyframe
// PCGStep1 launch (kernel_pcg.cu:1101-1112), i.e. kf_count times per inner step.
__global__ void __launch_bounds__(256) PcgInit2Kernel(uint32_t n, uint32_t a_index, float a, int kf_count, const float* __restrict__ r,
                                                      const float* __restrict__ M, float* __restrict__ delta, float* __restrict__ g,
                                                      float* __restrict__ p, double* __restrict__ scalars, int slot_alpha_n) {
  double alpha = 0.0, eps = 0.0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float r_value = r[i] + ((i == a_index) ? (-kAPriorWeight * kAPriorWeight * a) : 0.f);
    const float p_value = r_value / (M[i] + DiagExtra(i, a_index));
    p[i] = p_value;
    delta[i] = 0.f;
    g[i] = 0.f;
    alpha += static_cast<double>(r_value * p_value);
    eps += static_cast<double>(DiagExtra(i, a_index) * p_value * p_value);
  }
  GridOrderedAdd(scalars + slot_alpha_n, alpha, scalars + kPcgPartialsA, reinterpret_cast<unsigned int*>(scalars + kPcgCounters));
  GridOrderedAdd(scalars + 1, eps * kf_count, scalars + kPcgPartialsB, reinterpret_cast<unsigned int*>(scalars + kPcgCounters) + 1);
}

// PCGStep2CUDAKernel (kernel_pcg.cu:1115-1166)
__global__ void __launch_bounds__(256) PcgStep2Kernel(uint32_t n, uint32_t a_index, float* __restrict__ r, const float* __restrict__ M,
                                                      float* __restrict__ delta, float* __restrict__ g, const float* __restrict__ p,
                                                      double* __restrict__ scalars, int slot_alpha_n, int slot_beta_n) {
  const float alpha_n = static_cast<float>(scalars[slot_alpha_n]), alpha_d = static_cast<float>(scalars[1]);
  const float alpha = (alpha_d >= 1e-35f) ? (alpha_n / alpha_d) : 0.f;
  double beta = 0.0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float p_value = p[i];
    delta[i] += alpha * p_value;
    float r_value = r[i];
    r_value -= alpha * (g[i] + DiagExtra(i, a_index) * p_value);
    r[i] = r_value;
    const float z_value = r_value / (M[i] + DiagExtra(i, a_index));
    g[i] = z_value;
    beta += static_cast<double>(z_value * r_value);
  }
  GridOrderedAdd(scalars + slot_beta_n, beta, scalars + kPcgPartialsA, reinterpret_cast<unsigned int*>(scalars + kPcgCounters));
}

// PCGStep3CUDAKernel (kernel_pcg.cu:1206-1224) + the g = 0 of the next step (direct_ba_pcg.cc:379) + the next alpha_d's
// lambda/prior term (see PcgInit2Kernel).  scalars[1] must have been cleared before this launch.
__global__ void __launch_bounds__(256) PcgStep3Kernel(uint32_t n, uint32_t a_index, int kf_count, float* __restrict__ g, float* __restrict__ p,
                                                      double* __restrict__ scalars, int slot_alpha_n, int slot_beta_n) {
  const float alpha_n = static_cast<float>(scalars[slot_alpha_n]), beta_n = static_cast<float>(scalars[slot_beta_n]);
  const float beta = (alpha_n >= 1e-35f) ? (beta_n / alpha_n) : 0.f;
  double eps = 0.0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float p_value = g[i] + beta * p[i];
    p[i] = p_value;
    g[i] = 0.f;
    eps += static_cast<double>(DiagExtra(i, a_index) * p_value * p_value);
  }
  GridOrderedAdd(scalars + 1, eps * kf_count, scalars + kPcgPartialsB, reinterpret_cast<unsigned int*>(scalars + kPcgCounters) + 1);
}

// UpdateSurfelsFromPCGDeltaCUDAKernel (kernel_pcg.cu:1278-1308)
__global__ void __launch_bounds__(256) PcgUpdateSurfelsKernel(float* __restrict__ surfels, uint32_t pitch, uint32_t n, int use_desc,
                                                              uint32_t surfel_start, const float* __restrict__ delta) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t P = pitch;
  const uint32_t su = surfel_start + (use_desc ? 3u : 1u) * i;
  const float t = delta[su];
  if (t != 0.f) {
    const Vec3 nrm = UnpackNormal(__float_as_uint(surfels[kRowNormal * P + i]));
    surfels[kRowX * P + i] += t * nrm.x;
    surfels[kRowY * P + i] += t * nrm.y;
    surfels[kRowZ * P + i] += t * nrm.z;
  }
  if (use_desc) {
    surfels[kRowD1 * P + i] = fmaxf(-180.f, fminf(180.f, surfels[kRowD1 * P + i] + delta[su + 1]));
    surfels[kRowD2 * P + i] = fmaxf(-180.f, fminf(180.f, surfels[kRowD2 * P + i] + delta[su + 2]));
  }
}

// UpdateCFactorsFromPCGDeltaCUDAKernel (kernel_pcg.cu:1338-1351)
__global__ void __launch_bounds__(256) PcgUpdateCfactorKernel(float* __restrict__ cfactor, uint32_t cells, const float* __restrict__ delta) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cells) cfactor[i] += delta[i];
}

// Multi-GPU: this rank's part of p^T J^T W J p (fp64, scalars[3]) travels with g through the fp32 sum all-reduce as a
// (high, low) float pair appended to the vector; afterwards the total joins the lambda / prior term already waiting in scalars[1].
__global__ void PcgPackAlphaDKernel(const double* __restrict__ scalars, float* __restrict__ tail) {
  const double v = scalars[3];
  const float hi = static_cast<float>(v);
  tail[0] = hi;
  tail[1] = static_cast<float>(v - static_cast<double>(hi));
}
__global__ void PcgUnpackAlphaDKernel(double* __restrict__ scalars, const float* __restrict__ tail) {
  scalars[1] += static_cast<double>(tail[0]) + static_cast<double>(tail[1]);
  scalars[3] = 0.0;
}
LaunchResult LaunchPcgPackAlphaD(const double* scalars, float* tail, cudaStream_t stream) {
  PcgPackAlphaDKernel<<<1, 1, 0, stream>>>(scalars, tail);
  return {1};
}
LaunchResult LaunchPcgUnpackAlphaD(double* scalars, const float* tail, cudaStream_t stream) {
  PcgUnpackAlphaDKernel<<<1, 1, 0, stream>>>(scalars, tail);
  return {1};
}

// The pose-block terms' part of the products (soft pose priors, relative pose constraints), one thread per pose block with terms,
// after PcgAccumulateKernel.  A thread gathers its block's terms in list order and writes only its own block; the one block
// sums alpha_d's share in a fixed order (a few thousand keyframes at most).
template <bool INIT>
__global__ void __launch_bounds__(256) PcgPoseTermsKernel(const PcgPoseBlock* __restrict__ blocks, int block_count,
                                                          const PcgPoseTerm* __restrict__ terms, float* __restrict__ r,
                                                          float* __restrict__ M, const float* __restrict__ p, float* __restrict__ g,
                                                          double* __restrict__ alpha_d) {
  double pap = 0.0;
  for (int i = threadIdx.x; i < block_count; i += blockDim.x) {
    const PcgPoseBlock blk = blocks[i];
    if constexpr (INIT) {
      for (int e = blk.begin; e < blk.end; ++e) {
        const PcgPoseTerm& t = terms[e];
        int d = 0;
        for (int c = 0; c < 6; ++c) {
          r[blk.u + c] -= t.b[c];
          M[blk.u + c] += t.H[d];
          d += 6 - c;
        }
      }
    } else {
      float pv[6], hp[6];
      for (int c = 0; c < 6; ++c) {
        pv[c] = p[blk.u + c];
        hp[c] = 0.f;
      }
      for (int e = blk.begin; e < blk.end; ++e) {
        const PcgPoseTerm& t = terms[e];
        int idx = 0;
        for (int row = 0; row < 6; ++row)
          for (int col = row; col < 6; ++col) {
            const float h = t.H[idx++];
            hp[row] += h * pv[col];
            if (col != row) hp[col] += h * pv[row];
          }
        if (t.other >= 0) {
          float pj[6];
          for (int c = 0; c < 6; ++c) pj[c] = p[t.other + c];
          for (int row = 0; row < 6; ++row)
            for (int col = 0; col < 6; ++col) hp[row] += t.X[row * 6 + col] * pj[col];
        }
      }
      for (int c = 0; c < 6; ++c) {
        g[blk.u + c] += hp[c];
        pap += static_cast<double>(pv[c] * hp[c]);
      }
    }
  }
  if constexpr (!INIT) {
    pap = BlockSum(pap);
    if (threadIdx.x == 0) *alpha_d += pap;
  }
}

LaunchResult LaunchPcgPoseTerms(const PcgPoseBlock* blocks, int block_count, const PcgPoseTerm* terms, bool init, float* r, float* M,
                                const float* p, float* g, double* alpha_d, cudaStream_t stream) {
  if (block_count <= 0) return {};
  if (init) PcgPoseTermsKernel<true><<<1, 256, 0, stream>>>(blocks, block_count, terms, r, M, p, g, alpha_d);
  else PcgPoseTermsKernel<false><<<1, 256, 0, stream>>>(blocks, block_count, terms, r, M, p, g, alpha_d);
  return {1};
}

LaunchResult LaunchPcgAccumulate(const PcgArgs& a, int sm_count, bool init, cudaStream_t stream) {
  if (a.end <= a.begin || a.kf_count <= 0) return {};
  LaunchResult r{1, cudaMemsetAsync(a.queue, 0, sizeof(unsigned int), stream)};
  const uint64_t n_tiles = (a.end - a.begin + 31u) / 32u;
  const uint64_t n_items = n_tiles * ((a.kf_count + kGroup - 1) / kGroup);
  auto launch = [&](auto kernel) {
    int per_sm = 0;
    r += cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0);
    kernel<<<ItemGrid(per_sm, sm_count, n_items), kThreads, 0, stream>>>(a);
  };
  if (init) launch(PcgAccumulateKernel<true>);
  else launch(PcgAccumulateKernel<false>);
  return r;
}

static uint32_t VectorGrid(uint32_t n, int sm_count) {
  // (<= 2048 blocks: the workspace of the ordered grid sums, kPcgPartialsA / B)
  return static_cast<uint32_t>(std::min<uint64_t>(std::min<uint64_t>((static_cast<uint64_t>(n) + 255) / 256, static_cast<uint64_t>(sm_count) * 8), 2048));
}

LaunchResult LaunchPcgInit2(uint32_t n, uint32_t a_index, float a, int kf_count, const float* r, const float* M, float* delta, float* g,
                            float* p, double* scalars, int slot_alpha_n, int sm_count, cudaStream_t stream) {
  PcgInit2Kernel<<<VectorGrid(n, sm_count), 256, 0, stream>>>(n, a_index, a, kf_count, r, M, delta, g, p, scalars, slot_alpha_n);
  return {1};
}
LaunchResult LaunchPcgStep2(uint32_t n, uint32_t a_index, float* r, const float* M, float* delta, float* g, const float* p, double* scalars,
                            int slot_alpha_n, int slot_beta_n, int sm_count, cudaStream_t stream) {
  PcgStep2Kernel<<<VectorGrid(n, sm_count), 256, 0, stream>>>(n, a_index, r, M, delta, g, p, scalars, slot_alpha_n, slot_beta_n);
  return {1};
}
LaunchResult LaunchPcgStep3(uint32_t n, uint32_t a_index, int kf_count, float* g, float* p, double* scalars, int slot_alpha_n,
                            int slot_beta_n, int sm_count, cudaStream_t stream) {
  PcgStep3Kernel<<<VectorGrid(n, sm_count), 256, 0, stream>>>(n, a_index, kf_count, g, p, scalars, slot_alpha_n, slot_beta_n);
  return {1};
}
LaunchResult LaunchPcgUpdateSurfels(float* surfels, uint32_t pitch, uint32_t n, bool use_desc, uint32_t surfel_start, const float* delta,
                                    cudaStream_t stream) {
  if (n == 0) return {};
  PcgUpdateSurfelsKernel<<<(n + 255) / 256, 256, 0, stream>>>(surfels, pitch, n, use_desc ? 1 : 0, surfel_start, delta);
  return {1};
}
LaunchResult LaunchPcgUpdateCfactor(float* cfactor, uint32_t cells, const float* delta, cudaStream_t stream) {
  PcgUpdateCfactorKernel<<<(cells + 255) / 256, 256, 0, stream>>>(cfactor, cells, delta);
  return {1};
}

}  // namespace bba
