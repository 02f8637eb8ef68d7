// pose_solve.cu -- device-side Gauss-Newton step of DirectBA::EstimateFramePose for a list of keyframes.
//
// The reference downloads H (21 floats) and b (6 floats) per keyframe and iteration, solves on the CPU and
// re-uploads the pose (direct_ba_alternating.cc:153-233, one blocking cudaStreamSynchronize each).  Here one
// thread per keyframe does the fp64 LDLT (host_math.hpp SolveLDLT<6>), the Sophus update
// global_T_frame <- global_T_frame * exp(-x), the convergence test and the work-list compaction on the
// device, so a whole pose step needs no host round trip.
//
// This translation unit is compiled WITHOUT -use_fast_math.
#include "host_math.hpp"
#include "kernels.cuh"

namespace bba {

// DET (the deterministic mode): the accumulator record is read from the keyframe's exact sums, rounded to fp64, instead of acc.
template <bool DET>
__global__ void __launch_bounds__(256) PoseSolveKernel(const PoseSolveArgs a) {
  __shared__ int next_count;
  __shared__ unsigned long long tot[5];
  const int count = *a.count_in;
  if (threadIdx.x == 0) next_count = 0;
  if (threadIdx.x < 5) tot[threadIdx.x] = 0ull;
  __syncthreads();
  for (int i = threadIdx.x; i < count; i += blockDim.x) {
    const int kf = a.work_in[i];
    double* acc = a.acc + static_cast<size_t>(kf) * kPoseAccSize;
    double rounded[DET ? kPoseAccSize : 1];
    if constexpr (DET) {
      ExactSum* e = a.exact + static_cast<size_t>(kf) * kPoseAccSize;
      for (int j = 0; j < kPoseAccSize; ++j) {
        rounded[j] = ExactFinalize(e[j]);
        e[j] = ExactSum{};
      }
      acc = rounded;
    }
    // The reference's buffers are fp32 (PoseEstimationHelperBuffers, kernels.h:47-58); it casts to double for the
    // solve (direct_ba_alternating.cc:206).  Round to fp32 first to stay on its numerical path.
    double H[21], b[6], x[6];
    for (int j = 0; j < 21; ++j) H[j] = static_cast<double>(static_cast<float>(acc[j]));
    for (int j = 0; j < 6; ++j) b[j] = static_cast<double>(static_cast<float>(acc[21 + j]));
    if (a.iteration == 0) {
      double* fs = a.first_stats + static_cast<size_t>(kf) * 8;
      fs[0] = acc[27]; fs[1] = acc[28]; fs[2] = acc[29]; fs[3] = acc[30]; fs[4] = acc[31];
      fs[5] = static_cast<double>(a.stage_counts[2 * kf]);
      fs[6] = static_cast<double>(a.stage_counts[2 * kf + 1]);
      fs[7] = 0.0;
    }
    atomicAdd(&tot[0], 1ull);
    atomicAdd(&tot[1], a.stage_counts[2 * kf]);
    atomicAdd(&tot[2], a.stage_counts[2 * kf + 1]);
    atomicAdd(&tot[3], static_cast<unsigned long long>(acc[27] + 0.5));
    atomicAdd(&tot[4], static_cast<unsigned long long>(acc[28] + 0.5));
    for (int j = 0; j < kPoseAccSize; ++j) acc[j] = 0.0;
    a.stage_counts[2 * kf] = 0ull;
    a.stage_counts[2 * kf + 1] = 0ull;

    float* pe = a.pose_est + static_cast<size_t>(kf) * 7;
    if (a.term_offsets) {
      // the soft pose terms (a prior, the equivalent priors of relative pose constraints and their damping anchors), added to
      // the rounded sums in fp64 at the current estimate, in list order, each scaled by the weight of its loss there (w = 1.0
      // exactly for a trivial loss, so H + 1.0 * Hp = H + Hp)
      const int end = a.term_offsets[kf + 1];
      for (int t = a.term_offsets[kf]; t < end; ++t) {
        const PoseTerm& term = a.terms[t];
        double Hp[21], bp[6], cost, rho, w;
        PosePriorTerms(term.pose, pe, term.info, Hp, bp, &cost);
        RobustLoss(term.loss.type, term.loss.scale, 2.0 * cost, &rho, &w);
        for (int j = 0; j < 21; ++j) H[j] += w * Hp[j];
        for (int j = 0; j < 6; ++j) b[j] += w * bp[j];
      }
    }
    if (a.attitude && a.attitude[kf].has) {
      // the attitude prior (DESIGN §3.17), after the terms, weighted as they are
      const bba_attitude_prior& ap = a.attitude[kf].p;
      double Hp[21], bp[6], cost, rho, w;
      AttitudePriorTerms(ap.reference_direction, ap.measured_direction, ap.information, pe, Hp, bp, &cost);
      RobustLoss(ap.loss.type, ap.loss.scale, 2.0 * cost, &rho, &w);
      for (int j = 0; j < 21; ++j) H[j] += w * Hp[j];
      for (int j = 0; j < 6; ++j) b[j] += w * bp[j];
    }
    SolveLDLT<6>(H, b, x);
    float xf[6], neg[6];
    for (int j = 0; j < 6; ++j) {
      xf[j] = static_cast<float>(x[j]);
      neg[j] = -xf[j];
    }
    Pose est;
    est.q[0] = pe[0]; est.q[1] = pe[1]; est.q[2] = pe[2]; est.q[3] = pe[3];
    est.t[0] = pe[4]; est.t[1] = pe[5]; est.t[2] = pe[6];
    est = Compose(est, Exp(neg));   // direct_ba_alternating.cc:214 (kDamping = 1)
    pe[0] = est.q[0]; pe[1] = est.q[1]; pe[2] = est.q[2]; pe[3] = est.q[3];
    pe[4] = est.t[0]; pe[5] = est.t[1]; pe[6] = est.t[2];
    float M[12];
    ToMatrix3x4(Inverse(est), M);
    for (int j = 0; j < 12; ++j) a.kfs[kf].T[j] = M[j];

    const bool conv = IsScale1PoseEstimationConverged(xf);   // direct_ba_alternating.cc:231
    a.iterations[kf] = a.iteration + 1;
    a.converged[kf] = conv ? 1 : 0;
    if (!conv && a.iteration + 1 < a.max_iterations) {
      const int pos = atomicAdd(&next_count, 1);
      a.work_out[pos] = kf;
    }
  }
  __syncthreads();
  if (threadIdx.x < 5 && tot[threadIdx.x]) atomicAdd(a.totals + threadIdx.x, tot[threadIdx.x]);
  if (threadIdx.x == 0) {
    *a.queue = 0u;
    *a.count_out = next_count;
    // Publish progress to the host (zero-copy) so that it can stop enqueueing iterations once every keyframe
    // has converged, without ever blocking the stream.
    a.host_flag[1] = next_count;
    __threadfence_system();
    a.host_flag[0] = a.iteration + 1;
  }
}

LaunchResult LaunchPoseSolve(const PoseSolveArgs& args, cudaStream_t stream) {
  if (args.exact) PoseSolveKernel<true><<<1, 256, 0, stream>>>(args);
  else PoseSolveKernel<false><<<1, 256, 0, stream>>>(args);
  return {1};
}

}  // namespace bba
