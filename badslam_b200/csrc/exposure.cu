// exposure.cu -- keyframe exposure estimation and compensation (DESIGN.md §3.21): the host orchestration of
// bba_estimate_keyframe_exposures (the exposure walks of kernels.cu, the co-visibility Gram and the one-CTA fp64 solve kernel
// below) and bba_set_keyframe_exposures / bba_get_keyframe_exposures, which re-extract a keyframe's luma with its gain.
#include <cmath>
#include <limits>

#include "handle.hpp"

namespace bba {
namespace {

// ---- the solve (one CTA, fixed order) --------------------------------------------------------------------------------------------
// L x = r over the keyframes of the gauge keyframe's component of C > 0, with x[gauge] = 0: L = diag(rowsum(C) - diag C) -
// offdiag(C).  The CTA builds the CSR of C's off-diagonal non-zeros (columns in order), marks the component by sweeps of
// reachability to a fixpoint (the set does not depend on the sweeps' interleaving), then runs Jacobi-preconditioned CG in fp64 with
// block sums in a fixed order, so the result is the same bits on every run.
constexpr int kSolveThreads = 1024;

struct ExposureSolveArgs {
  const uint32_t* C;      // [n][n]
  const long long* r;     // [n]
  int n, gauge;
  int* row_start;         // [n + 1]
  int* reached;           // [n]
  int* iterations;        // [1]
  int* cols;              // [n * n]
  double* work;           // [6 n]: x, res, z, p, q, deg
  double* x_log;          // [n] out: x / 2^16 (NaN outside the component)
  int* xq;                // [n] out: rint(x) (0 outside the component)
  uint32_t* diag;         // [n] out: C's diagonal
  int max_iterations;
  double tol;             // on |res| / |r|
};

__device__ double BlockSum(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < kSolveThreads / 32 ? red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[32] = v;
  }
  __syncthreads();
  const double out = red[32];
  __syncthreads();
  return out;
}

__global__ void __launch_bounds__(kSolveThreads) ExposureSolveKernel(const __grid_constant__ ExposureSolveArgs a) {
  __shared__ double red[33];
  const int n = a.n, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const size_t N = static_cast<size_t>(n);
  // CSR of the off-diagonal non-zeros: counts, a serial scan (n <= max_keyframes), the columns in order
  for (int i = warp; i < n; i += kSolveThreads / 32) {
    int cnt = 0;
    for (int b = 0; b < n; b += 32) {
      const int j = b + lane;
      cnt += __popc(__ballot_sync(0xffffffffu, j < n && j != i && a.C[i * N + j] != 0u));
    }
    if (lane == 0) {
      a.row_start[i + 1] = cnt;
      a.diag[i] = a.C[i * N + i];
    }
  }
  __syncthreads();
  if (t == 0) {
    a.row_start[0] = 0;
    for (int i = 0; i < n; ++i) a.row_start[i + 1] += a.row_start[i];
  }
  __syncthreads();
  for (int i = warp; i < n; i += kSolveThreads / 32) {
    int pos = a.row_start[i];
    for (int b = 0; b < n; b += 32) {
      const int j = b + lane;
      const bool nz = j < n && j != i && a.C[i * N + j] != 0u;
      const unsigned m = __ballot_sync(0xffffffffu, nz);
      if (nz) a.cols[pos + __popc(m & ((1u << lane) - 1u))] = j;
      pos += __popc(m);
    }
  }
  for (int i = t; i < n; i += kSolveThreads) a.reached[i] = i == a.gauge;
  __syncthreads();
  // the gauge keyframe's component
  volatile int* reached = a.reached;
  for (;;) {
    int changed = 0;
    for (int i = t; i < n; i += kSolveThreads) {
      if (reached[i]) continue;
      for (int k = a.row_start[i]; k < a.row_start[i + 1]; ++k)
        if (reached[a.cols[k]]) {
          reached[i] = 1;
          changed = 1;
          break;
        }
    }
    if (!__syncthreads_or(changed)) break;
  }
  double* x = a.work;
  double* res = x + n;
  double* z = res + n;
  double* p = z + n;
  double* q = p + n;
  double* deg = q + n;
  // unknowns: reached and not the gauge; every vector is 0 elsewhere
  double rr0 = 0.0, rz = 0.0;
  for (int i = t; i < n; i += kSolveThreads) {
    const bool u = reached[i] && i != a.gauge;
    double d = 0.0;
    for (int k = a.row_start[i]; k < a.row_start[i + 1]; ++k) d += static_cast<double>(a.C[i * N + a.cols[k]]);
    deg[i] = d;
    x[i] = 0.0;
    res[i] = u ? static_cast<double>(a.r[i]) : 0.0;
    z[i] = u ? res[i] / d : 0.0;
    p[i] = z[i];
    rr0 += res[i] * res[i];
    rz += res[i] * z[i];
  }
  rr0 = BlockSum(rr0, red);
  rz = BlockSum(rz, red);
  int it = 0;
  if (rr0 > 0.0) {
    const double stop = a.tol * a.tol * rr0;
    for (; it < a.max_iterations;) {
      double pq = 0.0;
      for (int i = t; i < n; i += kSolveThreads) {
        double v = 0.0;
        if (reached[i] && i != a.gauge) {
          v = deg[i] * p[i];
          for (int k = a.row_start[i]; k < a.row_start[i + 1]; ++k) {
            const int j = a.cols[k];
            v -= static_cast<double>(a.C[i * N + j]) * p[j];
          }
        }
        q[i] = v;
        pq += p[i] * v;
      }
      pq = BlockSum(pq, red);
      const double alpha = rz / pq;
      double rr = 0.0;
      for (int i = t; i < n; i += kSolveThreads) {
        x[i] += alpha * p[i];
        res[i] -= alpha * q[i];
        rr += res[i] * res[i];
      }
      rr = BlockSum(rr, red);
      ++it;
      if (!(rr > stop)) break;
      double rz_new = 0.0;
      for (int i = t; i < n; i += kSolveThreads) {
        z[i] = reached[i] && i != a.gauge ? res[i] / deg[i] : 0.0;
        rz_new += res[i] * z[i];
      }
      rz_new = BlockSum(rz_new, red);
      const double beta = rz_new / rz;
      rz = rz_new;
      for (int i = t; i < n; i += kSolveThreads) p[i] = z[i] + beta * p[i];
      __syncthreads();
    }
  }
  for (int i = t; i < n; i += kSolveThreads) {
    const bool in = reached[i];
    a.x_log[i] = in ? x[i] * (1.0 / 65536.0) : __longlong_as_double(0x7ff8000000000000ll);
    a.xq[i] = in ? static_cast<int>(fmin(fmax(rint(x[i]), -2147483647.0), 2147483647.0)) : 0;
  }
  if (t == 0) *a.iterations = it;
}

LaunchResult LaunchExposureSolve(const ExposureSolveArgs& a, cudaStream_t stream) {
  if (a.n <= 0) return {};
  ExposureSolveKernel<<<1, kSolveThreads, 0, stream>>>(a);
  return {1};
}

// round(2^16 ln v), v = 1 .. 255 (entry 0 is never read: min_luma >= 1)
const int* LogQ16Table() {
  static const std::vector<int> table = [] {
    std::vector<int> t(256, 0);
    for (int v = 1; v < 256; ++v) t[v] = static_cast<int>(std::nearbyint(65536.0 * std::log(static_cast<double>(v))));
    return t;
  }();
  return table.data();
}

// The listed ids: known, no repeats.
bool CheckIds(bba_handle h, int count, const int* ids, const std::string& fn, bba_status* st) {
  const int K = static_cast<int>(h->keyframes.size());
  std::vector<char> seen(K, 0);
  for (int i = 0; i < count; ++i) {
    if (ids[i] < 0 || ids[i] >= K) {
      *st = Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "unknown keyframe id");
      return false;
    }
    if (seen[ids[i]]++) {
      *st = Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "repeated keyframe id");
      return false;
    }
  }
  return true;
}

constexpr int kMaxExposureRounds = 16;

bba_status EstimateKeyframeExposures(bba_handle h, const bba_exposure_options* o, int count, const int* ids, float* gains,
                                     uint32_t* observations, uint32_t* inliers, cudaStream_t s) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_estimate_keyframe_exposures: ";
  if (!o) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null options");
  if (count <= 0 || !ids || !gains) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "no keyframes listed, or a null array");
  bba_status st = BBA_OK;
  if (!CheckIds(h, count, ids, fn, &st)) return st;
  const int gauge_id = o->gauge_keyframe < 0 ? ids[0] : o->gauge_keyframe;
  const int gauge = static_cast<int>(std::find(ids, ids + count, gauge_id) - ids);
  if (gauge == count) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "the gauge keyframe is not listed");
  const int min_luma = o->min_luma == 0 ? 8 : o->min_luma, max_luma = o->max_luma == 0 ? 247 : o->max_luma;
  if (min_luma < 1 || max_luma > 255 || min_luma > max_luma) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad luma range");
  if (!std::isfinite(o->inlier_threshold)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "inlier_threshold is not finite");
  const double threshold = o->inlier_threshold <= 0.f ? 0.1 : static_cast<double>(o->inlier_threshold);
  if (threshold > 16.0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "inlier_threshold above 16");
  const int rounds = o->outer_iterations <= 0 ? 2 : o->outer_iterations;
  if (rounds > kMaxExposureRounds) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "more than 16 outer_iterations");
  for (int i = 0; i < count; ++i)
    if (h->keyframes[ids[i]].color_staged)
      return Fail(h, BBA_ERR_STATE, fn + "a listed keyframe's colour was updated through the staging image; its colour image is gone");
  const uint32_t n = h->surfels_size;
  if (n > 0)
    if (bba_status st2 = CheckSurfels(h)) return st2;
  auto& e = h->exposure;
  const size_t N = static_cast<size_t>(count);
  ReplicaWalk walk;   // (the co-visibility chunk rule over the listed rows)
  if (bba_status st2 = ReserveReplicaWalk(h, N, &walk)) return st2;
  const uint32_t chunk = walk.chunk;
  BBA_CUDA(h, e.d_ids.Reserve(N));
  BBA_CUDA(h, e.d_images.Reserve(N));
  BBA_CUDA(h, e.d_n.Reserve(chunk));
  BBA_CUDA(h, e.d_sum.Reserve(chunk));
  for (int b = 0; b < 2 && b < rounds - 1; ++b) {
    BBA_CUDA(h, e.d_test_n[b].Reserve(chunk));
    BBA_CUDA(h, e.d_test_sum[b].Reserve(chunk));
  }
  BBA_CUDA(h, e.d_C.Reserve(N * N));
  BBA_CUDA(h, e.d_r.Reserve(N));
  BBA_CUDA(h, e.d_xq.Reserve(N * rounds));
  BBA_CUDA(h, e.d_csr.Reserve(2 * N + 2 + N * N));
  BBA_CUDA(h, e.d_work.Reserve(7 * N));
  BBA_CUDA(h, e.d_diag.Reserve(2 * N));
  if (bba_status st2 = UploadKeyframes(h, s)) return st2;   // the current poses
  std::vector<ExposureImage> images(count);
  for (int i = 0; i < count; ++i) {
    const Keyframe& kf = h->keyframes[ids[i]];
    images[i] = ExposureImage{kf.rgba, static_cast<uint32_t>(kf.rgba_pitch), 0u};
  }
  BBA_CUDA(h, cudaMemcpyAsync(e.d_ids, ids, sizeof(int) * N, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemcpyAsync(e.d_images, images.data(), sizeof(ExposureImage) * N, cudaMemcpyHostToDevice, s));
  ExposureWalkArgs w{};
  w.images = e.d_images;
  std::copy(LogQ16Table(), LogQ16Table() + 256, w.log_q16);
  w.min_luma = min_luma;
  w.max_luma = max_luma;
  w.tau = std::llround(65536.0 * threshold);
  const auto xq = [&](int round) { return e.d_xq.get() + static_cast<size_t>(round - 1) * N; };   // round >= 1
  int* csr = e.d_csr;
  ExposureSolveArgs sa{e.d_C, e.d_r, count, gauge, csr, csr + N + 1, csr + 2 * N + 1, csr + 2 * N + 2, e.d_work,
                       e.d_work.get() + 6 * N, nullptr, e.d_diag.get() + N, 4 * count + 100, 1e-14};
  for (int k = 1; k <= rounds; ++k) {
    BBA_CUDA(h, cudaMemsetAsync(e.d_C, 0, sizeof(uint32_t) * N * N, s));
    BBA_CUDA(h, cudaMemsetAsync(e.d_r, 0, sizeof(long long) * N, s));
    // (the walk zeroes the bit rows at the start of a chunk; only the members' walk writes them)
    if (bba_status st2 = WalkReplica(h, walk, h->d_kfs, e.d_ids, count, s, [&](const GeometryArgs& g, uint32_t words) {
          const uint32_t len = g.end - g.begin;
          w.geo = g;
          w.words = words;
          // the test sums of rounds 2 .. k: stats_j = the members of round j - 1 with y - x_{j-1}, in d_test[j % 2]
          for (int j = 2; j <= k; ++j) {
            ExposureWalkArgs a = w;
            if (j >= 3) {
              a.test_n = e.d_test_n[(j - 1) % 2];
              a.test_sum = e.d_test_sum[(j - 1) % 2];
              a.test_x = xq(j - 2);
            }
            a.n = e.d_test_n[j % 2];
            a.sum = e.d_test_sum[j % 2];
            a.sub_x = xq(j - 1);
            BBA_CUDA(h, cudaMemsetAsync(a.n, 0, sizeof(uint32_t) * len, s));
            BBA_CUDA(h, cudaMemsetAsync(a.sum, 0, sizeof(long long) * len, s));
            BBA_LAUNCH(h, h->launches, LaunchExposureWalk, a, h->sm_count, s);
          }
          // the members of round k: their n and sum of y with the bit rows, then r
          ExposureWalkArgs a = w;
          if (k >= 2) {
            a.test_n = e.d_test_n[k % 2];
            a.test_sum = e.d_test_sum[k % 2];
            a.test_x = xq(k - 1);
          }
          a.n = e.d_n;
          a.sum = e.d_sum;
          a.bits = h->covis.d_bits;
          BBA_CUDA(h, cudaMemsetAsync(a.n, 0, sizeof(uint32_t) * len, s));
          BBA_CUDA(h, cudaMemsetAsync(a.sum, 0, sizeof(long long) * len, s));
          BBA_LAUNCH(h, h->launches, LaunchExposureWalk, a, h->sm_count, s);
          a.bits = nullptr;
          a.rhs = e.d_r;
          BBA_LAUNCH(h, h->launches, LaunchExposureWalk, a, h->sm_count, s);
          const CovisibilityGramArgs q{h->covis.d_bits, words, h->geo.d_all_list, count, count, e.d_C};
          BBA_LAUNCH(h, h->launches, LaunchCovisibilityGram, q, h->sm_count, s);
          return BBA_OK;
        }))
      return st2;
    sa.xq = xq(k);
    BBA_LAUNCH(h, h->launches, LaunchExposureSolve, sa, s);
    if (k == 1) BBA_CUDA(h, cudaMemcpyAsync(e.d_diag, e.d_diag.get() + N, sizeof(uint32_t) * N, cudaMemcpyDeviceToDevice, s));
  }
  std::vector<double> x(count);
  std::vector<uint32_t> diag(2 * N);
  BBA_CUDA(h, cudaMemcpyAsync(x.data(), sa.x_log, sizeof(double) * N, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaMemcpyAsync(diag.data(), e.d_diag, sizeof(uint32_t) * 2 * N, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  e.count = count;
  for (int i = 0; i < count; ++i) {
    const bool in = !std::isnan(x[i]);
    gains[i] = in ? static_cast<float>(std::exp(x[i])) : std::numeric_limits<float>::quiet_NaN();
    if (observations) observations[i] = diag[i];
    if (inliers) inliers[i] = in ? diag[N + i] : 0u;
  }
  return BBA_OK;
}

// Re-extracts the luma of keyframes ids[0 .. count) with the gains, in batches of MakeLumaTextures.
constexpr int kGainBatch = 16;

bba_status SetKeyframeExposures(bba_handle h, int count, const int* ids, const float* gains, cudaStream_t s) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_set_keyframe_exposures: ";
  if (count < 0 || (count > 0 && (!ids || !gains))) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad count or a null array");
  bba_status st = BBA_OK;
  if (!CheckIds(h, count, ids, fn, &st)) return st;
  for (int i = 0; i < count; ++i)
    if (!std::isfinite(gains[i]) || !(gains[i] > 0.f)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "a gain is not finite and positive");
  for (int i = 0; i < count; ++i)
    if (h->keyframes[ids[i]].color_staged)
      return Fail(h, BBA_ERR_STATE, fn + "a keyframe's colour was updated through the staging image; its colour image is gone");
  for (int b = 0; b < count; b += kGainBatch) {
    const int m = std::min(kGainBatch, count - b);
    LumaSource sources[kGainBatch];
    Texture* out[kGainBatch];
    for (int i = 0; i < m; ++i) {
      Keyframe& kf = h->keyframes[ids[b + i]];
      sources[i] = LumaSource{kf.rgba, kf.rgba_pitch, gains[b + i]};
      out[i] = &kf.luma;
    }
    if (bba_status st2 = MakeLumaTextures(h, /*front_end=*/false, m, sources, out, s)) return st2;
    for (int i = 0; i < m; ++i) h->keyframes[ids[b + i]].gain = gains[b + i];
  }
  return Publish(h, s, false);
}

}  // namespace
}  // namespace bba

using namespace bba;

extern "C" {

bba_status bba_estimate_keyframe_exposures(bba_handle h, const bba_exposure_options* options, int count, const int* keyframe_ids,
                                           float* gains, uint32_t* observations, uint32_t* inliers, void* stream) {
  return EstimateKeyframeExposures(h, options, count, keyframe_ids, gains, observations, inliers, static_cast<cudaStream_t>(stream));
}

bba_status bba_set_keyframe_exposures(bba_handle h, int count, const int* keyframe_ids, const float* gains, void* stream) {
  return SetKeyframeExposures(h, count, keyframe_ids, gains, static_cast<cudaStream_t>(stream));
}

bba_status bba_get_keyframe_exposures(bba_handle h, int count, const int* keyframe_ids, float* gains) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (count < 0 || (count > 0 && (!keyframe_ids || !gains))) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_get_keyframe_exposures: bad count or a null array");
  std::unique_lock<std::mutex> lock(h->fe.mu);
  const int K = static_cast<int>(h->fe.kfs.size());
  for (int i = 0; i < count; ++i)
    if (keyframe_ids[i] < 0 || keyframe_ids[i] >= K) {
      lock.unlock();
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_get_keyframe_exposures: unknown keyframe id");
    }
  for (int i = 0; i < count; ++i) gains[i] = h->fe.kfs[keyframe_ids[i]].gain;
  return BBA_OK;
}

bba_status bba_debug_get_exposure_system(bba_handle h, int count, uint32_t* C, int64_t* r) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (count <= 0 || count != h->exposure.count || !C || !r)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_get_exposure_system: count is not the last estimate's");
  BBA_CUDA(h, cudaMemcpy(C, h->exposure.d_C, sizeof(uint32_t) * count * count, cudaMemcpyDeviceToHost));
  BBA_CUDA(h, cudaMemcpy(r, h->exposure.d_r, sizeof(int64_t) * count, cudaMemcpyDeviceToHost));
  return BBA_OK;
}

}  // extern "C"
