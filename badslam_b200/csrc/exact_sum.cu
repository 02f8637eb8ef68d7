// exact_sum.cu -- the device side of bba_debug_exact_sum: the exact sum's deposits from many CTAs in a scrambled order, and its
// rounding (exact_sum.cuh).
//
// This translation unit is compiled WITHOUT -use_fast_math.
#include "kernels.cuh"

namespace bba {

// Thread t of the grid deposits the values (t + k T) * stride mod n (T threads in all, stride odd and coprime to n: a permutation),
// so that neighbouring values land from different CTAs in no particular order.
__global__ void __launch_bounds__(256) ExactSumDepositKernel(const float* __restrict__ values, uint64_t n, uint64_t stride, ExactSum* sum) {
  const uint64_t threads = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += threads)
    ExactDeposit(sum, values[(i * stride) % n]);
}

__global__ void ExactSumFinalizeKernel(const ExactSum* sum, double* out) { *out = ExactFinalize(*sum); }

LaunchResult LaunchExactSumDebug(const float* values, uint64_t n, ExactSum* sum, double* out, int sm_count, cudaStream_t stream) {
  uint64_t stride = 1;
  if (n > 1) {
    auto gcd = [](uint64_t x, uint64_t y) {
      while (y) {
        const uint64_t t = x % y;
        x = y;
        y = t;
      }
      return x;
    };
    stride = 2654435761ull % n;   // (i * stride stays below 2^64 for n < 2^32)
    while (gcd(stride, n) != 1) ++stride;
  }
  LaunchResult r;
  if (n) {
    ExactSumDepositKernel<<<4 * sm_count, 256, 0, stream>>>(values, n, stride, sum);
    r.kernels = 1;
  }
  ExactSumFinalizeKernel<<<1, 1, 0, stream>>>(sum, out);
  ++r.kernels;
  return r;
}

}  // namespace bba
