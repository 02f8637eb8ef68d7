// launch.hpp -- what every host-callable Launch* returns: the kernels it enqueued (memsets and copies are not kernels) and the
// first error of its runtime and library calls.  Errors of <<<>>> launches reach the caller through cudaGetLastError (BBA_LAUNCH).
#pragma once

#include <cuda_runtime.h>

namespace bba {

struct LaunchResult {
  int kernels = 0;                   // 0 when the launcher returned before its first launch
  cudaError_t error = cudaSuccess;   // the first error is kept

  LaunchResult& operator+=(cudaError_t e) {
    if (error == cudaSuccess) error = e;
    return *this;
  }
  LaunchResult& operator+=(const LaunchResult& r) {
    kernels += r.kernels;
    return *this += r.error;
  }
};

}  // namespace bba
