#!/usr/bin/env bash
# Compiles the reference's OWN, UNMODIFIED BA CUDA kernels from a checkout of the
# reference ($BADSLAM_REFERENCE) into oracle/_ref/ (git-ignored),
# then links them with oracle/ref_driver.cu (our Eigen-free restatement of the
# thin host wrappers kernel_opt_*.cc) into oracle/_ref/libbadslam_ref.so.
# Test / baseline infrastructure only -- never loaded by the product path.
#
# Flags follow applications/badslam/CMakeLists.txt:74-75 (-use_fast_math
# --expt-relaxed-constexpr, C++14); arch = sm_90a (H100).
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
REF="${BADSLAM_REFERENCE:?set BADSLAM_REFERENCE to a checkout of the reference}"
OUT="$HERE/_ref"
mkdir -p "$OUT/obj"
if [ ! -d "$REF/applications/badslam/src/badslam" ]; then
  echo "build_ref: reference not present at $REF; keeping prebuilt $OUT" >&2
  exit 0
fi
B="$REF/applications/badslam/src/badslam"
NVCC="${NVCC:-nvcc}"
FLAGS=(-std=c++14 -O3 -gencode arch=compute_90a,code=sm_90a -use_fast_math --expt-relaxed-constexpr
       -Xcompiler -fPIC -w
       -I "$HERE/ref_shim" -I "$REF/applications/badslam/src" -I "$REF/libvis/src"
       -I "$REF/libvis/third_party/loguru")
SRCS=("$B/kernel_opt_pose.cu" "$B/kernel_opt_geometry.cu" "$B/kernel_surfel_activation.cu"
      "$B/kernel_opt_intrinsics.cu" "$B/kernel_pcg.cu"
      "$B/kernel_delete_surfels.cu" "$B/kernel_supporting_surfels.cu"
      "$B/kernel_compact_surfels.cu" "$B/kernel_create_surfels.cu"
      "$B/cuda_depth_processing.cu" "$B/cuda_image_processing.cu" "$B/kernel_downsample.cu"
      "$REF/libvis/src/libvis/cuda/cuda_buffer.cu")
pids=()
for s in "${SRCS[@]}"; do
  o="$OUT/obj/$(basename "${s%.cu}").o"
  if [ ! -f "$o" ] || [ "$s" -nt "$o" ]; then
    extra=()
    # AccumulateIntrinsicsCoefficientsCUDAKernel is launched with 1024-thread blocks (CUDA_AUTO_TUNE_1D_TEMPLATED default,
    # kernel_opt_intrinsics.cu:239-242) but compiles to > 64 registers: "too many resources requested for
    # launch".  Same for PCGInitCUDAKernel (1024 threads, kernel_pcg.cu:538-541).  Cap the registers for these translation
    # units only (a build flag, the sources stay untouched).
    [[ "$s" == *kernel_opt_intrinsics.cu || "$s" == *kernel_pcg.cu ]] && extra=(-maxrregcount=64)
    ( "$NVCC" "${FLAGS[@]}" "${extra[@]}" -c "$s" -o "$o" && echo "built $o" ) &
    pids+=($!)
  fi
done
# loguru (LOG/CHECK macros used by the launch wrappers)
if [ ! -f "$OUT/obj/loguru.o" ]; then
  ( g++ -std=c++14 -O2 -fPIC -w -DLOGURU_REPLACE_GLOG=1 -DLOGURU_WITH_STREAMS=1 \
      -I "$REF/libvis/third_party/loguru" -c "$REF/libvis/third_party/loguru/loguru.cpp" \
      -o "$OUT/obj/loguru.o" && echo "built loguru.o" ) &
  pids+=($!)
fi
rc=0
for p in "${pids[@]:-}"; do [ -n "$p" ] && { wait "$p" || rc=1; }; done
[ $rc -eq 0 ] || { echo "build_ref: object compile failed" >&2; exit 1; }
if [ -f "$HERE/ref_driver.cu" ]; then
  "$NVCC" "${FLAGS[@]}" -shared -o "$OUT/libbadslam_ref.so" "$HERE/ref_driver.cu" \
      "$OUT"/obj/*.o -lcudart -ldl -lpthread
  echo "built $OUT/libbadslam_ref.so"
fi
