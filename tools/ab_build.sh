#!/usr/bin/env bash
# Builds a variant of libbadba_b200.so with extra nvcc flags for kernels.cu into tools/ab/<name>.so (A/B experiments).
#   tools/ab_build.sh ctas3 -DBBA_POSE_MIN_CTAS=3
set -euo pipefail
cd "$(dirname "${BASH_SOURCE[0]}")/.."
name="$1"; shift
mkdir -p tools/ab
C=badslam_b200/csrc
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr -use_fast_math "$@" \
     -c $C/kernels.cu -o tools/ab/$name.kernels.o
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o tools/ab/$name.so tools/ab/$name.kernels.o \
     badslam_b200/_obj/intrinsics.cu.o badslam_b200/_obj/pcg.cu.o badslam_b200/_obj/lifecycle.cu.o badslam_b200/_obj/preprocess.cu.o badslam_b200/_obj/odometry.cu.o badslam_b200/_obj/pose_solve.cu.o badslam_b200/_obj/badba.cu.o -cudart static
echo tools/ab/$name.so
