"""CPU-only: the local-group entry points of include/badba.h from C99, and badba::LocalGroup of include/badba_direct_ba.hpp
instantiated by a C++ program; both link against the library and exercise what needs no device (NULL arguments are refused)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "badslam_b200")


def test_local_group_declarations_compile_as_c99(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "group.c"
    src.write_text(r'''
#include "badba.h"
int main(void) {
  bba_local_group g = 0;
  bba_handle ranks[2] = {0, 0};
  if (bba_local_group_create(0, 2, 0, &g) != BBA_ERR_INVALID_ARGUMENT) return 1;
  if (bba_local_group_create(ranks, 2, 0, &g) != BBA_ERR_INVALID_ARGUMENT || g != 0) return 2;
  if (bba_local_group_create(ranks, 0, 1, &g) != BBA_ERR_INVALID_ARGUMENT) return 3;
  if (bba_local_group_reset(0) != BBA_ERR_INVALID_ARGUMENT || bba_local_group_poison(0) != BBA_ERR_INVALID_ARGUMENT) return 4;
  if (bba_debug_collective(0, BBA_COLLECTIVE_ALLREDUCE_SUM, 0, 0, 0) != BBA_ERR_INVALID_ARGUMENT) return 5;
  bba_local_group_destroy(0);
  return 0;
}''')
    exe = tmp_path / "group"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                           "-o", str(exe), "-L", LIBDIR, "-lbadba_b200", f"-Wl,-rpath,{LIBDIR}"])
    assert subprocess.call([str(exe)]) == 0


def test_cpp_local_group_compiles_and_fails_loudly_without_device(tmp_path):
    import torch
    gxx = shutil.which("g++")
    if gxx is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("no host compiler / CUDA headers")
    src = tmp_path / "group.cpp"
    src.write_text(r'''
#include "badba_direct_ba.hpp"
struct SE3 { float d[7]; float* data() { return d; } const float* data() const { return d; } };
struct Cam { int w, h; float p[4]; int width() const { return w; } int height() const { return h; } const float* parameters() const { return p; } };
using DA = badba::DirectBA<SE3, Cam>;
int main() {
  Cam c{64, 48, {30, 30, 32, 24}};
  try {
    std::vector<std::unique_ptr<DA>> members;
    for (int r = 0; r < 2; ++r)
      members.emplace_back(new DA(1000, 1e-3f, 40.f, 4, 0.8f, 1, 2, 3, c, c, 0, true, true, 16, 0, r, 2));
    badba::LocalGroup<DA> group(std::move(members), {0, 0});
    int ran = 0;
    group.RunOnRanks([&](int rank, DA& ba) { if (ba.handle() && rank >= 0) __atomic_add_fetch(&ran, 1, __ATOMIC_RELAXED); });
    if (ran != 2) return 2;
    bool thrown = false;
    try {
      group.RunOnRanks([](int rank, DA&) { if (rank == 1) throw std::runtime_error("rank 1 gives up"); });
    } catch (const std::runtime_error&) { thrown = true; }
    group.Reset();
    return thrown ? 0 : 3;
  }
  catch (const badba::Error& e) { return e.status == BBA_ERR_NO_DEVICE ? 42 : 1; }
}''')
    exe = tmp_path / "group"
    subprocess.check_call([gxx, "-std=c++17", "-pthread", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src),
                           "-o", str(exe), "-L", LIBDIR, "-lbadba_b200", f"-Wl,-rpath,{LIBDIR}", "-L", "/usr/local/cuda/lib64", "-lcudart",
                           "-Wl,-rpath,/usr/local/cuda/lib64"])   # (RunOnRanks sets each thread's device: the caller links cudart)
    assert subprocess.call([str(exe)], timeout=300) == (0 if torch.cuda.is_available() else 42)
