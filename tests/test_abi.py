"""The C-ABI library loads without a GPU and exports every symbol include/badba.h declares."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "badba.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = set(re.findall(r"\b(bba_[a-z_0-9]+)\s*\(", src))
    names -= {"bba_collective_fn", "bba_collective_op"}
    return sorted(names)


def test_header_declares_the_hot_path():
    names = declared_symbols()
    for required in ("bba_create", "bba_destroy", "bba_add_keyframe", "bba_set_surfels", "bba_accumulate_pose_coeffs",
                     "bba_estimate_frame_pose", "bba_update_surfel_activation", "bba_optimize_geometry_iteration",
                     "bba_optimize_intrinsics", "bba_bundle_adjust"):
        assert required in names


def declared_abi_version():
    src = open(os.path.join(ROOT, "include", "badba.h")).read()
    return int(re.search(r"^#define BBA_ABI_VERSION (\d+)$", src, flags=re.M).group(1))


def test_library_exports_every_declared_symbol_at_abi_version_10():
    from badslam_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "build libbadba_b200.so first (python -m badslam_b200.build)"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared_symbols():
        assert hasattr(lib, name), f"{name} declared in include/badba.h but not exported"
    # and the python binding types every one of them
    assert set(declared_symbols()) == set(_lib.SYMBOLS.keys())
    # library, header and binding are one version: v10 made bba_pcg_debug stop at any inner step (bba_pcg_probe)
    assert _lib.load().bba_abi_version() == declared_abi_version() == _lib.ABI_VERSION == 10


def test_no_cpu_fallback_without_a_device():
    """Without a GPU the product path must fail loudly, not fall back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from badslam_b200 import _lib
    lib = _lib.load()
    cfg = _lib.Config()
    cfg.depth_width = cfg.color_width = 64
    cfg.depth_height = cfg.color_height = 48
    cfg.depth_intrinsics[:] = [30, 30, 32, 24]
    cfg.color_intrinsics[:] = [30, 30, 32, 24]
    cfg.raw_to_float_depth, cfg.baseline_fx, cfg.sparse_surfel_cell_size = 1e-3, 40, 4
    cfg.max_surfel_count, cfg.max_keyframes = 1024, 4
    cfg.use_depth_residuals = cfg.use_descriptor_residuals = 1
    cfg.world_size = 1
    h = ctypes.c_void_p()
    assert lib.bba_create(ctypes.byref(cfg), ctypes.byref(h)) == _lib.ERR_NO_DEVICE
    from badslam_b200.direct_ba import DirectBA, PinholeCamera4f
    cam = PinholeCamera4f(64, 48, [30, 30, 32, 24])
    with pytest.raises(_lib.BadBAError):
        DirectBA(1024, 1e-3, 40, 4, color_camera_initial_estimate=cam, depth_camera_initial_estimate=cam)


def test_product_does_not_import_the_oracle():
    """Nothing under badslam_b200/ may reference oracle/ (the oracle is test infrastructure)."""
    pkg = os.path.join(ROOT, "badslam_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h", ".cpp")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", txt, flags=re.M), f
                assert '#include "../../oracle' not in txt and "oracle/host_math" not in txt, f


def test_cpp_adaptor_header_compiles_and_fails_loudly_without_device(tmp_path):
    """include/badba_direct_ba.hpp (the reference-signature adaptor of INTEGRATION.md) compiles against the library."""
    import shutil
    import subprocess
    import torch
    gxx = shutil.which("g++")
    if gxx is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("no host compiler / CUDA headers")
    src = tmp_path / "adaptor.cpp"
    src.write_text(r'''
#include "badba_direct_ba.hpp"
struct SE3 { float d[7]; float* data() { return d; } const float* data() const { return d; } };
struct Cam { int w, h; float p[4]; int width() const { return w; } int height() const { return h; } const float* parameters() const { return p; } };
int main(int argc, char**) {
  Cam c{64, 48, {30, 30, 32, 24}};
  try {
    badba::DirectBA<SE3, Cam> ba(1000, 1e-3f, 40.f, 4, 0.8f, 1, 2, 3, c, c, 0, true, true);
    if (argc > 100) {   // never taken: instantiates member templates that need real buffers to run
      float mn, mx;
      ba.PreprocessFrame(nullptr, 1.5f, 0.005f, 2.f, 3.f, {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, &mn, &mx);
      ba.CreateSurfelsForKeyframe(nullptr, true, 0);
      SE3 pose{};
      ba.EstimateFramePose(nullptr, pose, {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, &pose);
      badba::SaveCalibration(nullptr, ba.handle(), "/tmp/calib");
      badba::LoadCalibration(nullptr, ba.handle(), "/tmp/calib");
      { std::lock_guard<std::mutex> lock(ba.Mutex()); ba.SetA(ba.a() + ba.GetMinObservationCount()); }
      ba.Lock(); ba.IncreaseBAIterationCount(); ba.Unlock();
      int done; bool conv;
      ba.BundleAdjustment(nullptr, false, false, true, true, true, 1, 10, false, 0, 0, true, &done, &conv, 0, nullptr, 30, 2500,
                          [](int it) { return it < 3; });
    }
  }
  catch (const badba::Error& e) { return e.status == BBA_ERR_NO_DEVICE ? 42 : 1; }
  return 0;
}''')
    exe = tmp_path / "adaptor"
    libdir = os.path.join(ROOT, "badslam_b200")
    subprocess.check_call([gxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src), "-o", str(exe),
                           "-L", libdir, "-lbadba_b200", f"-Wl,-rpath,{libdir}"])
    rc = subprocess.call([str(exe)])
    assert rc == (0 if torch.cuda.is_available() else 42)


def test_header_is_plain_c_and_links_from_c(tmp_path):
    """include/badba.h is the FFI boundary: it must compile as C99 (cgo / JNI / ctypes-style bindings parse it as C) and a C
    program must link against the library and call a device-free entry point."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "binding.c"
    src.write_text(r'''
#include "badba.h"
#include <math.h>
int main(void) {
  bba_ba_options o;
  float tangent[6] = {0.1f, -0.2f, 0.3f, 0.0f, 0.0f, 0.0f}, pose[7], back[6];
  (void)o;
  if (bba_abi_version() != BBA_ABI_VERSION) return 1;
  bba_host_se3_exp(tangent, pose);            /* pure translation: q = (0, 0, 0, 1), t = tangent[0..2] */
  bba_host_se3_log(pose, back);
  if (fabsf(pose[3] - 1.0f) > 1e-6f || fabsf(pose[4] - 0.1f) > 1e-6f || fabsf(back[2] - 0.3f) > 1e-6f) return 2;
  return bba_create(0, 0) == BBA_ERR_INVALID_ARGUMENT ? 0 : 3;
}''')
    exe = tmp_path / "binding"
    libdir = os.path.join(ROOT, "badslam_b200")
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                           "-o", str(exe), "-L", libdir, "-lbadba_b200", "-lm", f"-Wl,-rpath,{libdir}"])
    assert subprocess.call([str(exe)]) == 0
