"""CPU-only: the soft pose prior's terms (bba_host_pose_prior_terms) against an independent numpy derivation, and the prior entry
points of include/badba.h from C99."""
import ctypes as C
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "badslam_b200")


def lib():
    from badslam_b200 import _lib
    return _lib.load()


def hat(w):
    return np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])


def so3_left_jacobian(phi):
    th = np.linalg.norm(phi)
    W = hat(phi)
    if th < 1e-8:
        return np.eye(3) + 0.5 * W
    return np.eye(3) + (1 - np.cos(th)) / th ** 2 * W + (th - np.sin(th)) / th ** 3 * W @ W


def to_rt(pose):
    q = np.asarray(pose[:4], np.float64)
    return Rotation.from_quat(q / np.linalg.norm(q)).as_matrix(), np.asarray(pose[4:], np.float64)


def log_rt(R, t):   # Sophus tangent order (translation, rotation), angle in [0, pi]
    phi = Rotation.from_matrix(R).as_rotvec()
    return np.concatenate([np.linalg.solve(so3_left_jacobian(phi), t), phi])


def exp_rt(xi):
    return Rotation.from_rotvec(xi[3:]).as_matrix(), so3_left_jacobian(xi[3:]) @ xi[:3]


def residual(P, T, delta=np.zeros(6)):   # log(P^-1 T exp(delta))
    Rp, tp = P
    Rt, tt = T
    Rd, td = exp_rt(delta)
    R, t = Rt @ Rd, tt + Rt @ td
    return log_rt(Rp.T @ R, Rp.T @ (t - tp))


def jacobian_fd(P, T, h=1e-6):
    J = np.zeros((6, 6))
    for i in range(6):
        e = np.zeros(6)
        e[i] = h
        J[:, i] = (residual(P, T, e) - residual(P, T, -e)) / (2 * h)
    return J


def upper(M):
    return np.array([M[i, j] for i in range(6) for j in range(i, 6)])


def host_terms(prior, pose, info):
    H, b, cost = np.zeros(21), np.zeros(6), C.c_double()
    p = np.ascontiguousarray(prior, np.float32)
    q = np.ascontiguousarray(pose, np.float32)
    L = np.ascontiguousarray(info, np.float32)
    lib().bba_host_pose_prior_terms(p.ctypes.data, q.ctypes.data, L.ctypes.data, H.ctypes.data, b.ctypes.data, C.byref(cost))
    return H, b, cost.value


def random_pose(rng, angle=None):
    rv = rng.normal(size=3)
    rv /= np.linalg.norm(rv)
    rv *= rng.uniform(0, np.pi) if angle is None else angle
    q = Rotation.from_rotvec(rv).as_quat()
    return np.concatenate([q, rng.normal(size=3)]).astype(np.float32)


def compose_tangent(pose, xi):   # pose * exp(xi) as float[7]
    R, t = to_rt(pose)
    Rd, td = exp_rt(np.asarray(xi, np.float64))
    return np.concatenate([Rotation.from_matrix(R @ Rd).as_quat(), t + R @ td]).astype(np.float32)


def random_info(rng):
    A = rng.normal(size=(6, 6))
    return A @ A.T + np.diag(rng.uniform(0.1, 10, 6))


def cases():
    rng = np.random.default_rng(7)
    out = []
    for i in range(12):   # general relative poses
        P = random_pose(rng)
        out.append((f"general{i}", P, random_pose(rng)))
    for ang in (1e-4, 0.03, 0.049, 0.051, 0.3):   # small rotations, both sides of the series switch
        P = random_pose(rng)
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        out.append((f"small{ang}", P, compose_tangent(P, np.concatenate([rng.normal(size=3) * 0.1, axis * ang]))))
    for d in (1e-2, 3e-3):   # rotations near pi
        P = random_pose(rng)
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        out.append((f"near_pi{d}", P, compose_tangent(P, np.concatenate([rng.normal(size=3), axis * (np.pi - d)]))))
    P = random_pose(rng)
    out.append(("zero", P, P.copy()))
    return out


@pytest.mark.parametrize("name,prior,pose", cases(), ids=[c[0] for c in cases()])
def test_terms_against_finite_differences(name, prior, pose):
    P, T = to_rt(prior), to_rt(pose)
    r = residual(P, T)
    J = jacobian_fd(P, T)
    if name == "zero":
        np.testing.assert_allclose(J, np.eye(6), atol=1e-8)
    # L = I: H = J^T J, b = J^T r, cost = |r|^2 / 2
    H, b, cost = host_terms(prior, pose, upper(np.eye(6)))
    scale = max(1.0, np.abs(J).max()) ** 2
    np.testing.assert_allclose(H, upper(J.T @ J), atol=2e-6 * scale, rtol=1e-6)
    np.testing.assert_allclose(b, J.T @ r, atol=2e-6 * scale * max(1.0, np.abs(r).max()), rtol=1e-6)
    np.testing.assert_allclose(cost, 0.5 * r @ r, rtol=1e-9, atol=1e-14)
    # a general information matrix (rounded to fp32 as the ABI takes it)
    L = random_info(np.random.default_rng(zlib.crc32(name.encode()))).astype(np.float32).astype(np.float64)
    L = np.triu(L) + np.triu(L, 1).T
    H, b, cost = host_terms(prior, pose, upper(L))
    np.testing.assert_allclose(H, upper(J.T @ L @ J), atol=2e-6 * scale * np.abs(L).max(), rtol=1e-6)
    np.testing.assert_allclose(b, J.T @ L @ r, atol=2e-6 * scale * np.abs(L).max() * max(1.0, np.abs(r).max()), rtol=1e-6)
    np.testing.assert_allclose(cost, 0.5 * r @ L @ r, rtol=1e-9, atol=1e-12)


def test_one_step_on_the_terms_alone_reaches_the_prior():
    """The solve's update T <- T exp(-x), H x = b, with the prior's terms alone lands on the prior (Jr(r) r = r)."""
    rng = np.random.default_rng(3)
    for _ in range(20):
        prior = random_pose(rng)
        pose = random_pose(rng)
        H, b, _ = host_terms(prior, pose, upper(np.eye(6)))
        Hm = np.zeros((6, 6))
        Hm[np.triu_indices(6)] = H
        Hm = Hm + np.triu(Hm, 1).T
        x = np.linalg.solve(Hm, b)
        stepped = compose_tangent(pose, -x)
        err = residual(to_rt(prior), to_rt(stepped))
        assert np.abs(err).max() < 1e-5


def test_prior_entry_points_compile_as_c99_and_refuse_bad_arguments(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "prior.c"
    src.write_text(r'''
#include "badba.h"
int main(void) {
  const float pose[7] = {0.f, 0.f, 0.f, 1.f, 1.f, 2.f, 3.f};
  float info[21] = {0};
  double H[21], b[6], cost = -1.0;
  int ids[1] = {0}, has = 7;
  info[0] = info[6] = info[11] = info[15] = info[18] = info[20] = 4.f;
  bba_host_pose_prior_terms(pose, pose, info, H, b, &cost);
  if (cost != 0.0 || H[0] != 4.0 || H[1] != 0.0 || b[0] != 0.0) return 1;
  if (bba_set_keyframe_pose_priors(0, 1, ids, pose, info) != BBA_ERR_INVALID_ARGUMENT) return 2;
  if (bba_clear_keyframe_pose_priors(0, -1, 0) != BBA_ERR_INVALID_ARGUMENT) return 3;
  if (bba_get_keyframe_pose_prior(0, 0, 0, 0, &has) != BBA_ERR_INVALID_ARGUMENT || has != 7) return 4;
  return 0;
}''')
    exe = tmp_path / "prior"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                           "-o", str(exe), "-L", LIBDIR, "-lbadba_b200", f"-Wl,-rpath,{LIBDIR}"])
    assert subprocess.call([str(exe)]) == 0
    exported = C.CDLL(os.path.join(LIBDIR, "libbadba_b200.so"))
    for name in ("bba_set_keyframe_pose_priors", "bba_clear_keyframe_pose_priors", "bba_get_keyframe_pose_prior",
                 "bba_host_pose_prior_terms"):
        assert hasattr(exported, name)


def test_cpp_adaptor_prior_methods_compile(tmp_path):
    gxx = shutil.which("g++")
    if gxx is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("no host compiler / CUDA headers")
    src = tmp_path / "prior.cpp"
    src.write_text(r'''
#include "badba_direct_ba.hpp"
struct SE3 { float d[7]; float* data() { return d; } const float* data() const { return d; } };
struct Cam { int w, h; float p[4]; int width() const { return w; } int height() const { return h; } const float* parameters() const { return p; } };
int main(int argc, char**) {
  Cam c{64, 48, {30, 30, 32, 24}};
  try {
    badba::DirectBA<SE3, Cam> ba(1000, 1e-3f, 40.f, 4, 0.8f, 1, 2, 3, c, c, 0, true, true);
    if (argc > 100) {   // never taken: instantiates the members
      const SE3 prior{{0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f}};
      const float info[21] = {1.f};
      ba.SetKeyframePosePrior(0, prior, info);
      ba.ClearKeyframePosePriors({0});
      ba.ClearKeyframePosePriors();
    }
  }
  catch (const badba::Error& e) { return e.status == BBA_ERR_NO_DEVICE ? 42 : 1; }
  return 0;
}''')
    exe = tmp_path / "prior"
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include",
                           str(src), "-o", str(exe), "-L", LIBDIR, "-lbadba_b200", f"-Wl,-rpath,{LIBDIR}"])
    assert subprocess.call([str(exe)]) in (0, 42)
