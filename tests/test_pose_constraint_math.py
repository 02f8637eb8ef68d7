"""CPU-only: the soft relative pose constraint's terms (bba_host_pose_constraint_terms) against numpy central differences, the two
prior forms a constraint takes when one end is held fixed, and the constraint entry points of include/badba.h from C99 and C++."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import test_pose_prior_math as M

ROOT = M.ROOT
LIBDIR = M.LIBDIR


def constraint_terms(Z, A, B, info):
    H, b, cost = np.zeros(78), np.zeros(12), C.c_double()
    z, a, bb, L = (np.ascontiguousarray(x, np.float32) for x in (Z, A, B, info))
    M.lib().bba_host_pose_constraint_terms(z.ctypes.data, a.ctypes.data, bb.ctypes.data, L.ctypes.data, H.ctypes.data, b.ctypes.data,
                                           C.byref(cost))
    return H, b, cost.value


def residual(Z, A, B, da=np.zeros(6), db=np.zeros(6)):   # log(Z^-1 (A exp(da))^-1 B exp(db))
    Rz, tz = Z
    Ra, ta = A
    Rb, tb = B
    Rda, tda = M.exp_rt(da)
    Rdb, tdb = M.exp_rt(db)
    Ra2, ta2 = Ra @ Rda, ta + Ra @ tda
    Rb2, tb2 = Rb @ Rdb, tb + Rb @ tdb
    Re, te = Ra2.T @ Rb2, Ra2.T @ (tb2 - ta2)        # A^-1 B
    return M.log_rt(Rz.T @ Re, Rz.T @ (te - tz))     # Z^-1 A^-1 B


def jacobian_fd(Z, A, B, h=1e-6):
    J = np.zeros((6, 12))
    for i in range(12):
        e = np.zeros(12)
        e[i] = h
        J[:, i] = (residual(Z, A, B, e[:6], e[6:]) - residual(Z, A, B, -e[:6], -e[6:])) / (2 * h)
    return J


def upper12(Hm):
    return np.array([Hm[i, j] for i in range(12) for j in range(i, 12)])


def matrix(H, n):
    Hm = np.zeros((n, n))
    Hm[np.triu_indices(n)] = H
    return Hm + np.triu(Hm, 1).T


def as_pose(R, t):
    return np.concatenate([Rotation.from_matrix(R).as_quat(), t]).astype(np.float32)


def compose(P, Q):
    (Rp, tp), (Rq, tq) = M.to_rt(P), M.to_rt(Q)
    return as_pose(Rp @ Rq, tp + Rp @ tq)


def inverse(P):
    R, t = M.to_rt(P)
    return as_pose(R.T, -R.T @ t)


def adjoint(P):   # Ad(P) in the tangent order (translation, rotation)
    R, t = M.to_rt(P)
    Ad = np.zeros((6, 6))
    Ad[:3, :3] = Ad[3:, 3:] = R
    Ad[:3, 3:] = M.hat(t) @ R
    return Ad


def cases():
    rng = np.random.default_rng(17)
    out = []
    for i in range(8):
        out.append((f"general{i}", M.random_pose(rng), M.random_pose(rng), M.random_pose(rng)))
    for ang in (0.0, 1e-4, 0.03, 0.3):   # near r = 0: B close to A Z
        Z, A = M.random_pose(rng), M.random_pose(rng)
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        xi = np.concatenate([rng.normal(size=3) * 0.1 * (ang > 0), axis * ang])
        out.append((f"small{ang}", Z, A, M.compose_tangent(compose(A, Z), xi)))
    for d in (1e-2, 3e-3):   # rotations of r near pi
        Z, A = M.random_pose(rng), M.random_pose(rng)
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        out.append((f"near_pi{d}", Z, A, M.compose_tangent(compose(A, Z), np.concatenate([rng.normal(size=3), axis * (np.pi - d)]))))
    return out


@pytest.mark.parametrize("name,Z,A,B", cases(), ids=[c[0] for c in cases()])
def test_terms_against_finite_differences(name, Z, A, B):
    Zr, Ar, Br = M.to_rt(Z), M.to_rt(A), M.to_rt(B)
    r = residual(Zr, Ar, Br)
    J = jacobian_fd(Zr, Ar, Br)
    scale = max(1.0, np.abs(J).max()) ** 2
    for seed in (None, 1):
        if seed is None:
            L = np.eye(6)
        else:
            L = M.random_info(np.random.default_rng(len(name))).astype(np.float32).astype(np.float64)
            L = np.triu(L) + np.triu(L, 1).T
        H, b, cost = constraint_terms(Z, A, B, M.upper(L))
        lmax = np.abs(L).max()
        np.testing.assert_allclose(H, upper12(J.T @ L @ J), atol=3e-6 * scale * lmax, rtol=1e-6, err_msg=name)
        np.testing.assert_allclose(b, J.T @ L @ r, atol=3e-6 * scale * lmax * max(1.0, np.abs(r).max()), rtol=1e-6, err_msg=name)
        np.testing.assert_allclose(cost, 0.5 * r @ L @ r, rtol=1e-9, atol=1e-12, err_msg=name)


def test_one_end_fixed_is_a_prior():
    """With A fixed the term in B is the prior at A Z with the same L.  With B fixed the term in A is the prior at B Z^-1, whose
    residual is -Ad(Z) r: its information is Ad(Z^-1)^T L Ad(Z^-1), which the same L matches only when Z has no rotation and no
    translation."""
    rng = np.random.default_rng(23)
    for i in range(10):
        Z, A = M.random_pose(rng), M.random_pose(rng)
        B = M.compose_tangent(compose(A, Z), rng.normal(size=6) * 0.2)
        L = M.random_info(rng)
        L = (np.triu(L) + np.triu(L, 1).T).astype(np.float32).astype(np.float64)
        H, b, cost = constraint_terms(Z, A, B, M.upper(L))
        Hm = matrix(H, 12)
        # B's end: the prior at A Z
        Hp, bp, cp = M.host_terms(compose(A, Z), B, M.upper(L))
        tol = 2e-4 * max(1.0, np.abs(Hm).max())
        np.testing.assert_allclose(matrix(Hp, 6), Hm[6:, 6:], atol=tol, rtol=1e-4)
        np.testing.assert_allclose(bp, b[6:], atol=tol, rtol=1e-4)
        np.testing.assert_allclose(cp, cost, rtol=1e-3, atol=1e-7)
        # A's end: the prior at B Z^-1 with L_a = Ad(Z^-1)^T L Ad(Z^-1)
        Ad = adjoint(inverse(Z))
        La = Ad.T @ L @ Ad
        Hp, bp, cp = M.host_terms(compose(B, inverse(Z)), A, M.upper(La))
        tol = 2e-4 * max(1.0, np.abs(Hm).max())
        np.testing.assert_allclose(matrix(Hp, 6), Hm[:6, :6], atol=tol, rtol=1e-4)
        np.testing.assert_allclose(bp, b[:6], atol=tol, rtol=1e-4)
        np.testing.assert_allclose(cp, cost, rtol=1e-3, atol=1e-7)
        # ... and not with L itself
        _, bp_same, _ = M.host_terms(compose(B, inverse(Z)), A, M.upper(L))
        assert np.abs(bp_same - b[:6]).max() > 1e-3 * np.abs(b[:6]).max()


def test_pure_rotation_edge_step():
    """The 12 x 12 terms at a consistent pair are zero in b and have a null space of the common motion: (Ad(B^-1 A) x, x) moves
    both ends rigidly and leaves r unchanged."""
    rng = np.random.default_rng(4)
    Z, A = M.random_pose(rng), M.random_pose(rng)
    B = compose(A, Z)
    H, b, cost = constraint_terms(Z, A, B, M.upper(np.eye(6)))
    assert cost < 1e-10 and np.abs(b).max() < 1e-5
    x = rng.normal(size=6)
    v = np.concatenate([x, adjoint(inverse(B)) @ adjoint(A) @ x])   # delta_b = Ad(B^-1 A) delta_a
    Hm = matrix(H, 12)
    assert np.abs(Hm @ v).max() < 1e-4 * np.abs(Hm).max() * np.abs(v).max()


def test_constraint_entry_points_compile_as_c99_and_refuse_bad_arguments(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "constraint.c"
    src.write_text(r'''
#include "badba.h"
int main(void) {
  const float pose[7] = {0.f, 0.f, 0.f, 1.f, 1.f, 2.f, 3.f};
  const float ident[7] = {0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f};
  bba_pose_constraint c;
  int i, id = -5, ids[1] = {0}, count = 9;
  double H[78], b[12], cost = -1.0;
  c.keyframe_a = 0;
  c.keyframe_b = 1;
  for (i = 0; i < 7; ++i) c.a_T_b[i] = ident[i];
  for (i = 0; i < 21; ++i) c.information[i] = 0.f;
  c.information[0] = c.information[6] = c.information[11] = c.information[15] = c.information[18] = c.information[20] = 4.f;
  bba_host_pose_constraint_terms(ident, pose, pose, c.information, H, b, &cost);
  if (cost != 0.0 || H[0] != 4.0 || H[6] != -4.0 || H[1] != 0.0 || b[0] != 0.0) return 1;
  cost = -1.0;
  bba_host_pose_constraint_terms(ident, pose, pose, c.information, 0, b, &cost);
  if (cost != -1.0) return 2;
  if (bba_add_keyframe_pose_constraints(0, 1, &c, &id) != BBA_ERR_INVALID_ARGUMENT || id != -5) return 3;
  if (bba_remove_keyframe_pose_constraints(0, 1, ids) != BBA_ERR_INVALID_ARGUMENT) return 4;
  if (bba_remove_keyframe_pose_constraints(0, -1, 0) != BBA_ERR_INVALID_ARGUMENT) return 5;
  if (bba_get_keyframe_pose_constraints(0, 1, ids, &c, &count) != BBA_ERR_INVALID_ARGUMENT || count != 9) return 6;
  return 0;
}''')
    exe = tmp_path / "constraint"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                           "-o", str(exe), "-L", LIBDIR, "-lbadba_b200", f"-Wl,-rpath,{LIBDIR}"])
    assert subprocess.call([str(exe)]) == 0


def test_cpp_adaptor_constraint_methods_compile(tmp_path):
    gxx = shutil.which("g++")
    if gxx is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("no host compiler / CUDA headers")
    src = tmp_path / "constraint.cpp"
    src.write_text(r'''
#include "badba_direct_ba.hpp"
struct SE3 { float d[7]; float* data() { return d; } const float* data() const { return d; } };
struct Cam { int w, h; float p[4]; int width() const { return w; } int height() const { return h; } const float* parameters() const { return p; } };
int main(int argc, char**) {
  Cam c{64, 48, {30, 30, 32, 24}};
  try {
    badba::DirectBA<SE3, Cam> ba(1000, 1e-3f, 40.f, 4, 0.8f, 1, 2, 3, c, c, 0, true, true);
    if (argc > 100) {   // never taken: instantiates the members
      const SE3 a_T_b{{0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f}};
      const float info[21] = {1.f};
      const int id = ba.AddKeyframePoseConstraint(0, 1, a_T_b, info);
      ba.RemoveKeyframePoseConstraints({id});
      ba.RemoveKeyframePoseConstraints();
    }
  }
  catch (const badba::Error& e) { return e.status == BBA_ERR_NO_DEVICE ? 42 : 1; }
  return 0;
}''')
    exe = tmp_path / "constraint"
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include",
                           str(src), "-o", str(exe), "-L", LIBDIR, "-lbadba_b200", f"-Wl,-rpath,{LIBDIR}"])
    assert subprocess.call([str(exe)]) in (0, 42)
