// host_math.hpp -- small dense maths shared by host orchestration and the device-side
// Gauss-Newton solve kernel of libbadba_b200 (product code; independent of oracle/).
//
// Semantics follow the reference's host code so that results stay within the parity budget:
//   SE3f update  global_T_frame * exp(-x)      direct_ba_alternating.cc:214
//   Sophus SE3/SO3 exp, log, inverse, product  libvis/third_party/sophus/sophus/{se3,so3}.hpp
//   fp64 LDLT of the upper triangle            direct_ba_alternating.cc:206, kernel_opt_intrinsics.cc:171,272
//   convergence test                           convergence_analysis.h:45-52
// Pose layout: float[7] = {qx,qy,qz,qw,tx,ty,tz} (Sophus::SE3f::data()).
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define BBA_HD __host__ __device__ __forceinline__
#else
#define BBA_HD inline
#endif

namespace bba {

constexpr float kSophusEpsilonF = 1e-5f;   // sophus/common.hpp:146-148

// Trigonometry evaluated in fp64 and rounded: these run once per keyframe per Gauss-Newton
// iteration, and must not degrade to the fast-math approximations the kernels are built with.
BBA_HD float PSin(float x) { return static_cast<float>(sin(static_cast<double>(x))); }
BBA_HD float PCos(float x) { return static_cast<float>(cos(static_cast<double>(x))); }
BBA_HD float PAtan(float x) { return static_cast<float>(atan(static_cast<double>(x))); }
BBA_HD float PSqrt(float x) { return static_cast<float>(sqrt(static_cast<double>(x))); }
BBA_HD float PDiv(float a, float b) { return static_cast<float>(static_cast<double>(a) / static_cast<double>(b)); }

struct Pose {  // global_T_frame or its inverse
  float q[4];  // x y z w
  float t[3];
};

BBA_HD void QuatRotate(const float q[4], const float v[3], float out[3]) {
  // Eigen::QuaternionBase::_transformVector
  const float ux = 2.f * (q[1] * v[2] - q[2] * v[1]);
  const float uy = 2.f * (q[2] * v[0] - q[0] * v[2]);
  const float uz = 2.f * (q[0] * v[1] - q[1] * v[0]);
  out[0] = v[0] + q[3] * ux + (q[1] * uz - q[2] * uy);
  out[1] = v[1] + q[3] * uy + (q[2] * ux - q[0] * uz);
  out[2] = v[2] + q[3] * uz + (q[0] * uy - q[1] * ux);
}

BBA_HD void QuatToMatrix(const float q[4], float R[9]) {
  // Eigen::QuaternionBase::toRotationMatrix
  const float tx = 2.f * q[0], ty = 2.f * q[1], tz = 2.f * q[2];
  const float twx = tx * q[3], twy = ty * q[3], twz = tz * q[3];
  const float txx = tx * q[0], txy = ty * q[0], txz = tz * q[0];
  const float tyy = ty * q[1], tyz = tz * q[1], tzz = tz * q[2];
  R[0] = 1.f - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
  R[3] = txy + twz; R[4] = 1.f - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.f - (txx + tyy);
}

BBA_HD Pose Inverse(const Pose& a) {   // se3.hpp:127-130
  Pose r;
  r.q[0] = -a.q[0]; r.q[1] = -a.q[1]; r.q[2] = -a.q[2]; r.q[3] = a.q[3];
  const float nt[3] = {-a.t[0], -a.t[1], -a.t[2]};
  QuatRotate(r.q, nt, r.t);
  return r;
}

BBA_HD Pose Compose(const Pose& a, const Pose& b) {   // se3.hpp:203-207, so3.hpp:215-232
  Pose r;
  float rt[3];
  QuatRotate(a.q, b.t, rt);
  r.t[0] = a.t[0] + rt[0]; r.t[1] = a.t[1] + rt[1]; r.t[2] = a.t[2] + rt[2];
  const float ax = a.q[0], ay = a.q[1], az = a.q[2], aw = a.q[3];
  const float bx = b.q[0], by = b.q[1], bz = b.q[2], bw = b.q[3];
  r.q[3] = aw * bw - ax * bx - ay * by - az * bz;
  r.q[0] = aw * bx + ax * bw + ay * bz - az * by;
  r.q[1] = aw * by + ay * bw + az * bx - ax * bz;
  r.q[2] = aw * bz + az * bw + ax * by - ay * bx;
  const float sn = r.q[0] * r.q[0] + r.q[1] * r.q[1] + r.q[2] * r.q[2] + r.q[3] * r.q[3];
  if (sn != 1.0f) {
    const float s = PDiv(2.0f, 1.0f + sn);
    r.q[0] *= s; r.q[1] *= s; r.q[2] *= s; r.q[3] *= s;
  }
  return r;
}

// Quaternion interpolation of the trajectory deformation, host only.  Eigen's 4-float dot product and squared norm reduce as its
// SSE packet code does, (x + z) + (y + w); sin / acos are the fp32 library functions std::sin / std::acos call for float.
inline float QuatDot(const float a[4], const float b[4]) { return (a[0] * b[0] + a[2] * b[2]) + (a[1] * b[1] + a[3] * b[3]); }

inline void QuatSlerp(const float q0[4], float t, const float q1[4], float out[4]) {   // Eigen QuaternionBase::slerp
  const float one = 1.0f - 1.1920928955078125e-7f;   // 1 - NumTraits<float>::epsilon()
  const float d = QuatDot(q0, q1);
  const float abs_d = fabsf(d);
  float scale0, scale1;
  if (abs_d >= one) {
    scale0 = 1.0f - t;
    scale1 = t;
  } else {
    const float theta = acosf(abs_d);
    const float sin_theta = sinf(theta);
    scale0 = sinf((1.0f - t) * theta) / sin_theta;
    scale1 = sinf(t * theta) / sin_theta;
  }
  if (d < 0.0f) scale1 = -scale1;
  for (int i = 0; i < 4; ++i) out[i] = scale0 * q0[i] + scale1 * q1[i];
}

inline void QuatNormalize(float q[4]) {   // so3.hpp:159-168 (SO3::normalize, behind setQuaternion)
  const float length = sqrtf(QuatDot(q, q));
  for (int i = 0; i < 4; ++i) q[i] /= length;
}

// Row-major 3x4 [R|t].
BBA_HD void ToMatrix3x4(const Pose& p, float M[12]) {
  float R[9];
  QuatToMatrix(p.q, R);
  M[0] = R[0]; M[1] = R[1]; M[2] = R[2]; M[3] = p.t[0];
  M[4] = R[3]; M[5] = R[4]; M[6] = R[5]; M[7] = p.t[1];
  M[8] = R[6]; M[9] = R[7]; M[10] = R[8]; M[11] = p.t[2];
}

BBA_HD void Hat(const float w[3], float O[9]) {
  O[0] = 0.f; O[1] = -w[2]; O[2] = w[1];
  O[3] = w[2]; O[4] = 0.f; O[5] = -w[0];
  O[6] = -w[1]; O[7] = w[0]; O[8] = 0.f;
}

BBA_HD void Mat3Mul(const float A[9], const float B[9], float C[9]) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}

BBA_HD Pose Exp(const float a[6]) {   // se3.hpp:293-313 + so3.hpp:282-312
  Pose r;
  const float* om = a + 3;
  const float theta_sq = om[0] * om[0] + om[1] * om[1] + om[2] * om[2];
  const float theta = PSqrt(theta_sq);
  float imag, real;
  if (theta < kSophusEpsilonF) {
    const float p4 = theta_sq * theta_sq;
    imag = 0.5f - (1.0f / 48.0f) * theta_sq + (1.0f / 3840.0f) * p4;
    real = 1.f - 0.5f * theta_sq + (1.0f / 384.0f) * p4;
  } else {
    const float h = 0.5f * theta;
    imag = PDiv(PSin(h), theta);
    real = PCos(h);
  }
  r.q[0] = imag * om[0]; r.q[1] = imag * om[1]; r.q[2] = imag * om[2]; r.q[3] = real;
  float O[9], O2[9], V[9];
  Hat(om, O);
  Mat3Mul(O, O, O2);
  if (theta < kSophusEpsilonF) {
    QuatToMatrix(r.q, V);
  } else {
    const float c1 = PDiv(1.f - PCos(theta), theta_sq);
    const float c2 = PDiv(theta - PSin(theta), theta_sq * theta);
    for (int i = 0; i < 9; ++i) V[i] = c1 * O[i] + c2 * O2[i];
    V[0] += 1.f; V[4] += 1.f; V[8] += 1.f;
  }
  for (int i = 0; i < 3; ++i) r.t[i] = V[i * 3] * a[0] + V[i * 3 + 1] * a[1] + V[i * 3 + 2] * a[2];
  return r;
}

BBA_HD void Log(const Pose& p, float out[6]) {   // se3.hpp:435-468 + so3.hpp:421-466
  const float sq_n = p.q[0] * p.q[0] + p.q[1] * p.q[1] + p.q[2] * p.q[2];
  const float n = PSqrt(sq_n);
  const float w = p.q[3];
  float f;
  if (n < kSophusEpsilonF) {
    f = PDiv(2.f, w) - PDiv(2.f * sq_n, w * w * w);
  } else if (fabsf(w) < kSophusEpsilonF) {
    f = PDiv(w > 0.f ? 3.14159265358979323846f : -3.14159265358979323846f, n);
  } else {
    f = PDiv(2.f * PAtan(PDiv(n, w)), n);
  }
  const float theta = f * n;
  const float om[3] = {f * p.q[0], f * p.q[1], f * p.q[2]};
  float O[9], O2[9];
  Hat(om, O);
  Mat3Mul(O, O, O2);
  float c2;
  if (fabsf(theta) < kSophusEpsilonF) {
    c2 = 1.f / 12.f;
  } else {
    const float h = 0.5f * theta;
    c2 = PDiv(1.f - PDiv(theta * PCos(h), 2.f * PSin(h)), theta * theta);
  }
  for (int i = 0; i < 3; ++i) {
    float v0 = -0.5f * O[i * 3] + c2 * O2[i * 3] + (i == 0 ? 1.f : 0.f);
    float v1 = -0.5f * O[i * 3 + 1] + c2 * O2[i * 3 + 1] + (i == 1 ? 1.f : 0.f);
    float v2 = -0.5f * O[i * 3 + 2] + c2 * O2[i * 3 + 2] + (i == 2 ? 1.f : 0.f);
    out[i] = v0 * p.t[0] + v1 * p.t[1] + v2 * p.t[2];
  }
  out[3] = om[0]; out[4] = om[1]; out[5] = om[2];
}

BBA_HD bool IsScale1PoseEstimationConverged(const float x[6]) {   // convergence_analysis.h:45-52
  const float s = 1e-06f / 1e-07f;
  const float sq = x[0] * x[0] + x[1] * x[1] + x[2] * x[2] + (s * x[3]) * (s * x[3]) + (s * x[4]) * (s * x[4]) +
                   (s * x[5]) * (s * x[5]);
  return sq < 1e-06f;
}

// x = A^-1 b for the symmetric N x N matrix whose upper triangle is packed row-major in `upper`
// (N(N+1)/2 entries, the layout of gauss_newton.cuh:59-73).  fp64, symmetric pivoting on the
// largest diagonal entry (what Eigen's LDLT does).  Rank-deficient directions get x = 0.
template <int N>
BBA_HD void SolveLDLT(const double* upper, const double* b, double* x) {
  double M[N * N];
  int perm[N];
  int idx = 0;
  for (int r = 0; r < N; ++r) {
    perm[r] = r;
    for (int c = r; c < N; ++c) {
      M[r * N + c] = upper[idx];
      M[c * N + r] = upper[idx];
      ++idx;
    }
  }
  for (int k = 0; k < N; ++k) {
    int p = k;
    double best = fabs(M[k * N + k]);
    for (int i = k + 1; i < N; ++i) {
      const double v = fabs(M[i * N + i]);
      if (v > best) { best = v; p = i; }
    }
    if (p != k) {
      for (int c = 0; c < N; ++c) { const double t = M[k * N + c]; M[k * N + c] = M[p * N + c]; M[p * N + c] = t; }
      for (int r = 0; r < N; ++r) { const double t = M[r * N + k]; M[r * N + k] = M[r * N + p]; M[r * N + p] = t; }
      const int t = perm[k]; perm[k] = perm[p]; perm[p] = t;
    }
    const double d = M[k * N + k];
    if (d == 0.0) {
      for (int i = k + 1; i < N; ++i) M[i * N + k] = 0.0;
      continue;
    }
    for (int i = k + 1; i < N; ++i) M[i * N + k] /= d;
    for (int i = k + 1; i < N; ++i)
      for (int j = k + 1; j <= i; ++j) {
        M[i * N + j] -= M[i * N + k] * d * M[j * N + k];
        M[j * N + i] = M[i * N + j];
      }
  }
  double y[N];
  for (int i = 0; i < N; ++i) y[i] = b[perm[i]];
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < i; ++j) y[i] -= M[i * N + j] * y[j];
  for (int i = 0; i < N; ++i) {
    const double d = M[i * N + i];
    y[i] = (fabs(d) > 2.2250738585072014e-308) ? y[i] / d : 0.0;
  }
  for (int i = N - 1; i >= 0; --i)
    for (int j = i + 1; j < N; ++j) y[i] -= M[j * N + i] * y[j];
  for (int i = 0; i < N; ++i) x[perm[i]] = y[i];
}

// ---- soft pose prior on a keyframe (bba_set_keyframe_pose_priors) ----
// 3x3 helpers in fp64 (row-major).
BBA_HD void HatD(const double w[3], double O[9]) {
  O[0] = 0.0; O[1] = -w[2]; O[2] = w[1];
  O[3] = w[2]; O[4] = 0.0; O[5] = -w[0];
  O[6] = -w[1]; O[7] = w[0]; O[8] = 0.0;
}
BBA_HD void Mat3MulD(const double A[9], const double B[9], double C[9]) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) C[r * 3 + c] = A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c] + A[r * 3 + 2] * B[6 + c];
}

// The inverse left Jacobian of SO(3) at the rotation vector w with angle theta = |w|: I - W/2 + c W^2.
BBA_HD void So3LeftJacobianInverse(const double w[3], double theta, double A[9]) {
  const double t2 = theta * theta;
  double c;
  if (theta < 0.05) {
    c = 1.0 / 12.0 + t2 / 720.0 + t2 * t2 / 30240.0;
  } else {
    const double h = 0.5 * theta;
    c = (1.0 - h * cos(h) / sin(h)) / t2;
  }
  double W[9], W2[9];
  HatD(w, W);
  Mat3MulD(W, W, W2);
  for (int i = 0; i < 9; ++i) A[i] = -0.5 * W[i] + c * W2[i];
  A[0] += 1.0; A[4] += 1.0; A[8] += 1.0;
}

// A pose in fp64 with its quaternion normalised: q (x, y, z, w) and t.
BBA_HD void LoadPoseD(const float p[7], double q[4], double t[3]) {
  double n = 0.0;
  for (int i = 0; i < 4; ++i) {
    q[i] = p[i];
    n += q[i] * q[i];
  }
  n = 1.0 / sqrt(n);
  for (int i = 0; i < 4; ++i) q[i] *= n;
  for (int i = 0; i < 3; ++i) t[i] = p[4 + i];
}

// P^-1 T of two poses in fp64: q = conj(qp) * qt, t = R(qp)^T (t_T - t_P).
BBA_HD void Se3BetweenD(const double qp[4], const double tp[3], const double qt[4], const double tt[3], double q[4], double t[3]) {
  const double ax = -qp[0], ay = -qp[1], az = -qp[2], aw = qp[3];
  const double bx = qt[0], by = qt[1], bz = qt[2], bw = qt[3];
  q[3] = aw * bw - ax * bx - ay * by - az * bz;
  q[0] = aw * bx + ax * bw + ay * bz - az * by;
  q[1] = aw * by + ay * bw + az * bx - ax * bz;
  q[2] = aw * bz + az * bw + ax * by - ay * bx;
  const double d[3] = {tt[0] - tp[0], tt[1] - tp[1], tt[2] - tp[2]};
  // rotate d by conj(qp): v + w u + v x u with u = 2 (qv x d), qv = -qp.xyz
  const double ux = 2.0 * (ay * d[2] - az * d[1]), uy = 2.0 * (az * d[0] - ax * d[2]), uz = 2.0 * (ax * d[1] - ay * d[0]);
  t[0] = d[0] + aw * ux + (ay * uz - az * uy);
  t[1] = d[1] + aw * uy + (az * ux - ax * uz);
  t[2] = d[2] + aw * uz + (ax * uy - ay * ux);
}

// A * B of two poses in fp64: q = qa * qb, t = R(qa) t_B + t_A.
BBA_HD void Se3ComposeD(const double qa[4], const double ta[3], const double qb[4], const double tb[3], double q[4], double t[3]) {
  const double ax = qa[0], ay = qa[1], az = qa[2], aw = qa[3];
  q[3] = aw * qb[3] - ax * qb[0] - ay * qb[1] - az * qb[2];
  q[0] = aw * qb[0] + ax * qb[3] + ay * qb[2] - az * qb[1];
  q[1] = aw * qb[1] + ay * qb[3] + az * qb[0] - ax * qb[2];
  q[2] = aw * qb[2] + az * qb[3] + ax * qb[1] - ay * qb[0];
  const double ux = 2.0 * (ay * tb[2] - az * tb[1]), uy = 2.0 * (az * tb[0] - ax * tb[2]), uz = 2.0 * (ax * tb[1] - ay * tb[0]);
  t[0] = ta[0] + tb[0] + aw * ux + (ay * uz - az * uy);
  t[1] = ta[1] + tb[1] + aw * uy + (az * ux - ax * uz);
  t[2] = ta[2] + tb[2] + aw * uz + (ax * uy - ay * ux);
}

// Ad(T) of a pose in the tangent order (translation, rotation): [[R, [t]x R], [0, R]], so that T exp(x) T^-1 = exp(Ad(T) x).
BBA_HD void Se3AdjointD(const double q[4], const double t[3], double Ad[36]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double R[9] = {1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - z * w), 2.0 * (x * z + y * w),
                       2.0 * (x * y + z * w), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - x * w),
                       2.0 * (x * z - y * w), 2.0 * (y * z + x * w), 1.0 - 2.0 * (x * x + y * y)};
  double T[9], TR[9];
  HatD(t, T);
  Mat3MulD(T, R, TR);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      Ad[i * 6 + j] = R[i * 3 + j];
      Ad[i * 6 + 3 + j] = TR[i * 3 + j];
      Ad[(3 + i) * 6 + j] = 0.0;
      Ad[(3 + i) * 6 + 3 + j] = R[i * 3 + j];
    }
}

// log of a pose with a unit quaternion, in the tangent order (translation, rotation), fp64, the rotation angle in [0, pi].
BBA_HD void Se3LogD(const double q_in[4], const double t[3], double r[6], double* theta_out) {
  double q[4] = {q_in[0], q_in[1], q_in[2], q_in[3]};
  if (q[3] < 0.0)
    for (int i = 0; i < 4; ++i) q[i] = -q[i];
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  const double theta = 2.0 * atan2(n, q[3]);
  const double f = (n > 1e-10) ? theta / n : 2.0 / q[3] * (1.0 - n * n / (3.0 * q[3] * q[3]));
  const double w[3] = {f * q[0], f * q[1], f * q[2]};
  double A[9];
  So3LeftJacobianInverse(w, theta, A);
  for (int i = 0; i < 3; ++i) {
    r[i] = A[i * 3] * t[0] + A[i * 3 + 1] * t[1] + A[i * 3 + 2] * t[2];
    r[3 + i] = w[i];
  }
  *theta_out = theta;
}

// r = log(P^-1 T) in the tangent order (translation, rotation), fp64, the rotation angle in [0, pi].  The quaternions are
// normalised first.
BBA_HD void PosePriorResidual(const float prior[7], const float pose[7], double r[6], double* theta_out) {
  double qp[4], tp[3], qt[4], tt[3], q[4], t[3];
  LoadPoseD(prior, qp, tp);
  LoadPoseD(pose, qt, tt);
  Se3BetweenD(qp, tp, qt, tt, q, t);
  Se3LogD(q, t, r, theta_out);
}

// J = Jr^-1(r), the inverse right Jacobian of SE(3) in the tangent order (rho, phi): d log(exp(r) exp(delta)) / d delta at 0.
// Jr^-1(r) = Jl^-1(-r) = [[A, -A Q A], [0, A]] with A = Jl^-1_SO3(-phi) and Q = Q(-rho, -phi) (Barfoot, eq. 7.86).
BBA_HD void Se3RightJacobianInverse(const double r[6], double theta, double J[36]) {
  const double rho[3] = {-r[0], -r[1], -r[2]}, phi[3] = {-r[3], -r[4], -r[5]};
  double A[9];
  So3LeftJacobianInverse(phi, theta, A);
  const double t2 = theta * theta;
  double c1, c2, c3;
  if (theta < 0.05) {
    c1 = 1.0 / 6.0 - t2 / 120.0 + t2 * t2 / 5040.0;
    c2 = 1.0 / 24.0 - t2 / 720.0 + t2 * t2 / 40320.0;
    c3 = 1.0 / 120.0 - t2 / 2520.0 + t2 * t2 / 120960.0;
  } else {
    const double s = sin(theta), c = cos(theta);
    c1 = (theta - s) / (t2 * theta);
    c2 = (t2 + 2.0 * c - 2.0) / (2.0 * t2 * t2);
    c3 = (2.0 * theta - 3.0 * s + theta * c) / (2.0 * t2 * t2 * theta);
  }
  double P[9], R[9], PR[9], RP[9], PRP[9], PP[9], PPR[9], RPP[9], PRPP[9], PPRP[9];
  HatD(phi, P);
  HatD(rho, R);
  Mat3MulD(P, R, PR);
  Mat3MulD(R, P, RP);
  Mat3MulD(PR, P, PRP);
  Mat3MulD(P, P, PP);
  Mat3MulD(PP, R, PPR);
  Mat3MulD(RP, P, RPP);
  Mat3MulD(PRP, P, PRPP);
  Mat3MulD(PP, RP, PPRP);
  double Q[9];
  for (int i = 0; i < 9; ++i)
    Q[i] = 0.5 * R[i] + c1 * (PR[i] + RP[i] + PRP[i]) + c2 * (PPR[i] + RPP[i] - 3.0 * PRP[i]) + c3 * (PRPP[i] + PPRP[i]);
  double AQ[9], AQA[9];
  Mat3MulD(A, Q, AQ);
  Mat3MulD(AQ, A, AQA);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      J[i * 6 + j] = A[i * 3 + j];
      J[i * 6 + 3 + j] = -AQA[i * 3 + j];
      J[(3 + i) * 6 + j] = 0.0;
      J[(3 + i) * 6 + 3 + j] = A[i * 3 + j];
    }
}

// The terms of 1/2 r^T L r with the 6 x N Jacobian J (row-major): H = J^T L J (upper triangle, N (N + 1) / 2), b = J^T L r (N),
// cost = r^T L r / 2.  info: L's upper triangle (21).  fp64 throughout.
template <int N>
BBA_HD void InformationTerms(const double r[6], const double* J, const float info[21], double* H, double* b, double* cost) {
  double L[36];
  int idx = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) {
      L[i * 6 + j] = L[j * 6 + i] = info[idx];
      ++idx;
    }
  double LJ[6 * N], Lr[6];
  for (int i = 0; i < 6; ++i) {
    Lr[i] = 0.0;
    for (int k = 0; k < 6; ++k) Lr[i] += L[i * 6 + k] * r[k];
    for (int j = 0; j < N; ++j) {
      double s = 0.0;
      for (int k = 0; k < 6; ++k) s += L[i * 6 + k] * J[k * N + j];
      LJ[i * N + j] = s;
    }
  }
  idx = 0;
  double c = 0.0;
  for (int i = 0; i < N; ++i) {
    double s = 0.0;
    for (int k = 0; k < 6; ++k) s += J[k * N + i] * Lr[k];
    b[i] = s;
    if (i < 6) c += r[i] * Lr[i];
    for (int j = i; j < N; ++j) {
      double h = 0.0;
      for (int k = 0; k < 6; ++k) h += J[k * N + i] * LJ[k * N + j];
      H[idx++] = h;
    }
  }
  *cost = 0.5 * c;
}

// The prior's terms at global_T_frame = pose, for an update pose <- pose * exp(delta): with r = log(P^-1 pose) and J = Jr^-1(r),
// H = J^T L J (upper triangle, 21), b = J^T L r (6), cost = r^T L r / 2.  fp64 throughout.
BBA_HD void PosePriorTerms(const float prior[7], const float pose[7], const float info[21], double H[21], double b[6], double* cost) {
  double r[6], theta, J[36];
  PosePriorResidual(prior, pose, r, &theta);
  Se3RightJacobianInverse(r, theta, J);
  InformationTerms<6>(r, J, info, H, b, cost);
}

// ---- attitude prior on a keyframe (bba_set_keyframe_attitude_priors, DESIGN §3.17) ----
// The attitude prior's terms at global_T_frame = pose, for an update pose <- pose * exp(delta).  p = R^-1 d_ref is the predicted
// direction in the camera frame and m = d_meas the measured one (both normalised here); theta in [0, pi] is their angle and the
// term costs L theta^2 / 2.  The residual is r = theta n with n = (p x m) / |p x m|, the rotation vector that turns p into m.
//   b = L theta n: the exact gradient (d theta = n . omega for the rotation part omega of delta; at theta = pi exactly, p x m = 0
//       and b = 0).
//   H = L (I - p p^T) in the rotation block: r's Gauss-Newton matrix at theta = 0, which stays finite at every angle (the exact one
//       grows as (theta / sin theta)^2 across the great circle through p and m).
// The translation rows of H and b are zero and p, the yaw axis about d_ref, is H's null direction.  H: upper triangle (21) in the
// tangent order (translation, rotation); cost = L theta^2 / 2.  fp64 throughout.
BBA_HD void AttitudePriorTerms(const float d_ref[3], const float d_meas[3], float information, const float pose[7], double H[21],
                               double b[6], double* cost) {
  double q[4], t[3], d[3], m[3], nd = 0.0, nm = 0.0;
  LoadPoseD(pose, q, t);
  for (int i = 0; i < 3; ++i) {
    d[i] = d_ref[i];
    m[i] = d_meas[i];
    nd += d[i] * d[i];
    nm += m[i] * m[i];
  }
  nd = 1.0 / sqrt(nd);
  nm = 1.0 / sqrt(nm);
  for (int i = 0; i < 3; ++i) {
    d[i] *= nd;
    m[i] *= nm;
  }
  // p = R^T d: rotate d by conj(q), as Se3BetweenD
  const double ax = -q[0], ay = -q[1], az = -q[2], aw = q[3];
  const double ux = 2.0 * (ay * d[2] - az * d[1]), uy = 2.0 * (az * d[0] - ax * d[2]), uz = 2.0 * (ax * d[1] - ay * d[0]);
  const double p[3] = {d[0] + aw * ux + (ay * uz - az * uy), d[1] + aw * uy + (az * ux - ax * uz), d[2] + aw * uz + (ax * uy - ay * ux)};
  const double x[3] = {p[1] * m[2] - p[2] * m[1], p[2] * m[0] - p[0] * m[2], p[0] * m[1] - p[1] * m[0]};   // p x m
  const double s = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]), c = p[0] * m[0] + p[1] * m[1] + p[2] * m[2];
  const double theta = atan2(s, c);
  const double f = s > 0.0 ? theta / s : 1.0;   // |x| = sin theta; p x m = 0 at 0 and pi, where b = 0
  const double L = information;
  int idx = 0;
  for (int r = 0; r < 6; ++r) {
    b[r] = r < 3 ? 0.0 : L * f * x[r - 3];
    for (int col = r; col < 6; ++col, ++idx)
      H[idx] = r < 3 ? 0.0 : L * ((r == col ? 1.0 : 0.0) - p[r - 3] * p[col - 3]);
  }
  *cost = 0.5 * L * theta * theta;
}

// The robust loss of a pose term (bba_robust_loss, Ceres' conventions): a term whose squared Mahalanobis norm is s = r^T L r costs
// rho(s) / 2 instead of s / 2, and IRLS scales its H and b by w = rho'(s).  type: 0 trivial (rho = s), 1 Huber, 2 Cauchy; scale =
// delta in units of sqrt(s).  An inlier under Huber (s <= delta^2) gets rho = s and w = 1.0 exactly, as the trivial loss does.
BBA_HD void RobustLoss(int type, float scale, double s, double* rho, double* w) {
  const double d = scale, d2 = d * d;
  if (type == 1 && s > d2) {
    const double root = sqrt(s);
    *rho = 2.0 * d * root - d2;
    *w = d / root;
  } else if (type == 2) {
    *rho = d2 * log1p(s / d2);
    *w = 1.0 / (1.0 + s / d2);
  } else {
    *rho = s;
    *w = 1.0;
  }
}

// Whether the symmetric 6x6 matrix with upper triangle info is positive semi-definite up to fp32 rounding: the pivoted LDLT of
// SolveLDLT (largest |diagonal| first) has no negative pivot, and a zero pivot leaves nothing in its column.  Host only: the test of
// every information matrix a caller passes (priors, constraints, the pose graph's odometry chain).
inline bool InformationPsd(const float info[21]) {
  double M[36];
  double scale = 0.0;
  int idx = 0;
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) {
      M[r * 6 + c] = M[c * 6 + r] = info[idx++];
      scale = fmax(scale, fabs(static_cast<double>(info[idx - 1])));
    }
  if (scale == 0.0) return true;
  const double pivot_tol = 1e-6 * scale, column_tol = 1e-3 * scale;
  bool done[6] = {};
  for (int k = 0; k < 6; ++k) {
    int p = -1;
    for (int i = 0; i < 6; ++i)
      if (!done[i] && (p < 0 || fabs(M[i * 6 + i]) > fabs(M[p * 6 + p]))) p = i;
    done[p] = true;
    const double d = M[p * 6 + p];
    if (d < -pivot_tol) return false;
    if (d <= pivot_tol) {
      for (int i = 0; i < 6; ++i)
        if (!done[i] && fabs(M[i * 6 + p]) > column_tol) return false;
      continue;
    }
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j)
        if (!done[i] && !done[j]) M[i * 6 + j] -= M[i * 6 + p] * M[p * 6 + j] / d;
  }
  return true;
}

// ---- soft relative pose constraint between two keyframes (bba_add_keyframe_pose_constraints) ----
// The index of (r, c), r <= c, in the row-major upper triangle of a 12 x 12 matrix (78 entries).
BBA_HD int Upper12(int r, int c) { return r * 12 - r * (r - 1) / 2 + (c - r); }

// The constraint's terms at global_T_frame = pose_a, pose_b, for the updates pose_a * exp(delta_a), pose_b * exp(delta_b): with
// r = log(Z^-1 pose_a^-1 pose_b), Z = a_T_b, J_b = Jr^-1(r) and J_a = -Jr^-1(r) Ad(pose_b^-1 pose_a), and J = [J_a | J_b]:
// H = J^T L J over (delta_a, delta_b) (12 x 12 upper triangle, 78), b = J^T L r (12), cost = r^T L r / 2.  fp64 throughout.
BBA_HD void PoseConstraintTerms(const float a_T_b[7], const float pose_a[7], const float pose_b[7], const float info[21], double r[6],
                                double H[78], double b[12], double* cost) {
  double qz[4], tz[3], qa[4], ta[3], qb[4], tb[3], qe[4], te[3], qx[4], tx[3];
  LoadPoseD(a_T_b, qz, tz);
  LoadPoseD(pose_a, qa, ta);
  LoadPoseD(pose_b, qb, tb);
  Se3BetweenD(qa, ta, qb, tb, qe, te);   // pose_a^-1 pose_b
  Se3BetweenD(qz, tz, qe, te, qx, tx);   // Z^-1 pose_a^-1 pose_b
  double theta, Jr[36], Ad[36], J[72];
  Se3LogD(qx, tx, r, &theta);
  Se3RightJacobianInverse(r, theta, Jr);
  Se3BetweenD(qb, tb, qa, ta, qe, te);   // pose_b^-1 pose_a
  Se3AdjointD(qe, te, Ad);
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double s = 0.0;
      for (int k = 0; k < 6; ++k) s += Jr[i * 6 + k] * Ad[k * 6 + j];
      J[i * 12 + j] = -s;
      J[i * 12 + 6 + j] = Jr[i * 6 + j];
    }
  InformationTerms<12>(r, J, info, H, b, cost);
}

// The information of the prior that stands for a constraint's term in pose_a while pose_b stays fixed.  That prior sits at
// P = pose_b Z^-1, and its residual log(P^-1 pose_a) = log(Z (Z^-1 pose_a^-1 pose_b)^-1 Z^-1) = -Ad(Z) r, so with
// L_a = Ad(Z^-1)^T L Ad(Z^-1) its cost equals the constraint's.  info_a: L_a's upper triangle (21).
BBA_HD void PoseConstraintInformationA(const float a_T_b[7], const float info[21], double info_a[21]) {
  double qz[4], tz[3], qi[4], ti[3], Ad[36], L[36];
  LoadPoseD(a_T_b, qz, tz);
  const double q_id[4] = {0.0, 0.0, 0.0, 1.0}, t_id[3] = {0.0, 0.0, 0.0};
  Se3BetweenD(qz, tz, q_id, t_id, qi, ti);   // Z^-1
  Se3AdjointD(qi, ti, Ad);
  int idx = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) {
      L[i * 6 + j] = L[j * 6 + i] = info[idx];
      ++idx;
    }
  idx = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) {
      double s = 0.0;
      for (int k = 0; k < 6; ++k)
        for (int l = 0; l < 6; ++l) s += Ad[k * 6 + i] * L[k * 6 + l] * Ad[l * 6 + j];
      info_a[idx++] = s;
    }
}

// ---- loop-closure verification (bba_verify_loop_closures), host only ----
// Eigen's Quaternion(Matrix3f) (Quaternion.h quaternionbase_assign_impl) on a row-major 3x3 matrix, fp32.
inline void QuatFromMatrix(const float R[9], float q[4]) {
  const auto m = [&](int r, int c) { return R[r * 3 + c]; };
  float t = m(0, 0) + m(1, 1) + m(2, 2);
  if (t > 0.f) {
    t = sqrtf(t + 1.0f);
    q[3] = 0.5f * t;
    t = 0.5f / t;
    q[0] = (m(2, 1) - m(1, 2)) * t;
    q[1] = (m(0, 2) - m(2, 0)) * t;
    q[2] = (m(1, 0) - m(0, 1)) * t;
  } else {
    int i = 0;
    if (m(1, 1) > m(0, 0)) i = 1;
    if (m(2, 2) > m(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrtf(m(i, i) - m(j, j) - m(k, k) + 1.0f);
    q[i] = 0.5f * t;
    t = 0.5f / t;
    q[3] = (m(k, j) - m(j, k)) * t;
    q[j] = (m(j, i) + m(i, j)) * t;
    q[k] = (m(k, i) + m(i, k)) * t;
  }
}

// The eigen-decomposition A = V diag(w) V^T of a symmetric 3x3 matrix (row-major) by cyclic Jacobi rotations in fp64, the
// eigenvalues in descending order and V's columns the unit eigenvectors.
inline void SymmetricEigen3(const double A_in[9], double w[3], double V[9]) {
  double A[9];
  for (int i = 0; i < 9; ++i) {
    A[i] = A_in[i];
    V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  }
  for (int sweep = 0; sweep < 50; ++sweep) {
    const double off = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
    const double diag = A[0] * A[0] + A[4] * A[4] + A[8] * A[8];
    if (off <= 1e-30 * diag || off == 0.0) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = A[p * 3 + q];
        if (apq == 0.0) continue;
        const double theta = (A[q * 3 + q] - A[p * 3 + p]) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) {   // A <- A G (columns p, q), then G^T A (rows p, q)
          const double akp = A[k * 3 + p], akq = A[k * 3 + q];
          A[k * 3 + p] = c * akp - s * akq;
          A[k * 3 + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {
          const double apk = A[p * 3 + k], aqk = A[q * 3 + k];
          A[p * 3 + k] = c * apk - s * aqk;
          A[q * 3 + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = V[k * 3 + p], vkq = V[k * 3 + q];
          V[k * 3 + p] = c * vkp - s * vkq;
          V[k * 3 + q] = s * vkp + c * vkq;
        }
      }
  }
  int order[3] = {0, 1, 2};
  for (int i = 0; i < 3; ++i)
    for (int j = i + 1; j < 3; ++j)
      if (A[order[j] * 4] > A[order[i] * 4]) { const int t = order[i]; order[i] = order[j]; order[j] = t; }
  double Vs[9];
  for (int c = 0; c < 3; ++c) {
    w[c] = A[order[c] * 4];
    for (int r = 0; r < 3; ++r) Vs[r * 3 + c] = V[r * 3 + order[c]];
  }
  for (int i = 0; i < 9; ++i) V[i] = Vs[i];
}

// AveragePose (util.cc:110-128): the rotation matrices and the translations of `count` poses summed in fp64; the rotation is U V^T
// of the SVD M = U S V^T of the rotation sum, rounded to fp32 and set as Sophus' setRotationMatrix does (Eigen's matrix-to-
// quaternion conversion, then normalised); the translation is the fp64 mean rounded to fp32.  The SVD comes from the
// eigen-decomposition M^T M = V S^2 V^T: u_i = M v_i / s_i.  U V^T is the orthogonal polar factor of M, the same matrix whatever
// signs an SVD routine picks for its singular vectors when M has full rank.  Like the reference, a sum with det < 0 is not
// corrected: U V^T is then a reflection.  (A sum of rank < 3 -- rotations that cancel -- completes U by cross products.)
inline Pose AveragePose(int count, const Pose* poses) {
  double M[9] = {}, t[3] = {};
  for (int i = 0; i < count; ++i) {
    float R[9];
    QuatToMatrix(poses[i].q, R);
    for (int j = 0; j < 9; ++j) M[j] += static_cast<double>(R[j]);
    for (int j = 0; j < 3; ++j) t[j] += static_cast<double>(poses[i].t[j]);
  }
  double MtM[9], s2[3], V[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) MtM[r * 3 + c] = M[r] * M[c] + M[3 + r] * M[3 + c] + M[6 + r] * M[6 + c];
  SymmetricEigen3(MtM, s2, V);
  double U[9] = {};
  int rank = 0;
  for (int c = 0; c < 3; ++c) {
    const double s = sqrt(fmax(s2[c], 0.0));
    if (!(s > 1e-12 * sqrt(fmax(s2[0], 0.0)))) break;
    for (int r = 0; r < 3; ++r) U[r * 3 + c] = (M[r * 3] * V[c] + M[r * 3 + 1] * V[3 + c] + M[r * 3 + 2] * V[6 + c]) / s;
    ++rank;
  }
  if (rank < 3) {   // complete U to an orthonormal basis
    if (rank == 0) { U[0] = 1.0; rank = 1; }
    if (rank == 1) {
      const double a = fabs(U[0]) < 0.9 ? 1.0 : 0.0, b = 1.0 - a;   // any vector not parallel to u_1
      double u[3] = {a - U[0] * (a * U[0] + b * U[3]), b - U[3] * (a * U[0] + b * U[3]), -U[6] * (a * U[0] + b * U[3])};
      const double n = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
      for (int r = 0; r < 3; ++r) U[r * 3 + 1] = u[r] / n;
    }
    U[2] = U[3] * U[7] - U[6] * U[4];
    U[5] = U[6] * U[1] - U[0] * U[7];
    U[8] = U[0] * U[4] - U[3] * U[1];
  }
  float Rf[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      Rf[r * 3 + c] = static_cast<float>(U[r * 3] * V[c * 3] + U[r * 3 + 1] * V[c * 3 + 1] + U[r * 3 + 2] * V[c * 3 + 2]);
  Pose out;
  QuatFromMatrix(Rf, out.q);
  QuatNormalize(out.q);
  for (int j = 0; j < 3; ++j) out.t[j] = static_cast<float>(t[j] / (1.0 * count));
  return out;
}

// The agreement test of three refined cur_T_old estimates (loop_detector.cc:575-609), in fp32 like Sophus: for the pairs (0, 1),
// (0, 2), (1, 2) in this order, the rotational distance acos(clamp(dot of the third columns of the two rotation matrices)) --
// blind to a roll about the optical axis, as in the reference -- is tested first, then the Euclidean distance of the translations.
// The 3-vector dot product and squared norm reduce as Eigen's unrolled redux does, a0 + (a1 + a2).  Returns 0 when every pair
// agrees, 2 (BBA_LOOP_ROTATION_DISAGREES) or 3 (BBA_LOOP_TRANSLATION_DISAGREES) for the first failed test; *angle and
// *translation receive the largest distances over all three pairs.
inline int LoopAgreement(const Pose refined[3], float max_angle, float max_translation, float* angle, float* translation) {
  int status = 0;
  *angle = 0.f;
  *translation = 0.f;
  for (int i = 0; i < 2; ++i)
    for (int k = i + 1; k < 3; ++k) {
      float Ri[9], Rk[9];
      QuatToMatrix(refined[i].q, Ri);
      QuatToMatrix(refined[k].q, Rk);
      const float dot = Ri[2] * Rk[2] + (Ri[5] * Rk[5] + Ri[8] * Rk[8]);
      const float rotational = acosf(fminf(1.f, fmaxf(-1.f, dot)));
      const float d[3] = {refined[i].t[0] - refined[k].t[0], refined[i].t[1] - refined[k].t[1], refined[i].t[2] - refined[k].t[2]};
      const float translational = sqrtf(d[0] * d[0] + (d[1] * d[1] + d[2] * d[2]));
      if (status == 0 && rotational > max_angle) status = 2;
      if (status == 0 && translational > max_translation) status = 3;
      *angle = fmaxf(*angle, rotational);
      *translation = fmaxf(*translation, translational);
    }
  return status;
}

// Camera frusta and their intersection test (co-visibility of keyframes), host only.
struct Frustum {   // libvis/src/libvis/camera_frustum.h:43-250
  float p[8][3];
  float bmin[3], bmax[3];
  float axes[6][3];
  float plane_n[6][3];
  float plane_d[6];
};

inline void Sub(const float a[3], const float b[3], float o[3]) { o[0] = a[0] - b[0]; o[1] = a[1] - b[1]; o[2] = a[2] - b[2]; }
inline void CrossP(const float a[3], const float b[3], float o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
inline float DotP(const float a[3], const float b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

inline void MakeFrustum(Frustum* f, const float K[4], int width, int height, float min_depth, float max_depth, const Pose& global_T_cam) {
  float M[12];
  ToMatrix3x4(global_T_cam, M);
  for (int i = 0; i < 3; ++i) {
    f->bmin[i] = INFINITY;
    f->bmax[i] = -INFINITY;
  }
  // corner order of camera_frustum.h:155-177: top-left, top-right, bottom-left, bottom-right; min then max depth
  const float cx[4] = {0.f, static_cast<float>(width), 0.f, static_cast<float>(width)};
  const float cy[4] = {0.f, 0.f, static_cast<float>(height), static_cast<float>(height)};
  for (int c = 0; c < 4; ++c) {
    const float dx = (cx[c] - K[2]) / K[0], dy = (cy[c] - K[3]) / K[1];   // UnprojectFromPixelCornerConv
    for (int d = 0; d < 2; ++d) {
      const float depth = d ? max_depth : min_depth;
      const float v[3] = {depth * dx, depth * dy, depth};
      float* o = f->p[2 * c + d];
      for (int r = 0; r < 3; ++r) {
        o[r] = M[r * 4] * v[0] + M[r * 4 + 1] * v[1] + M[r * 4 + 2] * v[2] + M[r * 4 + 3];
        f->bmin[r] = fminf(f->bmin[r], o[r]);
        f->bmax[r] = fmaxf(f->bmax[r], o[r]);
      }
    }
  }
  // camera_frustum.h:180-218
  Sub(f->p[7], f->p[6], f->axes[0]);
  Sub(f->p[3], f->p[2], f->axes[1]);
  Sub(f->p[5], f->p[4], f->axes[2]);
  Sub(f->p[1], f->p[0], f->axes[3]);
  Sub(f->p[2], f->p[6], f->axes[4]);
  Sub(f->p[0], f->p[2], f->axes[5]);
  float fwd[3];
  CrossP(f->axes[5], f->axes[4], fwd);
  for (int i = 0; i < 3; ++i) {
    f->plane_n[0][i] = fwd[i];
    f->plane_n[1][i] = -fwd[i];
  }
  f->plane_d[0] = -DotP(fwd, f->p[1]);
  f->plane_d[1] = DotP(fwd, f->p[0]);
  CrossP(f->axes[0], f->axes[4], f->plane_n[2]); f->plane_d[2] = -DotP(f->plane_n[2], f->p[6]);
  CrossP(f->axes[1], f->axes[5], f->plane_n[3]); f->plane_d[3] = -DotP(f->plane_n[3], f->p[2]);
  CrossP(f->axes[4], f->axes[2], f->plane_n[4]); f->plane_d[4] = -DotP(f->plane_n[4], f->p[4]);
  CrossP(f->axes[5], f->axes[0], f->plane_n[5]); f->plane_d[5] = -DotP(f->plane_n[5], f->p[6]);
}

inline bool AllOutside(const Frustum& planes_of, const Frustum& points_of) {
  for (int pl = 0; pl < 6; ++pl) {
    int v = 0;
    for (; v < 8; ++v)
      if (DotP(planes_of.plane_n[pl], points_of.p[v]) + planes_of.plane_d[pl] < 0) break;
    if (v == 8) return true;
  }
  return false;
}

inline bool FrustaIntersect(const Frustum& a, const Frustum& b) {   // camera_frustum.h:73-143
  for (int i = 0; i < 3; ++i)
    if (fmaxf(a.bmin[i], b.bmin[i]) > fminf(a.bmax[i], b.bmax[i])) return false;
  if (AllOutside(a, b) || AllOutside(b, a)) return false;
  // Separating-axis part.  The reference crosses two edge directions of the SAME frustum (camera_frustum.h:122
  // uses axes_[this_edge] and axes_[other_edge], both members of `this`); kept as is for parity.
  for (int e1 = 0; e1 < 6; ++e1)
    for (int e2 = 0; e2 < 6; ++e2) {
      float dir[3];
      CrossP(a.axes[e1], a.axes[e2], dir);
      if (DotP(dir, dir) < 1e-5f) continue;
      float amin = INFINITY, amax = -INFINITY, bmin = INFINITY, bmax = -INFINITY;
      for (int p = 0; p < 8; ++p) {
        const float va = DotP(dir, a.p[p]), vb = DotP(dir, b.p[p]);
        amin = fminf(amin, va); amax = fmaxf(amax, va);
        bmin = fminf(bmin, vb); bmax = fmaxf(bmax, vb);
      }
      if (amax <= bmin || amin >= bmax) return false;
    }
  return true;
}

}  // namespace bba
