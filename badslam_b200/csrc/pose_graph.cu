// pose_graph.cu -- the keyframe pose graph of bba_optimize_pose_graph (DESIGN §3.14): Gauss-Newton over the soft pose priors, the
// relative pose constraints and the call's odometry chain, with every linear system solved on the device.
//
// One Gauss-Newton iteration is one round of four kernels, and the host enqueues every round without synchronising: the state
// (PoseGraphState) decides on the device whether the last step is kept, and once it is done every later kernel returns at once.
//   PoseGraphLinearizeKernel  one thread per term: PosePriorTerms / PoseConstraintTerms at the fp32 poses, in fp64.
//   PoseGraphAssembleKernel   one thread per row block: H_kk, b_k, the block-CSR row and the coupling H_{k,k+1}, summed over the
//                             row's terms in term order.  A held keyframe's row is the identity with a zero right-hand side.
//   PoseGraphSolveKernel      one CTA: the cost at the current poses (a fixed-order sum) and the test of the last step, then
//                             H delta = -b by PCG.  The preconditioner M is the block-tridiagonal part of H in keyframe order,
//                             factorised by odd-even (cyclic) reduction; every 6x6 pivot is an LDLT in SolveLDLT's convention,
//                             so a direction without information gets 0.  No float atomics: every sum runs in a fixed order.
//   PoseGraphUpdateKernel     one thread per keyframe: T <- T exp(delta) (as PcgApplyDelta), keeping T for a revert.
//
// This translation unit is compiled WITHOUT -use_fast_math.
#include "host_math.hpp"
#include "kernels.cuh"

namespace bba {
namespace {

constexpr int kSolveThreads = 256;
constexpr double kRelativeResidual = 1e-10;
constexpr double kConvergedStep = 1e-7;
constexpr double kPoseResolution = 1.0 / 524288.0;   // 2^-19

// The Solve kernel's view of PoseGraphArgs::work.  Vectors of K blocks: x (delta), r, p, q; z is the reduction's level-0 solution.
// Levels: level l holds n_l blocks (n_0 = K, n_{l+1} = ceil(n_l / 2), the even positions of level l) at slots off_l ...
struct Work {
  double *x, *r, *p, *q;
  double *B, *A, *C;             // [slot][36]: the level's diagonal, lower and upper couplings
  double *Li, *Ri, *Bi;          // [slot][36] at odd positions and the top: B^-1 A, B^-1 C and B^-1
  double *d, *y, *xl;            // [slot][6]: right-hand side, B^-1 d at odd positions, solution
};

__device__ Work MakeWork(double* w, int K) {
  const size_t n = 6 * static_cast<size_t>(K), slots = 2 * static_cast<size_t>(K) + 32;
  Work v;
  v.x = w;
  v.r = w + n;
  v.p = w + 2 * n;
  v.q = w + 3 * n;
  double* c = w + 5 * n;
  v.B = c;
  v.A = c + 36 * slots;
  v.C = c + 72 * slots;
  v.Li = c + 108 * slots;
  v.Ri = c + 144 * slots;
  v.Bi = c + 180 * slots;
  v.d = c + 216 * slots;
  v.y = c + 222 * slots;
  v.xl = c + 228 * slots;
  return v;
}

__device__ void Upper6(const double* M, double u[21]) {
  int idx = 0;
  for (int r = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c) u[idx++] = M[r * 6 + c];
}

// x = A^-1 b for a symmetric 6x6 pivot block (upper triangle, packed) with SolveLDLT's convention -- fp64, symmetric pivoting on the
// largest remaining diagonal entry, a direction without information gets x = 0 -- except that a pivot at most 1e-12 of A's largest
// diagonal entry counts as zero.  In the reduction a direction without information (a constraint with information on translation
// only) leaves a Schur complement of rounding noise, not an exact zero, and dividing by that noise would not give 0.  Out of line:
// the solve kernel calls it from several phases, and inlined copies would spill.
__device__ __noinline__ void Solve6(const double* upper, const double* b, double* x) {
  double M[36];
  int perm[6];
  double scale = 0.0;
  int idx = 0;
  for (int r = 0; r < 6; ++r) {
    perm[r] = r;
    for (int c = r; c < 6; ++c) {
      M[r * 6 + c] = M[c * 6 + r] = upper[idx++];
      if (c == r) scale = fmax(scale, fabs(upper[idx - 1]));
    }
  }
  const double tol = 1e-12 * scale;
  bool zero[6];
  for (int k = 0; k < 6; ++k) {
    int p = k;
    double best = fabs(M[k * 6 + k]);
    for (int i = k + 1; i < 6; ++i) {
      const double v = fabs(M[i * 6 + i]);
      if (v > best) { best = v; p = i; }
    }
    if (p != k) {
      for (int c = 0; c < 6; ++c) { const double t = M[k * 6 + c]; M[k * 6 + c] = M[p * 6 + c]; M[p * 6 + c] = t; }
      for (int r = 0; r < 6; ++r) { const double t = M[r * 6 + k]; M[r * 6 + k] = M[r * 6 + p]; M[r * 6 + p] = t; }
      const int t = perm[k]; perm[k] = perm[p]; perm[p] = t;
    }
    const double d = M[k * 6 + k];
    zero[k] = !(d > tol);
    if (zero[k]) {
      for (int i = k + 1; i < 6; ++i) M[i * 6 + k] = 0.0;
      continue;
    }
    for (int i = k + 1; i < 6; ++i) M[i * 6 + k] /= d;
    for (int i = k + 1; i < 6; ++i)
      for (int j = k + 1; j <= i; ++j) {
        M[i * 6 + j] -= M[i * 6 + k] * d * M[j * 6 + k];
        M[j * 6 + i] = M[i * 6 + j];
      }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) y[i] = b[perm[i]];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < i; ++j) y[i] -= M[i * 6 + j] * y[j];
  for (int i = 0; i < 6; ++i) y[i] = zero[i] ? 0.0 : y[i] / M[i * 6 + i];
  for (int i = 5; i >= 0; --i)
    for (int j = i + 1; j < 6; ++j) y[i] -= M[j * 6 + i] * y[j];
  for (int i = 0; i < 6; ++i) x[perm[i]] = y[i];
}

// The size and first slot of level l of the reduction over K blocks.
__device__ void Level(int K, int l, int* n, int* off) {
  int m = K, o = 0;
  for (int i = 0; i < l; ++i) {
    o += m;
    m = (m + 1) / 2;
  }
  *n = m;
  *off = o;
}

// out (+)= s * A v for a 6x6 row-major A.
__device__ void MulVec6(const double* A, const double* v, double s, double* out) {
  for (int r = 0; r < 6; ++r) {
    double t = 0.0;
    for (int c = 0; c < 6; ++c) t += A[r * 6 + c] * v[c];
    out[r] += s * t;
  }
}

// out = base - X Y (6x6 row-major; base may be null for 0).
__device__ void MulSub6(const double* base, const double* X, const double* Y, double* out) {
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) {
      double t = base ? base[r * 6 + c] : 0.0;
      for (int k = 0; k < 6; ++k) t -= X[r * 6 + k] * Y[k * 6 + c];
      out[r * 6 + c] = t;
    }
}

// The sum of v over the CTA, in a fixed order (every thread gets it).
__device__ double BlockSum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kSolveThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const double total = sh[0];
  __syncthreads();
  return total;
}

__device__ double BlockMax(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kSolveThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] = fmax(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  const double m = sh[0];
  __syncthreads();
  return m;
}

// a . b over n doubles: each thread sums its strided elements in order, then the fixed tree.
__device__ double Dot(const double* a, const double* b, int n, double* sh) {
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kSolveThreads) s += a[i] * b[i];
  return BlockSum(s, sh);
}

__global__ void __launch_bounds__(64) PoseGraphLinearizeKernel(const PoseGraphArgs a) {
  if (a.state->done) return;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.term_count) return;
  const PoseGraphTerm& term = a.terms[t];
  PoseGraphTermBlocks& blk = a.blocks[t];
  if (term.b < 0) {
    PosePriorTerms(term.z, a.poses + 7 * term.a, term.info, blk.H, blk.b, &blk.cost);
  } else {
    double r[6];
    PoseConstraintTerms(term.z, a.poses + 7 * term.a, a.poses + 7 * term.b, term.info, r, blk.H, blk.b, &blk.cost);
  }
}

__global__ void __launch_bounds__(128) PoseGraphAssembleKernel(const PoseGraphArgs a) {
  if (a.state->done) return;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.K) return;
  double* D = a.csr_val + 36 * static_cast<size_t>(a.csr_off[k]);
  double* U = a.tri + 36 * static_cast<size_t>(k);
  double* bk = a.rhs + 6 * static_cast<size_t>(k);
  for (int i = 0; i < 36; ++i) {
    D[i] = 0.0;
    U[i] = 0.0;
  }
  for (int i = 0; i < 6; ++i) bk[i] = 0.0;
  const int first = a.csr_off[k] + 1, last = a.csr_off[k + 1];
  if (a.held[k]) {
    for (int i = 0; i < 6; ++i) D[i * 7] = 1.0;
    for (int e = first; e < last; ++e)
      for (int i = 0; i < 36; ++i) a.csr_val[36 * static_cast<size_t>(e) + i] = 0.0;
    return;
  }
  int e = first;
  for (int j = a.row_off[k]; j < a.row_off[k + 1]; ++j) {
    const int t = a.row_terms[2 * j], side = a.row_terms[2 * j + 1];
    const PoseGraphTerm& term = a.terms[t];
    const PoseGraphTermBlocks& blk = a.blocks[t];
    if (term.b < 0) {
      int idx = 0;
      for (int r = 0; r < 6; ++r) {
        bk[r] += blk.b[r];
        for (int c = r; c < 6; ++c, ++idx) {
          D[r * 6 + c] += blk.H[idx];
          if (c != r) D[c * 6 + r] += blk.H[idx];
        }
      }
      continue;
    }
    // the 12x12 upper triangle over (delta_a, delta_b)
    auto h12 = [&](int r, int c) { return blk.H[r * 12 - r * (r - 1) / 2 + (c - r)]; };
    const int o = side ? 6 : 0, other = side ? term.a : term.b;
    for (int r = 0; r < 6; ++r) {
      bk[r] += blk.b[o + r];
      for (int c = r; c < 6; ++c) {
        const double v = h12(o + r, o + c);
        D[r * 6 + c] += v;
        if (c != r) D[c * 6 + r] += v;
      }
    }
    double* X = a.csr_val + 36 * static_cast<size_t>(e++);
    const bool coupled = !a.held[other];
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 6; ++c) {
        const double v = coupled ? (side ? h12(c, 6 + r) : h12(r, 6 + c)) : 0.0;   // H_kb = H_ab (side a), H_ba = H_ab^T
        X[r * 6 + c] = v;
        if (other == k + 1) U[r * 6 + c] += v;
      }
  }
}

// w.xl (level 0: z) = M^-1 r by the reduction's forward and back sweeps over the factorisation of FactorPreconditioner: only
// 6x6 products, the pivots' LDLT ran once per factorisation.
__device__ void ApplyPreconditioner(const Work& w, int K, const double* r) {
  for (int i = threadIdx.x; i < 6 * K; i += kSolveThreads) w.d[i] = r[i];
  __syncthreads();
  int levels = 0;
  int n = K, off = 0;
  while (n > 1) {
    const int noff = off + n, nn = (n + 1) / 2;
    ++levels;
    for (int j = 2 * threadIdx.x + 1; j < n; j += 2 * kSolveThreads) {
      const size_t s = off + j;
      double v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      MulVec6(w.Bi + 36 * s, w.d + 6 * s, 1.0, v);
      for (int c = 0; c < 6; ++c) w.y[6 * s + c] = v[c];
    }
    __syncthreads();
    for (int q = threadIdx.x; q < nn; q += kSolveThreads) {
      const int i = 2 * q;
      const size_t s = off + i;
      double v[6];
      for (int c = 0; c < 6; ++c) v[c] = w.d[6 * s + c];
      if (i >= 1) MulVec6(w.A + 36 * s, w.y + 6 * (s - 1), -1.0, v);
      if (i + 1 < n) MulVec6(w.C + 36 * s, w.y + 6 * (s + 1), -1.0, v);
      for (int c = 0; c < 6; ++c) w.d[6 * static_cast<size_t>(noff + q) + c] = v[c];
    }
    __syncthreads();
    off = noff;
    n = nn;
  }
  if (threadIdx.x < 6) {   // the top level: one block
    const size_t s = off;
    double t = 0.0;
    for (int c = 0; c < 6; ++c) t += w.Bi[36 * s + threadIdx.x * 6 + c] * w.d[6 * s + c];
    w.xl[6 * s + threadIdx.x] = t;
  }
  __syncthreads();
  for (int l = levels - 1; l >= 0; --l) {   // back sweep: even positions take the next level's solution, odd ones solve for theirs
    int m, o;
    Level(K, l, &m, &o);
    const int no = o + m;
    for (int p = threadIdx.x; p < m; p += kSolveThreads) {
      const size_t s = o + p;
      double v[6];
      if ((p & 1) == 0) {
        for (int c = 0; c < 6; ++c) v[c] = w.xl[6 * static_cast<size_t>(no + p / 2) + c];
      } else {
        for (int c = 0; c < 6; ++c) v[c] = w.y[6 * s + c];
        MulVec6(w.Li + 36 * s, w.xl + 6 * static_cast<size_t>(no + (p - 1) / 2), -1.0, v);
        if (p + 1 < m) MulVec6(w.Ri + 36 * s, w.xl + 6 * static_cast<size_t>(no + (p + 1) / 2), -1.0, v);
      }
      for (int c = 0; c < 6; ++c) w.xl[6 * s + c] = v[c];
    }
    __syncthreads();
  }
}

// Factorises M, the block-tridiagonal part of H, by odd-even reduction: level 0 is (H_kk, H_{k,k-1}, H_{k,k+1}); at every level the
// odd positions j get B_j^-1 A_j, B_j^-1 C_j and B_j^-1 (Solve6 on their columns), and the even positions form the next level's
// blocks (no fill on a chain); the top block gets its B^-1.
__device__ void FactorPreconditioner(const PoseGraphArgs& a, const Work& w) {
  const int K = a.K;
  for (int k = threadIdx.x; k < K; k += kSolveThreads) {
    const double* D = a.csr_val + 36 * static_cast<size_t>(a.csr_off[k]);
    for (int i = 0; i < 36; ++i) {
      w.B[36 * static_cast<size_t>(k) + i] = D[i];
      w.C[36 * static_cast<size_t>(k) + i] = k + 1 < K ? a.tri[36 * static_cast<size_t>(k) + i] : 0.0;
      // H_{k,k-1} = H_{k-1,k}^T
      w.A[36 * static_cast<size_t>(k) + i] = k > 0 ? a.tri[36 * static_cast<size_t>(k - 1) + (i % 6) * 6 + i / 6] : 0.0;
    }
  }
  __syncthreads();
  int n = K, off = 0;
  while (n > 1) {
    const int noff = off + n, nn = (n + 1) / 2, tasks = 18 * (n / 2);
    for (int t = threadIdx.x; t < tasks; t += kSolveThreads) {   // B^-1 A, B^-1 C and B^-1, column by column
      const size_t j = off + 2 * (t / 18) + 1;
      const int col = t % 18, m = col / 6, c = col % 6;
      double u[21], rhs[6], x[6];
      Upper6(w.B + 36 * j, u);
      for (int r = 0; r < 6; ++r) rhs[r] = m == 0 ? w.A[36 * j + r * 6 + c] : m == 1 ? w.C[36 * j + r * 6 + c] : (r == c ? 1.0 : 0.0);
      Solve6(u, rhs, x);
      double* dst = (m == 0 ? w.Li : m == 1 ? w.Ri : w.Bi) + 36 * j;
      for (int r = 0; r < 6; ++r) dst[r * 6 + c] = x[r];
    }
    __syncthreads();
    for (int q = threadIdx.x; q < nn; q += kSolveThreads) {
      const int i = 2 * q;
      const size_t s = off + i, ns = noff + q;
      double Bn[36];
      for (int c = 0; c < 36; ++c) Bn[c] = w.B[36 * s + c];
      if (i >= 1) {
        MulSub6(Bn, w.A + 36 * s, w.Ri + 36 * (s - 1), Bn);
        MulSub6(nullptr, w.A + 36 * s, w.Li + 36 * (s - 1), w.A + 36 * ns);
      } else {
        for (int c = 0; c < 36; ++c) w.A[36 * ns + c] = 0.0;
      }
      if (i + 1 < n) {
        MulSub6(Bn, w.C + 36 * s, w.Li + 36 * (s + 1), Bn);
        MulSub6(nullptr, w.C + 36 * s, w.Ri + 36 * (s + 1), w.C + 36 * ns);
      } else {
        for (int c = 0; c < 36; ++c) w.C[36 * ns + c] = 0.0;
      }
      for (int c = 0; c < 36; ++c) w.B[36 * ns + c] = Bn[c];
    }
    __syncthreads();
    off = noff;
    n = nn;
  }
  if (threadIdx.x < 6) {   // the top level's B^-1
    double u[21], rhs[6], x[6];
    Upper6(w.B + 36 * static_cast<size_t>(off), u);
    for (int r = 0; r < 6; ++r) rhs[r] = r == static_cast<int>(threadIdx.x) ? 1.0 : 0.0;
    Solve6(u, rhs, x);
    for (int r = 0; r < 6; ++r) w.Bi[36 * static_cast<size_t>(off) + r * 6 + threadIdx.x] = x[r];
  }
  __syncthreads();
}

// H p, gathered per row over its block-CSR entries in order.
__device__ void MultiplyH(const PoseGraphArgs& a, const double* p, double* q) {
  for (int k = threadIdx.x; k < a.K; k += kSolveThreads) {
    double v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    MulVec6(a.csr_val + 36 * static_cast<size_t>(a.csr_off[k]), p + 6 * static_cast<size_t>(k), 1.0, v);
    for (int e = a.csr_off[k] + 1; e < a.csr_off[k + 1]; ++e)
      MulVec6(a.csr_val + 36 * static_cast<size_t>(e), p + 6 * static_cast<size_t>(a.csr_col[e]), 1.0, v);
    for (int c = 0; c < 6; ++c) q[6 * static_cast<size_t>(k) + c] = v[c];
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kSolveThreads) PoseGraphSolveKernel(const PoseGraphArgs a) {
  __shared__ double sh[kSolveThreads];
  __shared__ int skip;
  __shared__ double accepted;
  if (threadIdx.x == 0) {
    skip = a.state->done;
    accepted = a.state->cost;
  }
  __syncthreads();
  if (skip) return;
  // the cost at the current poses, and the test of the last step
  double c = 0.0;
  for (int t = threadIdx.x; t < a.term_count; t += kSolveThreads) c += a.blocks[t].cost;
  const double cost = BlockSum(c, sh);
  if (a.round > 0 && !(cost <= accepted)) {   // the step raised the cost (or made it NaN): revert it and stop
    for (int i = threadIdx.x; i < 7 * a.K; i += kSolveThreads) a.poses[i] = a.prev[i];
    if (threadIdx.x == 0) a.state->done = 1;
    return;
  }
  if (threadIdx.x == 0) {
    if (a.round == 0) a.state->initial_cost = cost;
    a.state->cost = cost;
    if (a.round >= a.max_iterations) a.state->done = 1;
  }
  if (a.round >= a.max_iterations) return;

  const Work w = MakeWork(a.work, a.K);
  const int n = 6 * a.K;
  FactorPreconditioner(a, w);
  double* z = w.xl;   // level 0 of the reduction's solution
  for (int i = threadIdx.x; i < n; i += kSolveThreads) {
    w.x[i] = 0.0;
    w.r[i] = -a.rhs[i];
  }
  __syncthreads();
  const double bb = Dot(w.r, w.r, n, sh);
  int its = 0;
  if (bb > 0.0) {
    ApplyPreconditioner(w, a.K, w.r);
    double rz = Dot(w.r, z, n, sh);
    for (int i = threadIdx.x; i < n; i += kSolveThreads) w.p[i] = z[i];
    __syncthreads();
    while (its < a.max_linear) {
      MultiplyH(a, w.p, w.q);
      const double pq = Dot(w.p, w.q, n, sh);
      if (!(pq > 0.0)) break;
      const double alpha = rz / pq;
      double rr = 0.0;
      for (int i = threadIdx.x; i < n; i += kSolveThreads) {
        w.x[i] += alpha * w.p[i];
        w.r[i] -= alpha * w.q[i];
        rr += w.r[i] * w.r[i];
      }
      rr = BlockSum(rr, sh);
      ++its;
      if (rr <= kRelativeResidual * kRelativeResidual * bb) break;
      ApplyPreconditioner(w, a.K, w.r);
      const double rz_next = Dot(w.r, z, n, sh);
      const double beta = rz_next / rz;
      rz = rz_next;
      for (int i = threadIdx.x; i < n; i += kSolveThreads) w.p[i] = z[i] + beta * w.p[i];
      __syncthreads();
    }
  }
  // the step's largest component against its pose's fp32 resolution: 1e-7, or 2^-19 of the pose's scale (1 for a rotation,
  // max(1, |t|_inf) for a translation) when that is larger.  A smaller step is the rounding noise of the fp32 poses and of their
  // fp32 update (a few ulps each): applied, it raises the cost as often as it lowers it.
  double m = 0.0;
  for (int i = threadIdx.x; i < n; i += kSolveThreads) {
    double scale = 1.0;
    if (i % 6 < 3) {
      const float* t = a.poses + 7 * (i / 6) + 4;
      scale = fmax(1.0, fmax(fabs(t[0]), fmax(fabs(t[1]), fabs(t[2]))));
    }
    m = fmax(m, fabs(w.x[i]) / fmax(kConvergedStep, kPoseResolution * scale));
  }
  m = BlockMax(m, sh);
  if (threadIdx.x == 0) {
    ++a.state->iterations;
    a.state->linear_iterations += its;
    if (m <= 1.0) {   // converged: the step is not applied
      a.state->converged = 1;
      a.state->done = 1;
    }
  }
}

__global__ void __launch_bounds__(128) PoseGraphUpdateKernel(const PoseGraphArgs a) {
  if (a.state->done) return;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.K || a.held[k]) return;
  float* pe = a.poses + 7 * k;
  float* pv = a.prev + 7 * k;
  const double* x = a.work + 6 * static_cast<size_t>(k);   // Work::x
  float d[6];
  for (int i = 0; i < 6; ++i) d[i] = static_cast<float>(x[i]);
  for (int i = 0; i < 7; ++i) pv[i] = pe[i];
  Pose T;
  T.q[0] = pe[0]; T.q[1] = pe[1]; T.q[2] = pe[2]; T.q[3] = pe[3];
  T.t[0] = pe[4]; T.t[1] = pe[5]; T.t[2] = pe[6];
  T = Compose(T, Exp(d));
  pe[0] = T.q[0]; pe[1] = T.q[1]; pe[2] = T.q[2]; pe[3] = T.q[3];
  pe[4] = T.t[0]; pe[5] = T.t[1]; pe[6] = T.t[2];
}

}  // namespace

LaunchResult LaunchPoseGraphRound(const PoseGraphArgs& a, cudaStream_t stream) {
  PoseGraphLinearizeKernel<<<(a.term_count + 63) / 64 > 0 ? (a.term_count + 63) / 64 : 1, 64, 0, stream>>>(a);
  PoseGraphAssembleKernel<<<(a.K + 127) / 128, 128, 0, stream>>>(a);
  PoseGraphSolveKernel<<<1, kSolveThreads, 0, stream>>>(a);
  if (a.round >= a.max_iterations) return {3};
  PoseGraphUpdateKernel<<<(a.K + 127) / 128, 128, 0, stream>>>(a);
  return {4};
}

}  // namespace bba
