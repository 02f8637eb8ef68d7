// pose_terms.cu -- the soft keyframe pose terms of libbadba_b200 (host side): the pose priors, attitude priors and relative pose
// constraints with their robust losses and entry points, their staging for the pose step (PoseSolveKernel) and the PCG products
// (LaunchPcgPoseTerms), and the keyframe pose graph (bba_optimize_pose_graph, bba_evaluate_keyframe_pose_terms, DESIGN §3.14).
#include <cmath>
#include <cstring>

#include "handle.hpp"

namespace bba {
namespace {

// Counts the priors and publishes the records.
bba_status CommitPosePriors(bba_handle h) {
  int count = 0;
  for (const PosePrior& p : h->pose_priors) count += p.has ? 1 : 0;
  h->pose_prior_count = count;
  return Publish(h, nullptr, false);
}

// The test of a robust loss a caller passes: a known type, and for HUBER / CAUCHY a finite scale > 0.
bool RobustLossValid(const bba_robust_loss& l) {
  if (l.type == BBA_LOSS_TRIVIAL) return true;
  return (l.type == BBA_LOSS_HUBER || l.type == BBA_LOSS_CAUCHY) && std::isfinite(l.scale) && l.scale > 0.f;
}

bool PoseRecordFinite(const float* pose, const float* info) {
  bool finite = true;
  for (int j = 0; j < 7; ++j) finite = finite && std::isfinite(pose[j]);
  for (int j = 0; j < 21; ++j) finite = finite && std::isfinite(info[j]);
  return finite;
}

// Reserves the staging buffers of the soft pose terms (pose step and PCG) for a prior on every keyframe and `constraints`
// constraints, with room to double the constraints before the next allocation, and with `attitude` for an attitude prior on every
// keyframe too.  The calls that add priors or constraints make it before they change anything; the staging repeats it, a no-op
// unless an earlier reservation failed.
bba_status ReservePoseTerms(bba_handle h, size_t constraints, bool attitude) {
  // pose step: a prior per keyframe, and per constraint an equivalent prior and a damping anchor at each end, the attitude priors
  // apart; PCG: a prior and an attitude prior per pose block and one term at each end of a constraint
  const size_t M = static_cast<size_t>(h->cfg.max_keyframes), grow = 2 * constraints;
  auto& p = h->pose;
  if (attitude) {
    BBA_CUDA(h, p.h_attitude.Reserve(M));
    BBA_CUDA(h, p.d_attitude.Reserve(M));
  }
  const size_t unary = attitude ? 2 * M : M;
  BBA_CUDA(h, p.h_term_offsets.Reserve(M + 1));
  BBA_CUDA(h, p.d_term_offsets.Reserve(M + 1));
  BBA_CUDA(h, p.h_terms.Reserve(M + 4 * constraints, M + 4 * grow));
  BBA_CUDA(h, p.d_terms.Reserve(M + 4 * constraints, M + 4 * grow));
  auto& pc = h->pcg;
  BBA_CUDA(h, pc.h_pose_blocks.Reserve(M));
  BBA_CUDA(h, pc.d_pose_blocks.Reserve(M));
  BBA_CUDA(h, pc.h_pose_terms.Reserve(unary + 2 * constraints, unary + 2 * grow));
  BBA_CUDA(h, pc.d_pose_terms.Reserve(unary + 2 * constraints, unary + 2 * grow));
  return BBA_OK;
}

bool HasAttitude(bba_handle h) { return h->attitude_prior_count > 0; }

// Counts the attitude priors and publishes the records.
bba_status CommitAttitudePriors(bba_handle h) {
  int count = 0;
  for (const AttitudePrior& p : h->attitude_priors) count += p.has ? 1 : 0;
  h->attitude_prior_count = count;
  return Publish(h, nullptr, false);
}

// An attitude prior's terms at global_T_frame = pose (AttitudePriorTerms), scaled by the robust weight of its loss there.
void WeightedAttitudeTerms(const AttitudePrior& a, const float pose[7], double H[21], double b[6]) {
  double cost, rho, w;
  AttitudePriorTerms(a.p.reference_direction, a.p.measured_direction, a.p.information, pose, H, b, &cost);
  RobustLoss(a.p.loss.type, a.p.loss.scale, 2.0 * cost, &rho, &w);
  for (int i = 0; i < 21; ++i) H[i] *= w;
  for (int i = 0; i < 6; ++i) b[i] *= w;
}

// The soft relative pose constraints that touch each of the first K keyframes, in id order: indices into h->pose_constraints,
// adj[off[k] .. off[k + 1]).
void ConstraintAdjacency(bba_handle h, int K, std::vector<int>* off, std::vector<int>* adj) {
  const std::vector<PoseConstraint>& cons = h->pose_constraints;
  off->assign(K + 1, 0);
  for (const PoseConstraint& c : cons) {
    ++(*off)[c.c.keyframe_a + 1];
    ++(*off)[c.c.keyframe_b + 1];
  }
  for (int k = 0; k < K; ++k) (*off)[k + 1] += (*off)[k];
  adj->resize(2 * cons.size());
  std::vector<int> fill(off->begin(), off->end() - 1);
  for (size_t i = 0; i < cons.size(); ++i) {   // in id order: cons is sorted by id
    (*adj)[fill[cons[i].c.keyframe_a]++] = static_cast<int>(i);
    (*adj)[fill[cons[i].c.keyframe_b]++] = static_cast<int>(i);
  }
}

// The terms of constraint c at global_T_frame = pa, pb (PoseConstraintTerms: H's 12 x 12 upper triangle and b over (delta_a,
// delta_b)), scaled by the robust weight of its loss there (w = 1 exactly for a trivial loss).  fp64.
void WeightedConstraintTerms(const PoseConstraint& c, const float pa[7], const float pb[7], double H[78], double b[12]) {
  double r[6], cost, rho, w;
  PoseConstraintTerms(c.c.a_T_b, pa, pb, c.c.information, r, H, b, &cost);
  RobustLoss(c.loss.type, c.loss.scale, 2.0 * cost, &rho, &w);
  for (int i = 0; i < 78; ++i) H[i] *= w;
  for (int i = 0; i < 12; ++i) b[i] *= w;
}

// ---- keyframe pose graph (bba_optimize_pose_graph, DESIGN §3.14) ----
// What the pose graph stages for K keyframes and C constraints: terms (a prior and an attitude prior per keyframe, the
// constraints, the chain), ints (held flags, row offsets, two ints per row entry, CSR offsets and columns) and doubles (the terms'
// blocks, the CSR blocks, b, the couplings and the solver's work).  A row holds its priors and one entry per end of a constraint or
// chain edge.
struct PoseGraphSizes {
  size_t terms, ints, doubles;
};
PoseGraphSizes PoseGraphCapacity(size_t K, size_t C) {
  const size_t terms = 3 * K + C, entries = 4 * K + 2 * C, nnz = 3 * K + 2 * C;
  const size_t block_doubles = sizeof(PoseGraphTermBlocks) / sizeof(double);
  return {terms, K + 2 * (K + 1) + 2 * entries + nnz, terms * block_doubles + 36 * nnz + 42 * K + PoseGraphWorkDoubles(K)};
}

// Sizes the pose graph's buffers for max_keyframes and `constraints` constraints, with room to double the constraints.
bba_status ReservePoseGraph(bba_handle h, size_t constraints) {
  const size_t M = static_cast<size_t>(h->cfg.max_keyframes);
  const PoseGraphSizes need = PoseGraphCapacity(M, constraints), alloc = PoseGraphCapacity(M, 2 * constraints);
  auto& g = h->graph;
  BBA_CUDA(h, g.h_terms.Reserve(need.terms, alloc.terms));
  BBA_CUDA(h, g.d_terms.Reserve(need.terms, alloc.terms));
  BBA_CUDA(h, g.h_ints.Reserve(need.ints, alloc.ints));
  BBA_CUDA(h, g.d_ints.Reserve(need.ints, alloc.ints));
  BBA_CUDA(h, g.h_eval.Reserve(2 * need.terms, 2 * alloc.terms));
  BBA_CUDA(h, g.d_eval.Reserve(2 * need.terms, 2 * alloc.terms));
  BBA_CUDA(h, g.d_doubles.Reserve(need.doubles, alloc.doubles));
  BBA_CUDA(h, g.h_poses.Reserve(7 * M));
  BBA_CUDA(h, g.d_poses.Reserve(14 * M));
  BBA_CUDA(h, g.h_hold_axes.Reserve(3 * M));
  BBA_CUDA(h, g.d_hold_axes.Reserve(3 * M));
  BBA_CUDA(h, g.d_state.Reserve(1));
  BBA_CUDA(h, g.h_state.Reserve(1));
  return BBA_OK;
}

int FindRoot(std::vector<int>& parent, int k) {
  while (parent[k] != k) k = parent[k] = parent[parent[k]];
  return k;
}

// Where StagePoseGraphTerms put the terms: keyframe k's prior and attitude prior (or -1), the first constraint and chain edge.
struct PoseGraphLayout {
  std::vector<int> prior_term, attitude_term;
  int first_constraint = 0, first_chain = 0;
};

// The pose graph's terms in h->graph.h_terms at the keyframe poses `poses`: the priors, the attitude priors, the constraints by
// id, then with odometry_information the odometry chain, whose Z are taken at `poses` and whose losses are TRIVIAL.  Returns the
// number of terms.
int StagePoseGraphTerms(bba_handle h, const float* poses, const float* odometry_information, PoseGraphLayout* layout) {
  auto& g = h->graph;
  const int K = static_cast<int>(h->keyframes.size());
  layout->prior_term.assign(K, -1);
  layout->attitude_term.assign(K, -1);
  int T = 0;
  auto add = [&](int a, int b, const float* z, const float* info, const bba_robust_loss& loss) {
    PoseGraphTerm& t = g.h_terms[T++];
    t.a = a;
    t.b = b;
    std::memcpy(t.z, z, sizeof(t.z));
    std::memcpy(t.info, info, sizeof(t.info));
    t.loss = loss;
  };
  for (int k = 0; k < K; ++k) {
    const PosePrior& p = h->pose_priors[k];
    if (!p.has) continue;
    layout->prior_term[k] = T;
    add(k, -1, p.pose, p.info, p.loss);
  }
  for (int k = 0; k < K && HasAttitude(h); ++k) {
    const AttitudePrior& p = h->attitude_priors[k];
    if (!p.has) continue;
    layout->attitude_term[k] = T;
    float z[7] = {}, info[21] = {};
    std::memcpy(z, p.p.reference_direction, sizeof(float) * 3);
    std::memcpy(z + 3, p.p.measured_direction, sizeof(float) * 3);
    info[0] = p.p.information;
    add(k, kPoseGraphAttitude, z, info, p.p.loss);
  }
  layout->first_constraint = T;
  for (const PoseConstraint& c : h->pose_constraints) add(c.c.keyframe_a, c.c.keyframe_b, c.c.a_T_b, c.c.information, c.loss);
  layout->first_chain = T;
  if (odometry_information)
    for (int k = 0; k + 1 < K; ++k) {
      double qa[4], ta[3], qb[4], tb[3], q[4], t[3];
      LoadPoseD(poses + 7 * k, qa, ta);
      LoadPoseD(poses + 7 * (k + 1), qb, tb);
      Se3BetweenD(qa, ta, qb, tb, q, t);   // T_k^-1 T_{k+1}
      float z[7];
      for (int j = 0; j < 4; ++j) z[j] = static_cast<float>(q[j]);
      for (int j = 0; j < 3; ++j) z[4 + j] = static_cast<float>(t[j]);
      add(k, k + 1, z, odometry_information, bba_robust_loss{BBA_LOSS_TRIVIAL, 0.f});
    }
  return T;
}

bba_status OptimizePoseGraph(bba_handle h, const bba_pose_graph_options* o, bba_pose_graph_result* result, cudaStream_t s) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_optimize_pose_graph: ";
  if (!o) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null options");
  const int K = static_cast<int>(h->keyframes.size());
  const int gauge = o->gauge_keyframe;
  if (gauge < -1 || gauge >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "gauge_keyframe out of range");
  if (o->use_odometry_chain) {
    for (int j = 0; j < 21; ++j)
      if (!std::isfinite(o->odometry_information[j])) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "non-finite odometry_information");
    if (!InformationPsd(o->odometry_information))
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "odometry_information is not positive semi-definite");
  }
  bba_pose_graph_result r{};
  if (result) *result = r;
  if (K < 2 && h->pose_prior_count == 0 && !HasAttitude(h)) return BBA_OK;
  const std::vector<PoseConstraint>& cons = h->pose_constraints;
  if (bba_status st = ReservePoseGraph(h, cons.size())) return st;
  auto& g = h->graph;
  const bool chain = o->use_odometry_chain != 0;
  const int max_iterations = o->max_iterations > 0 ? o->max_iterations : 20;   // pose_graph_optimizer.cc kMaxIterations

  // the terms: priors, constraints by id, then the chain at the poses the call starts from
  float* poses = g.h_poses;
  for (int k = 0; k < K; ++k) PoseToArray(h->keyframes[k].pose, poses + 7 * k);
  PoseGraphLayout layout;
  const int T = StagePoseGraphTerms(h, poses, chain ? o->odometry_information : nullptr, &layout);
  const std::vector<int>& prior_term = layout.prior_term;
  const std::vector<int>& attitude_term = layout.attitude_term;
  const int first_constraint = layout.first_constraint, first_chain = layout.first_chain;

  // the held keyframes: the gauge, the untouched ones, and the lowest id of every component without the gauge or a prior.  In
  // such a component with attitude priors the lowest id is held only in translation and, when the component's reference
  // directions are parallel, in rotation about them (held = 2, DESIGN §3.17): the priors fix the component's tilt, and holding
  // that keyframe's tilt too would bias every other keyframe toward it.
  std::vector<int> parent(K), lowest(K, -1), axis_of(K, -1);
  std::vector<char> touched(K, 0), anchored(K, 0), parallel(K, 1);
  for (int k = 0; k < K; ++k) parent[k] = k;
  for (int i = first_constraint; i < T; ++i) {
    const PoseGraphTerm& t = g.h_terms[i];
    touched[t.a] = touched[t.b] = 1;
    const int ra = FindRoot(parent, t.a), rb = FindRoot(parent, t.b);
    if (ra != rb) parent[std::max(ra, rb)] = std::min(ra, rb);
  }
  for (int k = 0; k < K; ++k) {
    const int root = FindRoot(parent, k);
    if (lowest[root] < 0) lowest[root] = k;
    if (prior_term[k] >= 0 || attitude_term[k] >= 0) touched[k] = 1;
    if (prior_term[k] >= 0 || k == gauge) anchored[root] = 1;
    if (attitude_term[k] < 0) continue;
    const float* d = h->attitude_priors[k].p.reference_direction;   // (unit)
    if (axis_of[root] < 0) {
      axis_of[root] = k;
    } else {
      const float* d0 = h->attitude_priors[axis_of[root]].p.reference_direction;
      const double cx = d[1] * d0[2] - d[2] * d0[1], cy = d[2] * d0[0] - d[0] * d0[2], cz = d[0] * d0[1] - d[1] * d0[0];
      if (cx * cx + cy * cy + cz * cz > 1e-12) parallel[root] = 0;
    }
  }
  int* held = g.h_ints;
  float* hold_axes = g.h_hold_axes;
  int held_count = 0, free_directions = 0;
  bool partial = false;
  for (int k = 0; k < K; ++k) {
    const int root = FindRoot(parent, k);
    const bool lowest_unanchored = !anchored[root] && lowest[root] == k;
    if (k == gauge || !touched[k] || (lowest_unanchored && axis_of[root] < 0)) {
      held[k] = 1;
      ++held_count;
    } else if (lowest_unanchored) {
      held[k] = 2;
      partial = true;
      for (int j = 0; j < 3; ++j) hold_axes[3 * k + j] = parallel[root] ? h->attitude_priors[axis_of[root]].p.reference_direction[j] : 0.f;
      free_directions += parallel[root] ? 2 : 3;
    } else {
      held[k] = 0;
      free_directions += 6;
    }
  }

  // row k: its prior, its constraints by id, the chain edges (k - 1, k) and (k, k + 1); the CSR row: the diagonal, then the other
  // end of every constraint and chain edge in the same order
  std::vector<int> off, adj;
  ConstraintAdjacency(h, K, &off, &adj);
  int* row_off = held + K;
  int entries = 0, nnz = 0;
  for (int k = 0; k < K; ++k) {
    row_off[k] = entries;
    const int binary = (off[k + 1] - off[k]) + (chain ? (k > 0) + (k + 1 < K) : 0);
    entries += (prior_term[k] >= 0) + (attitude_term[k] >= 0) + binary;
    nnz += 1 + binary;
  }
  row_off[K] = entries;
  int* row_terms = row_off + K + 1;
  int* csr_off = row_terms + 2 * entries;
  int* csr_col = csr_off + K + 1;
  int e = 0, c = 0;
  auto entry = [&](int term, int side, int col) {
    row_terms[2 * e] = term;
    row_terms[2 * e + 1] = side;
    ++e;
    if (col >= 0) csr_col[c++] = col;
  };
  for (int k = 0; k < K; ++k) {
    csr_off[k] = c;
    csr_col[c++] = k;
    if (prior_term[k] >= 0) entry(prior_term[k], 0, -1);
    if (attitude_term[k] >= 0) entry(attitude_term[k], 0, -1);
    for (int j = off[k]; j < off[k + 1]; ++j) {
      const bba_pose_constraint& pc = cons[adj[j]].c;
      const bool is_a = pc.keyframe_a == k;
      entry(first_constraint + adj[j], is_a ? 0 : 1, is_a ? pc.keyframe_b : pc.keyframe_a);
    }
    if (chain && k > 0) entry(first_chain + k - 1, 1, k - 1);
    if (chain && k + 1 < K) entry(first_chain + k, 0, k + 1);
  }
  csr_off[K] = c;
  const size_t ints = static_cast<size_t>(csr_col + nnz - held);

  const size_t M = static_cast<size_t>(h->cfg.max_keyframes);
  if (T) BBA_CUDA(h, cudaMemcpyAsync(g.d_terms, g.h_terms, sizeof(PoseGraphTerm) * T, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemcpyAsync(g.d_ints, g.h_ints, sizeof(int) * ints, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemcpyAsync(g.d_poses, poses, sizeof(float) * 7 * K, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemcpyAsync(g.d_poses + 7 * M, poses, sizeof(float) * 7 * K, cudaMemcpyHostToDevice, s));
  if (partial) BBA_CUDA(h, cudaMemcpyAsync(g.d_hold_axes, hold_axes, sizeof(float) * 3 * K, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemsetAsync(g.d_state, 0, sizeof(PoseGraphState), s));
  PoseGraphArgs a{};
  a.K = K;
  a.term_count = T;
  a.terms = g.d_terms;
  a.blocks = reinterpret_cast<PoseGraphTermBlocks*>(g.d_doubles.get());
  a.poses = g.d_poses;
  a.prev = g.d_poses + 7 * M;
  const int* d_ints = g.d_ints;
  a.held = d_ints;
  a.hold_axis = partial ? g.d_hold_axes.get() : nullptr;
  a.row_off = d_ints + (row_off - held);
  a.row_terms = d_ints + (row_terms - held);
  a.csr_off = d_ints + (csr_off - held);
  a.csr_col = d_ints + (csr_col - held);
  double* d = g.d_doubles.get() + static_cast<size_t>(T) * (sizeof(PoseGraphTermBlocks) / sizeof(double));
  a.csr_val = d;
  a.rhs = a.csr_val + 36 * static_cast<size_t>(nnz);
  a.tri = a.rhs + 6 * static_cast<size_t>(K);
  a.work = a.tri + 36 * static_cast<size_t>(K);
  a.state = g.d_state;
  a.max_iterations = max_iterations;
  a.max_linear = free_directions;   // 6 (K - held_count) without partial holds
  for (int round = 0; round <= max_iterations; ++round) {
    a.round = round;
    BBA_LAUNCH(h, h->launches, LaunchPoseGraphRound, a, s);
  }
  BBA_CUDA(h, cudaMemcpyAsync(g.h_state, g.d_state, sizeof(PoseGraphState), cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaMemcpyAsync(poses, g.d_poses, sizeof(float) * 7 * K, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  for (int k = 0; k < K; ++k)
    if (held[k] != 1) h->keyframes[k].pose = PoseFromArray(poses + 7 * k);
  const PoseGraphState& st = *g.h_state.get();
  r.iterations = st.iterations;
  r.converged = st.converged;
  r.linear_iterations = st.linear_iterations;
  r.held_keyframes = held_count;
  r.initial_cost = st.initial_cost;
  r.final_cost = st.cost;
  if (result) *result = r;
  return Publish(h, s, false);
}

// The pose graph's terms without the chain, linearised once at the current poses with a.eval set, which writes every term's
// {s, w} to h->graph.h_eval (bba_evaluate_keyframe_pose_terms, bba_evaluate_keyframe_attitude_priors).
bba_status EvaluateTerms(bba_handle h, PoseGraphLayout* layout, cudaStream_t s) {
  const int K = static_cast<int>(h->keyframes.size());
  if (bba_status st = ReservePoseGraph(h, h->pose_constraints.size())) return st;
  auto& g = h->graph;
  float* poses = g.h_poses;
  for (int k = 0; k < K; ++k) PoseToArray(h->keyframes[k].pose, poses + 7 * k);
  const int T = StagePoseGraphTerms(h, poses, nullptr, layout);
  if (T) {
    BBA_CUDA(h, cudaMemcpyAsync(g.d_terms, g.h_terms, sizeof(PoseGraphTerm) * T, cudaMemcpyHostToDevice, s));
    BBA_CUDA(h, cudaMemcpyAsync(g.d_poses, poses, sizeof(float) * 7 * K, cudaMemcpyHostToDevice, s));
    BBA_CUDA(h, cudaMemsetAsync(g.d_state, 0, sizeof(PoseGraphState), s));
    PoseGraphArgs a{};
    a.K = K;
    a.term_count = T;
    a.terms = g.d_terms;
    a.blocks = reinterpret_cast<PoseGraphTermBlocks*>(g.d_doubles.get());
    a.poses = g.d_poses;
    a.state = g.d_state;
    a.eval = g.d_eval;
    BBA_LAUNCH(h, h->launches, LaunchPoseGraphEvaluate, a, s);
    BBA_CUDA(h, cudaMemcpyAsync(g.h_eval, g.d_eval, sizeof(double) * 2 * T, cudaMemcpyDeviceToHost, s));
    BBA_CUDA(h, cudaStreamSynchronize(s));
  }
  return BBA_OK;
}

bba_status EvaluatePoseTerms(bba_handle h, int keyframe_capacity, double* prior_s, double* prior_weight, int constraint_capacity,
                             double* constraint_s, double* constraint_weight, cudaStream_t s) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (keyframe_capacity < 0 || constraint_capacity < 0)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_evaluate_keyframe_pose_terms: negative capacity");
  PoseGraphLayout layout;
  if (bba_status st = EvaluateTerms(h, &layout, s)) return st;
  const int K = static_cast<int>(h->keyframes.size());
  const std::vector<PoseConstraint>& cons = h->pose_constraints;
  const double* ev = h->graph.h_eval;
  for (int k = 0; k < std::min(keyframe_capacity, K); ++k) {
    const int t = layout.prior_term[k];
    if (prior_s) prior_s[k] = t >= 0 ? ev[2 * t] : std::nan("");
    if (prior_weight) prior_weight[k] = t >= 0 ? ev[2 * t + 1] : std::nan("");
  }
  for (int i = 0; i < std::min(constraint_capacity, static_cast<int>(cons.size())); ++i) {
    const int t = layout.first_constraint + i;
    if (constraint_s) constraint_s[i] = ev[2 * t];
    if (constraint_weight) constraint_weight[i] = ev[2 * t + 1];
  }
  return BBA_OK;
}

bba_status EvaluateAttitudePriors(bba_handle h, int keyframe_capacity, double* s_out, double* weight, cudaStream_t s) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (keyframe_capacity < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_evaluate_keyframe_attitude_priors: negative capacity");
  PoseGraphLayout layout;
  if (bba_status st = EvaluateTerms(h, &layout, s)) return st;
  const int K = static_cast<int>(h->keyframes.size());
  const double* ev = h->graph.h_eval;
  for (int k = 0; k < std::min(keyframe_capacity, K); ++k) {
    const int t = layout.attitude_term[k];
    if (s_out) s_out[k] = t >= 0 ? ev[2 * t] : std::nan("");
    if (weight) weight[k] = t >= 0 ? ev[2 * t + 1] : std::nan("");
  }
  return BBA_OK;
}

}  // namespace

// Keyframe k's list holds its prior, then for every constraint that touches it (in id order) the equivalent prior with the other
// end held at its start pose (T_b Z^-1 with the information of PoseConstraintInformationA, or T_a Z with L), then for every such
// constraint whose other end is in the step too a damping anchor, a prior at k's own start pose with the constraint's diagonal
// block for k at the start poses, scaled by the constraint's robust weight there, as its information (DESIGN.md 3.12, 3.15).  A
// term's loss is the prior's own, an equivalent prior's its constraint's, an anchor's TRIVIAL.  Every rank stages the same lists:
// they depend only on the start of the step.  The attitude priors go apart, as the per-keyframe array h->pose.d_attitude.
bba_status StagePoseTerms(bba_handle h, const std::vector<int>& ids, const std::vector<Pose>& init, cudaStream_t s, bool* staged,
                          bool* attitude) {
  auto& p = h->pose;
  *staged = *attitude = false;
  const int K = static_cast<int>(h->keyframes.size());
  if (HasAttitude(h)) {
    if (bba_status st = ReservePoseTerms(h, h->pose_constraints.size(), true)) return st;
    std::copy(h->attitude_priors.begin(), h->attitude_priors.begin() + K, p.h_attitude.get());
    BBA_CUDA(h, cudaMemcpyAsync(p.d_attitude, p.h_attitude, sizeof(AttitudePrior) * K, cudaMemcpyHostToDevice, s));
    *attitude = true;
  }
  if (h->pose_prior_count == 0 && h->pose_constraints.empty()) return BBA_OK;
  const std::vector<PoseConstraint>& cons = h->pose_constraints;
  if (bba_status st = ReservePoseTerms(h, cons.size(), HasAttitude(h))) return st;
  std::vector<int> pos(K, -1);   // index in ids
  for (size_t i = 0; i < ids.size(); ++i) pos[ids[i]] = static_cast<int>(i);
  auto start = [&](int k, float out[7]) { PoseToArray(pos[k] >= 0 ? init[pos[k]] : h->keyframes[k].pose, out); };
  std::vector<int> off, adj;
  ConstraintAdjacency(h, K, &off, &adj);
  // the anchors' information, once per constraint with both ends in the step: [a's diagonal block, b's] (upper triangles)
  std::vector<float> anchor_info;
  std::vector<int> anchor_of(cons.size(), -1);
  for (size_t i = 0; i < cons.size(); ++i) {
    const bba_pose_constraint& c = cons[i].c;
    if (pos[c.keyframe_a] < 0 || pos[c.keyframe_b] < 0) continue;
    float pa[7], pb[7];
    start(c.keyframe_a, pa);
    start(c.keyframe_b, pb);
    double H[78], b[12];
    WeightedConstraintTerms(cons[i], pa, pb, H, b);
    anchor_of[i] = static_cast<int>(anchor_info.size());
    for (int o = 0; o < 12; o += 6)   // the diagonal blocks in the 12 x 12 upper triangle
      for (int row = o; row < o + 6; ++row)
        for (int col = row; col < o + 6; ++col) anchor_info.push_back(static_cast<float>(H[Upper12(row, col)]));
  }
  int n = 0;
  for (int k = 0; k < K; ++k) {
    p.h_term_offsets[k] = n;
    if (pos[k] < 0) continue;
    const PosePrior& prior = h->pose_priors[k];
    if (prior.has) {
      PoseTerm& r = p.h_terms[n++];
      std::memcpy(r.pose, prior.pose, sizeof(r.pose));
      std::memcpy(r.info, prior.info, sizeof(r.info));
      r.loss = prior.loss;
    }
    for (int e = off[k]; e < off[k + 1]; ++e) {   // the equivalent priors
      const PoseConstraint& c = cons[adj[e]];
      const bool is_a = c.c.keyframe_a == k;
      float other[7];
      start(is_a ? c.c.keyframe_b : c.c.keyframe_a, other);
      double qz[4], tz[3], qo[4], to[3], q[4], t[3];
      LoadPoseD(c.c.a_T_b, qz, tz);
      LoadPoseD(other, qo, to);
      if (is_a) {   // T_b Z^-1
        double qi[4], ti[3];
        const double q_id[4] = {0.0, 0.0, 0.0, 1.0}, t_id[3] = {0.0, 0.0, 0.0};
        Se3BetweenD(qz, tz, q_id, t_id, qi, ti);
        Se3ComposeD(qo, to, qi, ti, q, t);
      } else {      // T_a Z
        Se3ComposeD(qo, to, qz, tz, q, t);
      }
      PoseTerm& r = p.h_terms[n++];
      for (int j = 0; j < 4; ++j) r.pose[j] = static_cast<float>(q[j]);
      for (int j = 0; j < 3; ++j) r.pose[4 + j] = static_cast<float>(t[j]);
      std::memcpy(r.info, is_a ? c.info_a : c.c.information, sizeof(r.info));
      r.loss = c.loss;
    }
    for (int e = off[k]; e < off[k + 1]; ++e) {   // the damping anchors
      const int a = anchor_of[adj[e]];
      if (a < 0) continue;
      PoseTerm& anchor = p.h_terms[n++];
      PoseToArray(init[pos[k]], anchor.pose);
      std::memcpy(anchor.info, anchor_info.data() + a + (cons[adj[e]].c.keyframe_a == k ? 0 : 21), sizeof(anchor.info));
      anchor.loss = bba_robust_loss{BBA_LOSS_TRIVIAL, 0.f};
    }
  }
  p.h_term_offsets[K] = n;
  BBA_CUDA(h, cudaMemcpyAsync(p.d_term_offsets, p.h_term_offsets, sizeof(int) * (K + 1), cudaMemcpyHostToDevice, s));
  if (n) BBA_CUDA(h, cudaMemcpyAsync(p.d_terms, p.h_terms, sizeof(PoseTerm) * n, cudaMemcpyHostToDevice, s));
  *staged = true;
  return BBA_OK;
}

// A keyframe's prior and, per constraint, H_aa / H_bb, H_ab and b_a / b_b of PoseConstraintTerms, gathered per pose block (every
// keyframe but the gauge) in the order prior, then constraints by id.  An edge to the gauge keeps only its other end's diagonal
// terms (p_gauge = 0).  Every term's H and b are scaled by its robust weight at these poses (one IRLS step per outer iteration).
// fp64, rounded to fp32.  Only rank 0 adds them: the sum all-reduce of r / M / g then counts each once.  A keyframe's attitude
// prior follows its prior.
bba_status StagePcgPoseTerms(bba_handle h, bool opt_poses, int gauge, cudaStream_t s) {
  auto& pc = h->pcg;
  pc.pose_blocks = 0;
  if (!opt_poses || (h->pose_prior_count == 0 && h->pose_constraints.empty() && !HasAttitude(h)) || h->cfg.rank != 0) return BBA_OK;
  const int K = static_cast<int>(h->keyframes.size());
  const size_t C = h->pose_constraints.size();
  if (bba_status st = ReservePoseTerms(h, C, HasAttitude(h))) return st;
  auto unknown = [&](int k) { return k == gauge ? -1 : 6 * (k < gauge ? k : k - 1); };
  std::vector<float> poses(7 * static_cast<size_t>(K));
  for (int k = 0; k < K; ++k) PoseToArray(h->keyframes[k].pose, poses.data() + 7 * k);
  // every constraint's terms at the current poses: [a's term, b's term]
  std::vector<PcgPoseTerm> edge(2 * C);
  for (size_t i = 0; i < C; ++i) {
    const bba_pose_constraint& c = h->pose_constraints[i].c;
    double H[78], b[12];
    WeightedConstraintTerms(h->pose_constraints[i], poses.data() + 7 * c.keyframe_a, poses.data() + 7 * c.keyframe_b, H, b);
    PcgPoseTerm& ta = edge[2 * i];
    PcgPoseTerm& tb = edge[2 * i + 1];
    ta.other = unknown(c.keyframe_b);
    tb.other = unknown(c.keyframe_a);
    int idx = 0;
    for (int row = 0; row < 6; ++row) {
      ta.b[row] = static_cast<float>(b[row]);
      tb.b[row] = static_cast<float>(b[6 + row]);
      for (int col = row; col < 6; ++col, ++idx) {
        ta.H[idx] = static_cast<float>(H[Upper12(row, col)]);
        tb.H[idx] = static_cast<float>(H[Upper12(6 + row, 6 + col)]);
      }
      for (int col = 0; col < 6; ++col) {
        const float x = static_cast<float>(H[Upper12(row, 6 + col)]);   // H_ab[row][col]
        ta.X[row * 6 + col] = x;
        tb.X[col * 6 + row] = x;                                       // H_ba = H_ab^T
      }
    }
  }
  std::vector<int> off, adj;
  ConstraintAdjacency(h, K, &off, &adj);
  int nb = 0, nt = 0;
  for (int k = 0; k < K; ++k) {
    if (k == gauge) continue;
    const int begin = nt;
    const PosePrior& prior = h->pose_priors[k];
    if (prior.has) {
      PcgPoseTerm& t = pc.h_pose_terms[nt++];
      t.other = -1;
      double H[21], b[6], cost, rho, w;
      PosePriorTerms(prior.pose, poses.data() + 7 * k, prior.info, H, b, &cost);
      RobustLoss(prior.loss.type, prior.loss.scale, 2.0 * cost, &rho, &w);
      for (int j = 0; j < 21; ++j) t.H[j] = static_cast<float>(w * H[j]);
      for (int j = 0; j < 6; ++j) t.b[j] = static_cast<float>(w * b[j]);
    }
    if (h->attitude_priors[k].has) {
      PcgPoseTerm& t = pc.h_pose_terms[nt++];
      t.other = -1;
      double H[21], b[6];
      WeightedAttitudeTerms(h->attitude_priors[k], poses.data() + 7 * k, H, b);
      for (int j = 0; j < 21; ++j) t.H[j] = static_cast<float>(H[j]);
      for (int j = 0; j < 6; ++j) t.b[j] = static_cast<float>(b[j]);
    }
    for (int e = off[k]; e < off[k + 1]; ++e) {
      const int i = adj[e];
      pc.h_pose_terms[nt++] = edge[2 * i + (h->pose_constraints[i].c.keyframe_a == k ? 0 : 1)];
    }
    if (nt > begin) pc.h_pose_blocks[nb++] = PcgPoseBlock{static_cast<uint32_t>(unknown(k)), begin, nt};
  }
  if (nb) {
    BBA_CUDA(h, cudaMemcpyAsync(pc.d_pose_blocks, pc.h_pose_blocks, sizeof(PcgPoseBlock) * nb, cudaMemcpyHostToDevice, s));
    BBA_CUDA(h, cudaMemcpyAsync(pc.d_pose_terms, pc.h_pose_terms, sizeof(PcgPoseTerm) * nt, cudaMemcpyHostToDevice, s));
  }
  pc.pose_blocks = nb;
  return BBA_OK;
}

}  // namespace bba

using namespace bba;

extern "C" {

// ---- soft pose priors ----
bba_status bba_set_keyframe_pose_priors(bba_handle h, int count, const int* ids, const float* poses, const float* information) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_set_keyframe_pose_priors: ";
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < 0");
  if (count > 0 && (!ids || !poses || !information)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  const int K = static_cast<int>(h->keyframes.size());
  for (int i = 0; i < count; ++i) {
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad keyframe id");
    const float* p = poses + 7 * static_cast<size_t>(i);
    const float* info = information + 21 * static_cast<size_t>(i);
    if (!PoseRecordFinite(p, info)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "non-finite pose or information");
    if (p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3] < 1e-12f) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "zero quaternion");
    if (!InformationPsd(info)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "information matrix is not positive semi-definite");
  }
  if (count > 0)
    if (bba_status st = ReservePoseTerms(h, h->pose_constraints.size(), HasAttitude(h))) return st;
  for (int i = 0; i < count; ++i) {
    PosePrior& r = h->pose_priors[ids[i]];
    std::memcpy(r.pose, poses + 7 * static_cast<size_t>(i), sizeof(r.pose));
    std::memcpy(r.info, information + 21 * static_cast<size_t>(i), sizeof(r.info));
    r.has = 1;
  }
  return CommitPosePriors(h);
}

bba_status bba_clear_keyframe_pose_priors(bba_handle h, int count, const int* ids) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_clear_keyframe_pose_priors: ";
  const int K = static_cast<int>(h->keyframes.size());
  if (count == -1) {
    std::fill(h->pose_priors.begin(), h->pose_priors.end(), PosePrior{});
    return CommitPosePriors(h);
  }
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < -1");
  if (count > 0 && !ids) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  for (int i = 0; i < count; ++i)
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad keyframe id");
  for (int i = 0; i < count; ++i) h->pose_priors[ids[i]] = PosePrior{};
  return CommitPosePriors(h);
}

bba_status bba_get_keyframe_pose_prior(bba_handle h, int id, float pose[7], float information[21], int* has_prior) {
  FrontEndScope front_end;
  if (!h || !has_prior) return BBA_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lock(h->fe.mu);
  if (id < 0 || id >= static_cast<int>(h->fe.kfs.size())) {
    lock.unlock();
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bad keyframe id");
  }
  const PosePrior& p = h->fe.kfs[id].prior;
  *has_prior = p.has;
  if (pose) std::memcpy(pose, p.pose, sizeof(p.pose));
  if (information) std::memcpy(information, p.info, sizeof(p.info));
  return BBA_OK;
}

bba_status bba_set_keyframe_pose_prior_losses(bba_handle h, int count, const int* ids, const bba_robust_loss* losses) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_set_keyframe_pose_prior_losses: ";
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < 0");
  if (count > 0 && (!ids || !losses)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  const int K = static_cast<int>(h->keyframes.size());
  for (int i = 0; i < count; ++i) {
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad keyframe id");
    if (!h->pose_priors[ids[i]].has) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "keyframe has no prior");
    if (!RobustLossValid(losses[i])) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "unknown loss type or bad scale");
  }
  for (int i = 0; i < count; ++i) h->pose_priors[ids[i]].loss = losses[i];
  return Publish(h, nullptr, false);
}

bba_status bba_get_keyframe_pose_prior_loss(bba_handle h, int id, bba_robust_loss* out) {
  FrontEndScope front_end;
  if (!h || !out) return BBA_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lock(h->fe.mu);
  if (id < 0 || id >= static_cast<int>(h->fe.kfs.size())) {
    lock.unlock();
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bad keyframe id");
  }
  *out = h->fe.kfs[id].prior.loss;
  return BBA_OK;
}

// ---- soft relative pose constraints ----
bba_status bba_add_keyframe_pose_constraints(bba_handle h, int count, const bba_pose_constraint* constraints, int* out_ids) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_add_keyframe_pose_constraints: ";
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < 0");
  if (count > 0 && !constraints) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  const int K = static_cast<int>(h->keyframes.size());
  for (int i = 0; i < count; ++i) {
    const bba_pose_constraint& c = constraints[i];
    if (c.keyframe_a < 0 || c.keyframe_a >= K || c.keyframe_b < 0 || c.keyframe_b >= K)
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad keyframe id");
    if (c.keyframe_a == c.keyframe_b) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "keyframe_a == keyframe_b");
    if (!PoseRecordFinite(c.a_T_b, c.information)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "non-finite pose or information");
    const float* q = c.a_T_b;
    if (q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] < 1e-12f) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "zero quaternion");
    if (!InformationPsd(c.information)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "information matrix is not positive semi-definite");
  }
  if (count == 0) return BBA_OK;
  if (bba_status st = ReservePoseTerms(h, h->pose_constraints.size() + count, HasAttitude(h))) return st;
  for (int i = 0; i < count; ++i) {
    PoseConstraint r{};
    r.id = h->next_pose_constraint_id++;
    r.c = constraints[i];
    double info_a[21];
    PoseConstraintInformationA(r.c.a_T_b, r.c.information, info_a);
    for (int j = 0; j < 21; ++j) r.info_a[j] = static_cast<float>(info_a[j]);
    h->pose_constraints.push_back(r);
    if (out_ids) out_ids[i] = r.id;
  }
  return Publish(h, nullptr, false);
}

bba_status bba_remove_keyframe_pose_constraints(bba_handle h, int count, const int* ids) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_remove_keyframe_pose_constraints: ";
  auto& cons = h->pose_constraints;
  if (count == -1) {
    cons.clear();
    return Publish(h, nullptr, false);
  }
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < -1");
  if (count > 0 && !ids) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  std::vector<char> drop(cons.size(), 0);
  for (int i = 0; i < count; ++i) {
    // ids increase along the list
    auto it = std::lower_bound(cons.begin(), cons.end(), ids[i], [](const PoseConstraint& c, int id) { return c.id < id; });
    if (it == cons.end() || it->id != ids[i]) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "unknown constraint id");
    drop[it - cons.begin()] = 1;
  }
  size_t n = 0;
  for (size_t i = 0; i < cons.size(); ++i)
    if (!drop[i]) cons[n++] = cons[i];
  cons.resize(n);
  return Publish(h, nullptr, false);
}

bba_status bba_get_keyframe_pose_constraints(bba_handle h, int capacity, int* ids, bba_pose_constraint* out, int* count) {
  FrontEndScope front_end;
  if (!h || !count) return BBA_ERR_INVALID_ARGUMENT;
  if (capacity < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_get_keyframe_pose_constraints: capacity < 0");
  std::lock_guard<std::mutex> lock(h->fe.mu);
  const std::vector<PoseConstraint>& cons = h->fe.constraints;
  *count = static_cast<int>(cons.size());
  const int n = std::min(capacity, *count);
  for (int i = 0; i < n; ++i) {
    if (ids) ids[i] = cons[i].id;
    if (out) out[i] = cons[i].c;
  }
  return BBA_OK;
}

bba_status bba_set_keyframe_pose_constraint_losses(bba_handle h, int count, const int* ids, const bba_robust_loss* losses) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_set_keyframe_pose_constraint_losses: ";
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < 0");
  if (count > 0 && (!ids || !losses)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  auto& cons = h->pose_constraints;
  std::vector<size_t> at(count);
  for (int i = 0; i < count; ++i) {
    auto it = std::lower_bound(cons.begin(), cons.end(), ids[i], [](const PoseConstraint& c, int id) { return c.id < id; });
    if (it == cons.end() || it->id != ids[i]) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "unknown constraint id");
    if (!RobustLossValid(losses[i])) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "unknown loss type or bad scale");
    at[i] = static_cast<size_t>(it - cons.begin());
  }
  for (int i = 0; i < count; ++i) cons[at[i]].loss = losses[i];
  return Publish(h, nullptr, false);
}

bba_status bba_get_keyframe_pose_constraint_losses(bba_handle h, int capacity, int* ids, bba_robust_loss* out, int* count) {
  FrontEndScope front_end;
  if (!h || !count) return BBA_ERR_INVALID_ARGUMENT;
  if (capacity < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_get_keyframe_pose_constraint_losses: capacity < 0");
  std::lock_guard<std::mutex> lock(h->fe.mu);
  const std::vector<PoseConstraint>& cons = h->fe.constraints;
  *count = static_cast<int>(cons.size());
  const int n = std::min(capacity, *count);
  for (int i = 0; i < n; ++i) {
    if (ids) ids[i] = cons[i].id;
    if (out) out[i] = cons[i].loss;
  }
  return BBA_OK;
}

// ---- attitude priors ----
bba_status bba_set_keyframe_attitude_priors(bba_handle h, int count, const int* ids, const bba_attitude_prior* priors) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_set_keyframe_attitude_priors: ";
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < 0");
  if (count > 0 && (!ids || !priors)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  const int K = static_cast<int>(h->keyframes.size());
  for (int i = 0; i < count; ++i) {
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad keyframe id");
    const bba_attitude_prior& p = priors[i];
    bool finite = std::isfinite(p.information);
    for (int j = 0; j < 3; ++j) finite = finite && std::isfinite(p.reference_direction[j]) && std::isfinite(p.measured_direction[j]);
    if (!finite) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "non-finite direction or information");
    for (const float* d : {p.reference_direction, p.measured_direction})
      if (std::sqrt(static_cast<double>(d[0]) * d[0] + static_cast<double>(d[1]) * d[1] + static_cast<double>(d[2]) * d[2]) < 1e-6)
        return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "direction of norm < 1e-6");
    if (!(p.information > 0.f)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "information is not > 0");
    if (!RobustLossValid(p.loss)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "unknown loss type or bad scale");
  }
  if (count > 0)
    if (bba_status st = ReservePoseTerms(h, h->pose_constraints.size(), true)) return st;
  for (int i = 0; i < count; ++i) {
    AttitudePrior& r = h->attitude_priors[ids[i]];
    r.p = priors[i];
    for (float* d : {r.p.reference_direction, r.p.measured_direction}) {
      const double n = std::sqrt(static_cast<double>(d[0]) * d[0] + static_cast<double>(d[1]) * d[1] + static_cast<double>(d[2]) * d[2]);
      for (int j = 0; j < 3; ++j) d[j] = static_cast<float>(d[j] / n);
    }
    r.has = 1;
  }
  return CommitAttitudePriors(h);
}

bba_status bba_clear_keyframe_attitude_priors(bba_handle h, int count, const int* ids) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_clear_keyframe_attitude_priors: ";
  const int K = static_cast<int>(h->keyframes.size());
  if (count == -1) {
    std::fill(h->attitude_priors.begin(), h->attitude_priors.end(), AttitudePrior{});
    return CommitAttitudePriors(h);
  }
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < -1");
  if (count > 0 && !ids) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  for (int i = 0; i < count; ++i)
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad keyframe id");
  for (int i = 0; i < count; ++i) h->attitude_priors[ids[i]] = AttitudePrior{};
  return CommitAttitudePriors(h);
}

bba_status bba_get_keyframe_attitude_prior(bba_handle h, int id, bba_attitude_prior* out, int* has) {
  FrontEndScope front_end;
  if (!h || !has) return BBA_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lock(h->fe.mu);
  if (id < 0 || id >= static_cast<int>(h->fe.kfs.size())) {
    lock.unlock();
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bad keyframe id");
  }
  const AttitudePrior& p = h->fe.kfs[id].attitude;
  *has = p.has;
  if (out) *out = p.p;
  return BBA_OK;
}

bba_status bba_evaluate_keyframe_attitude_priors(bba_handle h, int keyframe_capacity, double* s, double* weight, void* stream) {
  return EvaluateAttitudePriors(h, keyframe_capacity, s, weight, static_cast<cudaStream_t>(stream));
}

// ---- keyframe pose graph ----
bba_status bba_optimize_pose_graph(bba_handle h, const bba_pose_graph_options* options, bba_pose_graph_result* result, void* stream) {
  return OptimizePoseGraph(h, options, result, static_cast<cudaStream_t>(stream));
}

bba_status bba_evaluate_keyframe_pose_terms(bba_handle h, int keyframe_capacity, double* prior_s, double* prior_weight,
                                            int constraint_capacity, double* constraint_s, double* constraint_weight, void* stream) {
  return EvaluatePoseTerms(h, keyframe_capacity, prior_s, prior_weight, constraint_capacity, constraint_s, constraint_weight,
                           static_cast<cudaStream_t>(stream));
}

}  // extern "C"
