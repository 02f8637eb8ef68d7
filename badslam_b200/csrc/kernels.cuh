// kernels.cuh -- launch interface between the host orchestration (handle.hpp and its host units) and the sm_90a kernels.
// Every Launch* function returns the kernels it enqueued and the first error of its runtime calls (launch.hpp).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "device_math.cuh"
#include "exact_sum.cuh"
#include "launch.hpp"

namespace bba {

// One term of a keyframe's pose solve in the form of a soft pose prior (host_math.hpp PosePriorTerms): the prior global_T_frame
// and the upper triangle of its 6x6 information matrix.  The pose step stages a keyframe's prior, the equivalent priors of its
// relative pose constraints and their damping anchors as such terms (pose_step.cu StagePoseTerms).
struct PoseTerm {
  float pose[7];
  float info[21];
};

// Accumulator record per keyframe written by the pose kernel: 32 fp64 sums
//   [0..20] H upper triangle row-major, [21..26] b, [27] n_assoc, [28] n_photo,
//   [29] cost_depth, [30] cost_desc1, [31] cost_desc2
// followed (separately) by 2 u64 stage counters {n_inimg, n_depthok} for the byte model.
constexpr int kPoseAccSize = 32;

struct PoseAccumulateArgs {
  CameraParams cam;
  const float* surfels;      // 17-row SoA
  uint32_t pitch;            // floats per row
  uint32_t n;                // surfels_size
  const KfDevice* kfs;
  const int* work_list;      // keyframe ids to evaluate
  const int* work_count;     // device scalar
  const float* stream;       // kPoseStreamRows rows x stream_pitch, in spatial order (LaunchPoseStream); may be null
  uint32_t stream_pitch;     // floats per row
  const float* boxes;        // [n / kSpatialChunk rounded up][8] bounding box of every stream chunk (LaunchPoseStream)
  bool stream_sorted;        // the stream is in spatial order (perm), not in the caller's
  KfDevice* work_records;   // [max_kf] scratch: the work list's KfDevice records in list order (pad = keyframe id), filled by
                             // LaunchPoseAccumulate so that a work group's <= group records are ONE contiguous bulk copy
  int group;                 // keyframes per work item, 1 .. kPoseMaxGroup; 0: LaunchPoseAccumulate picks it
  double* acc;               // [max_kf][32]
  ExactSum* exact;           // deterministic mode: [max_kf][32] exact sums that take the warp totals instead of acc; else null
  unsigned long long* stage_counts;  // [max_kf][2]
  unsigned int* queue;       // global work-item counter, must be 0 at launch
};

constexpr int kPoseMaxGroup = 64;

// Persistent, TMA-staged pose residual/Jacobian/Hessian kernel (AccumulatePoseEstimationCoeffsCUDAKernel,
// kernel_opt_pose.cu:251-383, for a whole list of keyframes in one launch).
// with_stats: also accumulate residual costs + the stage counters (iteration 0 of a pose step, profiling, debug API).
// Spatial order of the surfels (spatial_order.cu).  The caller's surfels lie in creation order, raster order of the keyframe that
// made them: 256 consecutive ones form a band across a whole image.  Sorted by the Morton code of their positions (10 bits per axis
// inside the map's bounding box) they form compact chunks, most of which lie wholly outside a given keyframe's view.
// perm[s] = caller index of the surfel at sorted position s.  A stable radix sort: the same positions give the same permutation.
constexpr int kSpatialChunk = 256;   // surfels per bounding box of the pose stream
struct SpatialOrderBuffers {
  uint32_t* keys_in;     // [capacity]
  uint32_t* keys_out;    // [capacity]
  uint32_t* index_in;    // [capacity]
  uint32_t* perm;        // [capacity]
  unsigned int* bounds;  // [6] order-preserving encodings of the map's min / max
  void* temp;            // CUB scratch of SpatialOrderTempBytes(capacity) bytes
  size_t temp_bytes;
};
size_t SpatialOrderTempBytes(uint32_t capacity);
// Three launches: bounds, keys and the CUB radix sort, whose kernels count as one launch.
LaunchResult LaunchSpatialOrder(const float* surfels, uint32_t pitch, uint32_t n, const SpatialOrderBuffers& b, cudaStream_t stream);
// The pose step's surfel stream, in spatial order: stream row r, column s holds, for surfel perm[s], x y z d1 d2 (rows 0-4), the
// unpacked + re-normalised normal (rows 5-7, util_nvcc_only.cuh:83-95) and the tangent points gp + t1 / gp + t2 (rows 8-10 / 11-13,
// cost_function.cuh:115-133).  What the descriptor residual needs of a surfel alone is computed once per pose step (the surfels do
// not move while the keyframe poses are optimised) and the rows the kernel stages come from one buffer.  boxes[c] = min x y z, 0,
// max x y z, 0 over the finite positions of stream columns [256 c, 256 c + 256).  perm = null: the caller's order.
constexpr int kPoseStreamRows = 14;
LaunchResult LaunchPoseStream(const float* surfels, uint32_t pitch, uint32_t n, const uint32_t* perm, float* stream, uint32_t stream_pitch,
                              float* boxes, cudaStream_t cuda_stream);
// Instantiations of the pose kernel (surfel tile, PRE = stages the sorted stream); the values are bba_pose_variant's.
enum PoseVariant { kPoseVariantAuto = 0, kPoseVariant256Pre = 1, kPoseVariant512Pre = 2, kPoseVariant256 = 3, kPoseVariant512 = 4,
                   kPoseVariant1024 = 5 };
inline bool PoseVariantValid(int v) { return v >= kPoseVariantAuto && v <= kPoseVariant1024; }
inline bool PoseVariantPre(int v) { return v == kPoseVariant256Pre || v == kPoseVariant512Pre; }
// max_work: upper bound of *work_count known to the host (sizes the record-packing launch that precedes the kernel; both count).
// variant = kPoseVariantAuto: the tile follows from args.n and the SM count, and args.stream != null selects the variant that
// stages the sorted stream (and skips the chunks whose box lies outside a keyframe's view) instead of the caller's rows.  Any other
// variant forces that instantiation; a PRE variant needs args.stream and args.boxes, the others ignore them.  args.exact != null
// selects the deterministic instantiation of the same variant.  args.group = 0: 32 keyframes per work item on a stream in spatial
// order, 8 otherwise.
LaunchResult LaunchPoseAccumulate(const PoseAccumulateArgs& args, int sm_count, bool with_stats, int max_work, cudaStream_t stream,
                                  int variant = kPoseVariantAuto);
// Sets the dynamic shared-memory limit of every instantiation of the pose kernel on the current device (once per handle).
cudaError_t SetPoseAccumulateSmemLimits();

struct PoseSolveArgs {
  KfDevice* kfs;
  float* pose_est;             // [max_kf][7] global_T_frame estimates, updated in place
  double* acc;                 // consumed and re-zeroed
  ExactSum* exact;             // deterministic mode: consumed (rounded to fp64) and re-zeroed instead of acc; else null
  unsigned long long* stage_counts;
  const int* work_in;          // list consumed by this iteration
  const int* count_in;
  int* work_out;               // list of keyframes that need another iteration
  int* count_out;
  int* iterations;             // [max_kf]
  int* converged;              // [max_kf]
  double* first_stats;         // [max_kf][8]: n_assoc n_photo cost_depth cost_desc1 cost_desc2 n_inimg n_depthok (iteration 0)
  unsigned long long* totals;  // [8] cumulative: kf_evals, n_inimg, n_depthok, n_assoc, n_photo (over all iterations)
  volatile int* host_flag;     // mapped pinned memory: {iterations completed, work items left}
  unsigned int* queue;         // PoseAccumulateKernel's work-item counter, re-armed here
  int iteration;
  int max_iterations;
  // the soft pose terms by keyframe id: keyframe k's are terms[term_offsets[k] .. term_offsets[k + 1]), added in list order;
  // both null when no keyframe has one
  const int* term_offsets;     // [keyframes + 1]
  const PoseTerm* terms;
};
// Device-side Gauss-Newton step for every keyframe in the list (direct_ba_alternating.cc:173-233).
LaunchResult LaunchPoseSolve(const PoseSolveArgs& args, cudaStream_t stream);

// Keyframe pose graph (pose_graph.cu; bba_optimize_pose_graph, DESIGN §3.14).  One term of the cost: a soft pose prior on
// keyframe a (b = -1, z = the prior's global_T_frame), or a relative pose constraint (a, b, z = a_T_b): a handle constraint
// or an odometry-chain edge of the call.  info: the upper triangle of L.
struct PoseGraphTerm {
  int a, b;
  float z[7];
  float info[21];
};
// A term's linearisation at the current poses (host_math.hpp PosePriorTerms / PoseConstraintTerms): H's upper triangle (21 of
// a prior, 78 of a constraint over (delta_a, delta_b)), b = J^T L r (6 or 12) and the cost.
struct PoseGraphTermBlocks {
  double H[78];
  double b[12];
  double cost;
};
// The Gauss-Newton loop's state on the device.  Every kernel returns at once when done is set.
struct PoseGraphState {
  double initial_cost;   // at the poses the call starts from
  double cost;           // at the poses of the last accepted step
  int done;
  int iterations;        // Gauss-Newton iterations that solved a linear system
  int converged;
  int linear_iterations; // PCG iterations, summed
};
struct PoseGraphArgs {
  int K;                         // keyframes (row blocks)
  int term_count;
  const PoseGraphTerm* terms;    // [term_count]: priors, constraints by id, then the odometry chain
  PoseGraphTermBlocks* blocks;   // [term_count]
  float* poses;                  // [K][7] global_T_frame, updated in place
  float* prev;                   // [K][7] the poses before the last step (a rejected step reverts to them)
  const int* held;               // [K] 1: the keyframe keeps its pose (an identity row of H)
  const int* row_off;            // [K + 1] into row_terms
  const int* row_terms;          // [2 per entry] (term, side 0 = a / 1 = b): the terms of row block k in term order
  const int* csr_off;            // [K + 1] block-CSR of H: row k's blocks [csr_off[k], csr_off[k + 1]), the diagonal first,
  const int* csr_col;            //   then one block per constraint term of the row in term order
  double* csr_val;               // [nnz][36] row-major
  double* rhs;                   // [K][6] b
  double* tri;                   // [K][36] H_{k,k+1}: the upper coupling of the block-tridiagonal preconditioner M
  double* work;                  // the cyclic reduction's levels and the PCG vectors (PoseGraphWorkDoubles)
  PoseGraphState* state;
  int max_iterations;            // Gauss-Newton iterations
  int max_linear;                // PCG iterations per linear solve
  int round;                     // 0 .. max_iterations: the round of this launch
};
// The doubles of PoseGraphArgs::work for K keyframes: the reduction's levels (at most 2K + 32 blocks of six 6x6 matrices and
// three 6-vectors) and five PCG vectors of K blocks.
inline size_t PoseGraphWorkDoubles(size_t K) { return (2 * K + 32) * (6 * 36 + 3 * 6) + 5 * 6 * K; }
// One round of a Gauss-Newton iteration, four launches: linearise every term, assemble H / b / M per row block, solve (the cost
// test of the last step, then PCG with the block-tridiagonal preconditioner factorised by cyclic reduction, one CTA), and
// T <- T exp(delta).  round == max_iterations launches the first three only (the test of the last step).
LaunchResult LaunchPoseGraphRound(const PoseGraphArgs& a, cudaStream_t stream);

// Replicas of the surfel buffer / active flags on the OTHER ranks of a one-process-per-GPU job, mapped into this process
// (CUDA IPC) and written directly over NVLink by the geometry kernels: the owner of a surfel stores its updated rows into
// every replica, so the "all-gather" of the geometry step is fused into the kernels' own final stores.
constexpr int kMaxPeers = 7;
struct PeerSet {
  int count;                   // 0: no peers mapped (single GPU, or the host-collective exchange is used)
  float* surfels[kMaxPeers];   // same pitch / layout as the local buffer
  uint8_t* active[kMaxPeers];
};

// The geometry kernels visit the surfels in stream order: local index li -> stream position s = SurfelShardToGlobal(li) -> caller
// index perm[s] (s when perm is null).  Each launch first gathers its surfels' inputs into the geometry stream (LaunchGeo), so
// that a warp's 32 lanes read coalesced rows and hold a compact cluster of surfels; the partial sums parked between keyframe
// groups live in the caller's scratch rows 8..16 at column s, the results go to column perm[s] of the caller's rows.
struct GeometryArgs {
  CameraParams cam;
  float* surfels;
  uint32_t pitch;
  uint32_t n;
  uint32_t begin, end;         // range of this rank's LOCAL surfel indices (SurfelShardToGlobal maps them; 0 .. n on one GPU)
  uint32_t shard_rank, shard_world;
  const uint32_t* perm;        // spatial order (SpatialOrderBuffers::perm), or null: the caller's order
  float* stream;               // kGeoStreamRows x stream_pitch, filled by the launcher in stream order
  uint32_t stream_pitch;       // floats per row, >= n
  uint8_t* active;
  const KfDevice* kfs;
  const int* kf_list;          // non-inactive keyframes (ascending ids)
  int kf_count;
  unsigned int* queue;         // work-item counter (reset by the launcher)
  unsigned int* tile_epoch;    // [ceil(n / 32)] keyframe groups retired per tile (reset by the launcher)
  int tile_shift;              // log2(surfels per tile), 5..8; chosen by the launcher
  PeerSet peers;
};
// The geometry stream: x y z, packed normal, radius^2, d1, d2 and the active flags (as u32 bits) of the launch's surfels at their
// stream positions.  It shares the pose stream's buffer (the pose step rebuilds its own rows at its start).  desc_rows: also
// gather radius^2, d1, d2 (what the position / descriptor kernel reads with descriptors; the other launches read rows 0-3 + flags).
constexpr int kGeoStreamRows = 8;
static_assert(kGeoStreamRows <= kPoseStreamRows, "the geometry stream lives in the pose stream's buffer");
LaunchResult LaunchGeometryStream(const GeometryArgs& args, bool desc_rows, cudaStream_t stream);
// SetSurfelInactive + DetermineActiveSurfels (kernel_surfel_activation.cu:38-79) fused with the normal
// accumulation + update (kernel_opt_geometry.cu:527-597).
// Both launch the stream gather and the kernel, or nothing when there is nothing to do.
LaunchResult LaunchActivationAndNormals(const GeometryArgs& args, int sm_count, bool determine_activation, bool update_normals,
                                        cudaStream_t stream);
// Position (+ descriptor) accumulation and per-surfel solve (kernel_opt_geometry.cu:118-231,273-361 or :417-507).
LaunchResult LaunchPositionAndDescriptor(const GeometryArgs& args, int sm_count, cudaStream_t stream);

// Surfel deformation after an outside pose correction (bba_deform_surfels, DESIGN §3.13).  Per keyframe: D = global_T_frame (now)
// * original frame_T_global, row-major 3x4 from old global coordinates to new ones, and the original camera centre.
struct KfChange {
  float D[12];
  float centre[3];
  int unmoved;               // 1: D is the exact identity
};
struct DeformArgs {
  GeometryArgs geo;          // kfs: the keyframe records at their ORIGINAL poses; kf_list: 0 .. kf_count - 1
  const KfChange* changes;   // [kf_count] by keyframe id
  unsigned int* counts;      // [2] += surfels whose rows changed, surfels without an associated keyframe (zero at launch)
};
// The stream gather and the kernel, or nothing when there is nothing to do.  Deleted surfels (x = NaN) are skipped.
LaunchResult LaunchDeformSurfels(const DeformArgs& a, int sm_count, cudaStream_t stream);

// Multi-GPU surfel sharding: 256-surfel granules are dealt round-robin to the ranks (granule g belongs to rank g % world), so
// that every rank sees the same mix of well- and poorly-observed surfels (surfels are stored in creation order, and the
// cost of a surfel is the number of keyframes that see it).  A rank addresses its surfels through a dense local index.
constexpr uint32_t kShardGranuleShift = 8;
__host__ __device__ inline uint32_t SurfelShardToGlobal(uint32_t local, uint32_t rank, uint32_t world) {
  return world <= 1 ? local : ((((local >> kShardGranuleShift) * world + rank) << kShardGranuleShift) | (local & ((1u << kShardGranuleShift) - 1u)));
}
// Exchange of the shards: rows.count surfel rows, then the active flags as floats when rows.active, x shard_len floats per rank,
// in local index order.  The shards are granules of stream positions, surfel perm[s] at position s (perm null: the caller's order).
constexpr int kShardRows = 7;   // at most: x y z normal d1 d2 + active (the geometry step's)
struct ShardRows {
  int ids[kShardRows - 1];      // SurfelRow of each slice row
  int count;                    // of ids
  int active;                   // 1: one more slice row with the active flags
};
LaunchResult LaunchPackShard(const float* surfels, uint32_t pitch, const uint8_t* active, uint32_t n, ShardRows rows, const uint32_t* perm,
                             uint32_t rank, uint32_t world, uint32_t shard_len, float* slice, cudaStream_t stream);
LaunchResult LaunchUnpackShards(float* surfels, uint32_t pitch, uint8_t* active, uint32_t n, ShardRows rows, const uint32_t* perm,
                                uint32_t shard_len, int world, int skip_rank, const float* buffer, cudaStream_t stream);
// Pose results of the locally owned keyframes -> [K][17] floats (zeros elsewhere) for the sum all-reduce.
constexpr int kPoseSlot = 17;   // 7 pose, iterations, converged, 8 first-iteration statistics
LaunchResult LaunchPackPoseResults(const int* ids, int n, const float* pose_est, const int* iterations, const int* converged,
                                   const double* first_stats, float* out, cudaStream_t stream);

// Intrinsics + depth-deformation step (intrinsics.cu; OptimizeIntrinsicsCUDA, kernel_opt_intrinsics.cc:39-281).
constexpr int kIntrinsicsSums = 34;   // A (15) b1 (5) colour H (10) colour b (4), fp64
struct IntrinsicsArgs {
  CameraParams cam;
  const float* surfels;
  uint32_t pitch;
  uint32_t n;
  uint32_t begin, end;         // range of this rank's LOCAL surfel indices (SurfelShardToGlobal)
  uint32_t shard_rank, shard_world;
  const KfDevice* kfs;
  const int* kf_list;          // every keyframe (ascending ids)
  int kf_count;
  unsigned int* queue;         // work-item counter (reset by the launcher)
  double* sums;                // [kIntrinsicsSums]
  float* cell_B;               // [5][cell_count]
  float* cell_D;               // [cell_count]
  float* cell_b2;              // [cell_count]
  float* cell_obs;             // [cell_count] observation count (fp32 so that one sum all-reduce covers everything)
  uint32_t cell_count;
  // deterministic mode: exact sums that take the per-cell terms ([7][cell_count]: B rows 0-4, D, b2) and the global sums
  // ([kIntrinsicsSums]) instead of cell_B / cell_D / cell_b2 and sums (LaunchIntrinsicsFinalize rounds them); else null
  ExactSum* exact_cells;
  ExactSum* exact_sums;
};
LaunchResult LaunchIntrinsicsAccumulate(const IntrinsicsArgs& a, int sm_count, bool optimize_color, bool optimize_depth, cudaStream_t stream);
// Deterministic mode: cell_B / cell_D / cell_b2 (contiguous, [7][cell_count]) <- fp32 of the exact cell sums and sums <- the exact
// global sums, ahead of LaunchIntrinsicsSchur.
LaunchResult LaunchIntrinsicsFinalize(uint32_t cell_count, const ExactSum* exact_cells, float* cell_B, const ExactSum* exact_sums, double* sums,
                                      cudaStream_t stream);
LaunchResult LaunchIntrinsicsSchur(uint32_t cell_count, float* B, float* D, const float* b2, double* sums, cudaStream_t stream);
LaunchResult LaunchIntrinsicsConvertSums(double* sums, float* head, bool to_float, cudaStream_t stream);
LaunchResult LaunchIntrinsicsCellUpdate(uint32_t cell_count, const float* obs, const float* B, const float* D, const float* x1,
                                        float* cfactor, cudaStream_t stream);

// PCG Gauss-Newton step over all unknowns (pcg.cu; BundleAdjustmentPCG, direct_ba_pcg.cc:43-819).
struct PcgArgs {
  CameraParams cam;
  const float* surfels;
  uint32_t pitch;
  uint32_t begin, end;         // range of this rank's LOCAL surfel indices (SurfelShardToGlobal maps them; 0 .. n on one GPU)
  uint32_t n;                  // surfels_size
  uint32_t shard_rank, shard_world;
  int alpha_d_slot;            // scalars slot that receives this launch's p^T J^T W J p: 1 on one GPU, 3 (exchanged, then added to 1) otherwise
  const KfDevice* kfs;         // every keyframe, ids 0 .. kf_count-1
  int kf_count;
  int gauge_kf;                // keyframe whose pose is fixed (no unknowns), direct_ba_pcg.cc:315-333
  int opt_poses, opt_geometry, opt_depth_intr, opt_color_intr;
  uint32_t surfel_start, surfel_stride;   // first surfel unknown, unknowns per surfel (1 or 3)
  uint32_t depth_intr_start, color_intr_start;
  float* r;                    // INIT
  float* M;                    // INIT
  const float* p;              // STEP1
  float* g;                    // STEP1
  double* scalars;             // [0] / [2] alpha_n, beta_n (swapping roles), [1] alpha_d
  unsigned int* queue;         // work-item counter (reset by the launcher)
};
// Layout of the fp64 scalar block: [0] / [2] alpha_n, beta_n (swapping roles), [1] alpha_d, [3] this rank's part of alpha_d
// (multi-GPU), then the workspace of the fixed-order grid sums of the vector kernels.
constexpr int kPcgPartialsA = 8, kPcgPartialsB = 8 + 2048, kPcgCounters = 8 + 4096, kPcgScalarDoubles = 8 + 4096 + 2;
LaunchResult LaunchPcgAccumulate(const PcgArgs& a, int sm_count, bool init, cudaStream_t stream);
LaunchResult LaunchPcgPackAlphaD(const double* scalars, float* tail, cudaStream_t stream);
LaunchResult LaunchPcgUnpackAlphaD(double* scalars, const float* tail, cudaStream_t stream);
LaunchResult LaunchPcgInit2(uint32_t n, uint32_t a_index, float a, int kf_count, const float* r, const float* M, float* delta, float* g, float* p,
                            double* scalars, int slot_alpha_n, int sm_count, cudaStream_t stream);
LaunchResult LaunchPcgStep2(uint32_t n, uint32_t a_index, float* r, const float* M, float* delta, float* g, const float* p, double* scalars,
                            int slot_alpha_n, int slot_beta_n, int sm_count, cudaStream_t stream);
LaunchResult LaunchPcgStep3(uint32_t n, uint32_t a_index, int kf_count, float* g, float* p, double* scalars, int slot_alpha_n, int slot_beta_n,
                            int sm_count, cudaStream_t stream);
LaunchResult LaunchPcgUpdateSurfels(float* surfels, uint32_t pitch, uint32_t n, bool use_desc, uint32_t surfel_start, const float* delta,
                                    cudaStream_t stream);
LaunchResult LaunchPcgUpdateCfactor(float* cfactor, uint32_t cells, const float* delta, cudaStream_t stream);
// The pose-block terms of the PCG products (soft pose priors and relative pose constraints).  One term of pose block i: H_ii
// (upper triangle), b_i (J^T L r), and for a constraint whose other end j is a pose unknown, j's first unknown and H_ij
// (row-major, rows i); other = -1 for a prior or an edge to the gauge keyframe (p_gauge = 0).
struct PcgPoseTerm {
  int other;
  float H[21];
  float b[6];
  float X[36];
};
// A pose block with terms: its first unknown u and its terms [begin, end) in a fixed order.
struct PcgPoseBlock {
  uint32_t u;
  int begin, end;
};
// init: r_i -= sum b_i, M_i += sum diag(H_ii); else g_i += sum (H_ii p_i + H_ij p_j) and *alpha_d += sum_i p_i . (that
// contribution) = p^T A p over the terms, a fixed-order fp64 sum without atomics.
LaunchResult LaunchPcgPoseTerms(const PcgPoseBlock* blocks, int block_count, const PcgPoseTerm* terms, bool init, float* r, float* M,
                                const float* p, float* g, double* alpha_d, cudaStream_t stream);

// End-of-BA surfel maintenance (lifecycle.cu; PerformBASchemeEndTasks, direct_ba.cc:566-653).
struct KfRadius {
  const uint16_t* ptr;         // pitched u16 (IEEE half radius^2, keyframe.h radius_buffer)
  uint32_t pitch;              // bytes
  uint32_t pad;
};
struct SurfelStatsArgs {
  CameraParams cam;
  float* surfels;
  uint32_t pitch;
  uint32_t n;
  const KfDevice* kfs;         // every keyframe, ids 0 .. kf_count-1
  const KfRadius* radius;
  int kf_count;
  int min_observation_count;
  unsigned int* queue;
  unsigned int* tile_epoch;
  int tile_shift;              // chosen by the launcher
  unsigned int* deleted_count; // device scalar, += surfels deleted by this launch
  // multi-GPU: this rank handles the surfels of its granule shard (local indices [0, local_count)); with mapped peers the two
  // result rows (x = deletion marker, radius^2) are stored into every replica, like the geometry step's results
  uint32_t local_count, shard_rank, shard_world;
  PeerSet peers;
};
LaunchResult LaunchObservationStats(SurfelStatsArgs a, int sm_count, cudaStream_t stream);
// Exclusive scan of n u32 counts, shared by the compaction and the surfel creation: block_sums needs ScanScratchWords(n) words,
// and block_sums[ScanTotalIndex(n)] receives the sum of all counts.
uint32_t ScanScratchWords(uint32_t n);
uint32_t ScanTotalIndex(uint32_t n);
// Moves surviving surfels from the tail into the free spots; afterwards the first n - free_count slots are the surfels.
// active != nullptr: the active flags move with them (CompactSurfelsCUDA's adapt_active_surfels).
LaunchResult LaunchCompactSurfels(float* surfels, uint32_t pitch, uint32_t n, uint32_t free_count, unsigned int* block_sums, uint8_t* active,
                                  cudaStream_t stream);

// In-loop surfel lifecycle for ONE keyframe (CreateSurfelsForKeyframe / DetermineSupportingSurfelsAndMergeSurfels).
struct CovisEntry {              // one co-visible keyframe of the keyframe new surfels are created for
  float R[12];                   // covis_T_frame = covis.frame_T_global * keyframe.global_T_frame (direct_ba.cc:365-370)
  const uint16_t* depth;
  const uint16_t* normals;
  uint32_t depth_pitch, normals_pitch;
  uint32_t pad[2];
};
struct LifecycleArgs {
  CameraParams cam;
  float T[12];                   // frame_T_global of the keyframe
  float G[12];                   // global_T_frame
  const uint16_t* depth;
  const uint16_t* normals;
  const uint16_t* radius;
  uint32_t depth_pitch, normals_pitch, radius_pitch;
  cudaTextureObject_t tex;       // luma
  const uint8_t* rgba;           // the keyframe's uchar4 colour image (surfel colours)
  uint32_t rgba_pitch;
  float* surfels;
  uint32_t pitch, n;
  unsigned int* sup;             // [3][cells] supporting surfel indices
  unsigned int* cell_bits;       // [cells]
  uint32_t cells;
  unsigned int* flags;           // [w * h] new-surfel flag per pixel
  const CovisEntry* covis;
  int covis_count;
  int min_observation_count;
  float cell_merge_dist_squared;
  unsigned int* counter;         // device scalar (deleted surfels)
};
LaunchResult LaunchSupportSurfels(const LifecycleArgs& a, int sm_count, cudaStream_t stream);   // sup[0] only (occupancy for the creation)
LaunchResult LaunchMergeSurfels(const LifecycleArgs& a, int sm_count, cudaStream_t stream);     // supports + merge, += *counter
LaunchResult LaunchSeedNewSurfels(const LifecycleArgs& a, bool filter, cudaStream_t stream);    // a.flags after LaunchSupportSurfels
LaunchResult LaunchExclusiveScan(const unsigned int* in, uint32_t n, unsigned int* out, unsigned int* block_sums, cudaStream_t stream);
LaunchResult LaunchCreateSurfels(const LifecycleArgs& a, const unsigned int* index, cudaStream_t stream);

// bba_debug_exact_sum: deposits the n values into *sum (zero at launch) from many CTAs, each visiting the values in a scrambled
// order, and rounds the result into *out.
LaunchResult LaunchExactSumDebug(const float* values, uint64_t n, ExactSum* sum, double* out, int sm_count, cudaStream_t stream);

// uchar4 (.w = luma) -> u8 planes, `images` images in one launch: image i (first, or rest[i - 1] in device memory) -> rows
// [i * h, (i + 1) * h) of luma.  One image reads no table (rest may be null).
struct LumaSource {
  const uint8_t* rgba;
  size_t pitch;
};
LaunchResult LaunchExtractLuma(LumaSource first, const LumaSource* rest, int images, uint8_t* luma, size_t luma_pitch, int w, int h,
                               cudaStream_t stream);

}  // namespace bba
