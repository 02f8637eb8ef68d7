/* include/badba.h -- C ABI of libbadba_b200.so, the Hopper (sm_90a) direct
 * bundle-adjustment backend that drops in behind ETH3D/badslam's DirectBA.
 *
 * The reference has no FFI layer: its seam is the C++ class `DirectBA`
 * (applications/badslam/src/badslam/direct_ba.h:65-550) on top of the free functions of
 * applications/badslam/src/badslam/kernels.h:94-495.  Every entry point below names the
 * reference interface it replaces.  The header-only C++ adaptor include/badba_direct_ba.hpp
 * keeps the reference's own signatures on top of this ABI (see INTEGRATION.md).
 *
 * Conventions (mirroring SURVEY.md 8b):
 *  - plain pointers and sizes only; no C++/torch types cross the boundary;
 *  - device pointers are CALLER-OWNED and are NOT copied unless the function name ends in
 *    `_host` (those copy from host memory into library-owned device memory);
 *  - a pitched 2-D device buffer is (pointer, pitch in BYTES), i.e. the fields of the
 *    reference's CUDABuffer_<T> (libvis/src/libvis/cuda/cuda_buffer.cuh:112-118);
 *  - poses are float[7] = {qx,qy,qz,qw,tx,ty,tz} = Sophus::SE3f::data() of global_T_frame;
 *  - every call is stream-ordered on the cudaStream_t passed as `void* stream` (0 = default
 *    stream); calls that return host scalars synchronise that stream before returning, like
 *    the reference (kernel_opt_pose.cc:96, kernel_opt_intrinsics.cc:136,263);
 *  - one in-flight call per handle (DirectBA::Mutex(), direct_ba.h:196-208);
 *  - errors are status codes + bba_last_error(); nothing aborts (the reference LOG(FATAL)s,
 *    libvis/src/libvis/cuda/cuda_util.h:35-49) and nothing falls back to a CPU path.
 */
#ifndef BADBA_H
#define BADBA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BBA_ABI_VERSION 8

typedef struct bba_context* bba_handle;

typedef enum {
  BBA_OK = 0,
  BBA_ERR_INVALID_ARGUMENT = 1,
  BBA_ERR_CUDA = 2,
  BBA_ERR_STATE = 3,
  BBA_ERR_UNSUPPORTED = 4,
  BBA_ERR_NO_DEVICE = 5
} bba_status;

/* Keyframe::Activation (keyframe.h:54-67) */
typedef enum { BBA_KF_ACTIVE = 0, BBA_KF_COVISIBLE_ACTIVE = 1, BBA_KF_INACTIVE = 2 } bba_kf_activation;

/* DirectBA constructor arguments (direct_ba.h:73-88, direct_ba.cc:74-163). */
typedef struct {
  int depth_width, depth_height;
  int color_width, color_height;
  float depth_intrinsics[4];   /* fx, fy, cx, cy: PinholeCamera4f::parameters(), pixel-corner convention */
  float color_intrinsics[4];
  float raw_to_float_depth;
  float baseline_fx;
  int sparse_surfel_cell_size;
  uint32_t max_surfel_count;
  int max_keyframes;
  int use_depth_residuals;
  int use_descriptor_residuals;
  int device;                  /* CUDA device ordinal this handle lives on */
  int rank, world_size;        /* position in a one-process-per-GPU job (world_size 1 = single GPU) */
  /* surfel maintenance (direct_ba.h:73-88; defaults of bad_slam_config.h:143-158 are 1, 2, 3 and 0.8) */
  int min_observation_count_while_bootstrapping_1;   /* < 5 keyframes  */
  int min_observation_count_while_bootstrapping_2;   /* < 10 keyframes */
  int min_observation_count;
  float surfel_merge_dist_factor;                    /* DetermineSupportingSurfelsAndMergeSurfelsCUDA */
} bba_config;

/* Arguments of DirectBA::BundleAdjustment (direct_ba.h:143-162). */
typedef struct {
  int optimize_depth_intrinsics;
  int optimize_color_intrinsics;
  int do_surfel_updates;
  int optimize_poses;
  int optimize_geometry;
  int min_iterations;
  int max_iterations;
  int use_pcg;
  int active_keyframe_window_start;
  int active_keyframe_window_end;
  int increase_ba_iteration_count;
  double time_limit_seconds;   /* 0 = none (direct_ba_alternating.cc:704-709) */
  /* use_pcg only (direct_ba.h:158-160, direct_ba_pcg.cc:52-53) */
  int pcg_max_inner_iterations;   /* <= 0: 30 */
  int pcg_max_keyframes;          /* <= 0: 2500; keyframe_count must not exceed it */
  int pcg_gauge_keyframe;         /* keyframe whose pose is held fixed in every iteration; < 0: rand() % keyframe_count per
                                     iteration as the reference does (direct_ba_pcg.cc:324) */
  /* progress_function of direct_ba.h:160-162: called at the top of every iteration with the iteration index; returning 0
   * stops the optimisation before that iteration runs (direct_ba_alternating.cc:346-348, direct_ba_pcg.cc:174-176).
   * NULL = none.  With world_size > 1 it must return the same value on every rank. */
  int (*progress_function)(void* user, int iteration);
  void* progress_user;
} bba_ba_options;

typedef struct {
  int iterations_done;
  int converged;
  /* residual bookkeeping of the LAST executed iteration's pose step, taken at its starting state
   * (what the reference's debug counters report, kernel_opt_pose.cu:224-248) */
  uint64_t depth_residual_count;       /* associated (surfel, keyframe) pairs */
  uint64_t descriptor_residual_count;  /* 2 x pairs whose colour pixel is in bounds */
  double cost;                         /* sum Tukey(depth) + sum Huber(descriptor 1), reference convention */
  int pose_iterations_total;           /* Gauss-Newton iterations summed over keyframes and outer iterations */
  /* per-stage device time of the last iteration, reference stage names
   * (direct_ba_alternating.cc:629-689) */
  float ms_surfel_activation;
  float ms_geometry_optimization;
  float ms_pose_optimization;
  float ms_intrinsics_optimization;
  uint64_t kernel_launches;            /* kernels this call launched */
  /* use_pcg: inner PCG steps summed over the outer iterations, last residual norm sqrt(beta_n), device time of the
   * last iteration's PCG solve ("BA PCG step", direct_ba_pcg.cc:733-737) */
  int pcg_inner_iterations_total;
  float pcg_last_r_norm;
  float ms_pcg;
  /* PerformBASchemeEndTasks (direct_ba.cc:566-653): surfels deleted by this call, surfels_size afterwards (the surviving
   * surfels are compacted to the front of the caller's buffer) */
  uint32_t surfels_deleted;
  uint32_t surfels_size;
  /* do_surfel_updates: surfels appended by CreateSurfelsForKeyframe / marked by the in-loop merges during this call */
  uint32_t surfels_created;
  uint32_t surfels_merged;
} bba_ba_result;

/* Counters of one pose pass (superset of kernel_opt_pose.cu's debug outputs; the n_* feed the
 * algorithmic-bytes model of SURVEY.md 8d). */
typedef struct {
  float H[21];
  float b[6];
  uint64_t n_pair, n_inimg, n_depthok, n_assoc, n_photo;
  double cost_depth, cost_desc1, cost_desc2;
} bba_pose_coeffs;

/* Exchange step of a one-process-per-GPU job, implemented by the host (torch.distributed / NCCL in the harness, raw
 * ncclAllGather / ncclAllReduce in a C++ integration).  Both operate IN PLACE on a library-owned device buffer and are
 * enqueued on `stream`:
 *   BBA_COLLECTIVE_ALLGATHER      buffer = world_size slices of `count` BYTES; this rank's slice is slice[rank]
 *   BBA_COLLECTIVE_ALLREDUCE_SUM  buffer = `count` fp32 values, summed over ranks */
typedef enum { BBA_COLLECTIVE_ALLGATHER = 0, BBA_COLLECTIVE_ALLREDUCE_SUM = 1 } bba_collective_op;
typedef void (*bba_collective_fn)(void* user, int op, void* device_buffer, size_t count, void* stream);

/* ---- lifetime ---- */
int         bba_abi_version(void);
bba_status  bba_create(const bba_config* config, bba_handle* out);           /* DirectBA::DirectBA  direct_ba.cc:74 */
void        bba_destroy(bba_handle h);                                        /* DirectBA::~DirectBA direct_ba.cc:165 */
const char* bba_last_error(bba_handle h);                                     /* replaces LOG(FATAL) */

/* ---- scene model ---- */
/* surfels_ / surfels_size_ (direct_ba.cc:122, accessors direct_ba.h:300-340): 17-row pitched SoA. */
bba_status bba_set_surfels(bba_handle h, float* device_surfels, size_t pitch_bytes, uint32_t surfels_size);
/* active_surfels_ (direct_ba.cc:123) */
bba_status bba_set_active_flags(bba_handle h, uint8_t* device_flags);
/* Same two, from host memory into library-owned device buffers (e2e / harness path). */
bba_status bba_set_surfels_host(bba_handle h, const float* host_surfels, size_t pitch_bytes, uint32_t surfels_size, void* stream);
bba_status bba_get_surfels_host(bba_handle h, float* host_surfels, size_t pitch_bytes, int rows, void* stream);
bba_status bba_get_active_flags_host(bba_handle h, uint8_t* host_flags, void* stream);
bba_status bba_get_surfels_device(bba_handle h, float** device_surfels, size_t* pitch_bytes, uint32_t* surfels_size);

/* DirectBA::AddKeyframe (direct_ba.cc:197-205) with the Keyframe buffers of keyframe.h:160-200.
 * Computes frustum co-visibility against all earlier keyframes (direct_ba.cc:231-249). */
bba_status bba_add_keyframe(bba_handle h,
                            const uint16_t* device_depth, size_t depth_pitch,
                            const uint16_t* device_normals, size_t normals_pitch,
                            const uint16_t* device_radius, size_t radius_pitch,
                            const uint8_t* device_color_rgba, size_t color_pitch,
                            const float global_T_frame[7], float min_depth, float max_depth,
                            void* stream, int* out_keyframe_id);
bba_status bba_add_keyframe_host(bba_handle h,
                                 const uint16_t* host_depth, const uint16_t* host_normals,
                                 const uint16_t* host_radius, const uint8_t* host_color_rgba,
                                 const float global_T_frame[7], float min_depth, float max_depth,
                                 void* stream, int* out_keyframe_id);
int        bba_keyframe_count(bba_handle h);
bba_status bba_set_keyframe_pose(bba_handle h, int keyframe_id, const float global_T_frame[7]);   /* Keyframe::set_global_T_frame */
bba_status bba_get_keyframe_pose(bba_handle h, int keyframe_id, float global_T_frame[7]);         /* Keyframe::global_T_frame */
bba_status bba_set_keyframe_activation(bba_handle h, int keyframe_id, int activation);            /* Keyframe::SetActivation */
bba_status bba_get_keyframe_activation(bba_handle h, int keyframe_id, int* activation);
/* Bulk variants over keyframes [0, count): poses [count][7], activations [count] (either may be NULL). */
bba_status bba_set_keyframe_states(bba_handle h, int count, const float* global_T_frame, const int* activation);
bba_status bba_get_keyframe_states(bba_handle h, int count, float* global_T_frame, int* activation);
bba_status bba_get_covisibility(bba_handle h, int keyframe_id, uint8_t* out_row /* [keyframe_count] */);

/* depth_params_ / cameras (direct_ba.h:243-297; SetColorCamera etc.) */
bba_status bba_set_intrinsics(bba_handle h, const float depth_intrinsics[4], const float color_intrinsics[4], float depth_a);
bba_status bba_get_intrinsics(bba_handle h, float depth_intrinsics[4], float color_intrinsics[4], float* depth_a);
/* DirectBA::SetUseDepthResiduals / SetUseDescriptorResiduals (direct_ba.h:317-328; main.cc:853 switches the descriptor
 * residuals off for the final BA): takes effect from the next call.  At least one type must stay enabled. */
bba_status bba_set_residual_types(bba_handle h, int use_depth_residuals, int use_descriptor_residuals);
bba_status bba_get_residual_types(bba_handle h, int* use_depth_residuals, int* use_descriptor_residuals);
bba_status bba_set_cfactor_host(bba_handle h, const float* host_cfactor /* dense [cf_h][cf_w] */, void* stream);
bba_status bba_get_cfactor_host(bba_handle h, float* host_cfactor, void* stream);
bba_status bba_cfactor_size(bba_handle h, int* cf_width, int* cf_height);

/* ---- the hot path (kernels.h) ---- */
/* AccumulatePoseEstimationCoeffsCUDA (kernels.h:156-174, kernel_opt_pose.cc:39-97) for keyframe
 * `keyframe_id` evaluated at global_T_frame_estimate.  Synchronises the stream. */
bba_status bba_accumulate_pose_coeffs(bba_handle h, int keyframe_id, const float global_T_frame_estimate[7],
                                      bba_pose_coeffs* out, void* stream);
/* DirectBA::EstimateFramePose (direct_ba.h:122-129, direct_ba_alternating.cc:42-283) against a stored keyframe's
 * images.  iterations/converged may be NULL. */
bba_status bba_estimate_frame_pose(bba_handle h, int keyframe_id, const float global_T_frame_initial[7],
                                   float global_T_frame_out[7], int* iterations, int* converged, void* stream);
/* The same for a frame that is NOT a keyframe -- the buffer-taking signature of DirectBA::EstimateFramePose
 * (direct_ba.h:122-129: depth_buffer, normals_buffer, color_texture): frame-to-model tracking against the current surfels.
 * The colour image is the uchar4 buffer (.w = luma) the reference builds its texture from.  Needs one free keyframe slot
 * (keyframe_count < max_keyframes); nothing about the frame is kept after the call. */
bba_status bba_estimate_frame_pose_for_frame(bba_handle h, const uint16_t* device_depth, size_t depth_pitch,
                                             const uint16_t* device_normals, size_t normals_pitch,
                                             const uint8_t* device_color_rgba, size_t color_pitch,
                                             const float global_T_frame_initial[7], float global_T_frame_estimate[7],
                                             int* iterations, int* converged, void* stream);
/* UpdateSurfelActivationCUDA (kernels.h:262-269, kernel_surfel_activation.cc:39-67) */
bba_status bba_update_surfel_activation(bba_handle h, void* stream);
/* OptimizeGeometryIterationCUDA (kernels.h:234-244, kernel_opt_geometry.cc:80-201) */
bba_status bba_optimize_geometry_iteration(bba_handle h, void* stream);
/* DirectBA::PerformBASchemeEndTasks (direct_ba.cc:566-653): DeleteSurfelsAndUpdateRadiiCUDA over every keyframe (surfels
 * with fewer than GetMinObservationCount() observations, or more free-space violations than observations, are deleted; the
 * others get the smallest observed radius) + CompactSurfelsCUDA.  bba_bundle_adjust runs it like the reference does: at
 * the end when increase_ba_iteration_count is set, else at the start of the first call after the counter changed.
 * do_surfel_updates (the reference's second argument, direct_ba.h:435-437): first merge similar surfels using every keyframe
 * that was active in this BA iteration block (direct_ba.cc:577-601).
 * The keyframes' radius buffers must be valid.  *deleted / *surfels_size may be NULL. */
bba_status bba_perform_end_tasks(bba_handle h, int do_surfel_updates, uint32_t* deleted, uint32_t* surfels_size, void* stream);
/* surfels_size_ of the reference (the caller's buffer holds that many surfels at its front). */
uint32_t bba_surfels_size(bba_handle h);
/* ba_iteration_count_ / last_ba_iteration_count_ (direct_ba.h:373-377): the pair decides whether a call with
 * increase_ba_iteration_count = 0 first runs the end tasks (direct_ba_alternating.cc:313-319). */
bba_status bba_get_ba_iteration_counts(bba_handle h, int* ba_iteration_count, int* last_ba_iteration_count);
bba_status bba_set_ba_iteration_counts(bba_handle h, int ba_iteration_count, int last_ba_iteration_count);

/* In-loop surfel lifecycle (do_surfel_updates = 1 runs these inside bba_bundle_adjust on the reference's schedule,
 * direct_ba_alternating.cc:399-430,489-541, direct_ba.cc:577-601; with several ranks they run replicated -- they are deterministic).
 *  bba_create_surfels_for_keyframe: DirectBA::CreateSurfelsForKeyframe (direct_ba.h:114-117, direct_ba.cc:340-405): one new
 *    surfel per sparse cell of the keyframe that no existing surfel is associated with, optionally filtered by the
 *    observations / free-space violations in the co-visible keyframes, appended in raster order; surfels_size grows.
 *  bba_merge_surfels_for_keyframe: DetermineSupportingSurfelsAndMergeSurfelsCUDA (kernels.h, kernel_supporting_surfels.cc:
 *    40-118): surfels of a cell that are close to one of the cell's supporting surfels are marked deleted (x = NaN pattern).
 *  bba_compact_surfels: CompactSurfelsCUDA (kernel_compact_surfels.cu:159-279) for `free_count` marked surfels.
 * The reference resolves two races "first come" (which pixel of a cell seeds the new surfel, which surfels support a cell);
 * this library uses the outcome of executing the reference's threads in index order (smallest raster index / three smallest
 * surfel indices), which is reproducible and identical to the reference for sparse_surfel_cell_size = 1. */
bba_status bba_create_surfels_for_keyframe(bba_handle h, int keyframe_id, int filter_new_surfels, uint32_t* created, void* stream);
bba_status bba_merge_surfels_for_keyframe(bba_handle h, int keyframe_id, uint32_t* deleted, void* stream);
bba_status bba_compact_surfels(bba_handle h, uint32_t free_count, int with_active_flags, uint32_t* surfels_size, void* stream);

/* Parity hook for the PCG solver's building blocks (kernel_pcg.cu:179-1037): runs the init pass (PCGInitCUDA for every
 * keyframe) -> out_r, out_M; PCGInit2 -> out_p; one PCGStep1 sweep -> out_g, out_scalars = {alpha_n, alpha_d}.
 * Host output buffers of *unknown_count floats; call with out_r = NULL to query the count.  o->pcg_gauge_keyframe >= 0. */
bba_status bba_pcg_debug(bba_handle h, const bba_ba_options* o, uint32_t* unknown_count, float* out_r, float* out_M, float* out_p,
                         float* out_g, double out_scalars[2], void* stream);

/* OptimizeIntrinsicsCUDA (kernels.h:246-260, kernel_opt_intrinsics.cc:39-281) */
bba_status bba_optimize_intrinsics(bba_handle h, int optimize_depth_intrinsics, int optimize_color_intrinsics, void* stream);
/* DirectBA::BundleAdjustment (direct_ba.h:143-162, direct_ba.cc:407-453 -> direct_ba_alternating.cc:285-738) */
bba_status bba_bundle_adjust(bba_handle h, const bba_ba_options* options, bba_ba_result* result, void* stream);

/* ---- multi-GPU (one process per GPU; not present in the reference, SURVEY.md 8e) ---- */
/* Sharding (SURVEY.md 8e, DESIGN.md "Multi-GPU"): keyframe images and the surfel buffer are replicated on every rank.
 *  - geometry step: rank r updates the surfels of its shard (256-surfel granules dealt round-robin, see bba_shard_*); ONE
 *    all-gather of the updated rows (x, y, z, normal, descriptor 1/2, active flag) per outer iteration -- or direct stores into
 *    the peers' replicas, bba_peer_import -- makes every replica identical again;
 *  - pose step: the non-inactive keyframes are dealt to the ranks (balanced by measured work), each rank runs the Gauss-Newton
 *    loops of its keyframes locally, and ONE all-reduce (sum of disjoint slots, K x 17 floats) publishes the poses;
 *  - intrinsics step and PCG products: summed over each rank's surfel shard, completed by one sum all-reduce;
 *  - surfel creation / merging / compaction: replicated (deterministic); end tasks: statistics sharded, compaction replicated.
 * Registers the exchange callback; required before any hot-path call when world_size > 1. */
bba_status bba_set_collective(bba_handle h, bba_collective_fn fn, void* user);
/* Fused geometry exchange over NVLink peer memory (optional, <= 8 ranks on one node): every rank exports CUDA IPC handles
 * of its surfel buffer + active flags, the host passes the handles of ALL ranks (indexed by rank) to every rank, and from
 * then on the geometry kernels store a surfel's updated rows straight into every replica; the all-gather of the exchange
 * step degenerates to a 1-element all-reduce used as a barrier.  Without it the host-collective all-gather is used.
 * The mapping is dropped by bba_set_surfels / bba_set_surfels_host / bba_set_active_flags. */
typedef struct {
  unsigned char surfels_ipc[64];   /* cudaIpcMemHandle_t of the allocation holding the surfel buffer */
  uint64_t surfels_offset;         /* byte offset of the buffer inside that allocation */
  unsigned char active_ipc[64];
  uint64_t active_offset;
  uint64_t pitch_bytes;
  uint32_t surfels_size;
  int32_t rank;
} bba_peer_handle;
bba_status bba_peer_export(bba_handle h, bba_peer_handle* out);
bba_status bba_peer_import(bba_handle h, const bba_peer_handle* all_ranks, int count);
int bba_peer_count(bba_handle h);
/* Back to the host-collective exchange (all ranks must agree on the mode: a rank whose import failed makes everyone unmap). */
bba_status bba_peer_unmap(bba_handle h);
/* With mapped peers the geometry kernels of the OTHER ranks store into this rank's replica.  A caller that rewrites its replica
 * outside the library (restores a snapshot of the surfel rows, uploads new surfels in place, ...) must say so on every rank, in
 * the same place: the next kernel that stores into peer replicas is then preceded by a barrier across the ranks, so that no
 * rank's stores can land in a replica before its owner's rewrite has happened (and be overwritten by it).  No-op on one GPU
 * or with the host-collective exchange. */
bba_status bba_mark_replica_rewritten(bba_handle h);

/* The partition itself, exposed so that hosts and tests can reason about it.
 * Surfels: 256-surfel granules are dealt round-robin (granule g -> rank g % world_size), which gives every rank the same
 * mix of well- and poorly-observed surfels; a rank addresses its surfels through a dense local index, and the exchange
 * slices ([7][slice_length] floats per rank) are in local index order.
 * Keyframes: the DEFAULT owner rank of the i-th entry of a keyframe work list is round-robin.  Once a pose step has run, the
 * library balances the next one by the measured per-keyframe work (Gauss-Newton iterations x pairs projecting into the
 * image, replicated on all ranks) with a longest-first greedy assignment; any disjoint assignment is valid because the
 * results are published through disjoint slots of one sum all-reduce. */
int      bba_shard_surfel_owner(uint32_t surfel_index, int world_size);
uint32_t bba_shard_surfel_local_index(uint32_t surfel_index, int world_size);
uint32_t bba_shard_slice_length(uint32_t surfels_size, int world_size);
int  bba_shard_keyframe_owner(int list_index, int world_size);
/* The assignment rule itself (host-only, no device needed): cost[i] > 0 = measured work of work-list entry i, 0 = unknown
 * (mean of the known ones); all unknown or world_size 1 -> round-robin. */
void bba_balance_keyframes(const float* cost, int count, int world_size, int* owner);

/* Re-uploads the images of an existing keyframe from host memory (same sizes as at creation) -- the per-step
 * host->device input path of a live system, where a keyframe's RGB-D data arrives from the sensor thread
 * (BadSlam::CreateKeyframe, bad_slam.cc).  NULL pointers leave the corresponding buffer untouched. */
bba_status bba_update_keyframe_host(bba_handle h, int keyframe_id,
                                    const uint16_t* host_depth, const uint16_t* host_normals,
                                    const uint16_t* host_radius, const uint8_t* host_color_rgba, void* stream);

/* ---- keyframe preprocessing (SURVEY.md 8(f3)): raw RGB-D frame -> the keyframe buffers bba_add_keyframe takes ----
 * BadSlam::PreprocessFrame (bad_slam.cc:692-765): ComputeBrightnessCUDA (cuda_image_processing.cu:165-193),
 * BilateralFilteringAndDepthCutoffCUDA (cuda_depth_processing.cu:42-128), ComputeNormalsCUDA (:134-276),
 * ComputePointRadiiAndRemoveIsolatedPixelsCUDA (:295-383), and the ComputeMinMaxDepthCUDA (:390-465) of keyframe creation
 * (bad_slam.cc:978), fused into one kernel launch.  Uses the handle's depth camera, depth deformation (a, cfactor) and
 * raw_to_float_depth.  All images are device memory with byte pitches; raw depth: 0 = no measurement; rgb: uchar3.  The output
 * depth must not alias the raw depth.  device_rgb / device_color_rgba may both be NULL (depth only).  Pixels dropped by a stage
 * get depth 65535, normal 0 and radius 0 (the reference leaves their radius untouched).  min_depth / max_depth (metres, over
 * the valid output pixels; +inf / 0 when there is none) may be NULL; when given the call synchronises the stream like
 * ComputeMinMaxDepthCUDA does.  The reference's optional CPU median filter (preprocessing.cc:37-85, off by default) and the
 * depth / colour pyramids are not part of this call. */
typedef struct {
  float bilateral_filter_sigma_xy;         /* BadSlamConfig::bilateral_filter_sigma_xy          default 1.5   (bad_slam_config.h:113) */
  float bilateral_filter_sigma_inv_depth;  /* BadSlamConfig::bilateral_filter_sigma_inv_depth   default 0.005 (:122) */
  float bilateral_filter_radius_factor;    /* BadSlamConfig::bilateral_filter_radius_factor     default 2.0   (:118); radius <= 16 px */
  float max_depth;                         /* BadSlamConfig::max_depth, metres                  default 3.0   (:96) */
} bba_preprocess_options;
bba_status bba_preprocess_frame(bba_handle h, const bba_preprocess_options* options,
                                const uint16_t* device_raw_depth, size_t raw_depth_pitch,
                                const uint8_t* device_rgb, size_t rgb_pitch,
                                uint16_t* device_depth, size_t depth_pitch,
                                uint16_t* device_normals, size_t normals_pitch,
                                uint16_t* device_radius, size_t radius_pitch,
                                uint8_t* device_color_rgba, size_t color_pitch,
                                float* min_depth, float* max_depth, void* stream);

/* ---- image-pair odometry (SURVEY.md 8(f4)): a new frame tracked against a stored keyframe ----
 * BadSlam::RunOdometry (bad_slam.cc:829-950) -> TrackFramePairwise (pairwise_frame_tracking.cc:153-678): intensity (or Sobel
 * gradient magnitude) images of both frames (cuda_image_processing.cu:103-206), calibrated float depth of both, the base
 * keyframe's colour transformed to the depth intrinsics (kernel_downsample.cu:345-372), the depth / normal / colour pyramids
 * (kernel_downsample.cu:40-156), and on every level from coarse to fine: the cost comparison between the previous result and
 * the initial estimate (kernel_opt_pose.cu:939-1296, pairwise_frame_tracking.cc:427-508) and up to 30 damped Gauss-Newton
 * iterations on depth + descriptor (or gradient-magnitude) residuals of every base pixel projected into the tracked frame
 * (kernel_opt_pose.cu:422-885; fp64 LDLT + SE3 update pairwise_frame_tracking.cc:553-593; convergence_analysis.h:56-63).
 * The pyramids are one launch per level for both images; the whole coarse-to-fine optimisation is ONE persistent kernel
 * launch with no host round trip (the reference synchronises the stream once per iteration).
 * The tracked frame is given like in bba_estimate_frame_pose_for_frame (preprocessed depth, normals, uchar4 colour with
 * .w = luma); poses are base_T_frame as {qx,qy,qz,qw,tx,ty,tz}.  Uses the handle's cameras, depth deformation and residual types. */
typedef struct {
  int num_scales;                        /* BadSlamConfig::num_scales, default 5 (bad_slam_config.h:167); 1..8 */
  int use_pyramid_level_0;               /* RunOdometry passes true (bad_slam.cc:923) */
  int use_gradmag;                       /* RunOdometry passes false: separate x/y gradient components (bad_slam.cc:833) */
  int test_different_initial_estimates;  /* RunOdometry passes true: the two motion-model predictions are compared on the coarsest level */
  int max_iterations_per_scale;          /* kMaxIterationsPerScale = 30 (pairwise_frame_tracking.cc:247); <= 0 selects it */
} bba_odometry_options;
typedef struct {
  int iterations[8];        /* Gauss-Newton iterations per pyramid level (index = scale) */
  int chose_initial[8];     /* 1: the initial-estimate arm won the cost comparison on this level, 0: the other arm, -1: no comparison */
  uint32_t residual_count;  /* the reference's debug counters at the last accumulation (kernel_opt_pose.cu:619-657) */
  float residual_sum;
  uint32_t passes;          /* image passes (grid-wide barriers) of the persistent kernel */
  uint32_t kernel_launches; /* launches of the whole call */
} bba_odometry_result;
bba_status bba_track_frame_pairwise(bba_handle h, const bba_odometry_options* options, int base_keyframe_id,
                                    const uint16_t* device_depth, size_t depth_pitch,
                                    const uint16_t* device_normals, size_t normals_pitch,
                                    const uint8_t* device_color_rgba, size_t color_pitch,
                                    const float base_T_frame_initial_1[7], const float base_T_frame_initial_2[7],
                                    float base_T_frame_estimate[7], bba_odometry_result* result, void* stream);
/* Parity hooks (the pyramids and normal equations of the LAST bba_track_frame_pairwise call of this handle, device-resident):
 *  bba_odometry_get_level: one pyramid level of the base (which = 0) or tracked (1) image into dense host arrays
 *    [height][width] (any may be NULL); *width / *height return the level's size.
 *  bba_odometry_debug_coeffs: AccumulatePoseEstimationCoeffsFromImagesCUDA (kernels.h:181-203) at base_T_frame_a -> H[21], b[6],
 *    residual count / sum, and ComputeCostAndResidualCountFromImagesCUDA (kernels.h:205-223) at both poses -> counts[2], costs[2]. */
bba_status bba_odometry_get_level(bba_handle h, int which, int scale, float* host_depth, uint16_t* host_normals, uint8_t* host_color,
                                  int* width, int* height, void* stream);
bba_status bba_odometry_debug_coeffs(bba_handle h, int scale, int use_gradmag, const float base_T_frame_a[7], const float base_T_frame_b[7],
                                     float H[21], float b[6], uint32_t* residual_count, float* residual_sum,
                                     uint32_t counts[2], float costs[2], void* stream);

/* ---- host-side building blocks (no handle, no device) ----
 * The host arithmetic the backend runs between kernels, exported so that it can be checked without a GPU: Sophus'
 * SE3 exp / log / product / inverse on {qx,qy,qz,qw,tx,ty,tz} (se3.hpp:127-130,203-207,293-313,435-468), the convergence test of
 * convergence_analysis.h:45-52, the fp64 pivoted LDLT solve standing in for Eigen's (direct_ba_alternating.cc:206,
 * kernel_opt_intrinsics.cc:171,272; n = 4, 5 or 6, upper triangle packed row-major; returns 0 for another n), and the frustum
 * intersection behind the co-visibility lists (camera_frustum.h:73-143, direct_ba.cc:231-249). */
void bba_host_se3_exp(const float tangent[6], float out_pose[7]);
void bba_host_se3_log(const float pose[7], float out_tangent[6]);
void bba_host_se3_compose(const float a[7], const float b[7], float out_pose[7]);
void bba_host_se3_inverse(const float a[7], float out_pose[7]);
int  bba_host_pose_update_converged(const float x[6]);
int  bba_host_solve_ldlt(int n, const double* upper, const double* b, double* x);
int  bba_host_frusta_intersect(const float depth_intrinsics[4], int width, int height,
                               const float global_T_frame_a[7], float min_depth_a, float max_depth_a,
                               const float global_T_frame_b[7], float min_depth_b, float max_depth_b);

/* The constant-motion model in front of the image-pair odometry (BadSlam::PredictFramePose / RunOdometry / ClearMotionModel /
 * the rebase in BadSlam::ProcessFrame when a keyframe is created: bad_slam.cc:542-565, 767-827, 949-954, 1057-1068).  Host
 * arithmetic on at most three stored estimates of base_kf_tr_frame and, kept separately as in the reference, their inverses;
 * the caller owns the record.  One tracked frame of BadSlam::RunOdometry is
 *     bba_host_motion_model_predict(&m, use_motion_model, e1, e2);
 *     bba_track_frame_pairwise(..., e1, e2, estimate, ...);
 *     bba_host_motion_model_push(&m, estimate);
 * and bba_host_motion_model_rebase(&m) follows the creation of a keyframe from the frame tracked last. */
typedef struct {
  int   count;                       /* stored estimates, 0..3 (oldest first) */
  float base_kf_tr_frame[3][7];
  float frame_tr_base_kf[3][7];
} bba_motion_model;
/* ClearMotionModel: one stored estimate = last_kf_frame_T_global * global_T_frame, or identity if there is no keyframe yet
 * (last_kf_frame_T_global == NULL). */
void bba_host_motion_model_clear(bba_motion_model* m, const float last_kf_frame_T_global[7], const float global_T_frame[7]);
/* PredictFramePose: the two initial estimates TrackFramePairwise tries.  Returns 0 (and writes nothing) if m holds no estimate. */
int  bba_host_motion_model_predict(const bba_motion_model* m, int use_motion_model, float out_estimate_1[7], float out_estimate_2[7]);
/* The tail of RunOdometry: drop the oldest of three, append the new estimate and its inverse. */
void bba_host_motion_model_push(bba_motion_model* m, const float base_T_frame_estimate[7]);
/* A keyframe was created from the frame tracked last: re-express the older estimates relative to it; the last becomes identity. */
void bba_host_motion_model_rebase(bba_motion_model* m);

/* ---- instrumentation ---- */
uint64_t   bba_kernel_launch_count(bba_handle h);   /* kernels launched through this handle so far */

/* Per-kernel device timing (cudaEvents on the launching stream) and the counters of the algorithmic-bytes
 * model of SURVEY.md 8d, accumulated over every pose / geometry launch while profiling is enabled. */
typedef struct {
  uint64_t pose_launches;        /* PoseAccumulateKernel launches (non-empty work list) */
  double   pose_ms;              /* their summed device time */
  uint64_t kf_evals;             /* sum over launches of keyframes in the work list */
  uint64_t n_pair, n_inimg, n_depthok, n_assoc, n_photo;   /* summed over those launches */
  uint64_t geometry_launches;
  double   activation_normals_ms;
  double   position_descriptor_ms;
} bba_profile;
/* level 0 = off, 1 = per-launch cudaEvent timing, 2 = timing + byte-model counters (n_inimg, n_depthok) in every iteration */
bba_status bba_set_profiling(bba_handle h, int level);
bba_status bba_get_profile(bba_handle h, bba_profile* out, int reset);

#ifdef __cplusplus
}
#endif
#endif
