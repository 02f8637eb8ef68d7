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
 *  - two sides per handle, as BadSlam's default parallel_ba mode runs DirectBA (bad_slam.cc:643-765,
 *    831-950 beside BAThreadMain, bad_slam.cc:1196-1305):
 *      BA side: every entry point; one call in flight at a time (DirectBA::Mutex(),
 *        direct_ba.h:196-208);
 *      front-end side: one further thread may make one call at a time, on its own stream, while a
 *        BA-side call is in flight -- also from inside progress_function.  The front-end calls are
 *        bba_preprocess_frame, bba_preprocess_raw_frame, bba_track_frame_pairwise,
 *        bba_track_frame_pairwise_to_frame, bba_track_frames_pairwise, bba_odometry_get_level,
 *        bba_odometry_debug_coeffs, the
 *        bba_host_* functions (no handle) and the readers bba_keyframe_count, bba_get_keyframe_pose,
 *        bba_get_keyframe_states, bba_get_keyframe_activation, bba_get_intrinsics,
 *        bba_get_cfactor_host, bba_cfactor_size and bba_get_residual_types.
 *    Front-end calls read a snapshot of the state the BA side published last (cameras, a, cfactor,
 *    residual types, keyframe records and poses), never the state a running BA call is changing.
 *    The BA side publishes in every setter, bba_add_keyframe*, bba_update_keyframe_host, at the end
 *    of every pose step (all poses together), of every intrinsics step and of every BA call.  With
 *    one thread a front-end call therefore sees exactly the handle's current state.  The front end
 *    does not get a view in the middle of a BA iteration, nor any share of the SMs: its kernels
 *    queue behind the BA kernels that occupy them (INTEGRATION.md section 2);
 *  - several handles may be driven concurrently from different threads of one process (one BA side
 *    each); the members of a local group (bba_local_group_create) are such handles, with the
 *    threading contract given there;
 *  - errors are status codes + bba_last_error(), per calling thread; nothing aborts (the reference
 *    LOG(FATAL)s, libvis/src/libvis/cuda/cuda_util.h:35-49) and nothing falls back to a CPU path.
 */
#ifndef BADBA_H
#define BADBA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BBA_ABI_VERSION 10

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
  uint64_t kernel_launches;            /* kernels this call launched, as the launchers report them: the CUB radix sort of the
                                        * spatial order counts as one, memsets and copies are not counted */
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
/* Replaces LOG(FATAL): the message of the last failed call made on the calling thread on this handle (or the note of a call
 * that succeeded with a warning, such as surfel creation at the surfel limit).  Valid until that thread's next failure. */
const char* bba_last_error(bba_handle h);

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
/* The getters of keyframe state are front-end calls: they return the published state (see Conventions). */
int        bba_keyframe_count(bba_handle h);                                                      /* front end */
bba_status bba_set_keyframe_pose(bba_handle h, int keyframe_id, const float global_T_frame[7]);   /* Keyframe::set_global_T_frame */
bba_status bba_get_keyframe_pose(bba_handle h, int keyframe_id, float global_T_frame[7]);         /* Keyframe::global_T_frame; front end */
bba_status bba_set_keyframe_activation(bba_handle h, int keyframe_id, int activation);            /* Keyframe::SetActivation */
bba_status bba_get_keyframe_activation(bba_handle h, int keyframe_id, int* activation);           /* front end */
/* Bulk variants over keyframes [0, count): poses [count][7], activations [count] (either may be NULL).  The getter is a
 * front-end call: all poses of one publication. */
bba_status bba_set_keyframe_states(bba_handle h, int count, const float* global_T_frame, const int* activation);
bba_status bba_get_keyframe_states(bba_handle h, int count, float* global_T_frame, int* activation);
bba_status bba_get_covisibility(bba_handle h, int keyframe_id, uint8_t* out_row /* [keyframe_count] */);
/* Soft pose priors (not in the reference; g2o / Ceres / GTSAM offer the same term): a keyframe with a prior adds
 * 1/2 r^T L r to the cost, r = log(prior^-1 * global_T_frame) in the tangent order of the pose solve (translation, then
 * rotation, Sophus), L a 6x6 information matrix given as its upper triangle, row-major, in the layout of H (21 floats).  The
 * term enters only where the keyframe's pose is optimised: the pose step of the alternating scheme and bba_estimate_frame_pose
 * (a keyframe that is inactive in a BA iteration keeps its pose), and the pose unknowns of the PCG scheme (not the gauge
 * keyframe).  A handle without priors runs exactly the code it ran before they existed.  With several ranks every rank sets the
 * same priors, as it adds the same keyframes.
 *  bba_set_keyframe_pose_priors: ids [count], prior_global_T_frame [count][7], information [count][21]; replaces the prior of
 *    each listed keyframe.  BBA_ERR_INVALID_ARGUMENT for an unknown id, a non-finite value, a zero quaternion or an L that is not
 *    positive semi-definite (the pivoted LDLT of L has a negative pivot, or a zero pivot with a non-zero column); the arguments
 *    are checked before anything changes, and a failed call leaves the handle unchanged.
 *  bba_clear_keyframe_pose_priors: removes the priors of ids [count]; count = -1 removes every prior (ids is not read).
 *  bba_get_keyframe_pose_prior: front-end call (the published priors); *has_prior = 0 and zeros without a prior (pose /
 *    information may be NULL).
 * The setters are BA-side calls and publish. */
bba_status bba_set_keyframe_pose_priors(bba_handle h, int count, const int* keyframe_ids, const float* prior_global_T_frame,
                                        const float* information);
bba_status bba_clear_keyframe_pose_priors(bba_handle h, int count, const int* keyframe_ids);
bba_status bba_get_keyframe_pose_prior(bba_handle h, int keyframe_id, float prior_global_T_frame[7], float information[21],
                                       int* has_prior);
/* Soft relative pose constraints between two keyframes (not in the reference; the binary counterpart of the priors, as the edges
 * of a pose graph): a loop closure's relative pose (bba_track_frames_pairwise), wheel odometry or integrated IMU motion between
 * two keyframes, the fixed extrinsics of a camera rig.  A constraint (a, b, Z = a_T_b, L), a != b, adds 1/2 r^T L r to the cost,
 * r = log(Z^-1 * global_T_a^-1 * global_T_b) in the tangent order of the pose solve (translation, then rotation), L a 6x6
 * information matrix given as its upper triangle, row-major, in the layout of H (21 floats).  Unlike a prior it fixes no gauge.
 * Where it enters:
 *  - the pose step of the alternating scheme and bba_estimate_frame_pose: each end that is in the step's keyframe list sees the
 *    term as a prior, with the other end held at its pose at the start of the step; when both ends are in the list each also
 *    gets a damping anchor at its own start pose (DESIGN.md 3.12).  An end outside the list (inactive, or every keyframe but
 *    the one of bba_estimate_frame_pose) keeps its pose.  The frames of bba_estimate_frame_poses_for_frames get no terms.
 *  - the PCG scheme: the exact 12x12 terms of both pose unknowns, with the gauge keyframe fixed.
 * A handle without constraints runs exactly the code it ran before they existed.  With several ranks every rank makes the same
 * calls, as it adds the same keyframes, and so gets the same ids.
 *  bba_add_keyframe_pose_constraints: constraints [count]; writes the ids they get to out_ids [count] (may be NULL).  Ids come
 *    from a counter of the handle and are never reused.  BBA_ERR_INVALID_ARGUMENT for an unknown keyframe, a == b, a non-finite
 *    value, a zero quaternion or an L that is not positive semi-definite (the test of bba_set_keyframe_pose_priors); the
 *    arguments are checked before anything changes, and a failed call leaves the handle unchanged.  The call reserves what the
 *    bundle adjustment needs for the new count.
 *  bba_remove_keyframe_pose_constraints: removes ids [count]; count = -1 removes every constraint (ids is not read).  An
 *    unknown id refuses the whole call.
 *  bba_get_keyframe_pose_constraints: front-end call (the published constraints, in id order): *count = their number; at most
 *    capacity of them are written to ids / out (either may be NULL).
 * The add and remove calls are BA-side calls and publish. */
typedef struct {
  int keyframe_a, keyframe_b;
  float a_T_b[7];        /* Z = global_T_a^-1 * global_T_b at the constraint's optimum (qx qy qz qw tx ty tz) */
  float information[21]; /* L's upper triangle, row-major */
} bba_pose_constraint;
bba_status bba_add_keyframe_pose_constraints(bba_handle h, int count, const bba_pose_constraint* constraints, int* out_ids);
bba_status bba_remove_keyframe_pose_constraints(bba_handle h, int count, const int* ids);
bba_status bba_get_keyframe_pose_constraints(bba_handle h, int capacity, int* ids, bba_pose_constraint* out, int* count);

/* depth_params_ / cameras (direct_ba.h:243-297; SetColorCamera etc.).  The getters bba_get_intrinsics, bba_get_residual_types,
 * bba_get_cfactor_host and bba_cfactor_size are front-end calls (the published cameras, a, residual types and cfactor; the
 * cfactor read waits for its publication on `stream`). */
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
/* Parity hook for the pose kernel as the BA pose step runs it: one launch over a work list of `count` distinct keyframes
 * (ids [count], each evaluated at its own global_T_frame [count][7]), in groups of 8, with the record packing and -- for the
 * PRE variants -- the surfel stream in spatial order with per-chunk boxes that the pose step builds first (the spatial order
 * itself is rebuilt when the surfel count changed or new surfels were set since it was built).  variant = BBA_POSE_VARIANT_AUTO picks the instantiation
 * the pose step would (PRE from 4 keyframes with descriptor residuals, the tile from the surfel count and the SM count);
 * any other value forces that (surfel tile, PRE) instantiation.  with_stats = 0 runs the kernel without the residual costs
 * and stage counters, as the pose step does after its first Gauss-Newton iteration.
 * Outputs are indexed by KEYFRAME ID over all keyframe_count keyframes, listed or not (a keyframe outside the list reads back
 * zeros unless the kernel wrote to its record): H [keyframe_count][21] (upper triangle, row-major), b [keyframe_count][6],
 * counts [keyframe_count][4] = {in image, depth ok, associated, photometric} (the first two stay 0 without stats), costs
 * [keyframe_count][3] = {depth, descriptor 1, descriptor 2} (written only with stats; may be NULL without).  Every
 * keyframe's accumulator and counters are cleared before the launch and after the read-back.  Synchronises the stream. */
typedef enum {
  BBA_POSE_VARIANT_AUTO = 0,
  BBA_POSE_VARIANT_256_PRE = 1,   /* 256-surfel tiles, precomputed per-surfel frames in spatial order, culled chunks */
  BBA_POSE_VARIANT_512_PRE = 2,
  BBA_POSE_VARIANT_256 = 3,       /* 256-surfel tiles, tangent points derived per pair */
  BBA_POSE_VARIANT_512 = 4,
  BBA_POSE_VARIANT_1024 = 5
} bba_pose_variant;
bba_status bba_debug_pose_coeffs_batch(bba_handle h, int count, const int* keyframe_ids, const float* global_T_frame, int variant,
                                       int with_stats, double* H, double* b, uint64_t* counts, double* costs, void* stream);
/* Forces the number of keyframes that share one staged surfel tile in every later launch of the pose kernel (1 .. 64; 0, the
 * default: the library's choice).  The results do not depend on it beyond the order of the default mode's floating-point
 * sums; in the deterministic mode they are the same bits.  For tests and timing. */
bba_status bba_debug_set_pose_group(bba_handle h, int keyframes);
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
/* The device buffers of a frame that is not a keyframe, as bba_estimate_frame_pose_for_frame takes them. */
typedef struct {
  const uint16_t* depth;      size_t depth_pitch;
  const uint16_t* normals;    size_t normals_pitch;
  const uint8_t*  color_rgba; size_t color_pitch;   /* uchar4, .w = luma */
} bba_frame_buffers;
/* bba_estimate_frame_pose_for_frame for many entries in one call.  An entry is one (frame, initial pose) pair: entry i tracks
 * frames[frame_of_entry[i]] (frames[i] when frame_of_entry is NULL) from global_T_frame_initial[i] ([count][7]) against the
 * current surfels, with the Gauss-Newton loop, iteration limit (30) and convergence test of the single-frame call, and writes
 * global_T_frame_estimate[i] ([count][7]), iterations[i] and converged[i] (either array may be NULL).  A frame may appear in
 * several entries: several initial poses for one frame (relocalisation hypotheses), or one pose per frame of a trajectory.
 * With at_estimate ([count], may be NULL) entry i also gets what bba_accumulate_pose_coeffs returns at its returned pose -- H, b,
 * the stage counts and the costs -- to rank hypotheses by association count or cost; that costs one more pose-kernel launch per
 * chunk.
 * The entries ride through the pose step as temporary entries behind the keyframes, in chunks of at most
 * max_keyframes - keyframe_count entries, in entry order: one chunk runs one luma extraction launch for its distinct frames and
 * one pose step for all its entries.  With no free keyframe slot the call returns BBA_ERR_STATE; nothing is reallocated on the
 * pose path.  The frames' luma textures come from a library-owned pool, allocated on first use and never larger than the number
 * of free slots.  When the call returns the handle is as it was (keyframes, poses, activations, co-visibility, surfels); only the
 * spatial order of the surfels may have been rebuilt.  BBA_ERR_INVALID_ARGUMENT: a NULL array, count or frame_count < 1, a frame
 * index out of range (or count > frame_count without frame_of_entry), a NULL frame buffer or a pitch too small; BBA_ERR_UNSUPPORTED:
 * world_size > 1.  Arguments are checked before anything is enqueued, and a failed check leaves the handle unchanged.  A BA-side
 * call; synchronises the stream. */
bba_status bba_estimate_frame_poses_for_frames(bba_handle h, int frame_count, const bba_frame_buffers* frames, int count,
                                               const int* frame_of_entry, const float* global_T_frame_initial,
                                               float* global_T_frame_estimate, int* iterations, int* converged,
                                               bba_pose_coeffs* at_estimate, void* stream);
/* UpdateSurfelActivationCUDA (kernels.h:262-269, kernel_surfel_activation.cc:39-67) */
bba_status bba_update_surfel_activation(bba_handle h, void* stream);
/* OptimizeGeometryIterationCUDA (kernels.h:234-244, kernel_opt_geometry.cc:80-201) */
bba_status bba_optimize_geometry_iteration(bba_handle h, void* stream);
/* Carries the keyframes' pose changes since original_keyframe_T_global over to the surfel map (not in the reference; DESIGN.md
 * §3.13), after an outside pose correction written with bba_set_keyframe_states: a caller's pose graph after a loop closure, a
 * re-anchoring to GNSS or motion-capture priors, a relocalisation.
 * original_keyframe_T_global [count][7]: frame_T_global of keyframes 0 .. count-1 before the correction (RememberKeyframePoses).
 * Keyframe k's change is D_k = global_T_frame[k] * original_keyframe_T_global[k]; a keyframe whose current pose inverts
 * (bba_host_se3_inverse) to its original bit for bit is unmoved.  The voters of a surfel are the keyframes k < count it is
 * associated with at their original poses (the association test of the geometry passes, with the current cameras, a and
 * cfactor); without one, the keyframe whose original camera centre is nearest (the smaller id on a tie).  A surfel whose voters
 * are all unmoved keeps its bits; any other gets p + sum_k (D_k p - p) / |voters| and the packed normalised sum of R_k n.
 * Radius, colour, descriptors and active flags are not touched; deleted surfels (x = NaN) are skipped.  The result of a surfel
 * depends on nothing but its own row and the keyframes, bit for bit, with any number of ranks.
 * *moved: surfels whose rows changed; *unobserved: surfels without an associated keyframe.  Either may be NULL; a non-NULL one
 * synchronises the stream (with several ranks, every rank must pass the same NULL-ness: the counts are summed over the ranks).
 * BBA_ERR_INVALID_ARGUMENT: count < 0 or > the keyframe count, a NULL original_keyframe_T_global with count > 0, a non-finite
 * value or a zero quaternion; arguments are checked before anything is enqueued, and a failed check changes nothing.  count = 0
 * or an empty map: nothing to do.  A BA-side call. */
bba_status bba_deform_surfels(bba_handle h, int count, const float* original_keyframe_T_global, uint32_t* moved, uint32_t* unobserved,
                              void* stream);
/* Optimises the keyframe pose graph on the device (DESIGN.md §3.14): what the reference's PoseGraphOptimizer
 * (pose_graph_optimizer.cc, g2o + CSparse, called from loop_detector.cc after a loop closure) does, over the handle's own pose
 * terms.  It minimises over the keyframe poses
 *   sum_priors 1/2 r^T L r + sum_constraints 1/2 r^T L r + sum_chain 1/2 r^T L_o r
 * with the priors and constraints of bba_set_keyframe_pose_priors / bba_add_keyframe_pose_constraints (the pose-only terms of the
 * BA cost) and, with use_odometry_chain, one edge (k, k + 1) per consecutive pair of keyframe ids whose Z = T_k^-1 T_{k+1} is taken
 * at the poses the call starts from (fp64, rounded to fp32) and whose L is odometry_information (the reference's
 * add_current_state_odometry_constraints).  The chain lives for the call only.  A loop edge is a constraint added first; it stays
 * on the handle for the BA that follows (remove it afterwards for the reference's throw-away edge).
 * Held keyframes keep their poses bit for bit: gauge_keyframe (-1: none; 0 in a zero-initialised struct, the reference's "vertex
 * 0 fixed"), every keyframe that no term touches, and in every connected component of the edges (constraints and chain) with
 * neither the gauge nor a prior, its lowest id.  Every other keyframe is an unknown, whatever its activation.
 * Gauss-Newton as in the reference: at the current poses H delta = -b (the PCG scheme's update T <- T exp(delta)) is solved by
 * PCG to a relative residual of 1e-10 (at most 6 x unknowns iterations), with the block-tridiagonal part of H in keyframe order
 * as its preconditioner; a step that raises the cost is taken back and ends the call; the call stops after max_iterations (<= 0:
 * 20, the reference's kMaxIterations) or when every component of a step is at most 1e-7, or 2^-19 of its pose's scale (1 for a
 * rotation, max(1, |t|_inf) for a translation) when that is larger: the resolution of fp32 poses (converged; that step is not
 * applied).
 * Poses stay fp32 between iterations; linearisation and solve run in fp64.  No float atomics: the result is bit-identical from
 * run to run, in the deterministic mode or not, and on every rank (each rank solves the whole graph; there is no exchange).
 * The free keyframes' poses are written back and published once; activations, priors, constraints, surfels, co-visibility and
 * the spatial order are not touched.  Synchronises the stream once.  result (may be NULL): Gauss-Newton iterations that solved a
 * system, converged, the PCG iterations summed, the held keyframes, and the cost at the start and at the end (never above it).
 * BBA_ERR_INVALID_ARGUMENT: a NULL options, a gauge outside [-1, keyframe count), or use_odometry_chain with a non-finite
 * odometry_information or one that is not positive semi-definite (the test of bba_set_keyframe_pose_priors); checked before
 * anything is enqueued, and a refused call changes nothing.  Fewer than two keyframes and no prior: nothing to do, a zero
 * result.  A BA-side call. */
typedef struct {
  int gauge_keyframe;              /* -1: none */
  int max_iterations;              /* <= 0: 20 */
  int use_odometry_chain;
  float odometry_information[21];  /* L_o's upper triangle, row-major (translation, then rotation) */
} bba_pose_graph_options;
typedef struct {
  int iterations, converged, linear_iterations, held_keyframes;
  double initial_cost, final_cost;
} bba_pose_graph_result;
bba_status bba_optimize_pose_graph(bba_handle h, const bba_pose_graph_options* options, bba_pose_graph_result* result, void* stream);
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

/* Parity hook for the PCG solver (direct_ba_pcg.cc:312-638, kernel_pcg.cu:179-1351).  Runs the solver's own sequence on the
 * handle's state with the gauge keyframe o->pcg_gauge_keyframe (>= 0): the init pass (PCGInitCUDA for every keyframe), PCGInit2,
 * `step` complete inner steps (PCGStep1 sweep, PCGStep2, PCGStep3), then inner step `step` itself, copying its intermediate
 * states into *out.  With `apply` != 0 it then applies delta as the solver does: surfels, cfactors, poses, intrinsics.
 * Vectors are host buffers of *unknown_count floats; NULL vectors are not copied.  Call with out = NULL to query the count.
 * Single-GPU handles only (world_size 1).
 * step = 0 returns the building blocks of the first step: r and M of the init pass, p0, g = J^T W J p0, alpha_n, alpha_d. */
typedef struct bba_pcg_probe {
  /* after the PCGStep1 sweep of inner step `step` */
  float* r;                /* residual */
  float* M;                /* diag(J^T W J) of the init pass */
  float* p;                /* search direction */
  float* g;                /* J^T W J p */
  float* delta;            /* solution so far */
  double alpha_n;          /* r^T M^-1 r (before this step) */
  double alpha_d;          /* p^T (J^T W J + lambda) p, the lambda / prior term counted once per keyframe */
  /* after PCGStep2 */
  float* r_step2;
  float* delta_step2;
  float* z;                /* M^-1 r (held in the g vector) */
  double beta_n;           /* z^T r */
  /* after PCGStep3 */
  float* p_step3;
  float* g_step3;          /* cleared for the next sweep */
  double alpha_d_step3;    /* re-armed with the lambda / prior term of the next step */
} bba_pcg_probe;
bba_status bba_pcg_debug(bba_handle h, const bba_ba_options* o, int step, int apply, uint32_t* unknown_count, bba_pcg_probe* out,
                         void* stream);

/* OptimizeIntrinsicsCUDA (kernels.h:246-260, kernel_opt_intrinsics.cc:39-281) */
bba_status bba_optimize_intrinsics(bba_handle h, int optimize_depth_intrinsics, int optimize_color_intrinsics, void* stream);
/* Parity hook for the intrinsics step: the normal equations bba_optimize_intrinsics accumulates, read back before the Schur
 * complement touches them (in the deterministic mode: the rounded exact sums).  The first half of the step itself runs, nothing
 * of the handle's state changes.  sums [34] (host, fp64): [0..14] upper triangle of the 5x5 A over (fx^-1, fy^-1, cx^-1, cy^-1, a),
 * [15..19] b1, [20..29] upper triangle of the colour camera's 4x4 H, [30..33] its b.  cells [8][cf_width * cf_height] (host,
 * fp32): rows 0..4 = B, 5 = D, 6 = b2, 7 = the observation count of each sparse cell.  Without surfels or keyframes everything
 * reads back zero.  Synchronises the stream. */
bba_status bba_debug_intrinsics_coeffs(bba_handle h, int optimize_depth_intrinsics, int optimize_color_intrinsics, double* sums,
                                       float* cells, void* stream);
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

/* ---- local groups: the ranks of a multi-GPU job as handles of ONE process (DESIGN.md "Local groups") ----
 * Each member is driven by its own host thread; the library exchanges between them itself, through device memory and CUDA
 * events (no callback, NCCL, MPI or IPC), across the GPUs of one node or with several ranks on one GPU.  The all-reduce sums
 * the ranks' buffers in rank order 0..N-1 on every rank, so the replicas stay equal bit for bit.
 * Threading contract:
 *  - each member's BA-side calls run on its own thread, with that thread's current device set to the member's device;
 *  - all members make the same sequence of BA-side calls (as the ranks of a multi-process job do);
 *  - front-end calls stay per handle, as above.
 * A BA-side call on a member that returns an error poisons the group: every exchange of every member waiting in it, and every
 * later one, fails at once with BBA_ERR_STATE, so no rank waits for one that returned early.  bba_local_group_reset clears the
 * poison, once every member's thread has returned. */
typedef struct bba_local_group_s* bba_local_group;
/* ranks[i] is the handle of rank i (created with world_size == count, rank == i), all in this process, <= 9 ranks.  Devices must be
 * equal or peer-capable (else BBA_ERR_UNSUPPORTED).  peer_stores: map every replica into every rank (needs equal surfels_size and
 * pitch): the geometry kernels then store into every replica and the geometry exchange is a barrier, as after bba_peer_import;
 * replacing a member's surfel buffer or flags (bba_set_surfels*, bba_set_active_flags) then needs a new group.  Replaces each
 * member's collective; arguments are checked before anything changes.  bba_set_collective and bba_peer_import on a member
 * return BBA_ERR_STATE.  Enables peer access between the members' distinct devices (left enabled by destroy). */
bba_status bba_local_group_create(const bba_handle* ranks, int count, int peer_stores, bba_local_group* out);
bba_status bba_local_group_reset(bba_local_group g);   /* clears the poisoned state */
/* Poisons the group from outside the library: for a member's thread that gives up between calls (an exception of the caller's
 * own code), so that the other members' exchanges return instead of waiting for it. */
bba_status bba_local_group_poison(bba_local_group g);
void       bba_local_group_destroy(bba_local_group g); /* before bba_destroy of any member; restores "no collective" */
/* Parity hook: runs the handle's registered exchange (group or bba_set_collective) once on a caller device buffer, on every rank
 * (op: bba_collective_op; count as for bba_collective_fn).  Stream-ordered, does not synchronise. */
bba_status bba_debug_collective(bba_handle h, int op, void* device_buffer, size_t count, void* stream);

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
 * ComputeMinMaxDepthCUDA does.  The raw depth and rgb are used as they are; bba_preprocess_raw_frame below adds the
 * reference's median densify filter and depth / colour pyramid levels in front of the same stages.
 * Front-end call (both functions): the published depth camera, a and cfactor. */
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

/* The same preprocessing of a frame as the sensor delivers it: the rest of BadSlam::PreprocessFrame (bad_slam.cc:649-689), which
 * the reference runs on the host, is a stage 0 of the same kernel launch:
 *   median_filter_and_densify_iterations = n (1..8): n passes of MedianFilterAndDensifyDepthMap (preprocessing.cc:40-85) over
 *     the raw depth, a 3x3 median of the non-zero pixels wherever there are at least 2 (holes are filled);
 *   pyramid_level_for_depth = L (1..3): the raw depth is raw_depth_width x raw_depth_height and is downscaled to the depth
 *     camera's size, which must be Camera::Scaled(2^-L) of it (int(W / 2^L + 0.5) x int(H / 2^L + 0.5)), by the median of the
 *     non-zero pixels of each box (Image::DownscaleUsingMedianWhileExcluding(0, ...), libvis image.h:1003-1053).  Sizes whose
 *     boxes would exceed 2^L pixels per axis (W > w 2^L, e.g. W = 4k + 1 at L = 2) return BBA_ERR_UNSUPPORTED;
 *   pyramid_level_for_color = L (1..3): rgb is rgb_width x rgb_height = (color width 2^L) x (color height 2^L) and is halved L
 *     times with truncation (ImagePyramid, DownscaleToHalfSize: a/4 + b/4 + c/4 + d/4 per channel) before the luma.
 * Median filtering together with depth downscaling returns BBA_ERR_UNSUPPORTED, as the reference refuses it.  The outputs
 * have the depth / colour camera's size and are those of bba_preprocess_frame applied to the stage-0 images, which never exist
 * in memory; with every option 0 the call is bba_preprocess_frame.  Sizes, levels and counts are checked before anything is
 * enqueued (BBA_ERR_INVALID_ARGUMENT). */
typedef struct {
  bba_preprocess_options base;
  int median_filter_and_densify_iterations;   /* BadSlamConfig, default 0 (bad_slam_config.h:104-109); 0..8 */
  int pyramid_level_for_depth;                /* default 0 (:74-78); 0..3 */
  int pyramid_level_for_color;                /* default 0 (:80-86); 0..3 */
} bba_raw_frame_options;
bba_status bba_preprocess_raw_frame(bba_handle h, const bba_raw_frame_options* options,
                                    const uint16_t* device_raw_depth, size_t raw_depth_pitch,
                                    int raw_depth_width, int raw_depth_height,
                                    const uint8_t* device_rgb, size_t rgb_pitch, int rgb_width, int rgb_height,
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
 * .w = luma); poses are base_T_frame as {qx,qy,qz,qw,tx,ty,tz}.  Uses the handle's cameras, depth deformation and residual types.
 * Front-end calls (bba_track_frame_pairwise, bba_track_frame_pairwise_to_frame, bba_track_frames_pairwise and the two parity hooks): the published cameras,
 * a, cfactor, residual types and base keyframe records; a luma staging plane and a pool of frame luma textures of the front end. */
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
  uint32_t kernel_launches; /* kernels the whole call launched (memsets and copies are not counted) */
} bba_odometry_result;
bba_status bba_track_frame_pairwise(bba_handle h, const bba_odometry_options* options, int base_keyframe_id,
                                    const uint16_t* device_depth, size_t depth_pitch,
                                    const uint16_t* device_normals, size_t normals_pitch,
                                    const uint8_t* device_color_rgba, size_t color_pitch,
                                    const float base_T_frame_initial_1[7], const float base_T_frame_initial_2[7],
                                    float base_T_frame_estimate[7], bba_odometry_result* result, void* stream);
/* The same against a base frame that is not a keyframe (yet): its preprocessed depth, normals and uchar4 colour buffers, what
 * bba_add_keyframe takes -- the keyframe BadSlam's odometry tracks against while it still waits in the BA thread's queue
 * (bad_slam.cc:831-950).  The result equals that of bba_track_frame_pairwise against the same buffers registered as a
 * keyframe, bit for bit, with the same kernel_launches (one luma launch serves both frames).  Nothing of the base is kept.
 * Both single-pair calls are the one-entry case of bba_track_frames_pairwise below, with its checks: a failed check enqueues
 * nothing. */
bba_status bba_track_frame_pairwise_to_frame(bba_handle h, const bba_odometry_options* options,
                                             const uint16_t* base_depth, size_t base_depth_pitch,
                                             const uint16_t* base_normals, size_t base_normals_pitch,
                                             const uint8_t* base_color_rgba, size_t base_color_pitch,
                                             const uint16_t* device_depth, size_t depth_pitch,
                                             const uint16_t* device_normals, size_t normals_pitch,
                                             const uint8_t* device_color_rgba, size_t color_pitch,
                                             const float base_T_frame_initial_1[7], const float base_T_frame_initial_2[7],
                                             float base_T_frame_estimate[7], bba_odometry_result* result, void* stream);
/* bba_track_frame_pairwise / bba_track_frame_pairwise_to_frame for many independent (base, tracked frame) pairs in one call, all
 * with the same options: re-tracking every frame against its base keyframe from its deformed pose after the final BA,
 * verifying a frame against several keyframes, or trying more starting poses for one pair.  Entry i tracks
 * frames[entries[i].tracked_frame] against keyframe entries[i].base_keyframe_id (>= 0) or, with -1, against the frame
 * frames[entries[i].base_frame] given as buffers, from base_T_frame_initial_1 (and _2 with test_different_initial_estimates),
 * and writes base_T_frame_estimate[i] ([count][7]) and results[i] ([count], may be NULL).  A frame or keyframe may appear in
 * any number of entries.
 * The entries run in chunks of at most BBA_ODOMETRY_CHUNK_ENTRIES, in entry order.  A chunk runs one luma launch for its distinct
 * frames, one intensity launch, one level-0 launch and one launch per coarser level for all its pyramids, and one tracking
 * launch in which groups of CTAs take the entries in order: 4 + (num_scales - 1) launches per chunk whatever its entry count;
 * results[i].kernel_launches counts the launches of entry i's chunk, *kernel_launches (may be NULL) those of the whole call.
 * The pyramids come from a library-owned pool, allocated on first use and grown to the largest chunk: one pyramid per
 * distinct image and role of a chunk (a base keyframe tracked by ten entries has one base pyramid), at most
 * 2 x BBA_ODOMETRY_CHUNK_ENTRIES.  One pyramid holds the colour-sized intensity plane and, per level, float depth, u16 normals
 * (from level 1 on) and u8 intensity: 2.56 MB at 640x480 with 5 levels from the level sizes, plus the row padding of the
 * pitched allocations.
 * Each entry's result equals that of its own single-pair call up to the order of the sums; in the deterministic mode it equals
 * it bit for bit, whatever else the call holds and in whatever order.  A front-end call like the single-pair calls: every
 * keyframe an entry names must be in the published snapshot.  BBA_ERR_INVALID_ARGUMENT: a NULL array, count or frame_count < 1,
 * a frame index or keyframe id out of range, a NULL frame buffer, a bad pitch, bad num_scales; BBA_ERR_UNSUPPORTED: the depth /
 * colour pyramid combination the single-pair call rejects.  Arguments are checked before anything is enqueued, and a failed
 * check leaves the handle and the launch counter unchanged.  Afterwards the parity hooks below describe the call's last entry.
 * Synchronises the stream once per chunk. */
#define BBA_ODOMETRY_CHUNK_ENTRIES 64
typedef struct {
  int base_keyframe_id;                 /* >= 0: that keyframe is the base; -1: frames[base_frame] is */
  int base_frame;                       /* read only when base_keyframe_id < 0 */
  int tracked_frame;                    /* index into frames */
  float base_T_frame_initial_1[7];
  float base_T_frame_initial_2[7];      /* read only with options->test_different_initial_estimates */
} bba_odometry_entry;
bba_status bba_track_frames_pairwise(bba_handle h, const bba_odometry_options* options, int frame_count, const bba_frame_buffers* frames,
                                     int count, const bba_odometry_entry* entries, float* base_T_frame_estimate /* [count][7] */,
                                     bba_odometry_result* results /* [count], may be NULL */, uint32_t* kernel_launches /* may be NULL */,
                                     void* stream);
/* Parity hooks (the pyramids and normal equations of the LAST bba_track_frame_pairwise call of this handle, device-resident;
 * after bba_track_frames_pairwise, of its last entry):
 *  bba_odometry_get_level: one pyramid level of the base (which = 0) or tracked (1) image into dense host arrays
 *    [height][width] (any may be NULL); *width / *height return the level's size.
 *  bba_odometry_debug_coeffs: AccumulatePoseEstimationCoeffsFromImagesCUDA (kernels.h:181-203) at base_T_frame_a -> H[21], b[6],
 *    residual count / sum, and ComputeCostAndResidualCountFromImagesCUDA (kernels.h:205-223) at both poses -> counts[2], costs[2]. */
bba_status bba_odometry_get_level(bba_handle h, int which, int scale, float* host_depth, uint16_t* host_normals, uint8_t* host_color,
                                  int* width, int* height, void* stream);
bba_status bba_odometry_debug_coeffs(bba_handle h, int scale, int use_gradmag, const float base_T_frame_a[7], const float base_T_frame_b[7],
                                     float H[21], float b[6], uint32_t* residual_count, float* residual_sum,
                                     uint32_t counts[2], float costs[2], void* stream);

/* ---- deterministic mode ----
 * Off by default.  When on, every floating-point sum whose order depends on the scheduling of the GPU goes through an exact,
 * order-independent accumulator (or, in the odometry kernel, a fixed-order sum of per-CTA totals), so that the same inputs on the
 * same GPU model give the same results bit for bit in every run, whatever else runs beside them on other streams.  Covered:
 * bba_bundle_adjust (pose, geometry and intrinsics steps, surfel lifecycle), bba_estimate_frame_pose (both forms),
 * bba_estimate_frame_poses_for_frames, bba_accumulate_pose_coeffs, bba_debug_pose_coeffs_batch, bba_optimize_intrinsics, bba_track_frame_pairwise(_to_frame),
 * bba_track_frames_pairwise,
 * bba_odometry_debug_coeffs and the preprocessing.  The results differ from those of the default mode only by the rounding of
 * those sums.  Not covered: the PCG solver -- bba_bundle_adjust with use_pcg and bba_pcg_debug return BBA_ERR_UNSUPPORTED while
 * the mode is on -- and more than one rank (the setter returns BBA_ERR_UNSUPPORTED for world_size > 1).  A call with
 * time_limit_seconds > 0, or whose progress_function looks at the wall clock, is reproducible only up to the number of iterations
 * it ran; the ms_* timings are measurements, not results.
 * bba_set_deterministic is a BA-side call that takes effect from the next call and publishes; front-end calls use the mode of their
 * snapshot.  Switching it on for the first time allocates the exact sums: 80 bytes per value, max_keyframes x 32 values for the
 * pose kernel and 7 per sparse cell for the intrinsics step (about 11 MB at 640x480 with cell size 4).  bba_get_deterministic is a
 * front-end call (the published mode). */
bba_status bba_set_deterministic(bba_handle h, int on);
bba_status bba_get_deterministic(bba_handle h, int* on);
/* Parity hook for the exact accumulator: deposits the n (< 2^31) device values through the device path, from many CTAs in a
 * scrambled order, and returns the sum rounded to fp64 (bba_host_exact_sum's result).  Synchronises the stream. */
bba_status bba_debug_exact_sum(bba_handle h, const float* device_values, uint64_t n, double* out, void* stream);

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
/* The terms a soft pose prior adds to a keyframe's pose solve at global_T_frame = pose, for the update pose * exp(delta): with
 * r = log(prior^-1 * pose) and J = Jr^-1(r), the inverse right Jacobian of SE(3), H = J^T L J (upper triangle, 21), b = J^T L r
 * (6) and cost = r^T L r / 2, all in fp64.  information: L's upper triangle (21).  Writes nothing if a pointer is NULL. */
void bba_host_pose_prior_terms(const float prior_global_T_frame[7], const float global_T_frame[7], const float information[21],
                               double H[21], double b[6], double* cost);
/* The terms of a soft relative pose constraint at global_T_a = pose_a, global_T_b = pose_b, for the updates pose_a * exp(delta_a)
 * and pose_b * exp(delta_b): with r = log(a_T_b^-1 * pose_a^-1 * pose_b), J_b = Jr^-1(r) and J_a = -Jr^-1(r) Ad(pose_b^-1 pose_a),
 * H = J^T L J over (delta_a, delta_b) (12 x 12 upper triangle, 78), b = J^T L r (12) and cost = r^T L r / 2, all in fp64.
 * Writes nothing if a pointer is NULL. */
void bba_host_pose_constraint_terms(const float a_T_b[7], const float global_T_a[7], const float global_T_b[7],
                                    const float information[21], double H[78], double b[12], double* cost);
int  bba_host_frusta_intersect(const float depth_intrinsics[4], int width, int height,
                               const float global_T_frame_a[7], float min_depth_a, float max_depth_a,
                               const float global_T_frame_b[7], float min_depth_b, float max_depth_b);
/* The exact accumulator of the deterministic mode on the host: the sum of n fp32 values, computed exactly and rounded once to
 * fp64 (to nearest, ties to even), so the result does not depend on the order of the values.  An exact zero gives +0.0.  Non-finite
 * values follow IEEE addition: NaN if there is a NaN or both infinities, else the infinity there is. */
void bba_host_exact_sum(const float* values, size_t n, double* out);

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

/* ExtrapolateAndInterpolateKeyframePoseChanges (trajectory_deformation.cc:45-130) on caller arrays: after a bundle adjustment
 * moved the keyframes, every frame in [start_frame, end_frame] that is not a keyframe is moved with them.  A frame before the
 * first or after the last keyframe gets the change of the nearest keyframe; a frame between two keyframes gets the two
 * keyframes' "old frame to new frame" corrections interpolated by its frame index (translation linearly, rotation by Eigen's
 * Quaternion::slerp, renormalised like Sophus' setQuaternion).  SE3 arithmetic in fp32, like Sophus::SE3f.
 *   keyframe_frame_index        [K]: frame index of each keyframe, >= 0 and strictly increasing
 *   original_keyframe_T_global  [K][7]: each keyframe's frame_T_global before the BA call (RememberKeyframePoses)
 *   keyframe_global_T_frame     [K][7]: each keyframe's global_T_frame after it
 *   frame_global_T_frame        [end_frame + 1][7]: global_T_frame of every frame, updated in place for the non-keyframes in
 *                               [start_frame, end_frame]; nothing else is read or written.  The caller clamps end_frame to its
 *                               frame count - 1 (trajectory_deformation.cc:51).
 * Returns BBA_OK, or BBA_ERR_INVALID_ARGUMENT without writing anything if keyframe_count < 1, an array is NULL, the keyframe
 * frame indices are negative or not strictly increasing, start_frame < 0 or start_frame > end_frame. */
int  bba_host_deform_trajectory(int keyframe_count, const int* keyframe_frame_index, const float* original_keyframe_T_global,
                                const float* keyframe_global_T_frame, int start_frame, int end_frame, float* frame_global_T_frame);

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
