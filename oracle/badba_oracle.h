/* oracle/badba_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement (plain C + OpenMP) of the reference's direct bundle-adjustment
 * hot path (SURVEY.md section 8a).  It exists so that tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline leg can CHECK the CUDA product path; the product
 * never links, imports or calls it.
 *
 * PARITY STATUS: the reference holds NO golden vectors / known-answer tests for
 * this path (SURVEY.md 8c).  The oracle is pinned (a) on the GPU box against the
 * reference's own unmodified CUDA kernels compiled into oracle/_ref (see
 * build_ref.sh + ref_driver.cu; tests/test_gpu_parity.py), (b) against the
 * reference's symbolic residual definitions (scripts/jacobians_derivation.py)
 * through numeric differentiation (tests/test_oracle_jacobians.py) and (c) against
 * the convergence assertions of the reference's tests (tests/test_oracle_convergence.py).
 * The dense fp64 solves follow Eigen (not vendored) => "parity unpinned" for those.
 */
#ifndef BADBA_ORACLE_H
#define BADBA_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { ORC_KF_ACTIVE = 0, ORC_KF_COVIS_ACTIVE = 1, ORC_KF_INACTIVE = 2 };

/* Texture-filter emulation of cudaFilterModeLinear on a normalized-float u8
 * texture (keyframe.cc:67-73): 0 = exact float weights, 1 = weights rounded to
 * nearest 1/256 (CUDA programming guide: 9-bit fixed point, 8 fractional bits),
 * 2 = weights truncated to 1/256, 3 (default) = the measured hardware behaviour (8-bit rounded per-texel product
 * weights, unorm16 result; tools/tex_probe*.cu), 4 = same with the coordinate converted to fixed point first. */
void orc_set_tex_mode(int mode);
int  orc_get_tex_mode(void);
void orc_set_num_threads(int n);
int  orc_get_max_threads(void);

typedef struct {
  int depth_w, depth_h, color_w, color_h;
  float depth_K[4];            /* fx, fy, cx, cy  (PinholeCamera4f::parameters, pixel-corner conv.) */
  float color_K[4];
  float raw_to_float_depth;
  float baseline_fx;
  float a;                     /* depth deformation alpha_1 */
  int   cell;                  /* sparse_surfel_cell_size */
  int   cf_w, cf_h;            /* cfactor grid size = ((w-1)/cell+1, (h-1)/cell+1) */
  float* cfactor;              /* [cf_h][cf_w] dense row-major */
  int use_depth_residuals;
  int use_descriptor_residuals;
} orc_model;

/* Keyframe image set: K stacked dense row-major images. */
typedef struct {
  int K;
  const uint16_t* depth;       /* [K][h][w]   bit15 = invalid, 65535 unknown (kernels.cuh:38-41) */
  const uint16_t* normals;     /* [K][h][w]   2 x s8 (util.cuh:126-146) */
  const uint16_t* radius;      /* [K][h][w]   IEEE half r^2 (cuda_depth_processing.cu:355) */
  const uint8_t*  color;       /* [K][ch][cw][4] uchar4, .w = luma (cuda_image_processing.cu:165-176) */
  float* global_T_frame;       /* [K][7]  qx qy qz qw tx ty tz, updated in place by BA */
  int32_t* activation;         /* [K]     ORC_KF_*, updated in place */
  const float* min_depth;      /* [K] */
  const float* max_depth;      /* [K] */
  uint8_t* covis;              /* [K][K] adjacency (filled by orc_compute_covisibility) */
} orc_keyframes;

/* Per-pose-pass outputs (superset of the reference's debug counters,
 * kernel_opt_pose.cu:224-248, and of SURVEY 8d's byte-model counters). */
typedef struct {
  double H[21];
  double b[6];
  uint64_t n_pair;      /* surfels evaluated */
  uint64_t n_inimg;     /* z>0 and projects into the depth image */
  uint64_t n_depthok;   /* passed valid-depth + depth-threshold + facing tests (KF normal read) */
  uint64_t n_assoc;     /* associated == depth residual count */
  uint64_t n_photo;     /* associated and colour pixel in bounds (2 descriptor residuals each) */
  double cost_depth;    /* sum TukeyResidual */
  double cost_desc1;    /* sum weighted Huber of descriptor residual 1 (the only one the reference's debug sums) */
  double cost_desc2;
} orc_pose_stats;

void orc_compute_covisibility(const orc_model* m, orc_keyframes* kfs);

/* frame_T_global as row-major 3x4 from a global_T_frame pose. */
void orc_frame_T_global(const float global_T_frame[7], float out12[12]);

/* AccumulatePoseEstimationCoeffsCUDA (kernel_opt_pose.cc:39-97 + kernel_opt_pose.cu:251-383)
 * for keyframe k evaluated at pose frame_T_global (row-major 3x4). */
void orc_pose_coeffs(const orc_model* m, const orc_keyframes* kfs, int k,
                     const float frame_T_global[12],
                     const float* surfels, int pitch, uint32_t n,
                     orc_pose_stats* out);

/* DirectBA::EstimateFramePose (direct_ba_alternating.cc:42-283). Returns #iterations, sets *converged. */
int orc_estimate_frame_pose(const orc_model* m, const orc_keyframes* kfs, int k,
                            const float global_T_frame_init[7],
                            const float* surfels, int pitch, uint32_t n,
                            float global_T_frame_out[7], int* converged, int max_iterations);

/* UpdateSurfelActivationCUDA (kernel_surfel_activation.cc:39-67). */
void orc_update_activation(const orc_model* m, const orc_keyframes* kfs,
                           const float* surfels, int pitch, uint32_t n, uint8_t* active);

/* OptimizeGeometryIterationCUDA (kernel_opt_geometry.cc:80-201); rows 8..16 are scratch. */
void orc_optimize_geometry_iteration(const orc_model* m, const orc_keyframes* kfs,
                                     float* surfels, int pitch, uint32_t n, const uint8_t* active);

/* OptimizeIntrinsicsCUDA (kernel_opt_intrinsics.cc:39-281); updates m->depth_K / color_K / a / cfactor. */
void orc_optimize_intrinsics(orc_model* m, const orc_keyframes* kfs,
                             const float* surfels, int pitch, uint32_t n,
                             int optimize_depth_intrinsics, int optimize_color_intrinsics);

typedef struct {
  int optimize_depth_intrinsics, optimize_color_intrinsics;
  int do_surfel_updates;
  int optimize_poses, optimize_geometry;
  int min_iterations, max_iterations;
  int active_keyframe_window_start, active_keyframe_window_end;
  int max_pose_iterations;     /* 30 (direct_ba_alternating.cc:130) */
  /* do_surfel_updates: in-loop surfel creation / merge (direct_ba_alternating.cc:399-430,489-541) */
  int ba_iteration_count;
  int32_t* last_active_in_ba_iteration;   /* [K] keyframe.h:113-128, updated in place */
  int32_t* last_covis_in_ba_iteration;    /* [K] */
  float surfel_merge_dist_factor;
  int min_observation_count;
  uint32_t max_surfels;
} orc_ba_options;

typedef struct {
  int iterations_done;
  int converged;
  /* counts at the starting state of the LAST executed iteration's pose step */
  uint64_t n_assoc, n_photo;
  double cost;
  int pose_iterations_total;   /* sum over keyframes and outer iterations of GN iterations */
  uint32_t surfels_size, surfels_created, surfels_merged;
} orc_ba_result;

/* DirectBA::BundleAdjustmentAlternating (direct_ba_alternating.cc:285-738), without
 * the surfel lifecycle (creation / merge / delete / compaction). */
void orc_bundle_adjust(orc_model* m, orc_keyframes* kfs,
                       float* surfels, int pitch, uint32_t n, uint8_t* active,
                       const orc_ba_options* opt, orc_ba_result* res);

/* DirectBA::BundleAdjustmentPCG (direct_ba_pcg.cc:43-819; kernels kernel_pcg.cu:179-1372) without the surfel lifecycle.
 * gauge_keyframe: the keyframe held fixed (the reference draws rand() % K per iteration, direct_ba_pcg.cc:324). */
typedef struct {
  int optimize_poses, optimize_geometry, optimize_depth_intrinsics, optimize_color_intrinsics;
  int min_iterations, max_iterations, max_inner_iterations, gauge_keyframe;
  /* do_surfel_updates (direct_ba_pcg.cc:180-206,644-690,775-815); same meaning as in orc_ba_options */
  int do_surfel_updates;
  int increase_ba_iteration_count;        /* 0: the loop is followed by one more merge + compaction (:775-815) */
  int ba_iteration_count;
  int32_t* last_active_in_ba_iteration;   /* [K], updated */
  int32_t* last_covis_in_ba_iteration;    /* [K], updated */
  float surfel_merge_dist_factor;
  int min_observation_count;
  uint32_t max_surfels;
} orc_pcg_options;
typedef struct {
  int iterations_done, converged, inner_iterations_total;
  float last_r_norm;
  uint32_t surfels_size, surfels_created, surfels_merged;
} orc_pcg_result;
void orc_bundle_adjust_pcg(orc_model* m, orc_keyframes* kfs, float* surfels, int pitch, uint32_t n, uint8_t* active,
                           const orc_pcg_options* opt, orc_pcg_result* res);

/* DirectBA::PerformBASchemeEndTasks (direct_ba.cc:566-653) without the final merge: delete surfels with fewer than
 * min_observation_count observations or more free-space violations than observations, give the others the smallest observed
 * radius^2, compact.  Returns the number of deleted surfels; *n is updated to the new surfels_size. */
uint32_t orc_end_tasks(const orc_model* m, const orc_keyframes* kfs, float* surfels, int pitch, uint32_t* n,
                       int min_observation_count);
/* ... with do_surfel_updates: first the merge over the keyframes that were active in this BA iteration block (direct_ba.cc:577-601) */
uint32_t orc_end_tasks_with_merge(const orc_model* m, const orc_keyframes* kfs, float* surfels, int pitch, uint32_t* n,
                                  int min_observation_count, const int32_t* last_active_in_ba_iteration, int ba_iteration_count,
                                  float surfel_merge_dist_factor);

/* In-loop surfel lifecycle with the deterministic resolution of the reference's atomicCAS races described in badba_oracle.c:
 * DirectBA::CreateSurfelsForKeyframe (direct_ba.cc:340-405) -> returns the number of surfels appended (*n updated);
 * DetermineSupportingSurfelsAndMergeSurfelsCUDA (kernel_supporting_surfels.cc:40-118) -> returns the number deleted;
 * CompactSurfelsCUDA (kernel_compact_surfels.cu:159-279) -> returns the new surfels_size. */
uint32_t orc_create_surfels_for_keyframe(const orc_model* m, const orc_keyframes* kfs, int k, int filter_new_surfels,
                                         int min_observation_count, float* surfels, int pitch, uint32_t* n, uint32_t max_surfels);
uint32_t orc_merge_surfels_for_keyframe(const orc_model* m, const orc_keyframes* kfs, int k, float merge_dist_factor,
                                        float* surfels, int pitch, uint32_t n);
uint32_t orc_compact_surfels(float* surfels, int pitch, uint32_t n, uint8_t* active);

/* Parity hook for the PCG building blocks: r, M after the init pass, p0, g after one J^T W J p sweep, {alpha_n, alpha_d}. */
uint32_t orc_pcg_debug(const orc_model* m, const orc_keyframes* kfs, const float* surfels, int pitch, uint32_t n,
                       const orc_pcg_options* opt, float* out_r, float* out_M, float* out_p, float* out_g, double* out_scalars);

/* Residual-level access for Jacobian tests: evaluates the raw residuals of one
 * (surfel, keyframe) pair.  Returns bit0 = associated, bit1 = photometric valid.
 * r[0] = depth, r[1], r[2] = descriptor; J_pose (3 x 6) are the reference's
 * analytic pose Jacobians (kernel_opt_pose.cu:45-142); J_geom (3 x 3) its
 * Jacobians wrt (t along normal, d1, d2) (kernel_opt_geometry.cu:118-231). */
int orc_pair_residuals(const orc_model* m, const orc_keyframes* kfs, int k,
                       const float frame_T_global[12],
                       const float surfel[8], float r[3], float J_pose[18], float J_geom[9]);
/* Same, plus the intermediate quantities (for the known-answer tests):
 * dbg[16] = px, py, calibrated depth, inv_stddev, colour x, colour y, t1x, t1y, t2x, t2y, gx1, gy1, gx2, gy2, 0, 0 */
int orc_pair_residuals_debug(const orc_model* m, const orc_keyframes* kfs, int k,
                             const float frame_T_global[12],
                             const float surfel[8], float r[3], float J_pose[18], float J_geom[9], float dbg[16]);

/* Sampling helper exposed for the generator / hardware validation. */
float orc_tex_luma(const orc_model* m, const orc_keyframes* kfs, int k, float x, float y);

/* ---- keyframe preprocessing (preprocess_oracle.c; SURVEY.md 8(f3)) ---- dense row-major images */
uint16_t orc_float_to_half(float f);   /* __float2half_rn as bits */
void orc_bilateral_filter_and_depth_cutoff(int w, int h, float sigma_xy, float sigma_value, float radius_factor,
                                           uint16_t max_depth, float raw_to_float, const uint16_t* in, uint16_t* out);
void orc_compute_normals(const orc_model* m, const uint16_t* in_depth, uint16_t* out_depth, uint16_t* out_normals);
void orc_compute_point_radii_and_remove_isolated_pixels(const orc_model* m, const uint16_t* depth, uint16_t* radius, uint16_t* out_depth);
void orc_compute_min_max_depth(int w, int h, float raw_to_float, const uint16_t* depth, float* min_depth, float* max_depth);
void orc_compute_brightness(int w, int h, const uint8_t* rgb, uint8_t* rgba);
void orc_preprocess_frame(const orc_model* m, float sigma_xy, float sigma_inv_depth, float radius_factor, float max_depth_m,
                          const uint16_t* raw_depth, const uint8_t* rgb, uint16_t* out_depth, uint16_t* out_normals,
                          uint16_t* out_radius, uint8_t* out_rgba, float* min_depth, float* max_depth);

/* Small pose utilities for the python harness. */
void orc_se3_exp(const float a[6], float out[7]);
void orc_se3_log(const float T[7], float out[6]);
void orc_se3_mul(const float A[7], const float B[7], float out[7]);
void orc_se3_inverse(const float A[7], float out[7]);

#ifdef __cplusplus
}
#endif
#endif
