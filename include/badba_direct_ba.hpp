// include/badba_direct_ba.hpp -- header-only C++ adaptor that keeps the reference's own signatures on top of the
// C ABI of include/badba.h, so that BadSlam::RunBundleAdjustment (applications/badslam/src/badslam/bad_slam.cc:485-540)
// and the BA thread (bad_slam.cc:1196-1317) can call the sm_90a backend without source changes beyond the include.
//
// It mirrors  class vis::DirectBA  (applications/badslam/src/badslam/direct_ba.h:65-550):
//   ctor                      direct_ba.h:73-88
//   AddKeyframe               direct_ba.h:95      (takes the keyframe's device buffers, keyframe.h:160-200)
//   EstimateFramePose         direct_ba.h:122-129
//   BundleAdjustment          direct_ba.h:143-162
//   accessors                 direct_ba.h:243-377
// The reference passes Eigen / Sophus / libvis types; this adaptor is templated on them so that it compiles both
// inside the reference tree (SE3f = Sophus::SE3f, PinholeCamera4f = vis::PinholeCamera4f, CUDABuffer<T>) and in a
// tree without Eigen (any type with .data() returning {qx,qy,qz,qw,tx,ty,tz} and .parameters()).
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <exception>
#include <fstream>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>
#include <stdexcept>
#include <string>
#include <utility>

#include "badba.h"

namespace badba {

class Error : public std::runtime_error {
 public:
  Error(bba_status s, const std::string& what) : std::runtime_error(what), status(s) {}
  bba_status status;
};

// A pitched device image as the reference's CUDABuffer_<T> exposes it (cuda_buffer.cuh:112-118).
template <typename T>
struct DeviceImage {
  const T* address;
  size_t pitch_bytes;
};

// The buffers of a frame that is not a keyframe, as EstimateFramePose takes them.
struct FrameImages {
  DeviceImage<uint16_t> depth;
  DeviceImage<uint16_t> normals;
  DeviceImage<uint8_t> color_rgba;
};

template <typename T>
struct MutableDeviceImage {
  T* address;
  size_t pitch_bytes;
};

// Stand-in for libvis' Timer (timing.h:114) when the caller passes none: BundleAdjustment is templated on the timer type and
// only needs GetTimeSinceStart() (direct_ba_alternating.cc:703-709).
struct NoTimer {
  double GetTimeSinceStart() const { return 0; }
};

template <typename SE3f, typename PinholeCamera4f>
class DirectBA {
 public:
  DirectBA(int max_surfel_count, float raw_to_float_depth, float baseline_fx, int sparse_surfel_cell_size,
           float surfel_merge_dist_factor, int min_observation_count_while_bootstrapping_1,
           int min_observation_count_while_bootstrapping_2, int min_observation_count,
           const PinholeCamera4f& color_camera_initial_estimate, const PinholeCamera4f& depth_camera_initial_estimate,
           int /*pyramid_level_for_color*/, bool use_depth_residuals, bool use_descriptor_residuals, int max_keyframes = 2500,
           int device = 0, int rank = 0, int world_size = 1) {
    bba_config c{};
    c.depth_width = depth_camera_initial_estimate.width();
    c.depth_height = depth_camera_initial_estimate.height();
    c.color_width = color_camera_initial_estimate.width();
    c.color_height = color_camera_initial_estimate.height();
    for (int i = 0; i < 4; ++i) {
      c.depth_intrinsics[i] = depth_camera_initial_estimate.parameters()[i];
      c.color_intrinsics[i] = color_camera_initial_estimate.parameters()[i];
    }
    c.raw_to_float_depth = raw_to_float_depth;
    c.baseline_fx = baseline_fx;
    c.sparse_surfel_cell_size = sparse_surfel_cell_size;
    c.max_surfel_count = static_cast<uint32_t>(max_surfel_count);
    c.max_keyframes = max_keyframes;
    c.use_depth_residuals = use_depth_residuals;
    c.use_descriptor_residuals = use_descriptor_residuals;
    c.device = device;
    c.rank = rank;
    c.world_size = world_size;
    c.min_observation_count_while_bootstrapping_1 = min_observation_count_while_bootstrapping_1;
    c.min_observation_count_while_bootstrapping_2 = min_observation_count_while_bootstrapping_2;
    c.min_observation_count = min_observation_count;
    c.surfel_merge_dist_factor = surfel_merge_dist_factor;
    min_observation_counts_[0] = min_observation_count_while_bootstrapping_1;
    min_observation_counts_[1] = min_observation_count_while_bootstrapping_2;
    min_observation_counts_[2] = min_observation_count;
    Check(bba_create(&c, &h_), "bba_create");
  }
  ~DirectBA() { bba_destroy(h_); }
  DirectBA(const DirectBA&) = delete;
  DirectBA& operator=(const DirectBA&) = delete;

  // surfels_ / active_surfels_ are owned by the caller exactly as in the reference (direct_ba.cc:122-123).
  void SetSurfelBuffers(float* surfels, size_t pitch_bytes, uint32_t surfels_size, uint8_t* active_surfels) {
    Check(bba_set_surfels(h_, surfels, pitch_bytes, surfels_size), "bba_set_surfels");
    Check(bba_set_active_flags(h_, active_surfels), "bba_set_active_flags");
  }

  // DirectBA::AddKeyframe(const shared_ptr<Keyframe>&): pass keyframe->depth_buffer().ToCUDA() etc.
  int AddKeyframe(cudaStream_t stream, DeviceImage<uint16_t> depth, DeviceImage<uint16_t> normals, DeviceImage<uint16_t> radius,
                  DeviceImage<uint8_t> color_rgba, const SE3f& global_T_frame, float min_depth, float max_depth) {
    return AddKeyframe(stream, -1, depth, normals, radius, color_rgba, global_T_frame, min_depth, max_depth);
  }

  // ... recording the keyframe's frame index in the video (Keyframe::frame_index(), keyframe.h:95), which
  // ExtrapolateAndInterpolateKeyframePoseChanges needs.  The index stays in the adaptor; the library does not use it.
  int AddKeyframe(cudaStream_t stream, int frame_index, DeviceImage<uint16_t> depth, DeviceImage<uint16_t> normals,
                  DeviceImage<uint16_t> radius, DeviceImage<uint8_t> color_rgba, const SE3f& global_T_frame, float min_depth,
                  float max_depth) {
    int id = -1;
    Check(bba_add_keyframe(h_, depth.address, depth.pitch_bytes, normals.address, normals.pitch_bytes, radius.address,
                           radius.pitch_bytes, color_rgba.address, color_rgba.pitch_bytes, global_T_frame.data(), min_depth,
                           max_depth, stream, &id),
          "bba_add_keyframe");
    if (static_cast<size_t>(id) >= keyframe_frame_index_.size()) keyframe_frame_index_.resize(id + 1, -1);
    keyframe_frame_index_[id] = frame_index;
    return id;
  }
  // The frame index given to AddKeyframe (-1: added without one).
  int keyframe_frame_index(int keyframe_id) const { return keyframe_frame_index_.at(keyframe_id); }

  // direct_ba.h:122-129 (frame = an already added keyframe)
  void EstimateFramePose(cudaStream_t stream, const SE3f& global_T_frame_initial_estimate, int keyframe_id,
                         SE3f* out_global_T_frame_estimate, bool /*called_within_ba*/ = false) {
    float out[7];
    Check(bba_estimate_frame_pose(h_, keyframe_id, global_T_frame_initial_estimate.data(), out, nullptr, nullptr, stream),
          "bba_estimate_frame_pose");
    for (int i = 0; i < 7; ++i) out_global_T_frame_estimate->data()[i] = out[i];
  }

  // direct_ba.h:122-129 for a frame that is not a keyframe (depth_buffer, normals_buffer, colour image in place of the
  // texture): frame-to-model tracking against the current surfels.
  void EstimateFramePose(cudaStream_t stream, const SE3f& global_T_frame_initial_estimate, DeviceImage<uint16_t> depth_buffer,
                         DeviceImage<uint16_t> normals_buffer, DeviceImage<uint8_t> color_buffer_rgba,
                         SE3f* out_global_T_frame_estimate, bool /*called_within_ba*/ = false) {
    float out[7];
    Check(bba_estimate_frame_pose_for_frame(h_, depth_buffer.address, depth_buffer.pitch_bytes, normals_buffer.address,
                                            normals_buffer.pitch_bytes, color_buffer_rgba.address, color_buffer_rgba.pitch_bytes,
                                            global_T_frame_initial_estimate.data(), out, nullptr, nullptr, stream),
          "bba_estimate_frame_pose_for_frame");
    std::memcpy(out_global_T_frame_estimate->data(), out, sizeof(out));
  }

  // The same for many entries in one call (bba_estimate_frame_poses_for_frames): entry i tracks frames[frame_of_entry[i]]
  // (frames[i] when frame_of_entry is empty) from global_T_frame_initial_estimates[i]; *out_global_T_frame_estimates gets one
  // estimate per entry and, when given, *at_estimate the pose-kernel coefficients at each estimate.
  void EstimateFramePoses(cudaStream_t stream, const std::vector<FrameImages>& frames,
                          const std::vector<SE3f>& global_T_frame_initial_estimates, std::vector<SE3f>* out_global_T_frame_estimates,
                          const std::vector<int>& frame_of_entry = {}, std::vector<bba_pose_coeffs>* at_estimate = nullptr) {
    const size_t count = global_T_frame_initial_estimates.size();
    const std::vector<bba_frame_buffers> buffers = MakeFrameBuffers(frames);
    std::vector<float> init(7 * count), out(7 * count);
    for (size_t i = 0; i < count; ++i) std::memcpy(init.data() + 7 * i, global_T_frame_initial_estimates[i].data(), sizeof(float) * 7);
    if (at_estimate) at_estimate->resize(count);
    Check(bba_estimate_frame_poses_for_frames(h_, static_cast<int>(frames.size()), buffers.data(), static_cast<int>(count),
                                              frame_of_entry.empty() ? nullptr : frame_of_entry.data(), init.data(), out.data(), nullptr,
                                              nullptr, at_estimate ? at_estimate->data() : nullptr, stream),
          "bba_estimate_frame_poses_for_frames");
    out_global_T_frame_estimates->resize(count);
    for (size_t i = 0; i < count; ++i) std::memcpy((*out_global_T_frame_estimates)[i].data(), out.data() + 7 * i, sizeof(float) * 7);
  }

  // TrackFramePairwise (pairwise_frame_tracking.h:71-108) as BadSlam::RunOdometry calls it (bad_slam.cc:911-938): the frame's
  // preprocessed depth / normals / colour (uchar4, .w = luma) tracked against keyframe `base_keyframe_id`.  The reference's
  // intermediate images (calibrated depth, colour in depth intrinsics, intensity images, pyramids) are built inside the call.
  void TrackFramePairwise(cudaStream_t stream, int base_keyframe_id, bool use_pyramid_level_0, bool use_gradmag,
                          DeviceImage<uint16_t> tracked_depth_buffer, DeviceImage<uint16_t> tracked_normals_buffer,
                          DeviceImage<uint8_t> tracked_color_buffer_rgba, bool test_different_initial_estimates,
                          const SE3f& base_T_frame_initial_estimate_1, const SE3f& base_T_frame_initial_estimate_2,
                          SE3f* out_base_T_frame_estimate, int num_scales = 5, bba_odometry_result* result = nullptr) {
    const bba_odometry_options o = MakeOdometryOptions(num_scales, use_pyramid_level_0, use_gradmag, test_different_initial_estimates);
    float out[7];
    Check(bba_track_frame_pairwise(h_, &o, base_keyframe_id, tracked_depth_buffer.address, tracked_depth_buffer.pitch_bytes,
                                   tracked_normals_buffer.address, tracked_normals_buffer.pitch_bytes, tracked_color_buffer_rgba.address,
                                   tracked_color_buffer_rgba.pitch_bytes, base_T_frame_initial_estimate_1.data(),
                                   base_T_frame_initial_estimate_2.data(), out, result, stream),
          "bba_track_frame_pairwise");
    std::memcpy(out_base_T_frame_estimate->data(), out, sizeof(out));
  }

  // The same against a base frame that is not a keyframe yet, given by the buffers AddKeyframe takes: the keyframe that still
  // waits in the BA thread's queue while the odometry thread tracks against it (parallel BA, INTEGRATION.md section 2).
  void TrackFramePairwise(cudaStream_t stream, DeviceImage<uint16_t> base_depth_buffer, DeviceImage<uint16_t> base_normals_buffer,
                          DeviceImage<uint8_t> base_color_buffer_rgba, bool use_pyramid_level_0, bool use_gradmag,
                          DeviceImage<uint16_t> tracked_depth_buffer, DeviceImage<uint16_t> tracked_normals_buffer,
                          DeviceImage<uint8_t> tracked_color_buffer_rgba, bool test_different_initial_estimates,
                          const SE3f& base_T_frame_initial_estimate_1, const SE3f& base_T_frame_initial_estimate_2,
                          SE3f* out_base_T_frame_estimate, int num_scales = 5, bba_odometry_result* result = nullptr) {
    const bba_odometry_options o = MakeOdometryOptions(num_scales, use_pyramid_level_0, use_gradmag, test_different_initial_estimates);
    float out[7];
    Check(bba_track_frame_pairwise_to_frame(h_, &o, base_depth_buffer.address, base_depth_buffer.pitch_bytes, base_normals_buffer.address,
                                            base_normals_buffer.pitch_bytes, base_color_buffer_rgba.address,
                                            base_color_buffer_rgba.pitch_bytes, tracked_depth_buffer.address,
                                            tracked_depth_buffer.pitch_bytes, tracked_normals_buffer.address,
                                            tracked_normals_buffer.pitch_bytes, tracked_color_buffer_rgba.address,
                                            tracked_color_buffer_rgba.pitch_bytes, base_T_frame_initial_estimate_1.data(),
                                            base_T_frame_initial_estimate_2.data(), out, result, stream),
          "bba_track_frame_pairwise_to_frame");
    std::memcpy(out_base_T_frame_estimate->data(), out, sizeof(out));
  }

  // Both forms above for many independent pairs in one call (bba_track_frames_pairwise), all with the same options: entry i
  // tracks frames[entries[i].tracked_frame] against keyframe entries[i].base_keyframe_id, or with -1 against
  // frames[entries[i].base_frame].  *out_base_T_frame_estimates gets one estimate per entry and, when given, *results one result.
  void TrackFramesPairwise(cudaStream_t stream, const std::vector<FrameImages>& frames, const std::vector<bba_odometry_entry>& entries,
                           bool use_pyramid_level_0, bool use_gradmag, bool test_different_initial_estimates,
                           std::vector<SE3f>* out_base_T_frame_estimates, int num_scales = 5,
                           std::vector<bba_odometry_result>* results = nullptr) {
    const bba_odometry_options o = MakeOdometryOptions(num_scales, use_pyramid_level_0, use_gradmag, test_different_initial_estimates);
    const std::vector<bba_frame_buffers> buffers = MakeFrameBuffers(frames);
    const size_t count = entries.size();
    std::vector<float> out(7 * count);
    if (results) results->resize(count);
    Check(bba_track_frames_pairwise(h_, &o, static_cast<int>(frames.size()), buffers.data(), static_cast<int>(count), entries.data(),
                                    out.data(), results ? results->data() : nullptr, nullptr, stream),
          "bba_track_frames_pairwise");
    out_base_T_frame_estimates->resize(count);
    for (size_t i = 0; i < count; ++i) std::memcpy((*out_base_T_frame_estimates)[i].data(), out.data() + 7 * i, sizeof(float) * 7);
  }

  // LoopDetector's verification of loop-closure candidates (loop_detector.cc:436-668, bba_verify_loop_closures): each candidate's
  // initial old_T_cur is refined against the matched keyframe and its two neighbours, the three estimates are tested for agreement
  // and averaged, and the correction is tested for necessity.  Thresholds <= 0 select the reference's.  out->at(i).status is a
  // bba_loop_status; on BBA_LOOP_ACCEPTED, cur_T_old is the loop edge for AddKeyframePoseConstraint(current, matched, ...).
  void VerifyLoopClosures(cudaStream_t stream, const std::vector<bba_loop_candidate>& candidates, bool use_pyramid_level_0,
                          bool use_gradmag, std::vector<bba_loop_verification>* out, int num_scales = 5,
                          float max_angle_difference = 0, float max_translation_difference = 0, float max_pixel_distance = 0) {
    bba_loop_verification_options o{};
    o.odometry = MakeOdometryOptions(num_scales, use_pyramid_level_0, use_gradmag, /*test_different_initial_estimates=*/false);
    o.max_angle_difference = max_angle_difference;
    o.max_translation_difference = max_translation_difference;
    o.max_pixel_distance = max_pixel_distance;
    out->resize(candidates.size());
    Check(bba_verify_loop_closures(h_, &o, static_cast<int>(candidates.size()), candidates.data(), out->data(), stream),
          "bba_verify_loop_closures");
  }

  // The randomized-fern place index (bba_index_keyframes, DESIGN.md §3.18; not in the reference): encodes the keyframes `ids`
  // (every keyframe when empty) from their current images.  Options that differ from the current ones reset the index first.
  void IndexKeyframes(cudaStream_t stream, const std::vector<int>& ids = {}, int num_ferns = 512, float min_depth = 0.5f,
                      float max_depth = 3.0f) {
    std::vector<int> all = ids;
    if (all.empty())
      for (int k = 0; k < bba_keyframe_count(h_); ++k) all.push_back(k);
    const bba_place_index_options o{num_ferns, min_depth, max_depth};
    Check(bba_index_keyframes(h_, &o, static_cast<int>(all.size()), all.data(), stream), "bba_index_keyframes");
  }
  // bba_query_place_index: per query, the ids and differences of at most max_matches candidates in (difference, id) order.
  void QueryPlaceIndex(cudaStream_t stream, const std::vector<bba_place_query>& queries, const std::vector<bba_frame_buffers>& frames,
                       int max_matches, std::vector<std::vector<int>>* ids, std::vector<std::vector<int>>* differences) {
    const size_t n = queries.size();
    std::vector<int> flat_ids(n * max_matches), flat_diffs(n * max_matches), counts(n);
    Check(bba_query_place_index(h_, static_cast<int>(frames.size()), frames.empty() ? nullptr : frames.data(), static_cast<int>(n),
                                queries.data(), max_matches, flat_ids.data(), flat_diffs.data(), counts.data(), stream),
          "bba_query_place_index");
    ids->assign(n, {});
    differences->assign(n, {});
    for (size_t q = 0; q < n; ++q) {
      (*ids)[q].assign(flat_ids.begin() + q * max_matches, flat_ids.begin() + q * max_matches + counts[q]);
      (*differences)[q].assign(flat_diffs.begin() + q * max_matches, flat_diffs.begin() + q * max_matches + counts[q]);
    }
  }
  // bba_get_place_index_codes: num_ferns / 8 words per keyframe of `ids`, num_ferns of the published index.
  std::vector<uint32_t> PlaceIndexCodes(cudaStream_t stream, const std::vector<int>& ids) {
    int num_ferns = 0;
    Check(bba_get_place_index_options(h_, &num_ferns, nullptr, nullptr), "bba_get_place_index_options");
    std::vector<uint32_t> out(ids.size() * static_cast<size_t>(num_ferns / 8));
    Check(bba_get_place_index_codes(h_, static_cast<int>(ids.size()), ids.data(), num_ferns / 8, out.data(), stream),
          "bba_get_place_index_codes");
    return out;
  }

  // bba_measure_keyframe_covisibility (not in the reference): counts [ids.size()][K], entry (i, b) the surfels associated with both
  // keyframe ids[i] and keyframe b at their current poses; an empty ids: every keyframe in id order.  A BA-side call; synchronises
  // the stream.
  void MeasureKeyframeCovisibility(cudaStream_t stream, const std::vector<int>& ids, std::vector<uint32_t>* counts) {
    const int K = bba_keyframe_count(h_);
    const int rows = ids.empty() ? K : static_cast<int>(ids.size());
    counts->assign(static_cast<size_t>(rows) * K, 0u);
    if (rows == 0) return;
    Check(bba_measure_keyframe_covisibility(h_, ids.empty() ? -1 : static_cast<int>(ids.size()), ids.empty() ? nullptr : ids.data(), K,
                                            counts->data(), stream),
          "bba_measure_keyframe_covisibility");
  }

  // bba_estimate_keyframe_exposures (not in the reference): the gains of keyframes ids relative to the gauge keyframe (an empty
  // ids: every keyframe in id order), and optionally each one's observations and inliers.  A BA-side call that changes nothing;
  // synchronises the stream.
  void EstimateKeyframeExposures(cudaStream_t stream, const bba_exposure_options& options, const std::vector<int>& ids,
                                 std::vector<float>* gains, std::vector<uint32_t>* observations = nullptr,
                                 std::vector<uint32_t>* inliers = nullptr) {
    const std::vector<int> list = ids.empty() ? AllKeyframeIds() : ids;
    gains->assign(list.size(), 0.f);
    if (observations) observations->assign(list.size(), 0u);
    if (inliers) inliers->assign(list.size(), 0u);
    Check(bba_estimate_keyframe_exposures(h_, &options, static_cast<int>(list.size()), list.data(), gains->data(),
                                          observations ? observations->data() : nullptr, inliers ? inliers->data() : nullptr, stream),
          "bba_estimate_keyframe_exposures");
  }
  // bba_set_keyframe_exposures: keyframe ids[i] gets gains[i] (an empty ids: every keyframe in id order); its luma is re-extracted.
  void SetKeyframeExposures(cudaStream_t stream, const std::vector<int>& ids, const std::vector<float>& gains) {
    const std::vector<int> list = ids.empty() ? AllKeyframeIds() : ids;
    if (gains.size() != list.size()) throw std::invalid_argument("SetKeyframeExposures: one gain per keyframe id");
    Check(bba_set_keyframe_exposures(h_, static_cast<int>(list.size()), list.data(), gains.data(), stream), "bba_set_keyframe_exposures");
  }
  // bba_get_keyframe_exposures: the published gains (an empty ids: every keyframe).  Front end.
  void GetKeyframeExposures(const std::vector<int>& ids, std::vector<float>* gains) const {
    const std::vector<int> list = ids.empty() ? AllKeyframeIds() : ids;
    gains->assign(list.size(), 1.f);
    Check(bba_get_keyframe_exposures(h_, static_cast<int>(list.size()), list.data(), gains->data()), "bba_get_keyframe_exposures");
  }

  // bba_measure_frame_overlap (not in the reference): per query, what the surfel map already explains of a frame that is not a
  // keyframe (*out, one record per query) and, with a non-null shared, the surfels it shares with every keyframe ([queries][K]).
  // A BA-side call; synchronises the stream.
  void MeasureFrameOverlap(cudaStream_t stream, const std::vector<bba_frame_buffers>& frames,
                           const std::vector<bba_frame_overlap_query>& queries, std::vector<bba_frame_overlap>* out,
                           std::vector<uint32_t>* shared = nullptr) {
    const int K = bba_keyframe_count(h_);
    out->assign(queries.size(), bba_frame_overlap{});
    if (shared) shared->assign(queries.size() * static_cast<size_t>(K), 0u);
    Check(bba_measure_frame_overlap(h_, static_cast<int>(frames.size()), frames.data(), static_cast<int>(queries.size()), queries.data(), K,
                                    shared && K > 0 ? shared->data() : nullptr, out->data(), stream),
          "bba_measure_frame_overlap");
  }

  // direct_ba.h:143-162, same argument order and defaults (Timer* is any type with GetTimeSinceStart()).
  template <typename TimerT = NoTimer>
  void BundleAdjustment(cudaStream_t stream, bool optimize_depth_intrinsics, bool optimize_color_intrinsics, bool do_surfel_updates,
                        bool optimize_poses, bool optimize_geometry, int min_iterations, int max_iterations, bool use_pcg,
                        int active_keyframe_window_start, int active_keyframe_window_end, bool increase_ba_iteration_count,
                        int* iterations_done = nullptr, bool* converged = nullptr, double time_limit = 0, TimerT* timer = nullptr,
                        int pcg_max_inner_iterations = 30, int pcg_max_keyframes = 2500,
                        std::function<bool(int)> progress_function = nullptr) {
    bba_ba_options o{};
    o.optimize_depth_intrinsics = optimize_depth_intrinsics;
    o.optimize_color_intrinsics = optimize_color_intrinsics;
    o.do_surfel_updates = do_surfel_updates;
    o.optimize_poses = optimize_poses;
    o.optimize_geometry = optimize_geometry;
    o.min_iterations = min_iterations;
    o.max_iterations = max_iterations;
    o.use_pcg = use_pcg;
    o.active_keyframe_window_start = active_keyframe_window_start;
    o.active_keyframe_window_end = active_keyframe_window_end;
    o.increase_ba_iteration_count = increase_ba_iteration_count;
    // direct_ba_alternating.cc:703-709: the limit is tested only when a timer is given, against timer->GetTimeSinceStart(),
    // i.e. counted from the timer's own start: hand the backend what is left of the budget at the time of the call
    // (0 = no limit; an already exhausted budget still runs one iteration, like the reference's test at the loop's end).
    o.time_limit_seconds = 0;
    if (timer != nullptr) {
      const double left = time_limit - timer->GetTimeSinceStart();
      o.time_limit_seconds = left > 1e-9 ? left : 1e-9;
    }
    o.pcg_max_inner_iterations = pcg_max_inner_iterations;
    o.pcg_max_keyframes = pcg_max_keyframes;
    o.pcg_gauge_keyframe = pcg_gauge_keyframe_;   // -1: rand() % K per iteration like direct_ba_pcg.cc:324
    if (progress_function) {
      o.progress_function = [](void* user, int iteration) -> int { return (*static_cast<std::function<bool(int)>*>(user))(iteration) ? 1 : 0; };
      o.progress_user = &progress_function;
    }
    bba_ba_result r{};
    Check(bba_bundle_adjust(h_, &o, &r, stream), "bba_bundle_adjust");
    if (iterations_done) *iterations_done = r.iterations_done;
    if (converged) *converged = r.converged != 0;
    last_result_ = r;
  }

  // ... and with a literal nullptr in the timer position (no type to deduce): no time limit, like the reference without a timer
  void BundleAdjustment(cudaStream_t stream, bool optimize_depth_intrinsics, bool optimize_color_intrinsics, bool do_surfel_updates,
                        bool optimize_poses, bool optimize_geometry, int min_iterations, int max_iterations, bool use_pcg,
                        int active_keyframe_window_start, int active_keyframe_window_end, bool increase_ba_iteration_count,
                        int* iterations_done, bool* converged, double time_limit, std::nullptr_t,
                        int pcg_max_inner_iterations = 30, int pcg_max_keyframes = 2500,
                        std::function<bool(int)> progress_function = nullptr) {
    BundleAdjustment<NoTimer>(stream, optimize_depth_intrinsics, optimize_color_intrinsics, do_surfel_updates, optimize_poses,
                              optimize_geometry, min_iterations, max_iterations, use_pcg, active_keyframe_window_start,
                              active_keyframe_window_end, increase_ba_iteration_count, iterations_done, converged, time_limit,
                              static_cast<NoTimer*>(nullptr), pcg_max_inner_iterations, pcg_max_keyframes, std::move(progress_function));
  }

  // direct_ba.h:114-117 (frame = an already added keyframe); returns the number of surfels created
  uint32_t CreateSurfelsForKeyframe(cudaStream_t stream, bool filter_new_surfels, int keyframe_id) {
    uint32_t created = 0;
    Check(bba_create_surfels_for_keyframe(h_, keyframe_id, filter_new_surfels, &created, stream), "bba_create_surfels_for_keyframe");
    return created;
  }

  // BadSlam::PreprocessFrame (bad_slam.cc:692-765: ComputeBrightnessCUDA, BilateralFilteringAndDepthCutoffCUDA,
  // ComputeNormalsCUDA, ComputePointRadiiAndRemoveIsolatedPixelsCUDA) + ComputeMinMaxDepthCUDA (bad_slam.cc:978) in one
  // launch.  depth_cutoff = BadSlamConfig::max_depth (metres); rgb: uchar3; the outputs are the buffers AddKeyframe takes.  min_depth / max_depth may be nullptr (no sync).
  void PreprocessFrame(cudaStream_t stream, float bilateral_filter_sigma_xy, float bilateral_filter_sigma_inv_depth,
                       float bilateral_filter_radius_factor, float depth_cutoff,
                       DeviceImage<uint16_t> raw_depth, DeviceImage<uint8_t> rgb,
                       MutableDeviceImage<uint16_t> depth, MutableDeviceImage<uint16_t> normals,
                       MutableDeviceImage<uint16_t> radius, MutableDeviceImage<uint8_t> color_rgba,
                       float* min_depth, float* max_depth) {
    const bba_preprocess_options o{bilateral_filter_sigma_xy, bilateral_filter_sigma_inv_depth, bilateral_filter_radius_factor, depth_cutoff};
    Check(bba_preprocess_frame(h_, &o, raw_depth.address, raw_depth.pitch_bytes, rgb.address, rgb.pitch_bytes, depth.address,
                               depth.pitch_bytes, normals.address, normals.pitch_bytes, radius.address, radius.pitch_bytes,
                               color_rgba.address, color_rgba.pitch_bytes, min_depth, max_depth, stream),
          "bba_preprocess_frame");
  }

  // ... of the frame as the sensor delivers it, with the rest of BadSlam::PreprocessFrame (bad_slam.cc:649-689) in the same
  // launch: BadSlamConfig::median_filter_and_densify_iterations, pyramid_level_for_depth (raw_depth is raw_width x raw_height,
  // the depth camera Camera::Scaled(2^-level) of it) and pyramid_level_for_color (rgb is rgb_width x rgb_height, the colour
  // camera x 2^level).  The outputs have the cameras' sizes.
  void PreprocessFrame(cudaStream_t stream, float bilateral_filter_sigma_xy, float bilateral_filter_sigma_inv_depth,
                       float bilateral_filter_radius_factor, float depth_cutoff, int median_filter_and_densify_iterations,
                       int pyramid_level_for_depth, int pyramid_level_for_color,
                       DeviceImage<uint16_t> raw_depth, int raw_width, int raw_height,
                       DeviceImage<uint8_t> rgb, int rgb_width, int rgb_height,
                       MutableDeviceImage<uint16_t> depth, MutableDeviceImage<uint16_t> normals,
                       MutableDeviceImage<uint16_t> radius, MutableDeviceImage<uint8_t> color_rgba,
                       float* min_depth, float* max_depth) {
    const bba_raw_frame_options o{{bilateral_filter_sigma_xy, bilateral_filter_sigma_inv_depth, bilateral_filter_radius_factor, depth_cutoff},
                                  median_filter_and_densify_iterations, pyramid_level_for_depth, pyramid_level_for_color};
    Check(bba_preprocess_raw_frame(h_, &o, raw_depth.address, raw_depth.pitch_bytes, raw_width, raw_height, rgb.address,
                                   rgb.pitch_bytes, rgb_width, rgb_height, depth.address, depth.pitch_bytes, normals.address,
                                   normals.pitch_bytes, radius.address, radius.pitch_bytes, color_rgba.address,
                                   color_rgba.pitch_bytes, min_depth, max_depth, stream),
          "bba_preprocess_raw_frame");
  }

  // direct_ba.cc:566-653 (runs inside BundleAdjustment on the reference's schedule; exposed like the reference does)
  void PerformBASchemeEndTasks(cudaStream_t stream, bool do_surfel_updates) {   // direct_ba.h:435-437
    Check(bba_perform_end_tasks(h_, do_surfel_updates ? 1 : 0, nullptr, nullptr, stream), "bba_perform_end_tasks");
  }

  void GetKeyframePose(int keyframe_id, SE3f* global_T_frame) const {
    float p[7];
    Check(bba_get_keyframe_pose(h_, keyframe_id, p), "bba_get_keyframe_pose");
    for (int i = 0; i < 7; ++i) global_T_frame->data()[i] = p[i];
  }
  void SetKeyframePose(int keyframe_id, const SE3f& global_T_frame) {
    Check(bba_set_keyframe_pose(h_, keyframe_id, global_T_frame.data()), "bba_set_keyframe_pose");
  }
  // Soft pose priors (not in the reference; badba.h): anchors keyframe_id to `prior` with the cost 1/2 r^T L r,
  // r = log(prior^-1 global_T_frame), L given as its upper triangle (translation, then rotation).
  void SetKeyframePosePrior(int keyframe_id, const SE3f& prior, const float (&information)[21]) {
    Check(bba_set_keyframe_pose_priors(h_, 1, &keyframe_id, prior.data(), information), "bba_set_keyframe_pose_priors");
  }
  // Removes the priors of keyframe_ids, or every prior when the list is empty.
  void ClearKeyframePosePriors(const std::vector<int>& keyframe_ids = {}) {
    Check(bba_clear_keyframe_pose_priors(h_, keyframe_ids.empty() ? -1 : static_cast<int>(keyframe_ids.size()), keyframe_ids.data()),
          "bba_clear_keyframe_pose_priors");
  }
  // Soft relative pose constraints (not in the reference; badba.h): the cost 1/2 r^T L r, r = log(a_T_b^-1 global_T_a^-1
  // global_T_b), L given as its upper triangle (translation, then rotation).  Returns the constraint's id.
  int AddKeyframePoseConstraint(int keyframe_a, int keyframe_b, const SE3f& a_T_b, const float (&information)[21]) {
    bba_pose_constraint c;
    c.keyframe_a = keyframe_a;
    c.keyframe_b = keyframe_b;
    std::memcpy(c.a_T_b, a_T_b.data(), sizeof(c.a_T_b));
    std::memcpy(c.information, information, sizeof(c.information));
    int id = -1;
    Check(bba_add_keyframe_pose_constraints(h_, 1, &c, &id), "bba_add_keyframe_pose_constraints");
    return id;
  }
  // Removes the constraints `ids`, or every constraint when the list is empty.
  void RemoveKeyframePoseConstraints(const std::vector<int>& ids = {}) {
    Check(bba_remove_keyframe_pose_constraints(h_, ids.empty() ? -1 : static_cast<int>(ids.size()), ids.data()),
          "bba_remove_keyframe_pose_constraints");
  }
  // Robust losses (not in the reference; badba.h): the prior of keyframe_id, or constraint `id`, costs 1/2 rho(r^T L r) with
  // rho of type (BBA_LOSS_TRIVIAL / HUBER / CAUCHY) and scale delta in units of sqrt(r^T L r).
  void SetKeyframePosePriorLoss(int keyframe_id, int type, float scale) {
    const bba_robust_loss loss{type, scale};
    Check(bba_set_keyframe_pose_prior_losses(h_, 1, &keyframe_id, &loss), "bba_set_keyframe_pose_prior_losses");
  }
  void SetKeyframePoseConstraintLoss(int id, int type, float scale) {
    const bba_robust_loss loss{type, scale};
    Check(bba_set_keyframe_pose_constraint_losses(h_, 1, &id, &loss), "bba_set_keyframe_pose_constraint_losses");
  }
  // s = r^T L r and the robust weight of every prior (indexed by keyframe id, NaN without a prior) and constraint (in id order)
  // at the current poses; a loop closure that a robust pose graph rejected has a weight near 0.  Synchronises the stream.
  void EvaluateKeyframePoseTerms(cudaStream_t stream, std::vector<double>* prior_s, std::vector<double>* prior_weight,
                                 std::vector<double>* constraint_s, std::vector<double>* constraint_weight) {
    int constraints = 0;
    Check(bba_get_keyframe_pose_constraints(h_, 0, nullptr, nullptr, &constraints), "bba_get_keyframe_pose_constraints");
    const int K = bba_keyframe_count(h_);
    prior_s->resize(K);
    prior_weight->resize(K);
    constraint_s->resize(constraints);
    constraint_weight->resize(constraints);
    Check(bba_evaluate_keyframe_pose_terms(h_, K, prior_s->data(), prior_weight->data(), constraints, constraint_s->data(),
                                           constraint_weight->data(), stream),
          "bba_evaluate_keyframe_pose_terms");
  }
  // Attitude priors (not in the reference; badba.h): the angle theta between R^-1 d_ref and d_meas costs 1/2 rho(L theta^2), with
  // d_ref in the map frame (e.g. gravity), d_meas in the keyframe's camera frame (e.g. the negated accelerometer reading at rest).
  void SetKeyframeAttitudePriors(const std::vector<int>& ids, const std::vector<bba_attitude_prior>& priors) {
    if (ids.size() != priors.size()) throw Error(BBA_ERR_INVALID_ARGUMENT, "SetKeyframeAttitudePriors: one prior per id");
    Check(bba_set_keyframe_attitude_priors(h_, static_cast<int>(ids.size()), ids.data(), priors.data()), "bba_set_keyframe_attitude_priors");
  }
  // Removes the attitude priors of `ids`, or every one when the list is empty.
  void ClearKeyframeAttitudePriors(const std::vector<int>& ids = {}) {
    Check(bba_clear_keyframe_attitude_priors(h_, ids.empty() ? -1 : static_cast<int>(ids.size()), ids.data()),
          "bba_clear_keyframe_attitude_priors");
  }
  // A keyframe's attitude prior as last published; false without one.
  bool GetKeyframeAttitudePrior(int keyframe_id, bba_attitude_prior* out) {
    int has = 0;
    Check(bba_get_keyframe_attitude_prior(h_, keyframe_id, out, &has), "bba_get_keyframe_attitude_prior");
    return has != 0;
  }
  // s = L theta^2 and the robust weight of every attitude prior (indexed by keyframe id, NaN without one) at the current poses.
  // Synchronises the stream.
  void EvaluateKeyframeAttitudePriors(cudaStream_t stream, std::vector<double>* s, std::vector<double>* weight) {
    const int K = bba_keyframe_count(h_);
    s->resize(K);
    weight->resize(K);
    Check(bba_evaluate_keyframe_attitude_priors(h_, K, s->data(), weight->data(), stream), "bba_evaluate_keyframe_attitude_priors");
  }
  // The keyframe pose graph (bba_optimize_pose_graph; the reference's PoseGraphOptimizer, here on the device): Gauss-Newton over
  // the priors, the constraints and, with add_current_state_odometry_constraints, one edge per consecutive pair of keyframes at
  // their current relative pose with `information` (identity when null).  The defaults are the reference's: vertex 0 fixed, 20
  // iterations.  Synchronises the stream.
  bba_pose_graph_result OptimizePoseGraph(cudaStream_t stream, bool add_current_state_odometry_constraints = true, int gauge_keyframe = 0,
                                          int max_iterations = 20, const float (*information)[21] = nullptr) {
    bba_pose_graph_options o{};
    o.gauge_keyframe = gauge_keyframe;
    o.max_iterations = max_iterations;
    o.use_odometry_chain = add_current_state_odometry_constraints ? 1 : 0;
    for (int i = 0, idx = 0; i < 6; ++i)
      for (int j = i; j < 6; ++j, ++idx) o.odometry_information[idx] = information ? (*information)[idx] : (i == j ? 1.f : 0.f);
    bba_pose_graph_result r{};
    Check(bba_optimize_pose_graph(h_, &o, &r, stream), "bba_optimize_pose_graph");
    return r;
  }
  uint32_t surfels_size() const { return bba_surfels_size(h_); }   // direct_ba.h:265
  void GetIntrinsics(float depth[4], float color[4], float* a) const { Check(bba_get_intrinsics(h_, depth, color, a), "bba_get_intrinsics"); }
  void SetPCGGaugeKeyframe(int keyframe_id) { pcg_gauge_keyframe_ = keyframe_id; }

  // direct_ba.h:195-211: the mutex callers on other threads take around reads of poses / intrinsics / surfel counts while a
  // BundleAdjustment call is running (the backend itself is one-call-at-a-time per handle)
  void Lock() const { mutex_.lock(); }
  void Unlock() const { mutex_.unlock(); }
  std::mutex& Mutex() const { return mutex_; }

  // direct_ba.h:220-226, 290-300, 311
  int GetMinObservationCount() const {
    const int K = bba_keyframe_count(h_);
    return (K < 10) ? ((K < 5) ? min_observation_counts_[0] : min_observation_counts_[1]) : min_observation_counts_[2];
  }
  float a() const { float d[4], c[4], a = 0.f; bba_get_intrinsics(h_, d, c, &a); return a; }
  void SetA(float a) { float d[4], c[4], old = 0.f; GetIntrinsics(d, c, &old); Check(bba_set_intrinsics(h_, d, c, a), "bba_set_intrinsics"); }
  void IncreaseBAIterationCount() {
    int count = 0, last = 0;
    Check(bba_get_ba_iteration_counts(h_, &count, &last), "bba_get_ba_iteration_counts");
    Check(bba_set_ba_iteration_counts(h_, count + 1, last), "bba_set_ba_iteration_counts");
  }

  // direct_ba.h:317-328
  bool use_depth_residuals() const { int d = 0, c = 0; bba_get_residual_types(h_, &d, &c); return d != 0; }
  bool use_descriptor_residuals() const { int d = 0, c = 0; bba_get_residual_types(h_, &d, &c); return c != 0; }
  void SetUseDepthResiduals(bool v) { Check(bba_set_residual_types(h_, v, use_descriptor_residuals()), "bba_set_residual_types"); }
  void SetUseDescriptorResiduals(bool v) { Check(bba_set_residual_types(h_, use_depth_residuals(), v), "bba_set_residual_types"); }
  // The deterministic mode (bba_set_deterministic): bitwise reproducible BA, frame pose estimation and odometry on one GPU.
  void SetDeterministic(bool on) { Check(bba_set_deterministic(h_, on ? 1 : 0), "bba_set_deterministic"); }
  bool deterministic() const { int on = 0; bba_get_deterministic(h_, &on); return on != 0; }
  const bba_ba_result& last_result() const { return last_result_; }
  bba_handle handle() const { return h_; }

 private:
  void Check(bba_status s, const char* where) const {
    if (s != BBA_OK) throw Error(s, std::string(where) + ": " + (h_ ? bba_last_error(h_) : "no handle"));
  }
  std::vector<int> AllKeyframeIds() const {
    std::vector<int> ids(static_cast<size_t>(std::max(0, bba_keyframe_count(h_))));
    for (size_t i = 0; i < ids.size(); ++i) ids[i] = static_cast<int>(i);
    return ids;
  }
  // The odometry options of the TrackFramePairwise forms: the reference's 30 iterations per scale.
  static bba_odometry_options MakeOdometryOptions(int num_scales, bool use_pyramid_level_0, bool use_gradmag,
                                                  bool test_different_initial_estimates) {
    bba_odometry_options o{};
    o.num_scales = num_scales;
    o.use_pyramid_level_0 = use_pyramid_level_0;
    o.use_gradmag = use_gradmag;
    o.test_different_initial_estimates = test_different_initial_estimates;
    o.max_iterations_per_scale = 30;
    return o;
  }
  static std::vector<bba_frame_buffers> MakeFrameBuffers(const std::vector<FrameImages>& frames) {
    std::vector<bba_frame_buffers> buffers(frames.size());
    for (size_t f = 0; f < frames.size(); ++f)
      buffers[f] = {frames[f].depth.address, frames[f].depth.pitch_bytes, frames[f].normals.address, frames[f].normals.pitch_bytes,
                    frames[f].color_rgba.address, frames[f].color_rgba.pitch_bytes};
    return buffers;
  }
  bba_handle h_ = nullptr;
  bba_ba_result last_result_{};
  std::vector<int> keyframe_frame_index_;   // by keyframe id; written by AddKeyframe (BA side)
  int pcg_gauge_keyframe_ = -1;
  int min_observation_counts_[3] = {1, 2, 3};
  mutable std::mutex mutex_;
};

// The ranks of a multi-GPU bundle adjustment as DirectBA members of one process (bba_local_group_create): the library exchanges
// between them itself, so a BA thread can drive several GPUs without NCCL, MPI or IPC.  members[r] must have been constructed
// with rank r, world_size members.size() and device devices[r].  The group is destroyed before its members.
//
//   group.RunOnRanks([&](int rank, DA& ba) { ba.BundleAdjustment(streams[rank], ...); });
//
// RunOnRanks runs fn on one thread per rank with that thread's current device set to the rank's device, joins them and rethrows
// the first exception; any exception poisons the group first, so that no other rank waits for one that gave up.  Reset()
// restores service afterwards.
template <typename DA>
class LocalGroup {
 public:
  LocalGroup(std::vector<std::unique_ptr<DA>> members, std::vector<int> devices, bool peer_stores = false)
      : members_(std::move(members)), devices_(std::move(devices)) {
    if (devices_.size() != members_.size()) throw Error(BBA_ERR_INVALID_ARGUMENT, "LocalGroup: one device per member");
    std::vector<bba_handle> handles;
    for (const auto& m : members_) handles.push_back(m->handle());
    const bba_status s = bba_local_group_create(handles.data(), static_cast<int>(handles.size()), peer_stores ? 1 : 0, &g_);
    if (s != BBA_OK) {
      std::string msg = "bba_local_group_create";
      for (bba_handle h : handles)
        if (h && std::strncmp(bba_last_error(h), "bba_local_group_create", 22) == 0) msg = bba_last_error(h);
      throw Error(s, msg);
    }
  }
  ~LocalGroup() { bba_local_group_destroy(g_); }   // (members_ go after the group)
  LocalGroup(const LocalGroup&) = delete;
  LocalGroup& operator=(const LocalGroup&) = delete;

  void RunOnRanks(const std::function<void(int, DA&)>& fn) {
    std::vector<std::exception_ptr> errors(members_.size());
    std::vector<std::thread> threads;
    for (size_t r = 0; r < members_.size(); ++r)
      threads.emplace_back([&, r] {
        try {
          if (cudaSetDevice(devices_[r]) != cudaSuccess) throw Error(BBA_ERR_CUDA, "LocalGroup: cudaSetDevice");
          fn(static_cast<int>(r), *members_[r]);
        } catch (...) {
          errors[r] = std::current_exception();
          bba_local_group_poison(g_);
        }
      });
    for (auto& t : threads) t.join();
    for (auto& e : errors)
      if (e) std::rethrow_exception(e);
  }
  void Reset() {
    if (bba_local_group_reset(g_) != BBA_OK) throw Error(BBA_ERR_INVALID_ARGUMENT, "bba_local_group_reset");
  }
  int size() const { return static_cast<int>(members_.size()); }
  DA& member(int rank) { return *members_.at(rank); }

 private:
  std::vector<std::unique_ptr<DA>> members_;
  std::vector<int> devices_;
  bba_local_group g_ = nullptr;
};

// SaveCalibration / LoadCalibration (io.h:60-72, io.cc:570-700), same three text files: <base>.depth_intrinsics.txt and
// <base>.color_intrinsics.txt ("fx fy cx-0.5 cy-0.5") and <base>.deformation.txt ("w h", a, then the cfactor grid row by row).
inline bool SaveCalibration(cudaStream_t stream, bba_handle h, const std::string& export_base_path) {
  float d[4], c[4], a;
  int w = 0, hh = 0;
  if (bba_get_intrinsics(h, d, c, &a) != BBA_OK || bba_cfactor_size(h, &w, &hh) != BBA_OK) return false;
  std::vector<float> cf(static_cast<size_t>(w) * hh);
  if (bba_get_cfactor_host(h, cf.data(), stream) != BBA_OK) return false;   // synchronises the stream
  const float* cams[2] = {d, c};
  const char* names[2] = {".depth_intrinsics.txt", ".color_intrinsics.txt"};
  for (int i = 0; i < 2; ++i) {
    std::ofstream f(export_base_path + names[i], std::ios::out);
    if (!f) return false;
    f << cams[i][0] << " " << cams[i][1] << " " << (cams[i][2] - 0.5) << " " << (cams[i][3] - 0.5);
  }
  std::ofstream f(export_base_path + ".deformation.txt", std::ios::out);
  if (!f) return false;
  f.precision(8);
  f << w << " " << hh << std::endl << a << std::endl;
  for (float v : cf) f << v << std::endl;
  return true;
}

inline bool LoadCalibration(cudaStream_t stream, bba_handle h, const std::string& import_base_path) {
  float cams[2][4], a = 0.f;
  const char* names[2] = {".depth_intrinsics.txt", ".color_intrinsics.txt"};
  for (int i = 0; i < 2; ++i) {
    std::ifstream f(import_base_path + names[i], std::ios::in);
    if (!f || !(f >> cams[i][0] >> cams[i][1] >> cams[i][2] >> cams[i][3])) return false;
    cams[i][2] += 0.5f;
    cams[i][3] += 0.5f;
  }
  std::ifstream f(import_base_path + ".deformation.txt", std::ios::in);
  int w = 0, hh = 0, fw = 0, fh = 0;
  if (!f || !(f >> fw >> fh) || bba_cfactor_size(h, &w, &hh) != BBA_OK || fw != w || fh != hh) return false;   // io.cc:676-680
  if (!(f >> a)) return false;
  std::vector<float> cf(static_cast<size_t>(w) * hh);
  for (float& v : cf)
    if (!(f >> v)) return false;
  return bba_set_intrinsics(h, cams[0], cams[1], a) == BBA_OK && bba_set_cfactor_host(h, cf.data(), stream) == BBA_OK;   // synchronises
}

// The motion model BadSlam keeps in front of TrackFramePairwise (members base_kf_tr_frame_ / frame_tr_base_kf_, bad_slam.h:346-347),
// with the reference's method names.  RunOdometry (bad_slam.cc:829-955) becomes
//   motion_model.PredictFramePose(&e1, &e2);  direct_ba.TrackFramePairwise(..., e1, e2, &estimate);  motion_model.Push(estimate);
// and ProcessFrame calls motion_model.Rebase() where it re-expresses the lists after creating a keyframe (bad_slam.cc:1057-1068).
template <typename SE3f>
class MotionModel {
 public:
  explicit MotionModel(bool use_motion_model = true) : use_motion_model_(use_motion_model) { bba_host_motion_model_clear(&m_, nullptr, nullptr); }

  // BadSlam::ClearMotionModel (bad_slam.cc:542-565); last_kf_frame_T_global == nullptr: no keyframe yet
  void ClearMotionModel(const SE3f* last_kf_frame_T_global, const SE3f* global_T_frame) {
    bba_host_motion_model_clear(&m_, last_kf_frame_T_global ? last_kf_frame_T_global->data() : nullptr,
                                global_T_frame ? global_T_frame->data() : nullptr);
  }
  // BadSlam::PredictFramePose (bad_slam.cc:767-827)
  void PredictFramePose(SE3f* base_kf_tr_frame_initial_estimate, SE3f* base_kf_tr_frame_initial_estimate_2) const {
    float e1[7], e2[7];
    if (!bba_host_motion_model_predict(&m_, use_motion_model_, e1, e2)) throw Error(BBA_ERR_INVALID_ARGUMENT, "motion model holds no estimate");
    std::memcpy(base_kf_tr_frame_initial_estimate->data(), e1, sizeof(e1));
    std::memcpy(base_kf_tr_frame_initial_estimate_2->data(), e2, sizeof(e2));
  }
  void Push(const SE3f& base_T_frame_estimate) { bba_host_motion_model_push(&m_, base_T_frame_estimate.data()); }
  void Rebase() { bba_host_motion_model_rebase(&m_); }
  int stored_frames() const { return m_.count; }
  const bba_motion_model& record() const { return m_; }

 private:
  bba_motion_model m_{};
  bool use_motion_model_;
};

// The trajectory deformation around a BA call (trajectory_deformation.h:43-58), under the reference's names so that
// BadSlam::RunBundleAdjustment and BAThreadMain (bad_slam.cc:505-533, 1267-1301) keep their shape:
//   std::vector<SE3f> original_keyframe_T_global;
//   RememberKeyframePoses(*direct_ba_, &original_keyframe_T_global);
//   direct_ba_->BundleAdjustment(...);
//   ExtrapolateAndInterpolateKeyframePoseChanges(start_frame, last_frame_index, *direct_ba_, original_keyframe_T_global, rgbd_video);

// frame_T_global of every keyframe, all from one publication of the poses (bba_get_keyframe_states): a front-end call, so the
// odometry thread may make it while a BA call runs.
template <typename SE3f, typename PinholeCamera4f>
void RememberKeyframePoses(const DirectBA<SE3f, PinholeCamera4f>& dense_ba, std::vector<SE3f>* original_keyframe_T_global) {
  const int K = bba_keyframe_count(dense_ba.handle());
  std::vector<float> poses(7 * static_cast<size_t>(K));
  if (bba_get_keyframe_states(dense_ba.handle(), K, poses.data(), nullptr) != BBA_OK)
    throw Error(BBA_ERR_INVALID_ARGUMENT, "RememberKeyframePoses: bba_get_keyframe_states failed");
  original_keyframe_T_global->resize(K);
  for (int k = 0; k < K; ++k) bba_host_se3_inverse(poses.data() + 7 * k, (*original_keyframe_T_global)[k].data());
}

// The deformation on explicit keyframe data: keyframe_frame_index[k], original_keyframe_T_global[k] (before the BA call) and
// keyframe_global_T_frame[k] (after it) for the same K keyframes.  RGBDVideo is any type with frame_count() and
// depth_frame_mutable(i) / color_frame_mutable(i) pointing to frames with global_T_frame() and SetGlobalTFrame() (libvis
// RGBDVideo<Vec3u8, u16>).  Only frames in [start_frame, end_frame] that are not keyframes are set, depth and colour frame alike.
template <typename SE3f, typename RGBDVideo>
void ExtrapolateAndInterpolateKeyframePoseChanges(uint32_t start_frame, uint32_t end_frame, const std::vector<int>& keyframe_frame_index,
                                                  const std::vector<SE3f>& original_keyframe_T_global,
                                                  const std::vector<SE3f>& keyframe_global_T_frame, RGBDVideo* rgbd_video) {
  const int K = static_cast<int>(keyframe_frame_index.size());
  if (original_keyframe_T_global.size() != keyframe_frame_index.size() || keyframe_global_T_frame.size() != keyframe_frame_index.size())
    throw Error(BBA_ERR_INVALID_ARGUMENT, "ExtrapolateAndInterpolateKeyframePoseChanges: one frame index and two poses per keyframe");
  const int64_t last = std::min<int64_t>(end_frame, static_cast<int64_t>(rgbd_video->frame_count()) - 1);   // trajectory_deformation.cc:51
  if (last < static_cast<int64_t>(start_frame)) return;
  const int first = static_cast<int>(start_frame), end = static_cast<int>(last);
  std::vector<float> original(7 * static_cast<size_t>(K)), current(7 * static_cast<size_t>(K));
  for (int k = 0; k < K; ++k) {
    std::memcpy(&original[7 * k], original_keyframe_T_global[k].data(), 7 * sizeof(float));
    std::memcpy(&current[7 * k], keyframe_global_T_frame[k].data(), 7 * sizeof(float));
  }
  std::vector<float> frames(7 * (static_cast<size_t>(end) + 1));
  for (int i = first; i <= end; ++i) std::memcpy(&frames[7 * i], rgbd_video->depth_frame_mutable(i)->global_T_frame().data(), 7 * sizeof(float));
  if (bba_host_deform_trajectory(K, keyframe_frame_index.data(), original.data(), current.data(), first, end, frames.data()) != BBA_OK)
    throw Error(BBA_ERR_INVALID_ARGUMENT, "ExtrapolateAndInterpolateKeyframePoseChanges: no keyframe, or frame indices not increasing");
  for (int i = first; i <= end; ++i) {
    if (std::binary_search(keyframe_frame_index.begin(), keyframe_frame_index.end(), i)) continue;
    SE3f new_global_T_frame;
    std::memcpy(new_global_T_frame.data(), &frames[7 * i], 7 * sizeof(float));
    rgbd_video->depth_frame_mutable(i)->SetGlobalTFrame(new_global_T_frame);
    rgbd_video->color_frame_mutable(i)->SetGlobalTFrame(new_global_T_frame);
  }
}

// ... with the keyframes of `dense_ba`: the first original_keyframe_T_global.size() keyframes, their current (published) poses
// and the frame indices given to AddKeyframe.  Called where BadSlam calls it, with the BA side idle (under DirectBA::Lock()).
template <typename SE3f, typename PinholeCamera4f, typename RGBDVideo>
void ExtrapolateAndInterpolateKeyframePoseChanges(uint32_t start_frame, uint32_t end_frame, const DirectBA<SE3f, PinholeCamera4f>& dense_ba,
                                                  const std::vector<SE3f>& original_keyframe_T_global, RGBDVideo* rgbd_video) {
  const int K = static_cast<int>(original_keyframe_T_global.size());
  std::vector<int> frame_index(K);
  for (int k = 0; k < K; ++k) {
    frame_index[k] = dense_ba.keyframe_frame_index(k);
    if (frame_index[k] < 0) throw Error(BBA_ERR_STATE, "ExtrapolateAndInterpolateKeyframePoseChanges: keyframe added without a frame index");
  }
  std::vector<float> poses(7 * static_cast<size_t>(K));
  if (bba_get_keyframe_states(dense_ba.handle(), K, poses.data(), nullptr) != BBA_OK)
    throw Error(BBA_ERR_INVALID_ARGUMENT, "ExtrapolateAndInterpolateKeyframePoseChanges: bba_get_keyframe_states failed");
  std::vector<SE3f> current(K);
  for (int k = 0; k < K; ++k) std::memcpy(current[k].data(), poses.data() + 7 * k, 7 * sizeof(float));
  ExtrapolateAndInterpolateKeyframePoseChanges(start_frame, end_frame, frame_index, original_keyframe_T_global, current, rgbd_video);
}

// The same pose changes carried over to the surfel map (bba_deform_surfels, not in the reference): after an outside correction of
// the keyframe poses (a pose graph after a loop closure, written with bba_set_keyframe_states), the surfels move with the
// keyframes they are associated with at the remembered poses.  A BA-side call; does not synchronise the stream.
template <typename SE3f, typename PinholeCamera4f>
void DeformSurfelsWithKeyframePoseChanges(DirectBA<SE3f, PinholeCamera4f>& dense_ba, const std::vector<SE3f>& original_keyframe_T_global,
                                          cudaStream_t stream) {
  const int K = static_cast<int>(original_keyframe_T_global.size());
  std::vector<float> original(7 * static_cast<size_t>(K));
  for (int k = 0; k < K; ++k) std::memcpy(&original[7 * k], original_keyframe_T_global[k].data(), 7 * sizeof(float));
  if (bba_status s = bba_deform_surfels(dense_ba.handle(), K, original.data(), nullptr, nullptr, stream))
    throw Error(s, std::string("DeformSurfelsWithKeyframePoseChanges: ") + bba_last_error(dense_ba.handle()));
}

}  // namespace badba
