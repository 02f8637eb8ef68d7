// loop_verification.cu -- bba_verify_loop_closures (DESIGN.md §3.16): LoopDetector's verification of loop-closure candidates
// (loop_detector.cc:436-668) on the published snapshot.  The host orchestration (neighbours, initial estimates, the tracking through
// the batched odometry of frames.cu with stored keyframes as the tracked images, the agreement test and AveragePose of
// host_math.hpp) and the one kernel of the necessity test.
#include <cmath>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include "handle.hpp"
#include "persistent.cuh"

namespace bba {
namespace {

constexpr int kNecessityThreads = 256;
constexpr int kNecessityPixelsPerThread = 8;
constexpr float kDefaultMaxAngle = 3.14159265358979323846f / 180.f * 10.f;   // kMaxAngleDifference (loop_detector.cc:577)
constexpr float kDefaultMaxTranslation = 0.02f;                              // kMaxEuclideanDistance (:578)
constexpr float kDefaultMaxPixelDistance = 1.0f;                             // kAveragePixelDistanceThreshold (:656)
constexpr uint32_t kMinNecessityPixels = 5;                                  // distance_count >= 5 (:657)

struct NecessityArgs {
  CameraParams cam;                            // depth unprojection, colour projection, a and the cfactor slot of the snapshot
  const LoopNecessityCandidate* candidates;    // [gridDim.y]
  double* partial_sum;                         // [candidates][gridDim.x]
  unsigned int* partial_count;                 // [candidates][gridDim.x]
};

// The colour camera's ProjectToPixelCornerConvIfVisible with pixel_border 0 (libvis camera.h:458-469, 1017-1029).
__device__ __forceinline__ bool ProjectColorCorner(const CameraParams& cam, float x, float y, float z, float* u, float* v) {
  if (z <= 0.f) return false;
  *u = cam.cfx * (x / z) + cam.ccx;
  *v = cam.cfy * (y / z) + cam.ccy;
  return *u >= 0.f && *v >= 0.f && *u < static_cast<float>(cam.cw) && *v < static_cast<float>(cam.ch);
}

// The necessity test of one candidate (blockIdx.y) over a fixed slice of the current keyframe's pixels per CTA: every pixel
// without the invalid-depth bit is unprojected at its centre with the calibrated depth, moved, and both points are projected by
// the colour camera; the CTA's fp64 distance sum and pixel count go to its partial slot.  The grid depends on the image size
// only, so a candidate's partials are the same bits whatever else the launch holds.
__global__ void __launch_bounds__(kNecessityThreads) LoopNecessityKernel(NecessityArgs a) {
  const int c = blockIdx.y;
  const LoopNecessityCandidate& cand = a.candidates[c];
  float T[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) T[i] = cand.T[i];
  const uint16_t* depth = cand.depth;
  const uint32_t depth_pitch = cand.depth_pitch;
  const int w = a.cam.w, n = a.cam.w * a.cam.h;
  double sum = 0.0;
  unsigned int count = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int px = i % w, py = i / w;
    const uint16_t measured = LoadPixelU16(depth, depth_pitch, px, py);
    if (measured & kInvalidDepthBit) continue;
    const float cf = a.cam.cfactor[SparseCell(a.cam, px, py)];
    const float d = RawToCalibratedDepth(a.cam.a, cf, a.cam.raw_to_float, measured);
    // UnprojectFromPixelCornerConv at (px + 0.5, py + 0.5): the pixel-centre unprojector of the kernels
    const float x = d * (a.cam.fx_inv * px + a.cam.cx_inv), y = d * (a.cam.fy_inv * py + a.cam.cy_inv), z = d;
    const float mx = T[0] * x + T[1] * y + T[2] * z + T[3];
    const float my = T[4] * x + T[5] * y + T[6] * z + T[7];
    const float mz = T[8] * x + T[9] * y + T[10] * z + T[11];
    float ue, ve, uc, vc;
    if (ProjectColorCorner(a.cam, mx, my, mz, &ue, &ve) && ProjectColorCorner(a.cam, x, y, z, &uc, &vc)) {
      const float du = ue - uc, dv = ve - vc;
      sum += static_cast<double>(sqrtf(du * du + dv * dv));
      ++count;
    }
  }
  sum = BlockSum(sum);
  __syncthreads();
  count = BlockSum(count);
  if (threadIdx.x == 0) {
    a.partial_sum[static_cast<size_t>(c) * gridDim.x + blockIdx.x] = sum;
    a.partial_count[static_cast<size_t>(c) * gridDim.x + blockIdx.x] = count;
  }
}

int NecessityBlocks(int pixels) {
  const int per_block = kNecessityThreads * kNecessityPixelsPerThread;
  return (pixels + per_block - 1) / per_block;
}

LaunchResult LaunchLoopNecessity(const NecessityArgs& a, int candidates, cudaStream_t s) {
  LaunchResult r;
  const dim3 grid(NecessityBlocks(a.cam.w * a.cam.h), candidates);
  LoopNecessityKernel<<<grid, kNecessityThreads, 0, s>>>(a);
  r.kernels = 1;
  return r;
}

bool FinitePose(const float p[7]) {
  for (int i = 0; i < 7; ++i)
    if (!std::isfinite(p[i])) return false;
  return p[0] != 0.f || p[1] != 0.f || p[2] != 0.f || p[3] != 0.f;
}

// The neighbours of loop_detector.cc:455-496 with K published keyframes (ids are contiguous): ids[0..2] = matched, next, previous
// (or the second next after keyframe 0).  Returns false (NO_NEIGHBOUR) when next or the third keyframe does not exist; the ids
// found so far are written, -1 elsewhere.
bool LoopNeighbours(int matched, int K, int ids[3]) {
  ids[0] = matched;
  ids[1] = ids[2] = -1;
  if (matched + 1 >= K) return false;
  ids[1] = matched + 1;
  const int previous = matched > 0 ? matched - 1 : ids[1] + 1;
  if (previous >= K) return false;
  ids[2] = previous;
  return true;
}

Pose ToPose(const float p[7]) {
  Pose r;
  std::memcpy(r.q, p, sizeof(float) * 4);
  std::memcpy(r.t, p + 4, sizeof(float) * 3);
  return r;
}
void FromPose(const Pose& r, float p[7]) {
  std::memcpy(p, r.q, sizeof(float) * 4);
  std::memcpy(p + 4, r.t, sizeof(float) * 3);
}

float Threshold(float v, float fallback) { return v > 0.f ? v : fallback; }

bba_status VerifyLoopClosures(bba_handle h, const bba_loop_verification_options* o, int count, const bba_loop_candidate* candidates,
                              bba_loop_verification* out, cudaStream_t s) {
  const char* fn = "bba_verify_loop_closures";
  const std::string name(fn);
  if (!o || !candidates || !out) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": null argument");
  if (count < 1) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": count must be at least 1");
  if (o->odometry.test_different_initial_estimates)   // loop_detector.cc:541
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": test_different_initial_estimates must be 0 (one initial estimate per pair)");
  if (!std::isfinite(o->max_angle_difference) || !std::isfinite(o->max_translation_difference) || !std::isfinite(o->max_pixel_distance))
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": non-finite threshold");
  if (bba_status st = CheckOdometryOptions(h, fn, o->odometry)) return st;
  int max_id = -1;
  for (int c = 0; c < count; ++c) {
    const bba_loop_candidate& k = candidates[c];
    const std::string which = " in candidate " + std::to_string(c);
    if (k.current_keyframe_id < 0 || k.matched_keyframe_id < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": no such keyframe" + which);
    if (k.current_keyframe_id == k.matched_keyframe_id)
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": the current and the matched keyframe are the same" + which);
    if (!FinitePose(k.old_T_cur_initial))
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": non-finite old_T_cur_initial or zero quaternion" + which);
    max_id = std::max(max_id, std::max(k.current_keyframe_id, k.matched_keyframe_id));
  }
  const float max_angle = Threshold(o->max_angle_difference, kDefaultMaxAngle);
  const float max_translation = Threshold(o->max_translation_difference, kDefaultMaxTranslation);
  const float max_pixels = Threshold(o->max_pixel_distance, kDefaultMaxPixelDistance);

  std::lock_guard<std::mutex> call(h->fe.call);
  FrontEndCall view(h);
  std::vector<KeyframeView> kfs;
  if (bba_status st = view.Snapshot(s, -1, fn, max_id, &kfs)) return st;   // (refuses ids outside the published keyframes)
  const int K = static_cast<int>(kfs.size());

  // neighbours and the three tracked pairs of every candidate that has them
  std::memset(out, 0, sizeof(bba_loop_verification) * count);
  std::vector<bba_odometry_entry> entries;
  std::vector<int> tracked_ids, entry_candidate;
  std::vector<Pose> matched_T_this;
  for (int c = 0; c < count; ++c) {
    const bba_loop_candidate& k = candidates[c];
    bba_loop_verification& v = out[c];
    v.average_pixel_distance = std::numeric_limits<float>::quiet_NaN();
    if (!LoopNeighbours(k.matched_keyframe_id, K, v.tracked_keyframe_ids)) {
      v.status = BBA_LOOP_NO_NEIGHBOUR;
      continue;
    }
    const Pose matched_T_global = Inverse(kfs[k.matched_keyframe_id].pose);
    const Pose cur_T_old_initial_inv = Inverse(ToPose(k.old_T_cur_initial));
    for (int i = 0; i < 3; ++i) {
      Pose m;   // identity for the matched keyframe itself
      if (i == 0) {
        m.q[0] = m.q[1] = m.q[2] = 0.f; m.q[3] = 1.f;
        m.t[0] = m.t[1] = m.t[2] = 0.f;
      } else {
        m = Compose(matched_T_global, kfs[v.tracked_keyframe_ids[i]].pose);
      }
      bba_odometry_entry e{};
      e.base_keyframe_id = k.current_keyframe_id;
      e.base_frame = -1;
      e.tracked_frame = -1;
      FromPose(Compose(cur_T_old_initial_inv, m), e.base_T_frame_initial_1);   // base_T_tracked_initial_estimate (:516)
      std::memcpy(e.base_T_frame_initial_2, e.base_T_frame_initial_1, sizeof(float) * 7);
      entries.push_back(e);
      tracked_ids.push_back(v.tracked_keyframe_ids[i]);
      entry_candidate.push_back(c);
      matched_T_this.push_back(m);
    }
  }

  // tracking: the old keyframes against the current one, through the odometry chunks
  const int n_entries = static_cast<int>(entries.size());
  std::vector<float> tracked(7 * static_cast<size_t>(n_entries));
  std::vector<bba_odometry_result> results(n_entries);
  if (n_entries > 0)
    if (bba_status st = TrackPairsOnSnapshot(h, o->odometry, view, kfs, 0, nullptr, n_entries, entries.data(), tracked_ids.data(),
                                             /*release_slot=*/false, tracked.data(), results.data(), s))
      return st;

  // refined estimates, agreement, average; the move of the necessity test for every candidate that agrees
  std::vector<int> tested;
  std::vector<LoopNecessityCandidate> moves;
  for (int j = 0; j < n_entries; j += 3) {
    const int c = entry_candidate[j];
    bba_loop_verification& v = out[c];
    Pose refined[3];
    for (int i = 0; i < 3; ++i) {
      const Pose cur_T_tracked = ToPose(&tracked[7 * static_cast<size_t>(j + i)]);
      const Pose old_T_cur_refined = Compose(matched_T_this[j + i], Inverse(cur_T_tracked));   // :546
      refined[i] = Inverse(old_T_cur_refined);                                                // :547
      FromPose(refined[i], v.cur_T_old_refined[i]);
      v.tracking[i] = results[j + i];
    }
    v.status = LoopAgreement(refined, max_angle, max_translation, &v.angle_difference, &v.translation_difference);
    const Pose average = AveragePose(3, refined);
    FromPose(average, v.cur_T_old);
    if (v.status != BBA_LOOP_ACCEPTED) continue;
    // cur_estimate_TR_cur_actual = (cur_T_old_averaged * matched.frame_T_global) * current.global_T_frame (:630-635)
    const bba_loop_candidate& k = candidates[c];
    const Pose move = Compose(Compose(average, Inverse(kfs[k.matched_keyframe_id].pose)), kfs[k.current_keyframe_id].pose);
    LoopNecessityCandidate m{};
    ToMatrix3x4(move, m.T);
    m.depth = kfs[k.current_keyframe_id].depth;
    m.depth_pitch = static_cast<uint32_t>(kfs[k.current_keyframe_id].depth_pitch);
    moves.push_back(m);
    tested.push_back(c);
  }

  // necessity: one launch for every candidate that agrees (grid.y = candidate)
  const int n_tested = static_cast<int>(tested.size());
  if (n_tested > 0) {
    auto& lv = h->fe.loop;
    const int blocks = NecessityBlocks(h->cfg.depth_width * h->cfg.depth_height);
    const size_t slots = static_cast<size_t>(n_tested) * blocks;
    BBA_CUDA(h, lv.h_candidates.Reserve(n_tested));
    BBA_CUDA(h, lv.d_candidates.Reserve(n_tested));
    BBA_CUDA(h, lv.d_sum.Reserve(slots));
    BBA_CUDA(h, lv.h_sum.Reserve(slots));
    BBA_CUDA(h, lv.d_count.Reserve(slots));
    BBA_CUDA(h, lv.h_count.Reserve(slots));
    std::copy(moves.begin(), moves.end(), lv.h_candidates.get());
    BBA_CUDA(h, cudaMemcpyAsync(lv.d_candidates, lv.h_candidates, sizeof(LoopNecessityCandidate) * n_tested, cudaMemcpyHostToDevice, s));
    NecessityArgs a{};
    a.cam = MakeCamera(h, view.cams, view.cfactor);
    a.candidates = lv.d_candidates;
    a.partial_sum = lv.d_sum;
    a.partial_count = lv.d_count;
    BBA_LAUNCH(h, h->front_end_launches, LaunchLoopNecessity, a, n_tested, s);
    if (bba_status st = view.ReleaseSlot()) return st;   // (the last reader of the cfactor)
    BBA_CUDA(h, cudaMemcpyAsync(lv.h_sum, lv.d_sum, sizeof(double) * slots, cudaMemcpyDeviceToHost, s));
    BBA_CUDA(h, cudaMemcpyAsync(lv.h_count, lv.d_count, sizeof(unsigned int) * slots, cudaMemcpyDeviceToHost, s));
    BBA_CUDA(h, cudaStreamSynchronize(s));
    for (int t = 0; t < n_tested; ++t) {
      bba_loop_verification& v = out[tested[t]];
      double sum = 0.0;
      uint32_t pixels = 0;
      for (int b = 0; b < blocks; ++b) {   // in block order
        sum += lv.h_sum[static_cast<size_t>(t) * blocks + b];
        pixels += lv.h_count[static_cast<size_t>(t) * blocks + b];
      }
      v.pixel_count = pixels;
      // the reference's float distance_sum / distance_count, here an fp64 sum rounded once
      v.average_pixel_distance = pixels > 0 ? static_cast<float>(sum / pixels) : std::numeric_limits<float>::quiet_NaN();
      if (pixels >= kMinNecessityPixels && v.average_pixel_distance <= max_pixels) v.status = BBA_LOOP_CORRECTION_TOO_SMALL;
    }
  }
  return BBA_OK;
}

}  // namespace
}  // namespace bba

using namespace bba;

extern "C" {

bba_status bba_verify_loop_closures(bba_handle h, const bba_loop_verification_options* options, int count,
                                    const bba_loop_candidate* candidates, bba_loop_verification* out, void* stream) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  return VerifyLoopClosures(h, options, count, candidates, out, static_cast<cudaStream_t>(stream));
}

void bba_host_average_pose(int count, const float* poses, float out[7]) {
  if (count < 1 || !poses || !out) return;
  std::vector<Pose> p(count);
  for (int i = 0; i < count; ++i) p[i] = ToPose(poses + 7 * static_cast<size_t>(i));
  FromPose(AveragePose(count, p.data()), out);
}

int bba_host_loop_agreement(const float cur_T_old_refined[21], float max_angle, float max_translation, float out_average[7],
                            float* angle_difference, float* translation_difference) {
  if (!cur_T_old_refined) return -1;
  Pose refined[3];
  for (int i = 0; i < 3; ++i) refined[i] = ToPose(cur_T_old_refined + 7 * i);
  float angle = 0.f, translation = 0.f;
  const int status = LoopAgreement(refined, Threshold(max_angle, kDefaultMaxAngle), Threshold(max_translation, kDefaultMaxTranslation),
                                   &angle, &translation);
  if (out_average) FromPose(AveragePose(3, refined), out_average);
  if (angle_difference) *angle_difference = angle;
  if (translation_difference) *translation_difference = translation;
  return status;
}

}  // extern "C"
