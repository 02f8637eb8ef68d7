// pose_step.cu -- the pose step of libbadba_b200 (host side): the spatial order of the surfels, the batched Gauss-Newton loop of
// EstimateFramePose over all keyframes at once, and the entry points that evaluate the pose kernel or track one frame.
#include <cstring>
#include <thread>

#include "handle.hpp"

namespace bba {

// Sizes the pose stream for surfels_size surfels and, with sort, makes the spatial order of the surfels current (see
// PoseStep::order_stale); with rebuild it is sorted again even when it is current.
bba_status EnsureSpatialOrder(bba_handle h, bool sort, bool rebuild, cudaStream_t s) {
  auto& p = h->pose;
  const uint32_t n = h->surfels_size;
  if (n > p.order.capacity) {
    p.order = {};   // frees the old buffers before the larger ones are allocated
    p.order_stale = true;
    const uint32_t cap = (n + 511u) / 512u * 512u;   // a multiple of the largest pose tile: 16-byte aligned stream rows
    const size_t sort_bytes = SpatialOrderTempBytes(cap);
    BBA_CUDA(h, p.order.words.Reserve(4 * static_cast<size_t>(cap) + 8));
    BBA_CUDA(h, p.order.temp.Reserve(sort_bytes));
    BBA_CUDA(h, p.order.stream.Reserve(kPoseStreamRows * static_cast<size_t>(cap)));
    BBA_CUDA(h, p.order.boxes.Reserve(8 * static_cast<size_t>(cap / kSpatialChunk)));
    uint32_t* words = p.order.words;
    p.order.view.keys_in = words;
    p.order.view.keys_out = words + cap;
    p.order.view.index_in = words + 2 * static_cast<size_t>(cap);
    p.order.view.perm = words + 3 * static_cast<size_t>(cap);
    p.order.view.bounds = words + 4 * static_cast<size_t>(cap);
    p.order.view.temp = p.order.temp;
    p.order.view.temp_bytes = sort_bytes;
    p.order.capacity = cap;
  }
  if (sort && (rebuild || p.order_stale || p.order_n != n)) {
    BBA_LAUNCH(h, h->launches, LaunchSpatialOrder, h->surfels, SurfelPitch(h), n, p.order.view, s);
    p.order_n = n;
    p.order_stale = false;
  }
  return BBA_OK;
}

namespace {

// Launch setup of the pose kernel, shared by the pose step and the entry points that evaluate it at a fixed state: arguments
// over the handle's buffers (the caller sets work_list / work_count) and, for a PRE variant, the pose stream built on s.
// The surfels do not move during a pose step: what the descriptor residual needs of a surfel alone (unpacked normal, the two
// tangent points) is computed once here instead of once per (surfel, keyframe, Gauss-Newton iteration) pair, and the surfels are
// put into spatial order with a bounding box per chunk, so that the kernel skips whole chunks outside a keyframe's view.  Not
// worth a launch + 14 rows of traffic for a handful of keyframes (frame tracking): the kernel then derives the frames per pair.
// variant = kPoseVariantAuto: that choice, from the number of keyframes n_work; any other: forced (bba_debug_pose_coeffs_batch).
// stream_current: the last pose step built the stream for the same surfels and the same choice, and nothing has changed the
// surfels since; it is used as it is.
bba_status PreparePoseAccumulate(bba_handle h, int n_work, int variant, cudaStream_t s, PoseAccumulateArgs* acc,
                                 bool stream_current = false) {
  auto& p = h->pose;
  SetSurfelFields(h, acc);
  acc->kfs = h->d_kfs;
  acc->work_records = p.d_work_records;
  acc->acc = p.d_acc;
  acc->exact = h->deterministic ? p.d_exact.get() : nullptr;
  acc->stage_counts = p.d_stage_counts;
  acc->queue = p.d_queue;
  acc->group = p.group;
  acc->stream = nullptr;
  acc->stream_pitch = 0;
  acc->boxes = nullptr;
  acc->stream_sorted = false;
  const bool pre = variant == kPoseVariantAuto ? h->cfg.use_descriptor_residuals && n_work >= 4 : PoseVariantPre(variant);
  // The rebuild (bounds, keys, radix sort) has a fixed cost of ~0.1 ms, most of it launch overhead at the start of a pose step
  // whose stream has just drained: measured on cfg2 (20 keyframes x 200 k surfels) it cost more than the culling it buys, on
  // cfg3_rank8 (200 x 375 k) it paid for itself many times over.  Below kSpatialOrderMinPairs (surfel, keyframe) pairs per
  // launch the stream keeps the caller's order; its chunk boxes are culled all the same.  A forced variant always sorts.  (In a
  // BA iteration the geometry step has usually made the order current already.)
  const bool sort = variant != kPoseVariantAuto ||
                    static_cast<uint64_t>(h->surfels_size) * static_cast<uint64_t>(n_work) >= kSpatialOrderMinPairs;
  if (pre && h->surfels_size > 0 && stream_current) {
    acc->stream = p.order.stream;
    acc->stream_pitch = p.order.capacity;
    acc->boxes = p.order.boxes;
    acc->stream_sorted = sort;
  } else if (pre && h->surfels_size > 0) {
    if (bba_status st = EnsureSpatialOrder(h, sort, /*rebuild=*/false, s)) return st;
    BBA_LAUNCH(h, h->launches, LaunchPoseStream, h->surfels, acc->pitch, h->surfels_size, sort ? p.order.view.perm : nullptr, p.order.stream,
               p.order.capacity, p.order.boxes, s);
    acc->stream = p.order.stream;
    acc->stream_pitch = p.order.capacity;
    acc->boxes = p.order.boxes;
    acc->stream_sorted = sort;
  }
  return BBA_OK;
}

// Stages one evaluation of the pose kernel on s: every keyframe's record at its own pose except keyframe ids[i] at poses[i]; the
// work list (the ids this rank owns, all of them without `owner`) and its count in h_work and on the device; zeroed
// accumulators, stage counts and work queue.  *n_work: the length of the work list.
bba_status StagePoseWork(bba_handle h, const std::vector<int>& ids, const std::vector<Pose>& poses, const int* owner, cudaStream_t s,
                         int* n_work) {
  auto& p = h->pose;
  const int K = static_cast<int>(h->keyframes.size()), M = h->cfg.max_keyframes;
  if (bba_status st = WaitStaging(h)) return st;
  for (int k = 0; k < K; ++k) FillKfDevice(h->keyframes[k], h->keyframes[k].pose, h->staging.h_kfs + k);
  int n = 0;
  for (size_t i = 0; i < ids.size(); ++i) {
    FillKfDevice(h->keyframes[ids[i]], poses[i], h->staging.h_kfs + ids[i]);
    if (!owner || owner[i] == h->cfg.rank) p.h_work[n++] = ids[i];
  }
  p.h_work[M] = n;
  p.h_work[M + 1] = 0;
  BBA_CUDA(h, cudaMemcpyAsync(h->d_kfs, h->staging.h_kfs, sizeof(KfDevice) * K, cudaMemcpyHostToDevice, s));
  if (n) BBA_CUDA(h, cudaMemcpyAsync(p.d_work[0], p.h_work, sizeof(int) * n, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemcpyAsync(p.d_count, p.h_work + M, sizeof(int) * 2, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemsetAsync(p.d_acc, 0, sizeof(double) * kPoseAccSize * K, s));
  if (h->deterministic) BBA_CUDA(h, cudaMemsetAsync(p.d_exact, 0, sizeof(ExactSum) * kPoseAccSize * K, s));
  BBA_CUDA(h, cudaMemsetAsync(p.d_stage_counts, 0, sizeof(unsigned long long) * 2 * K, s));
  BBA_CUDA(h, cudaMemsetAsync(p.d_queue, 0, sizeof(unsigned int), s));
  *n_work = n;
  return BBA_OK;
}

// One launch of the pose kernel for keyframes ids at poses; on return (stream synchronised) rec / sc hold every keyframe's
// accumulator record (in the deterministic mode its exact sums rounded to fp64) and its two stage counts, and the device records
// are zero again.  stream_current: see PreparePoseAccumulate.
bba_status PoseCoeffsBatch(bba_handle h, const std::vector<int>& ids, const std::vector<Pose>& poses, int variant, bool with_stats,
                           cudaStream_t s, std::vector<double>* rec, std::vector<unsigned long long>* sc, bool stream_current = false) {
  auto& p = h->pose;
  const int K = static_cast<int>(h->keyframes.size());
  int count = 0;
  if (bba_status st = StagePoseWork(h, ids, poses, nullptr, s, &count)) return st;
  PoseAccumulateArgs acc;
  if (bba_status st = PreparePoseAccumulate(h, count, variant, s, &acc, stream_current)) return st;
  acc.work_list = p.d_work[0];
  acc.work_count = p.d_count;
  BBA_LAUNCH(h, h->launches, LaunchPoseAccumulate, acc, h->sm_count, with_stats, count, s, variant);
  rec->resize(static_cast<size_t>(kPoseAccSize) * K);
  sc->resize(2 * static_cast<size_t>(K));
  std::vector<ExactSum> exact(h->deterministic ? rec->size() : 0);
  if (h->deterministic) {
    BBA_CUDA(h, cudaMemcpyAsync(exact.data(), p.d_exact, sizeof(ExactSum) * exact.size(), cudaMemcpyDeviceToHost, s));
    BBA_CUDA(h, cudaMemsetAsync(p.d_exact, 0, sizeof(ExactSum) * exact.size(), s));
  } else {
    BBA_CUDA(h, cudaMemcpyAsync(rec->data(), p.d_acc, sizeof(double) * rec->size(), cudaMemcpyDeviceToHost, s));
  }
  BBA_CUDA(h, cudaMemcpyAsync(sc->data(), p.d_stage_counts, sizeof(unsigned long long) * sc->size(), cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaMemsetAsync(p.d_acc, 0, sizeof(double) * rec->size(), s));
  BBA_CUDA(h, cudaMemsetAsync(p.d_stage_counts, 0, sizeof(unsigned long long) * sc->size(), s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  h->staging.pending = false;
  for (size_t i = 0; i < exact.size(); ++i) (*rec)[i] = ExactFinalize(exact[i]);
  return BBA_OK;
}

// The result of RunPoseStep for keyframe slot id.
void FramePoseResult(bba_handle h, int id, float out[7], int* iterations, int* converged) {
  std::memcpy(out, h->pose.h_pose_est + 7 * id, sizeof(float) * 7);
  if (iterations) *iterations = h->pose.h_iterations[id];
  if (converged) *converged = h->pose.h_converged[id];
}

// Keyframe slot id's coefficients out of what PoseCoeffsBatch read back (with stats).
void FillPoseCoeffs(bba_handle h, const std::vector<double>& rec, const std::vector<unsigned long long>& sc, int id, bba_pose_coeffs* out) {
  const double* r = rec.data() + static_cast<size_t>(id) * kPoseAccSize;
  for (int i = 0; i < 21; ++i) out->H[i] = static_cast<float>(r[i]);
  for (int i = 0; i < 6; ++i) out->b[i] = static_cast<float>(r[21 + i]);
  out->n_pair = h->surfels_size;
  out->n_inimg = sc[2 * id];
  out->n_depthok = sc[2 * id + 1];
  out->n_assoc = static_cast<uint64_t>(r[27] + 0.5);
  out->n_photo = static_cast<uint64_t>(r[28] + 0.5);
  out->cost_depth = r[29];
  out->cost_desc1 = r[30];
  out->cost_desc2 = r[31];
}

// Frame-to-model pose estimation (EstimateFramePose) of `count` entries, entry i = frame frame_of_entry[i] (i without the map)
// from init[i]; the arguments are valid.  The entries ride through the pose step as temporary entries behind the keyframes, in
// chunks of as many entries as there are free keyframe slots, in entry order: each chunk's distinct frames get a luma texture of
// the pool (one extraction launch), then one pose step runs every entry's Gauss-Newton loop and, with at_estimate, one more
// pose-kernel launch with stats evaluates every entry at its result.  The temporary entries take part in nothing else (no
// co-visibility, no activation state), own nothing and are removed before the next chunk; their slots' cost statistics are reset.
// Serves both entry points: bba_estimate_frame_pose_for_frame is the one-entry, one-frame case.
bba_status EstimateFramePoses(bba_handle h, int frame_count, const bba_frame_buffers* frames, int count, const int* frame_of_entry,
                              const float* init, float* out, int* iterations, int* converged, bba_pose_coeffs* at_estimate,
                              cudaStream_t s, const char* fn) {
  const int K = static_cast<int>(h->keyframes.size());
  const int free_slots = h->cfg.max_keyframes - K;
  if (free_slots < 1) return Fail(h, BBA_ERR_STATE, std::string(fn) + " needs one free keyframe slot (max_keyframes reached)");
  // the frames' luma memory stays bounded by the free slots: the pool (entries without an array hold no memory) and the BA
  // side's staging planes (released when they hold more; the next user allocates as many as it needs)
  auto& pool = h->frame_luma;
  pool.resize(free_slots);
  LumaStaging& staging = h->staging.luma;
  if (staging.planes > free_slots) {
    staging.plane = PitchedBuffer();
    staging.planes = 0;
  }
  std::vector<cudaTextureObject_t> luma(frame_count);   // the luma textures of the current chunk's frames
  std::vector<int> frame_of_chunk_entry;
  std::vector<int> ids;
  std::vector<Pose> poses;
  std::vector<double> rec;
  std::vector<unsigned long long> sc;
  for (int begin = 0; begin < count; begin += free_slots) {
    const int n = std::min(free_slots, count - begin);
    frame_of_chunk_entry.resize(n);
    for (int i = 0; i < n; ++i) frame_of_chunk_entry[i] = frame_of_entry ? frame_of_entry[begin + i] : begin + i;
    bba_status st = MakeFrameLumaTextures(h, /*front_end=*/false, frames, frame_of_chunk_entry, &pool, luma.data(), s);
    ids.resize(n);
    poses.resize(n);
    for (int i = 0; st == BBA_OK && i < n; ++i) {
      const int f = frame_of_chunk_entry[i];
      Keyframe entry{};
      entry.depth = frames[f].depth; entry.depth_pitch = frames[f].depth_pitch;
      entry.normals = frames[f].normals; entry.normals_pitch = frames[f].normals_pitch;
      entry.tex = luma[f];
      entry.pose = PoseFromArray(init + 7 * static_cast<size_t>(begin + i));
      entry.activation = BBA_KF_ACTIVE;
      ids[i] = K + i;
      poses[i] = entry.pose;
      h->keyframes.push_back(std::move(entry));
    }
    if (st == BBA_OK) st = RunPoseStep(h, ids, poses, 30, s);
    if (st == BBA_OK) {
      for (int i = 0; i < n; ++i) {
        const size_t e = static_cast<size_t>(begin + i);
        FramePoseResult(h, K + i, out + 7 * e, iterations ? iterations + e : nullptr, converged ? converged + e : nullptr);
        poses[i] = PoseFromArray(out + 7 * e);
      }
      // the pose step's surfel stream is still current: same surfels, same entry count and so the same variant
      if (at_estimate) st = PoseCoeffsBatch(h, ids, poses, kPoseVariantAuto, /*with_stats=*/true, s, &rec, &sc, /*stream_current=*/true);
    }
    h->keyframes.erase(h->keyframes.begin() + K, h->keyframes.end());
    for (int i = 0; i < n; ++i)   // the slots' cost statistics belong to future keyframes
      if (K + i < static_cast<int>(h->kf_cost.size())) h->kf_cost[K + i] = 0.f;
    if (st) return st;
    if (at_estimate)
      for (int i = 0; i < n; ++i) FillPoseCoeffs(h, rec, sc, K + i, at_estimate + begin + i);
  }
  return BBA_OK;
}

}  // namespace

// Runs the Gauss-Newton loop of EstimateFramePose for the keyframes in `ids`, all at once, starting from
// `init` poses.  On return (stream synchronised) h_pose_est / h_iterations / h_converged / h_first_stats hold the results.
bba_status RunPoseStep(bba_handle h, const std::vector<int>& ids, const std::vector<Pose>& init, int max_iterations, cudaStream_t s) {
  auto& p = h->pose;
  auto& x = h->xchg;
  const int K = static_cast<int>(h->keyframes.size());
  const int n = static_cast<int>(ids.size());
  if (n == 0) return BBA_OK;
  // Multi-GPU: the work list is dealt to the ranks (AssignKeyframes); every rank runs the Gauss-Newton loops of its own
  // keyframes and the results are published with one sum all-reduce over disjoint slots (below).
  const int world = h->cfg.world_size;
  if (bba_status st = CheckCollective(h)) return st;
  std::vector<int> owner(n, 0);
  if (world > 1) AssignKeyframes(h, ids, &owner);
  int n_local = 0;
  if (bba_status st = StagePoseWork(h, ids, init, owner.data(), s, &n_local)) return st;
  for (int k = 0; k < K; ++k) PoseToArray(h->keyframes[k].pose, p.h_pose_est + 7 * k);
  for (int i = 0; i < n; ++i) PoseToArray(init[i], p.h_pose_est + 7 * ids[i]);
  BBA_CUDA(h, cudaMemcpyAsync(p.d_pose_est, p.h_pose_est, sizeof(float) * 7 * K, cudaMemcpyHostToDevice, s));
  if (world > 1 && n_local) BBA_CUDA(h, cudaMemcpyAsync(x.d_local_ids, p.h_work, sizeof(int) * n_local, cudaMemcpyHostToDevice, s));
  bool terms = false, attitude = false;
  if (bba_status st = StagePoseTerms(h, ids, init, s, &terms, &attitude)) return st;
  BBA_CUDA(h, cudaMemsetAsync(p.d_iterations, 0, sizeof(int) * K, s));
  BBA_CUDA(h, cudaMemsetAsync(p.d_converged, 0, sizeof(int) * K, s));
  if (bba_status st = MarkStaging(h, s)) return st;

  PoseAccumulateArgs acc;
  if (bba_status st = PreparePoseAccumulate(h, n_local, kPoseVariantAuto, s, &acc)) return st;
  PoseSolveArgs sol;
  sol.kfs = h->d_kfs;
  sol.pose_est = p.d_pose_est;
  sol.acc = p.d_acc;
  sol.exact = acc.exact;
  sol.stage_counts = p.d_stage_counts;
  sol.iterations = p.d_iterations;
  sol.converged = p.d_converged;
  sol.first_stats = p.d_first_stats;
  sol.max_iterations = max_iterations;
  sol.totals = p.d_totals;
  sol.host_flag = p.d_flag;
  sol.queue = p.d_queue;
  sol.term_offsets = terms ? p.d_term_offsets.get() : nullptr;
  sol.terms = terms ? p.d_terms.get() : nullptr;
  sol.attitude = attitude ? p.d_attitude.get() : nullptr;
  p.h_flag[0] = 0;
  p.h_flag[1] = n_local;
  if (h->profiling) BBA_CUDA(h, cudaMemsetAsync(p.d_totals, 0, sizeof(unsigned long long) * 8, s));
  int enqueued = 0;
  for (int it = 0; it < max_iterations; ++it) {
    const int cur = it & 1;
    acc.work_list = p.d_work[cur];
    acc.work_count = p.d_count + cur;
    if (h->surfels_size > 0) {
      if (h->profiling && it < 32) BBA_CUDA(h, cudaEventRecord(h->prof_ev[2 * it], s));
      BBA_LAUNCH(h, h->launches, LaunchPoseAccumulate, acc, h->sm_count, /*with_stats=*/it == 0 || h->profiling >= 2, n_local, s);
      if (h->profiling && it < 32) BBA_CUDA(h, cudaEventRecord(h->prof_ev[2 * it + 1], s));
    }
    sol.work_in = p.d_work[cur];
    sol.count_in = p.d_count + cur;
    sol.work_out = p.d_work[cur ^ 1];
    sol.count_out = p.d_count + (cur ^ 1);
    sol.iteration = it;
    BBA_LAUNCH(h, h->launches, LaunchPoseSolve, sol, s);
    ++enqueued;
    // Keep kDepth iterations queued ahead of the one executing: wait (host poll on zero-copy memory, the stream is never
    // blocked) until iteration it-kDepth has finished, and stop as soon as an iteration left no unconverged keyframe.  (An
    // iteration whose list turned out empty costs three immediately-returning launches, ~10 us; the depth rides out a host
    // thread that is descheduled for a moment -- on a box whose cores were oversubscribed, 2 CPUs for 4 ranks, a depth of one
    // left the GPU idle between iterations.)
    // In the deterministic mode nothing is queued ahead: how many iterations the host had enqueued when the last one finished
    // depends on its timing, and with it the number of launches the call reports (bba_ba_result::kernel_launches).
    const int depth = h->deterministic ? 0 : 3;
    if (it >= depth) {
      unsigned int polls = 0;
      while (p.h_flag[0] < it - depth + 1) {
        // cudaSuccess: everything drained; any other result than "not ready" is a (sticky) device fault that would
        // otherwise leave this loop spinning for ever -- the BBA_CUDA check below reports it
        if (cudaStreamQuery(s) != cudaErrorNotReady) break;
        if (++polls > 256 && (polls & 15) == 0) std::this_thread::yield();   // let the other ranks' host threads run
      }
    }
    if (it >= 1 && p.h_flag[0] >= 1 && p.h_flag[1] == 0) break;   // (h_flag[1] belongs to the last finished iteration)
  }
  if (world > 1) {
    // ONE all-reduce per pose step: every rank contributes the slots of its keyframes, all others are zero.
    BBA_CUDA(h, cudaMemsetAsync(x.d_pose_pack, 0, sizeof(float) * kPoseSlot * K, s));
    BBA_LAUNCH(h, h->launches, LaunchPackPoseResults, x.d_local_ids, n_local, p.d_pose_est, p.d_iterations, p.d_converged, p.d_first_stats,
               x.d_pose_pack, s);
    if (bba_status st = Collective(h, BBA_COLLECTIVE_ALLREDUCE_SUM, x.d_pose_pack, static_cast<size_t>(kPoseSlot) * K, s)) return st;
    x.replicated_pass_pending = false;   // (every rank's earlier work on this stream precedes its contribution)
    BBA_CUDA(h, cudaMemcpyAsync(x.h_pose_pack, x.d_pose_pack, sizeof(float) * kPoseSlot * K, cudaMemcpyDeviceToHost, s));
  } else {
    BBA_CUDA(h, cudaMemcpyAsync(p.h_pose_est, p.d_pose_est, sizeof(float) * 7 * K, cudaMemcpyDeviceToHost, s));
    BBA_CUDA(h, cudaMemcpyAsync(p.h_iterations, p.d_iterations, sizeof(int) * K, cudaMemcpyDeviceToHost, s));
    BBA_CUDA(h, cudaMemcpyAsync(p.h_converged, p.d_converged, sizeof(int) * K, cudaMemcpyDeviceToHost, s));
    BBA_CUDA(h, cudaMemcpyAsync(p.h_first_stats, p.d_first_stats, sizeof(double) * 8 * K, cudaMemcpyDeviceToHost, s));
  }
  if (h->profiling) BBA_CUDA(h, cudaMemcpyAsync(p.h_totals, p.d_totals, sizeof(unsigned long long) * 8, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  h->staging.pending = false;
  if (world > 1) {
    for (int i = 0; i < n; ++i) {
      const int kf = ids[i];
      const float* slot = x.h_pose_pack + static_cast<size_t>(kf) * kPoseSlot;
      std::memcpy(p.h_pose_est + 7 * kf, slot, sizeof(float) * 7);
      p.h_iterations[kf] = static_cast<int>(slot[7] + 0.5f);
      p.h_converged[kf] = static_cast<int>(slot[8] + 0.5f);
      for (int j = 0; j < 8; ++j) p.h_first_stats[8 * kf + j] = slot[9 + j];
    }
  }
  // cost model for the next assignment: a culled pair costs ~6 % of a pair that projects into the image
  if (h->kf_cost.size() < static_cast<size_t>(K)) h->kf_cost.resize(h->cfg.max_keyframes, 0.f);
  for (int kf : ids)
    h->kf_cost[kf] = static_cast<float>(std::max(1, p.h_iterations[kf]) * (0.06 * h->surfels_size + p.h_first_stats[8 * kf + 5]));
  if (h->profiling && h->surfels_size > 0) {
    int real_iterations = 0;   // iterations that had a non-empty work list (h_work: this rank's keyframes)
    for (int i = 0; i < n_local; ++i) real_iterations = std::max(real_iterations, p.h_iterations[p.h_work[i]]);
    for (int it = 0; it < std::min(real_iterations, std::min(enqueued, 32)); ++it) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, h->prof_ev[2 * it], h->prof_ev[2 * it + 1]);
      h->profile.pose_ms += ms;
      ++h->profile.pose_launches;
    }
    h->profile.kf_evals += p.h_totals[0];
    h->profile.n_pair += p.h_totals[0] * static_cast<uint64_t>(h->surfels_size);
    h->profile.n_inimg += p.h_totals[1];
    h->profile.n_depthok += p.h_totals[2];
    h->profile.n_assoc += p.h_totals[3];
    h->profile.n_photo += p.h_totals[4];
  }
  return BBA_OK;
}

}  // namespace bba

using namespace bba;

extern "C" {

bba_status bba_accumulate_pose_coeffs(bba_handle h, int id, const float pose[7], bba_pose_coeffs* out, void* stream) {
  CHECK_KF(h, id);
  if (!pose || !out) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckSurfels(h)) return st;
  std::vector<double> rec;
  std::vector<unsigned long long> sc;
  if (bba_status st = PoseCoeffsBatch(h, std::vector<int>(1, id), std::vector<Pose>(1, PoseFromArray(pose)), kPoseVariantAuto,
                                      /*with_stats=*/true, static_cast<cudaStream_t>(stream), &rec, &sc))
    return st;
  FillPoseCoeffs(h, rec, sc, id, out);
  return BBA_OK;
}

bba_status bba_debug_pose_coeffs_batch(bba_handle h, int count, const int* ids, const float* poses, int variant, int with_stats,
                                       double* H, double* b, uint64_t* counts, double* costs, void* stream) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (!ids || !poses || !H || !b || !counts || (with_stats && !costs))
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_pose_coeffs_batch: null argument");
  if (count < 1 || count > h->cfg.max_keyframes)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_pose_coeffs_batch: count out of range");
  if (!PoseVariantValid(variant)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_pose_coeffs_batch: unknown variant");
  const int K = static_cast<int>(h->keyframes.size());
  std::vector<char> listed(K, 0);
  for (int i = 0; i < count; ++i) {
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_pose_coeffs_batch: bad keyframe id");
    if (listed[ids[i]]) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_pose_coeffs_batch: keyframe listed twice");
    listed[ids[i]] = 1;
  }
  if (bba_status st = CheckSurfels(h)) return st;
  std::vector<Pose> pose_list(count);
  for (int i = 0; i < count; ++i) pose_list[i] = PoseFromArray(poses + 7 * i);
  // every keyframe's record, listed or not: a record written outside the work list shows up in the caller's rows
  std::vector<double> rec;
  std::vector<unsigned long long> sc;
  if (bba_status st = PoseCoeffsBatch(h, std::vector<int>(ids, ids + count), pose_list, variant, with_stats != 0,
                                      static_cast<cudaStream_t>(stream), &rec, &sc))
    return st;
  for (int k = 0; k < K; ++k) {
    const double* r = rec.data() + static_cast<size_t>(k) * kPoseAccSize;
    std::memcpy(H + 21 * static_cast<size_t>(k), r, sizeof(double) * 21);
    std::memcpy(b + 6 * static_cast<size_t>(k), r + 21, sizeof(double) * 6);
    uint64_t* c = counts + 4 * static_cast<size_t>(k);
    c[0] = sc[2 * k];
    c[1] = sc[2 * k + 1];
    c[2] = static_cast<uint64_t>(r[27] + 0.5);
    c[3] = static_cast<uint64_t>(r[28] + 0.5);
    if (with_stats) std::memcpy(costs + 3 * static_cast<size_t>(k), r + 29, sizeof(double) * 3);
  }
  return BBA_OK;
}

bba_status bba_debug_set_pose_group(bba_handle h, int keyframes) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (keyframes < 0 || keyframes > kPoseMaxGroup)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_set_pose_group: keyframes out of range (0 .. " + std::to_string(kPoseMaxGroup) + ")");
  h->pose.group = keyframes;
  return BBA_OK;
}

bba_status bba_estimate_frame_pose(bba_handle h, int id, const float init[7], float out[7], int* iterations, int* converged,
                                   void* stream) {
  CHECK_KF(h, id);
  if (!init || !out) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckSurfels(h)) return st;
  std::vector<int> ids(1, id);
  std::vector<Pose> poses(1, PoseFromArray(init));
  if (bba_status st = RunPoseStep(h, ids, poses, 30, static_cast<cudaStream_t>(stream))) return st;
  FramePoseResult(h, id, out, iterations, converged);
  return BBA_OK;
}

bba_status bba_estimate_frame_pose_for_frame(bba_handle h, const uint16_t* device_depth, size_t depth_pitch,
                                             const uint16_t* device_normals, size_t normals_pitch,
                                             const uint8_t* device_color_rgba, size_t color_pitch, const float init[7], float out[7],
                                             int* iterations, int* converged, void* stream) {
  if (!h || !device_depth || !device_normals || !device_color_rgba || !init || !out) return BBA_ERR_INVALID_ARGUMENT;
  if (!FramePitchesOk(h, depth_pitch, normals_pitch, color_pitch)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "frame buffer pitch too small");
  if (bba_status st = CheckSurfels(h)) return st;
  const bba_frame_buffers frame{device_depth, depth_pitch, device_normals, normals_pitch, device_color_rgba, color_pitch};
  return EstimateFramePoses(h, 1, &frame, 1, nullptr, init, out, iterations, converged, nullptr, static_cast<cudaStream_t>(stream),
                            "bba_estimate_frame_pose_for_frame");
}

bba_status bba_estimate_frame_poses_for_frames(bba_handle h, int frame_count, const bba_frame_buffers* frames, int count,
                                               const int* frame_of_entry, const float* global_T_frame_initial,
                                               float* global_T_frame_estimate, int* iterations, int* converged,
                                               bba_pose_coeffs* at_estimate, void* stream) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_estimate_frame_poses_for_frames: ";
  if (!frames || !global_T_frame_initial || !global_T_frame_estimate) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  if (count < 1 || frame_count < 1) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count and frame_count must be at least 1");
  if (!frame_of_entry && count > frame_count)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "without frame_of_entry entry i uses frame i: count > frame_count");
  for (int f = 0; f < frame_count; ++f) {
    const bba_frame_buffers& b = frames[f];
    if (!b.depth || !b.normals || !b.color_rgba) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null frame buffer");
    if (!FramePitchesOk(h, b.depth_pitch, b.normals_pitch, b.color_pitch))
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "frame buffer pitch too small");
  }
  for (int i = 0; frame_of_entry && i < count; ++i)
    if (frame_of_entry[i] < 0 || frame_of_entry[i] >= frame_count) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "frame index out of range");
  if (h->cfg.world_size > 1) return Fail(h, BBA_ERR_UNSUPPORTED, fn + "runs on one rank only (world_size > 1)");
  if (bba_status st = CheckSurfels(h)) return st;
  return EstimateFramePoses(h, frame_count, frames, count, frame_of_entry, global_T_frame_initial, global_T_frame_estimate, iterations,
                            converged, at_estimate, static_cast<cudaStream_t>(stream), "bba_estimate_frame_poses_for_frames");
}

}  // extern "C"
