// bundle_adjust.cu -- bundle adjustment in libbadba_b200 (host side): the alternating scheme and the PCG scheme, the geometry and
// intrinsics steps, the PCG phases, and the surfel lifecycle (creation, merging, compaction, end tasks) with their entry points.
#include <chrono>
#include <cmath>
#include <cstring>
#include <limits>

#include "handle.hpp"

namespace bba {
namespace {

// direct_ba.cc:549-564
void DetermineCovisibleActiveKeyframes(bba_handle h) {
  for (Keyframe& kf : h->keyframes) {
    if (kf.activation != BBA_KF_ACTIVE) continue;
    for (int o : kf.covis) {
      Keyframe& other = h->keyframes[o];
      if (other.activation == BBA_KF_INACTIVE) other.activation = BBA_KF_COVISIBLE_ACTIVE;
    }
  }
}

// The per-tile group epochs of the geometry kernels for surfels_size surfels, with room for max_surfel_count when they grow.
bba_status ReserveTileEpochs(bba_handle h) {
  const uint32_t need = (h->surfels_size + 31u) / 32u;
  BBA_CUDA(h, h->geo.d_tile_epoch.Reserve(need, std::max<uint32_t>((h->cfg.max_surfel_count + 31u) / 32u, need) + 1));
  return BBA_OK;
}

// In which order the geometry launches visit the surfels.  kCaller: the caller's (the in-loop creation's two launches address the
// old and the new surfels by caller index, the PCG scheme's shards are the caller's granules).  kByPairs: the spatial order from
// kSpatialOrderMinPairs (surfel, keyframe) pairs per launch, the pose step's rule (the pose step then reuses the order).
// kSpatial: always the spatial order (the standalone entry points, like the forced pose variants).
enum class GeoOrder { kCaller, kByPairs, kSpatial };

bba_status BuildGeometryArgs(bba_handle h, bba::GeometryArgs* g, cudaStream_t s, GeoOrder order) {
  const int K = static_cast<int>(h->keyframes.size());
  int cnt = 0;
  for (int k = 0; k < K; ++k)
    if (h->keyframes[k].activation != BBA_KF_INACTIVE) h->geo.h_list[cnt++] = k;
  if (cnt) BBA_CUDA(h, cudaMemcpyAsync(h->geo.d_list, h->geo.h_list, sizeof(int) * cnt, cudaMemcpyHostToDevice, s));
  // With several ranks the order is rebuilt here from the replicated positions, so that every rank deals the same granules (the
  // pose step sorts by its own share of the keyframes, so a current order need not be the same on every rank).  With peer stores
  // (into the other ranks' replicas) the launches keep the caller's order: in spatial order that mode left about 3 % of
  // the surfels different from the one-GPU result in a two-rank run, for a reason not yet found, while the host-collective
  // exchange in spatial order reproduces it bit for bit.
  const bool sort = !PeerStores(h) && (order == GeoOrder::kSpatial ||
                                       (order == GeoOrder::kByPairs &&
                                        static_cast<uint64_t>(h->surfels_size) * static_cast<uint64_t>(cnt) >= kSpatialOrderMinPairs));
  if (bba_status st = EnsureSpatialOrder(h, sort, /*rebuild=*/h->cfg.world_size > 1, s)) return st;
  if (bba_status st = PeerFence(h, s)) return st;
  SetSurfelFields(h, g);
  SetShardFields(h, g);
  g->perm = sort && h->surfels_size > 0 ? h->pose.order.view.perm : nullptr;
  g->stream = h->pose.order.stream;
  g->stream_pitch = h->pose.order.capacity;
  h->geo.perm = g->perm;
  g->active = h->active;
  g->kfs = h->d_kfs;
  g->kf_list = h->geo.d_list;
  g->kf_count = cnt;
  g->queue = h->geo.d_queue;
  g->tile_shift = 8;
  g->peers = KernelPeers(h);
  if (bba_status st = ReserveTileEpochs(h)) return st;
  g->tile_epoch = h->geo.d_tile_epoch;
  return BBA_OK;
}

// geo.d_all_list, the keyframe list 0 .. max_keyframes - 1, made on first use.
bba_status MakeAllKeyframeList(bba_handle h) {
  if (h->geo.d_all_list) return BBA_OK;   // (set only once it is filled)
  DeviceBuffer<int> all;
  BBA_CUDA(h, all.Reserve(h->cfg.max_keyframes));
  std::vector<int> iota(h->cfg.max_keyframes);
  for (int i = 0; i < h->cfg.max_keyframes; ++i) iota[i] = i;
  BBA_CUDA(h, cudaMemcpy(all, iota.data(), sizeof(int) * iota.size(), cudaMemcpyHostToDevice));
  h->geo.d_all_list = std::move(all);
  return BBA_OK;
}

// The normal equations of the intrinsics step as AccumulateIntrinsics leaves them on the device: the kIntrinsicsSums global sums
// in geo.d_intr_sums and the cell rows, P floats each, in geo.d_intr.
struct IntrinsicsEquations {
  uint32_t P;
  float *cell_B, *cell_D, *cell_b2, *cell_obs, *d_x1;   // B: 5 rows
  bba::CameraParams cam;
};

// The first half of OptimizeIntrinsics (kernel_opt_intrinsics.cc:69-108): accumulate over EVERY keyframe; in the deterministic
// mode the exact sums are rounded into the same buffers.  The handle has keyframes and surfels.
bba_status AccumulateIntrinsics(bba_handle h, bool opt_depth, bool opt_color, cudaStream_t s, IntrinsicsEquations* eq) {
  const int K = static_cast<int>(h->keyframes.size());
  const uint32_t P = static_cast<uint32_t>(h->cf_w) * h->cf_h;
  const size_t intr_floats = 64 + static_cast<size_t>(8) * P + 8;
  BBA_CUDA(h, h->geo.d_intr.Reserve(intr_floats));
  BBA_CUDA(h, h->geo.d_intr_sums.Reserve(bba::kIntrinsicsSums));
  if (bba_status st = MakeAllKeyframeList(h)) return st;
  BBA_CUDA(h, h->geo.h_intr_sums.Reserve(bba::kIntrinsicsSums));
  BBA_CUDA(h, h->geo.h_intr_x1.Reserve(8));
  if (bba_status st = UploadKeyframes(h, s)) return st;
  BBA_CUDA(h, cudaMemsetAsync(h->geo.d_intr, 0, sizeof(float) * intr_floats, s));                      // :69-80
  BBA_CUDA(h, cudaMemsetAsync(h->geo.d_intr_sums, 0, sizeof(double) * bba::kIntrinsicsSums, s));
  const size_t exact_count = static_cast<size_t>(7) * P + bba::kIntrinsicsSums;
  if (h->deterministic) BBA_CUDA(h, cudaMemsetAsync(h->geo.d_intr_exact, 0, sizeof(bba::ExactSum) * exact_count, s));
  float* cell_B = h->geo.d_intr + 64;
  float* cell_D = cell_B + static_cast<size_t>(5) * P;
  float* cell_b2 = cell_D + P;
  float* cell_obs = cell_b2 + P;
  float* d_x1 = cell_obs + P;

  bba::IntrinsicsArgs a;
  SetSurfelFields(h, &a);
  SetShardFields(h, &a);
  a.kfs = h->d_kfs;
  a.kf_list = h->geo.d_all_list;
  a.kf_count = K;
  a.queue = h->geo.d_queue;
  a.sums = h->geo.d_intr_sums;
  a.cell_B = cell_B;
  a.cell_D = cell_D;
  a.cell_b2 = cell_b2;
  a.cell_obs = cell_obs;
  a.cell_count = P;
  a.exact_cells = h->deterministic ? h->geo.d_intr_exact.get() : nullptr;
  a.exact_sums = h->deterministic ? a.exact_cells + static_cast<size_t>(7) * P : nullptr;
  BBA_LAUNCH(h, h->launches, LaunchIntrinsicsAccumulate, a, h->sm_count, opt_color, opt_depth, s);   // :84-108, one launch for all keyframes
  if (h->deterministic) BBA_LAUNCH(h, h->launches, LaunchIntrinsicsFinalize, P, a.exact_cells, cell_B, a.exact_sums, h->geo.d_intr_sums, s);
  if (h->cfg.world_size > 1) {
    // every rank accumulated its surfel shard: one sum all-reduce over [34 global sums | B | D | b2 | obs]
    BBA_LAUNCH(h, h->launches, LaunchIntrinsicsConvertSums, h->geo.d_intr_sums, h->geo.d_intr, true, s);
    if (bba_status st = Collective(h, BBA_COLLECTIVE_ALLREDUCE_SUM, h->geo.d_intr, 64 + static_cast<size_t>(8) * P, s)) return st;
    BBA_LAUNCH(h, h->launches, LaunchIntrinsicsConvertSums, h->geo.d_intr_sums, h->geo.d_intr, false, s);
  }
  *eq = IntrinsicsEquations{P, cell_B, cell_D, cell_b2, cell_obs, d_x1, a.cam};
  return BBA_OK;
}

// OptimizeIntrinsicsCUDA (kernel_opt_intrinsics.cc:39-281): accumulate over EVERY keyframe, Schur-complement the
// per-cell cfactors away, solve the 5x5 / 4x4 systems in fp64 on the host, update intrinsics, a and the cfactors.
bba_status OptimizeIntrinsics(bba_handle h, bool opt_depth, bool opt_color, cudaStream_t s) {
  if (h->surfels_size == 0 || h->keyframes.empty()) return BBA_OK;   // :56-58
  IntrinsicsEquations eq;
  if (bba_status st = AccumulateIntrinsics(h, opt_depth, opt_color, s, &eq)) return st;
  const uint32_t P = eq.P;
  float *cell_B = eq.cell_B, *cell_D = eq.cell_D, *cell_b2 = eq.cell_b2, *cell_obs = eq.cell_obs, *d_x1 = eq.d_x1;
  if (opt_depth) BBA_LAUNCH(h, h->launches, LaunchIntrinsicsSchur, P, cell_B, cell_D, cell_b2, h->geo.d_intr_sums, s);   // :120-127
  BBA_CUDA(h, cudaMemcpyAsync(h->geo.h_intr_sums, h->geo.d_intr_sums, sizeof(double) * bba::kIntrinsicsSums, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));   // :136

  if (opt_depth) {
    // the reference keeps A and b1 in fp32 buffers and solves in fp64 (:130-171)
    double A[15], b1[5], x1[5];
    for (int i = 0; i < 15; ++i) A[i] = static_cast<double>(static_cast<float>(h->geo.h_intr_sums[i]));
    for (int i = 0; i < 5; ++i) b1[i] = static_cast<double>(static_cast<float>(h->geo.h_intr_sums[15 + i]));
    constexpr float kAPriorWeight = 10;   // :153-155
    A[14] = static_cast<double>(static_cast<float>(A[14]) + kAPriorWeight * kAPriorWeight);
    b1[4] = static_cast<double>(static_cast<float>(b1[4]) + kAPriorWeight * kAPriorWeight * h->depth_a);
    bba::SolveLDLT<5>(A, b1, x1);
    float x1f[5];
    for (int i = 0; i < 5; ++i) x1f[i] = static_cast<float>(x1[i]);
    const bba::CameraParams& c = eq.cam;   // :183-194
    const float new_fx = 1.0f / (c.fx_inv - x1f[0]);
    const float new_fy = 1.0f / (c.fy_inv - x1f[1]);
    const float new_cx = -(new_fx * (c.cx_inv - x1f[2])) + 0.5f;
    const float new_cy = -(new_fy * (c.cy_inv - x1f[3])) + 0.5f;
    for (int i = 0; i < 5; ++i) h->geo.h_intr_x1[i] = x1f[i];
    BBA_CUDA(h, cudaMemcpyAsync(d_x1, h->geo.h_intr_x1, sizeof(float) * 5, cudaMemcpyHostToDevice, s));   // :196
    BBA_LAUNCH(h, h->launches, LaunchIntrinsicsCellUpdate, P, cell_obs, cell_B, cell_D, d_x1, h->d_cfactor, s);   // :205-212
    BBA_CUDA(h, cudaStreamSynchronize(s));   // h_intr_x1 is reused by the next call
    h->depth_K[0] = new_fx; h->depth_K[1] = new_fy; h->depth_K[2] = new_cx; h->depth_K[3] = new_cy;
    h->depth_a -= x1f[4];
  }
  if (opt_color) {   // :256-280
    double H[10], b[4], x[4];
    for (int i = 0; i < 10; ++i) H[i] = static_cast<double>(static_cast<float>(h->geo.h_intr_sums[20 + i]));
    for (int i = 0; i < 4; ++i) b[i] = static_cast<double>(static_cast<float>(h->geo.h_intr_sums[30 + i]));
    bba::SolveLDLT<4>(H, b, x);
    for (int i = 0; i < 4; ++i) h->color_K[i] -= static_cast<float>(x[i]);
  }
  return Publish(h, s, opt_depth);   // cameras, a and (depth) the cfactor together
}

// ---- in-loop surfel lifecycle ---------------------------------------------------------------------------------------------
// direct_ba.h:220-226
int GetMinObservationCount(bba_handle h) {
  const size_t K = h->keyframes.size();
  return (K < 10) ? ((K < 5) ? h->cfg.min_observation_count_while_bootstrapping_1 : h->cfg.min_observation_count_while_bootstrapping_2)
                  : h->cfg.min_observation_count;
}

uint32_t SurfelCapacity(bba_handle h) {
  return std::min<uint32_t>(h->cfg.max_surfel_count, SurfelPitch(h));
}

// Copies the device counter d_count to the host through life.h_count (the caller reserves it before its launches) and waits.
bba_status ReadCount(bba_handle h, const unsigned int* d_count, cudaStream_t s, uint32_t* count) {
  BBA_CUDA(h, cudaMemcpyAsync(h->life.h_count, d_count, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  *count = *h->life.h_count;
  return BBA_OK;
}

// size of life.d_scan_sums: the surfel creation scans the pixels, the compaction the surfels
size_t ScanSumsAlloc(bba_handle h) {
  return bba::ScanScratchWords(std::max(static_cast<uint32_t>(h->cfg.depth_width) * h->cfg.depth_height, SurfelCapacity(h)));
}

bba_status MakeLifecycleArgs(bba_handle h, int k, bba::LifecycleArgs* a, cudaStream_t s) {
  const uint32_t cells = static_cast<uint32_t>(h->cf_w) * h->cf_h;
  const uint32_t pixels = static_cast<uint32_t>(h->cfg.depth_width) * h->cfg.depth_height;
  auto& l = h->life;
  BBA_CUDA(h, l.d_sup.Reserve(3 * static_cast<size_t>(cells)));
  BBA_CUDA(h, l.d_cell_bits.Reserve(cells));
  BBA_CUDA(h, l.d_flags.Reserve(pixels));
  BBA_CUDA(h, l.d_scan_out.Reserve(pixels));
  BBA_CUDA(h, l.d_scan_sums.Reserve(bba::ScanScratchWords(pixels), ScanSumsAlloc(h)));
  BBA_CUDA(h, l.d_covis.Reserve(h->cfg.max_keyframes));
  BBA_CUDA(h, l.h_covis.Reserve(h->cfg.max_keyframes));
  BBA_CUDA(h, l.d_deleted_count.Reserve(1));
  BBA_CUDA(h, l.h_count.Reserve(1));
  const Keyframe& kf = h->keyframes[k];
  SetSurfelFields(h, a);
  bba::ToMatrix3x4(bba::Inverse(kf.pose), a->T);
  bba::ToMatrix3x4(kf.pose, a->G);
  a->depth = kf.depth;
  a->normals = kf.normals;
  a->radius = kf.radius;
  a->depth_pitch = static_cast<uint32_t>(kf.depth_pitch);
  a->normals_pitch = static_cast<uint32_t>(kf.normals_pitch);
  a->radius_pitch = static_cast<uint32_t>(kf.radius_pitch);
  a->tex = kf.tex;
  a->rgba = kf.rgba;
  a->rgba_pitch = static_cast<uint32_t>(kf.rgba_pitch);
  a->sup = h->life.d_sup;
  a->cell_bits = h->life.d_cell_bits;
  a->cells = cells;
  a->flags = h->life.d_flags;
  a->covis = h->life.d_covis;
  a->covis_count = 0;
  a->min_observation_count = GetMinObservationCount(h);
  const float c = static_cast<float>(h->cfg.sparse_surfel_cell_size);
  a->cell_merge_dist_squared = c * c * h->cfg.surfel_merge_dist_factor * h->cfg.surfel_merge_dist_factor;   // kernel_supporting_surfels.cc:76-78
  a->counter = h->life.d_deleted_count;
  (void)s;
  return BBA_OK;
}

// DirectBA::CreateSurfelsForKeyframe (direct_ba.cc:340-405)
bba_status CreateSurfelsForKeyframe(bba_handle h, int k, bool filter, cudaStream_t s, uint32_t* new_count) {
  *new_count = 0;
  const Keyframe& kf = h->keyframes[k];
  if (!kf.radius || !kf.rgba) return Fail(h, BBA_ERR_STATE, "surfel creation needs the keyframe's radius and colour buffers");
  BBA_TRACE("create: enter");
  h->xchg.replicated_pass_pending = true;
  if (bba_status st = WaitStaging(h)) return st;
  bba::LifecycleArgs a;
  if (bba_status st = MakeLifecycleArgs(h, k, &a, s)) return st;
  BBA_TRACE("create: args made");
  if (filter) {   // covis_T_frame for every co-visible keyframe (direct_ba.cc:365-370)
    int cnt = 0;
    for (int c : kf.covis) {
      const Keyframe& other = h->keyframes[c];
      bba::CovisEntry& e = h->life.h_covis[cnt++];
      bba::ToMatrix3x4(bba::Compose(bba::Inverse(other.pose), kf.pose), e.R);
      e.depth = other.depth;
      e.normals = other.normals;
      e.depth_pitch = static_cast<uint32_t>(other.depth_pitch);
      e.normals_pitch = static_cast<uint32_t>(other.normals_pitch);
      e.pad[0] = e.pad[1] = 0;
    }
    a.covis_count = cnt;
    if (cnt) BBA_CUDA(h, cudaMemcpyAsync(h->life.d_covis, h->life.h_covis, sizeof(bba::CovisEntry) * cnt, cudaMemcpyHostToDevice, s));
  }
  BBA_TRACE("create: covis uploaded");
  const uint32_t pixels = static_cast<uint32_t>(h->cfg.depth_width) * h->cfg.depth_height;
  BBA_LAUNCH(h, h->launches, LaunchSupportSurfels, a, h->sm_count, s);   // DetermineSupportingSurfelsCUDA: is the cell supported at all
  BBA_LAUNCH(h, h->launches, LaunchSeedNewSurfels, a, filter, s);
  BBA_LAUNCH(h, h->launches, LaunchExclusiveScan, h->life.d_flags, pixels, h->life.d_scan_out, h->life.d_scan_sums, s);
  uint32_t created = 0;
  if (bba_status st = ReadCount(h, h->life.d_scan_sums + bba::ScanTotalIndex(pixels), s, &created)) return st;   // kernel_create_surfels.cu:466-474
  h->staging.pending = false;
  BBA_TRACE("create: counted");
  if (created == 0) return BBA_OK;
  if (h->surfels_size + static_cast<uint64_t>(created) > SurfelCapacity(h)) {
    // the reference logs "Maximum surfel count exceeded" and creates nothing (kernel_create_surfels.cc:163-166)
    SetError(h, "maximum surfel count exceeded: no surfels created for this keyframe");
    return BBA_OK;
  }
  BBA_LAUNCH(h, h->launches, LaunchCreateSurfels, a, h->life.d_scan_out, s);
  BBA_TRACE("create: appended");
  h->surfels_size += created;
  *new_count = created;
  return MarkStaging(h, s);
}

// DetermineSupportingSurfelsAndMergeSurfelsCUDA (kernel_supporting_surfels.cc:40-118); deleted surfels are only marked
bba_status MergeSurfelsForKeyframe(bba_handle h, int k, cudaStream_t s, uint32_t* deleted) {
  *deleted = 0;
  if (h->surfels_size == 0) return BBA_OK;
  h->xchg.replicated_pass_pending = true;
  bba::LifecycleArgs a;
  if (bba_status st = MakeLifecycleArgs(h, k, &a, s)) return st;
  BBA_CUDA(h, cudaMemsetAsync(h->life.d_deleted_count, 0, sizeof(unsigned int), s));
  BBA_LAUNCH(h, h->launches, LaunchMergeSurfels, a, h->sm_count, s);
  return ReadCount(h, h->life.d_deleted_count, s, deleted);   // kernel_supporting_surfels.cc:93-96
}

bba_status CompactSurfels(bba_handle h, uint32_t free_count, bool with_active, cudaStream_t s) {
  const uint32_t N = h->surfels_size;
  if (free_count == 0 || N == 0) return BBA_OK;
  h->xchg.replicated_pass_pending = true;
  BBA_CUDA(h, h->life.d_scan_sums.Reserve(bba::ScanScratchWords(N), ScanSumsAlloc(h)));
  BBA_LAUNCH(h, h->launches, LaunchCompactSurfels, h->surfels, SurfelPitch(h), N, free_count, h->life.d_scan_sums,
             with_active ? h->active : nullptr, s);
  h->surfels_size = N - free_count;
  return BBA_OK;
}

// DirectBA::PerformBASchemeEndTasks (direct_ba.cc:566-653) without the final merge (do_surfel_updates is not supported yet):
// DeleteSurfelsAndUpdateRadiiCUDA over every keyframe, then CompactSurfelsCUDA.  Replicated on every rank of a multi-GPU
// job (once per BA call, deterministic, identical inputs -> identical surfel buffers without an exchange).
bba_status PerformEndTasks(bba_handle h, cudaStream_t s, uint32_t* deleted_out, bool do_surfel_updates = false) {
  if (deleted_out) *deleted_out = 0;
  const int K = static_cast<int>(h->keyframes.size());
  const uint32_t N = h->surfels_size;
  if (N == 0) return BBA_OK;   // kernel_delete_surfels.cc:52-54
  h->xchg.replicated_pass_pending = true;
  BBA_CUDA(h, h->life.d_kf_radius.Reserve(h->cfg.max_keyframes));
  BBA_CUDA(h, h->life.h_kf_radius.Reserve(h->cfg.max_keyframes));
  BBA_CUDA(h, h->life.d_deleted_count.Reserve(1));
  BBA_CUDA(h, h->life.h_count.Reserve(1));
  BBA_TRACE("end tasks");
  // merge similar surfels using all keyframes which were active in this BA iteration block (direct_ba.cc:577-601)
  uint32_t merged = 0;
  if (do_surfel_updates) {
    for (int k = 0; k < K; ++k) {
      if (h->keyframes[k].last_active_in_ba_iteration != h->ba_iteration_count) continue;
      uint32_t d = 0;
      if (bba_status st = MergeSurfelsForKeyframe(h, k, s, &d)) return st;
      merged += d;
    }
  }
  if (bba_status st = UploadKeyframes(h, s)) return st;   // (waits for the previous use of the staging buffers)
  for (int k = 0; k < K; ++k) {
    if (!h->keyframes[k].radius) return Fail(h, BBA_ERR_STATE, "end tasks need the keyframes' radius buffers");
    h->life.h_kf_radius[k].ptr = h->keyframes[k].radius;
    h->life.h_kf_radius[k].pitch = static_cast<uint32_t>(h->keyframes[k].radius_pitch);
    h->life.h_kf_radius[k].pad = 0;
  }
  if (K) BBA_CUDA(h, cudaMemcpyAsync(h->life.d_kf_radius, h->life.h_kf_radius, sizeof(bba::KfRadius) * K, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemsetAsync(h->life.d_deleted_count, 0, sizeof(unsigned int), s));
  if (bba_status st = ReserveTileEpochs(h)) return st;
  bba::SurfelStatsArgs a;
  SetSurfelFields(h, &a);
  a.kfs = h->d_kfs;
  a.radius = h->life.d_kf_radius;
  a.kf_count = K;
  a.min_observation_count = GetMinObservationCount(h);
  a.queue = h->geo.d_queue;
  a.tile_epoch = h->geo.d_tile_epoch;
  a.tile_shift = 8;
  a.deleted_count = h->life.d_deleted_count;
  // Multi-GPU: every rank evaluates the surfels of its granule shard (the launch is as expensive as a geometry pass over every
  // keyframe); the two result rows reach the other replicas through peer stores or one all-gather, the deleted counts through a
  // sum all-reduce (which is also the barrier behind the peer stores).  The compaction then runs replicated on identical replicas.
  const int world = h->cfg.world_size, rank = h->cfg.rank;
  a.shard_rank = static_cast<uint32_t>(rank);
  a.shard_world = static_cast<uint32_t>(world);
  ShardSurfels(N, rank, world, &a.local_count, nullptr);
  a.peers = KernelPeers(h);
  if (world > 1) {
    if (bba_status st = CheckCollective(h)) return st;
    if (bba_status st = PeerFence(h, s)) return st;   // (e.g. the merges above rewrote whole replicas)
  }
  if (K > 0) BBA_LAUNCH(h, h->launches, LaunchObservationStats, a, h->sm_count, s);
  // (with no keyframe at all the reference still runs MarkDeletedSurfels on zero counts; not reachable through this API,
  // a BA call without keyframes has nothing to optimise)
  if (world > 1 && !PeerStores(h) && K > 0) {
    if (bba_status st = ExchangeShards(h, bba::ShardRows{{bba::kRowX, bba::kRowRadiusSq}, 2, 0}, nullptr, s)) return st;
  }
  uint32_t deleted_total = 0;
  if (bba_status st = ReadCount(h, h->life.d_deleted_count, s, &deleted_total)) return st;   // kernel_delete_surfels.cc:93-96
  if (world > 1) {
    if (bba_status st = SumOverRanks(h, deleted_total, s, &deleted_total)) return st;
    h->xchg.replicated_pass_pending = true;   // the compaction below rewrites every replica as a whole
  }
  h->staging.pending = false;
  BBA_TRACE("stats done");
  const uint32_t deleted = deleted_total + merged;
  if (deleted_out) *deleted_out = deleted;
  // kernel_compact_surfels.cu:167-169; direct_ba.cc:618: no active flags
  return CompactSurfels(h, deleted, /*with_active=*/false, s);
}

// Merges the new surfels of `keyframes` into the map and compacts it (direct_ba_alternating.cc:489-541, direct_ba_pcg.cc:644-690,
// 775-815); *merged: the number of surfels the merges deleted.
bba_status MergeAndCompact(bba_handle h, const std::vector<int>& keyframes, cudaStream_t s, uint32_t* merged) {
  *merged = 0;
  for (int k : keyframes) {
    uint32_t d = 0;
    if (bba_status st = MergeSurfelsForKeyframe(h, k, s, &d)) return st;
    *merged += d;
  }
  return CompactSurfels(h, *merged, /*with_active=*/true, s);
}

// Start of a BA call (direct_ba_alternating.cc:313-319, direct_ba_pcg.cc:157-161): the end tasks that the previous call left
// for this one when it did not advance the BA iteration count.
bba_status BeginBundleAdjust(bba_handle h, const bba_ba_options* o, bba_ba_result* res, cudaStream_t s) {
  if (!o->increase_ba_iteration_count && h->ba_iteration_count != h->last_ba_iteration_count) {
    h->last_ba_iteration_count = h->ba_iteration_count;
    uint32_t deleted = 0;
    if (bba_status st = PerformEndTasks(h, s, &deleted, o->do_surfel_updates != 0)) return st;
    res->surfels_deleted += deleted;
  }
  return BBA_OK;
}

// End of a BA call (direct_ba_alternating.cc:725-735, direct_ba_pcg.cc:771-776): the end tasks when the call advances the BA
// iteration count, then the map size and the launches of the call in the result.
bba_status EndBundleAdjust(bba_handle h, const bba_ba_options* o, uint64_t launches_before, bba_ba_result* res, cudaStream_t s) {
  if (o->increase_ba_iteration_count) {
    uint32_t deleted = 0;
    if (bba_status st = PerformEndTasks(h, s, &deleted, o->do_surfel_updates != 0)) return st;
    res->surfels_deleted += deleted;
    ++h->ba_iteration_count;
  }
  res->surfels_size = h->surfels_size;
  res->kernel_launches = h->launches - launches_before;
  return BBA_OK;
}

// The in-loop surfel creation of either scheme (direct_ba_alternating.cc:399-430, direct_ba_pcg.cc:183-206) when the call
// optimises the geometry with surfel updates: the keyframes that became active for the first time within BA iteration block
// `ba_iteration` get their surfels in ascending id order and make up *keyframes; the co-visible ones are marked as seen in it.
bba_status CreateInLoopSurfels(bba_handle h, const bba_ba_options* o, int ba_iteration, cudaStream_t s, bba_ba_result* res,
                               std::vector<int>* keyframes) {
  keyframes->clear();
  if (!o->optimize_geometry || !o->do_surfel_updates) return BBA_OK;
  for (int k = 0; k < static_cast<int>(h->keyframes.size()); ++k) {
    Keyframe& kf = h->keyframes[k];
    if (kf.activation == BBA_KF_ACTIVE && kf.last_active_in_ba_iteration != ba_iteration) {
      kf.last_active_in_ba_iteration = ba_iteration;
      keyframes->push_back(k);
    } else if (kf.activation == BBA_KF_COVISIBLE_ACTIVE && kf.last_covis_in_ba_iteration != ba_iteration) {
      kf.last_covis_in_ba_iteration = ba_iteration;
    }
  }
  for (int k : *keyframes) {
    uint32_t created = 0;
    if (bba_status st = CreateSurfelsForKeyframe(h, k, /*filter_new_surfels=*/true, s, &created)) return st;
    res->surfels_created += created;
  }
  return BBA_OK;
}

// The stop test at the end of an outer iteration of either scheme (direct_ba_alternating.cc:693-709, direct_ba_pcg.cc:757-766):
// converged (res->converged) or past the time limit.
bool StopIterating(const bba_ba_options* o, int iteration, int num_converged, int K,
                   std::chrono::steady_clock::time_point t_start, bba_ba_result* res) {
  if (iteration >= o->min_iterations - 1 && (num_converged == K || !o->optimize_poses)) {
    res->converged = 1;
    return true;
  }
  return o->time_limit_seconds > 0 &&
         std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count() > o->time_limit_seconds;
}

// Unknown layout of the PCG solver (direct_ba_pcg.cc:273-309) + the vectors sized for it.
struct PcgLayout {
  bool opt_poses, opt_geometry, opt_depth_intr, opt_color_intr, use_desc;
  uint32_t surfel_start, stride, depth_start, a_index, color_start, unknown_count;
};

bba_status MakePcgLayout(bba_handle h, const bba_ba_options* o, PcgLayout* L) {
  constexpr uint32_t kInvalid = 0xffffffffu;
  const int K = static_cast<int>(h->keyframes.size());
  const uint32_t N = h->surfels_size, P = static_cast<uint32_t>(h->cf_w) * h->cf_h;
  L->opt_depth_intr = o->optimize_depth_intrinsics && h->cfg.use_depth_residuals;   // direct_ba.cc:427-434
  L->opt_color_intr = o->optimize_color_intrinsics && h->cfg.use_descriptor_residuals;
  L->opt_poses = o->optimize_poses != 0;
  L->opt_geometry = o->optimize_geometry != 0;
  L->use_desc = h->cfg.use_descriptor_residuals != 0;
  L->stride = L->use_desc ? 3u : 1u;
  uint32_t cur = 0;
  if (L->opt_poses) cur += 6u * static_cast<uint32_t>(K - 1);
  L->surfel_start = L->depth_start = L->a_index = L->color_start = kInvalid;
  if (L->opt_geometry) { L->surfel_start = cur; cur += L->stride * N; }
  if (L->opt_depth_intr) { L->depth_start = cur; cur += 5u + P; L->a_index = L->depth_start + 4u; }
  if (L->opt_color_intr) { L->color_start = cur; cur += 4u; }
  L->unknown_count = cur;
  if (!h->pcg.d_scalars) {   // scalars + the ordered-sum workspace, zeroed once (set only once it is zeroed)
    DeviceBuffer<double> scalars;
    BBA_CUDA(h, scalars.Reserve(bba::kPcgScalarDoubles));
    BBA_CUDA(h, cudaMemset(scalars, 0, sizeof(double) * bba::kPcgScalarDoubles));
    h->pcg.d_scalars = std::move(scalars);
  }
  BBA_CUDA(h, h->pcg.h_scalars.Reserve(4));
  BBA_CUDA(h, h->pcg.h_delta.Reserve(6 * static_cast<size_t>(h->cfg.max_keyframes) + 16));
  const size_t cap = std::max<size_t>(L->unknown_count, 6 * static_cast<size_t>(h->cfg.max_keyframes) +
                                                            3 * static_cast<size_t>(std::max(h->cfg.max_surfel_count, N)) + 9 + P);
  for (auto& v : h->pcg.d_vec)   // (+ 8: the alpha_d pair that travels with g, multi-GPU)
    BBA_CUDA(h, v.Reserve(static_cast<size_t>(L->unknown_count) + 8, cap + 8));
  return BBA_OK;
}

bba::PcgArgs MakePcgArgs(bba_handle h, const PcgLayout& L, int gauge) {
  bba::PcgArgs a;
  SetSurfelFields(h, &a);
  SetShardFields(h, &a);   // this rank's surfels (all of them on one GPU)
  a.alpha_d_slot = h->cfg.world_size > 1 ? 3 : 1;
  a.kfs = h->d_kfs;
  a.kf_count = static_cast<int>(h->keyframes.size());
  a.gauge_kf = gauge;
  a.opt_poses = L.opt_poses;
  a.opt_geometry = L.opt_geometry;
  a.opt_depth_intr = L.opt_depth_intr;
  a.opt_color_intr = L.opt_color_intr;
  a.surfel_start = L.surfel_start;
  a.surfel_stride = L.stride;
  a.depth_intr_start = L.depth_start;
  a.color_intr_start = L.color_start;
  a.r = h->pcg.d_vec[0];
  a.M = h->pcg.d_vec[1];
  a.p = h->pcg.d_vec[4];
  a.g = h->pcg.d_vec[3];
  a.scalars = h->pcg.d_scalars;
  a.queue = h->geo.d_queue;
  return a;
}

// The pose-block terms of the products at the poses the init pass sees, staged for LaunchPcgPoseTerms: a keyframe's prior and,
// per constraint, H_aa / H_bb, H_ab and b_a / b_b of PoseConstraintTerms, gathered per pose block (every keyframe but the
// gauge) in the order prior, then constraints by id.  An edge to the gauge keeps only its other end's diagonal terms (p_gauge = 0).
// fp64, rounded to fp32.  Only rank 0 adds them: the sum all-reduce of r / M / g then counts each once.
bba_status StagePcgPoseTerms(bba_handle h, const PcgLayout& L, int gauge, cudaStream_t s) {
  auto& pc = h->pcg;
  pc.pose_blocks = 0;
  if (!L.opt_poses || (h->pose_prior_count == 0 && h->pose_constraints.empty()) || h->cfg.rank != 0) return BBA_OK;
  const int K = static_cast<int>(h->keyframes.size());
  const size_t C = h->pose_constraints.size();
  if (bba_status st = ReservePoseTerms(h, C)) return st;
  auto unknown = [&](int k) { return k == gauge ? -1 : 6 * (k < gauge ? k : k - 1); };
  std::vector<float> poses(7 * static_cast<size_t>(K));
  for (int k = 0; k < K; ++k) PoseToArray(h->keyframes[k].pose, poses.data() + 7 * k);
  // every constraint's terms at the current poses: [a's term, b's term]
  std::vector<bba::PcgPoseTerm> edge(2 * C);
  for (size_t i = 0; i < C; ++i) {
    const bba_pose_constraint& c = h->pose_constraints[i].c;
    double r[6], H[78], b[12], cost;
    PoseConstraintTerms(c.a_T_b, poses.data() + 7 * c.keyframe_a, poses.data() + 7 * c.keyframe_b, c.information, r, H, b, &cost);
    auto upper = [&](int row, int col) { return H[row * 12 - row * (row - 1) / 2 + (col - row)]; };
    bba::PcgPoseTerm& ta = edge[2 * i];
    bba::PcgPoseTerm& tb = edge[2 * i + 1];
    ta.other = unknown(c.keyframe_b);
    tb.other = unknown(c.keyframe_a);
    int idx = 0;
    for (int row = 0; row < 6; ++row) {
      ta.b[row] = static_cast<float>(b[row]);
      tb.b[row] = static_cast<float>(b[6 + row]);
      for (int col = row; col < 6; ++col, ++idx) {
        ta.H[idx] = static_cast<float>(upper(row, col));
        tb.H[idx] = static_cast<float>(upper(6 + row, 6 + col));
      }
      for (int col = 0; col < 6; ++col) {
        const float x = static_cast<float>(upper(row, 6 + col));   // H_ab[row][col]
        ta.X[row * 6 + col] = x;
        tb.X[col * 6 + row] = x;                                  // H_ba = H_ab^T
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
      bba::PcgPoseTerm& t = pc.h_pose_terms[nt++];
      t.other = -1;
      double H[21], b[6], cost;
      bba::PosePriorTerms(prior.pose, poses.data() + 7 * k, prior.info, H, b, &cost);
      for (int j = 0; j < 21; ++j) t.H[j] = static_cast<float>(H[j]);
      for (int j = 0; j < 6; ++j) t.b[j] = static_cast<float>(b[j]);
    }
    for (int e = off[k]; e < off[k + 1]; ++e) {
      const int i = adj[e];
      pc.h_pose_terms[nt++] = edge[2 * i + (h->pose_constraints[i].c.keyframe_a == k ? 0 : 1)];
    }
    if (nt > begin) pc.h_pose_blocks[nb++] = bba::PcgPoseBlock{static_cast<uint32_t>(unknown(k)), begin, nt};
  }
  if (nb) {
    BBA_CUDA(h, cudaMemcpyAsync(pc.d_pose_blocks, pc.h_pose_blocks, sizeof(bba::PcgPoseBlock) * nb, cudaMemcpyHostToDevice, s));
    BBA_CUDA(h, cudaMemcpyAsync(pc.d_pose_terms, pc.h_pose_terms, sizeof(bba::PcgPoseTerm) * nt, cudaMemcpyHostToDevice, s));
  }
  pc.pose_blocks = nb;
  return BBA_OK;
}

// The PCG solver's phases, shared by BundleAdjustPCG and the parity hook bba_pcg_debug.  Vectors: d_pcg = {r, M, delta, g, p};
// scalars = {alpha_n or beta_n (slot an), alpha_d (1), beta_n or alpha_n (slot bn), this rank's alpha_d (3, multi-GPU)}.
// Init: r = -J^T W F and M = diag(J^T W J) over every keyframe (:312-361), then PCGInit2 (:363-373) into slot `an`.
bba_status PcgInit(bba_handle h, const PcgLayout& L, const bba::PcgArgs& a, int an, cudaStream_t s) {
  const uint32_t U = L.unknown_count;
  BBA_CUDA(h, cudaMemsetAsync(h->pcg.d_vec[0], 0, sizeof(float) * U, s));
  BBA_CUDA(h, cudaMemsetAsync(h->pcg.d_vec[1], 0, sizeof(float) * U, s));
  BBA_CUDA(h, cudaMemsetAsync(h->pcg.d_scalars, 0, sizeof(double) * 4, s));
  BBA_LAUNCH(h, h->launches, LaunchPcgAccumulate, a, h->sm_count, true, s);   // PCGInitCUDA for every keyframe
  if (bba_status st = StagePcgPoseTerms(h, L, a.gauge_kf, s)) return st;
  BBA_LAUNCH(h, h->launches, LaunchPcgPoseTerms, h->pcg.d_pose_blocks, h->pcg.pose_blocks, h->pcg.d_pose_terms, true, a.r, a.M, nullptr,
             nullptr, nullptr, s);
  if (h->cfg.world_size > 1) {
    if (bba_status st = Collective(h, BBA_COLLECTIVE_ALLREDUCE_SUM, h->pcg.d_vec[0], U, s)) return st;
    if (bba_status st = Collective(h, BBA_COLLECTIVE_ALLREDUCE_SUM, h->pcg.d_vec[1], U, s)) return st;
    h->xchg.replicated_pass_pending = false;
  }
  BBA_LAUNCH(h, h->launches, LaunchPcgInit2, U, L.a_index, h->depth_a, a.kf_count, h->pcg.d_vec[0], h->pcg.d_vec[1], h->pcg.d_vec[2],
             h->pcg.d_vec[3], h->pcg.d_vec[4], h->pcg.d_scalars, an, h->sm_count, s);
  return BBA_OK;
}

// Inner step, first half: g += J^T W J p and alpha_d += p^T J^T W J p over every keyframe (PCGStep1CUDA, :392-419).
bba_status PcgStep1(bba_handle h, const PcgLayout& L, const bba::PcgArgs& a, cudaStream_t s) {
  BBA_LAUNCH(h, h->launches, LaunchPcgAccumulate, a, h->sm_count, false, s);
  BBA_LAUNCH(h, h->launches, LaunchPcgPoseTerms, h->pcg.d_pose_blocks, h->pcg.pose_blocks, h->pcg.d_pose_terms, false, nullptr, nullptr,
             a.p, a.g, a.scalars + a.alpha_d_slot, s);
  if (h->cfg.world_size > 1) {   // g and this rank's part of alpha_d: one all-reduce
    float* g = h->pcg.d_vec[3];
    BBA_LAUNCH(h, h->launches, LaunchPcgPackAlphaD, h->pcg.d_scalars, g + L.unknown_count, s);
    if (bba_status st = Collective(h, BBA_COLLECTIVE_ALLREDUCE_SUM, g, static_cast<size_t>(L.unknown_count) + 2, s)) return st;
    BBA_LAUNCH(h, h->launches, LaunchPcgUnpackAlphaD, h->pcg.d_scalars, g + L.unknown_count, s);
  }
  return BBA_OK;
}

// Inner step, second half: delta += alpha p, r -= alpha A p, z = M^-1 r (into g), beta_n = z^T r into slot `bn` (:421-437).
bba_status PcgStep2(bba_handle h, const PcgLayout& L, int an, int bn, cudaStream_t s) {
  BBA_CUDA(h, cudaMemsetAsync(h->pcg.d_scalars + bn, 0, sizeof(double), s));
  BBA_LAUNCH(h, h->launches, LaunchPcgStep2, L.unknown_count, L.a_index, h->pcg.d_vec[0], h->pcg.d_vec[1], h->pcg.d_vec[2], h->pcg.d_vec[3],
             h->pcg.d_vec[4], h->pcg.d_scalars, an, bn, h->sm_count, s);
  return BBA_OK;
}

// Before the next inner step: p = z + beta p, g = 0, alpha_d re-armed with its lambda / prior term (:456-464).
bba_status PcgStep3(bba_handle h, const PcgLayout& L, int an, int bn, cudaStream_t s) {
  BBA_CUDA(h, cudaMemsetAsync(h->pcg.d_scalars + 1, 0, sizeof(double), s));
  BBA_LAUNCH(h, h->launches, LaunchPcgStep3, L.unknown_count, L.a_index, static_cast<int>(h->keyframes.size()), h->pcg.d_vec[3],
             h->pcg.d_vec[4], h->pcg.d_scalars, an, bn, h->sm_count, s);
  return BBA_OK;
}

// Applies pcg_delta (:552-638): surfels, cfactors, poses (all but the gauge keyframe), intrinsics.  *num_converged counts the
// keyframes whose pose update is below the convergence threshold (the gauge keyframe included).
bba_status PcgApplyDelta(bba_handle h, const PcgLayout& L, int gauge, cudaStream_t s, int* num_converged) {
  const int K = static_cast<int>(h->keyframes.size());
  const uint32_t N = h->surfels_size, P = static_cast<uint32_t>(h->cf_w) * h->cf_h;
  const float* pcg_delta = h->pcg.d_vec[2];
  size_t n_host = 0;
  const size_t pose_floats = L.opt_poses ? 6 * static_cast<size_t>(K - 1) : 0;
  if (pose_floats) BBA_CUDA(h, cudaMemcpyAsync(h->pcg.h_delta, pcg_delta, sizeof(float) * pose_floats, cudaMemcpyDeviceToHost, s));
  n_host = pose_floats;
  float* h_di = h->pcg.h_delta + n_host;
  if (L.opt_depth_intr) {
    BBA_CUDA(h, cudaMemcpyAsync(h_di, pcg_delta + L.depth_start, sizeof(float) * 5, cudaMemcpyDeviceToHost, s));
    n_host += 5;
  }
  float* h_ci = h->pcg.h_delta + n_host;
  if (L.opt_color_intr) BBA_CUDA(h, cudaMemcpyAsync(h_ci, pcg_delta + L.color_start, sizeof(float) * 4, cudaMemcpyDeviceToHost, s));
  if (L.opt_geometry && N > 0) {
    BBA_LAUNCH(h, h->launches, LaunchPcgUpdateSurfels, h->surfels, SurfelPitch(h), N, L.use_desc, L.surfel_start, pcg_delta, s);
    h->xchg.replicated_pass_pending = true;   // every rank rewrites its whole replica (PeerFence)
  }
  if (L.opt_depth_intr) BBA_LAUNCH(h, h->launches, LaunchPcgUpdateCfactor, h->d_cfactor, P, pcg_delta + L.depth_start + 5, s);
  BBA_CUDA(h, cudaStreamSynchronize(s));
  if (L.opt_poses) {
    for (int k = 0; k < K; ++k) {
      if (k == gauge) {
        ++*num_converged;
        continue;
      }
      const float* d6 = h->pcg.h_delta + 6 * static_cast<size_t>(k < gauge ? k : k - 1);
      const Pose delta = bba::Exp(d6);
      h->keyframes[k].pose = bba::Compose(h->keyframes[k].pose, delta);   // :569-570
      float lg[6];
      bba::Log(delta, lg);
      if (bba::IsScale1PoseEstimationConverged(lg)) ++*num_converged;
    }
  }
  if (L.opt_depth_intr) {   // :590-612
    const double old_fx_inv = 1. / h->depth_K[0], old_fy_inv = 1. / h->depth_K[1];
    const double old_cx_inv = -(h->depth_K[2] - 0.5) * old_fx_inv, old_cy_inv = -(h->depth_K[3] - 0.5) * old_fy_inv;
    const double new_fx = 1. / (old_fx_inv + h_di[0]);
    const double new_fy = 1. / (old_fy_inv + h_di[1]);
    const double new_cx = -(new_fx * (old_cx_inv + h_di[2])) + 0.5;
    const double new_cy = -(new_fy * (old_cy_inv + h_di[3])) + 0.5;
    h->depth_K[0] = static_cast<float>(new_fx);
    h->depth_K[1] = static_cast<float>(new_fy);
    h->depth_K[2] = static_cast<float>(new_cx);
    h->depth_K[3] = static_cast<float>(new_cy);
    h->depth_a += h_di[4];
  }
  if (L.opt_color_intr)   // :623-638
    for (int c = 0; c < 4; ++c) h->color_K[c] = static_cast<float>(h->color_K[c] + h_ci[c]);
  return Publish(h, s, L.opt_depth_intr);   // poses, cameras, a and (depth) the cfactor together
}

// DirectBA::BundleAdjustmentPCG (direct_ba_pcg.cc:43-819) without the surfel lifecycle branches.
bba_status BundleAdjustPCG(bba_handle h, const bba_ba_options* o, bba_ba_result* res, cudaStream_t s) {
  const int K = static_cast<int>(h->keyframes.size());
  // Multi-GPU: the matrix-free products J^T W F / diag(J^T W J) / J^T W J p are summed over THIS rank's surfels (granule
  // sharding of the geometry step); one sum all-reduce of the vector per product makes every rank hold the full result (a
  // surfel's entries are non-zero on its owner only, pose / intrinsics entries are true sums), and the vector kernels, the
  // scalars and the updates then run replicated and bit-identically on every rank (fixed-order sums, pcg.cu GridOrderedAdd).
  const int world = h->cfg.world_size;
  if (bba_status st = CheckCollective(h)) return st;
  if (world > 1 && o->pcg_gauge_keyframe < 0)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "use_pcg with more than one rank needs pcg_gauge_keyframe >= 0 (the reference draws rand() % K)");
  if (K == 0) return Fail(h, BBA_ERR_STATE, "use_pcg: no keyframes");
  const int max_inner = o->pcg_max_inner_iterations > 0 ? o->pcg_max_inner_iterations : 30;
  const int max_keyframes = o->pcg_max_keyframes > 0 ? o->pcg_max_keyframes : 2500;
  if (K > max_keyframes) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "use_pcg: more keyframes than pcg_max_keyframes");   // :232
  if (o->pcg_gauge_keyframe >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "pcg_gauge_keyframe out of range");
  PcgLayout L;
  if (bba_status st = MakePcgLayout(h, o, &L)) return st;
  const bool opt_poses = L.opt_poses, opt_geometry = L.opt_geometry;
  const uint64_t launches_before = h->launches;
  const auto t_start = std::chrono::steady_clock::now();
  if (bba_status st = BeginBundleAdjust(h, o, res, s)) return st;
  std::vector<int> keyframes_with_new_surfels;

  for (int iteration = 0; iteration < o->max_iterations; ++iteration) {
    if (o->progress_function && !o->progress_function(o->progress_user, iteration)) break;
    ++res->iterations_done;
    // (pose.order_stale stays as it is: a new spatial order would change the last bits of later pose-kernel sums)
    if (bba_status st = CreateInLoopSurfels(h, o, h->ba_iteration_count, s, res, &keyframes_with_new_surfels)) return st;
    const uint32_t N = h->surfels_size;
    if (N > 0) BBA_CUDA(h, cudaMemsetAsync(h->active, bba::kSurfelActiveFlag, N, s));   // :209-212
    if (bba_status st = UploadKeyframes(h, s)) return st;
    BBA_CUDA(h, cudaEventRecord(h->ev[0], s));
    if (opt_geometry && N > 0) {   // UpdateSurfelNormalsCUDA, :215-227
      bba::GeometryArgs g;
      if (bba_status st = BuildGeometryArgs(h, &g, s, GeoOrder::kCaller)) return st;
      BBA_LAUNCH(h, h->launches, LaunchActivationAndNormals, g, h->sm_count, false, true, s);
      if (bba_status st = ExchangeGeometry(h, s)) return st;   // multi-GPU: every replica gets the other shards' normals
    }
    BBA_CUDA(h, cudaEventRecord(h->ev[1], s));

    if (bba_status st = MakePcgLayout(h, o, &L)) return st;   // unknown layout (:273-309)
    const uint32_t unknown_count = L.unknown_count;
    const int gauge = o->pcg_gauge_keyframe >= 0 ? o->pcg_gauge_keyframe : (rand() % K);   // :324

    int num_converged = 0;
    if (unknown_count > 0) {
      const bba::PcgArgs a = MakePcgArgs(h, L, gauge);
      int an = 0, bn = 2;
      if (bba_status st = PcgInit(h, L, a, an, s)) return st;
      float prev_r_norm = std::numeric_limits<float>::infinity();
      int without_improvement = 0;
      for (int step = 0; step < max_inner; ++step) {
        if (step > 0) std::swap(an, bn);   // alpha_n <- beta_n (:386); g was cleared and alpha_d re-armed by PcgStep3Kernel
        if (bba_status st = PcgStep1(h, L, a, s)) return st;
        if (bba_status st = PcgStep2(h, L, an, bn, s)) return st;
        BBA_CUDA(h, cudaMemcpyAsync(h->pcg.h_scalars, h->pcg.d_scalars, sizeof(double) * 4, cudaMemcpyDeviceToHost, s));
        BBA_CUDA(h, cudaStreamSynchronize(s));   // :436-437
        ++res->pcg_inner_iterations_total;
        const float r_norm = std::sqrt(static_cast<float>(h->pcg.h_scalars[bn]));
        res->pcg_last_r_norm = r_norm;
        if (static_cast<double>(r_norm) < static_cast<double>(prev_r_norm) - 1e-3) {   // :442-449
          without_improvement = 0;
        } else if (++without_improvement >= 3) {
          break;
        }
        prev_r_norm = r_norm;
        if (step < max_inner - 1) {   // :456-464
          if (bba_status st = PcgStep3(h, L, an, bn, s)) return st;
        }
      }
      BBA_CUDA(h, cudaEventRecord(h->ev[2], s));
      if (bba_status st = PcgApplyDelta(h, L, gauge, s, &num_converged)) return st;
      // surfel merge + compaction (:644-690) for the keyframes that received new surfels
      if (o->do_surfel_updates && !keyframes_with_new_surfels.empty()) {
        uint32_t merged = 0;
        if (bba_status st = MergeAndCompact(h, keyframes_with_new_surfels, s, &merged)) return st;
        res->surfels_merged += merged;
      }
    } else {
      BBA_CUDA(h, cudaEventRecord(h->ev[2], s));
      BBA_CUDA(h, cudaStreamSynchronize(s));
      num_converged = opt_poses ? 1 : 0;
    }
    cudaEventElapsedTime(&res->ms_geometry_optimization, h->ev[0], h->ev[1]);   // "BA normals update", :722-727
    cudaEventElapsedTime(&res->ms_pcg, h->ev[1], h->ev[2]);
    if (StopIterating(o, iteration, num_converged, K, t_start, res)) break;
  }
  if (!o->increase_ba_iteration_count && o->do_surfel_updates && !keyframes_with_new_surfels.empty()) {
    // :775-815: without the end tasks, the keyframes of the last iteration's creation step are merged (and the map compacted) once more
    uint32_t merged = 0;
    if (bba_status st = MergeAndCompact(h, keyframes_with_new_surfels, s, &merged)) return st;
    res->surfels_merged += merged;
  }
  return EndBundleAdjust(h, o, launches_before, res, s);
}

// The standalone geometry passes over every keyframe that is not inactive, in spatial order: the surfel activation
// (bba_update_surfel_activation), or the normals and then the positions and descriptors (bba_optimize_geometry_iteration).
bba_status GeometryPass(bba_handle h, bool activation, cudaStream_t s) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckSurfels(h)) return st;
  if (h->surfels_size == 0) return BBA_OK;
  if (bba_status st = UploadKeyframes(h, s)) return st;
  bba::GeometryArgs g;
  if (bba_status st = BuildGeometryArgs(h, &g, s, GeoOrder::kSpatial)) return st;
  if (bba_status st = CheckCollective(h)) return st;
  BBA_LAUNCH(h, h->launches, LaunchActivationAndNormals, g, h->sm_count, activation, !activation, s);
  if (!activation) BBA_LAUNCH(h, h->launches, LaunchPositionAndDescriptor, g, h->sm_count, s);
  if (bba_status st = ExchangeGeometry(h, s)) return st;
  return MarkStaging(h, s);
}

// Rotation matrix of a quaternion (x y z w), normalised in fp64.
void QuatToMatrix64(const float q[4], double R[9]) {
  const double n = std::sqrt(static_cast<double>(q[0]) * q[0] + static_cast<double>(q[1]) * q[1] + static_cast<double>(q[2]) * q[2] +
                             static_cast<double>(q[3]) * q[3]);
  const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w); R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w); R[7] = 2 * (y * z + x * w); R[8] = 1 - 2 * (x * x + y * y);
}

// Keyframe k's change for the surfel deformation (DESIGN §3.13): D = global_T_frame (now) * original frame_T_global and the
// original camera centre, in fp64 and rounded; a keyframe whose current pose inverts to the original bit for bit is unmoved.
KfChange KeyframeChange(const Pose& global_T_frame, const float original[7]) {
  KfChange c{};
  float inv[7];
  PoseToArray(Inverse(global_T_frame), inv);
  c.unmoved = std::memcmp(inv, original, sizeof(inv)) == 0;
  double Rc[9], Ro[9];
  QuatToMatrix64(global_T_frame.q, Rc);
  QuatToMatrix64(original, Ro);
  for (int r = 0; r < 3; ++r) {
    for (int col = 0; col < 3; ++col)
      c.D[4 * r + col] = static_cast<float>(Rc[3 * r] * Ro[col] + Rc[3 * r + 1] * Ro[3 + col] + Rc[3 * r + 2] * Ro[6 + col]);
    c.D[4 * r + 3] = static_cast<float>(Rc[3 * r] * original[4] + Rc[3 * r + 1] * original[5] + Rc[3 * r + 2] * original[6] +
                                        global_T_frame.t[r]);
    c.centre[r] = static_cast<float>(-(Ro[r] * original[4] + Ro[3 + r] * original[5] + Ro[6 + r] * original[6]));
  }
  if (c.unmoved)
    for (int i = 0; i < 12; ++i) c.D[i] = (i % 5 == 0) ? 1.f : 0.f;
  return c;
}

// bba_deform_surfels.  Every argument is checked before anything is enqueued.
bba_status DeformSurfels(bba_handle h, int count, const float* original, uint32_t* moved, uint32_t* unobserved, cudaStream_t s) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_deform_surfels: ";
  if (count < 0 || count > static_cast<int>(h->keyframes.size())) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad count");
  if (count > 0 && !original) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  for (int k = 0; k < count; ++k) {
    const float* p = original + 7 * static_cast<size_t>(k);
    for (int j = 0; j < 7; ++j)
      if (!std::isfinite(p[j])) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "non-finite pose");
    if (p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3] < 1e-12f) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "zero quaternion");
  }
  if (moved) *moved = 0;
  if (unobserved) *unobserved = 0;
  if (count == 0 || h->surfels_size == 0) return BBA_OK;
  if (bba_status st = CheckSurfels(h)) return st;
  if (bba_status st = CheckCollective(h)) return st;
  auto& d = h->deform;
  BBA_CUDA(h, d.h_kfs.Reserve(count, h->cfg.max_keyframes));
  BBA_CUDA(h, d.d_kfs.Reserve(count, h->cfg.max_keyframes));
  BBA_CUDA(h, d.h_changes.Reserve(count, h->cfg.max_keyframes));
  BBA_CUDA(h, d.d_changes.Reserve(count, h->cfg.max_keyframes));
  BBA_CUDA(h, d.d_counts.Reserve(2));
  BBA_CUDA(h, d.h_counts.Reserve(2));
  if (bba_status st = MakeAllKeyframeList(h)) return st;
  if (bba_status st = WaitStaging(h)) return st;
  for (int k = 0; k < count; ++k) {
    const Keyframe& kf = h->keyframes[k];
    const float* p = original + 7 * static_cast<size_t>(k);
    FillKfDevice(kf, kf.pose, d.h_kfs + k);
    ToMatrix3x4(PoseFromArray(p), d.h_kfs[k].T);   // the association runs at the original pose
    d.h_changes[k] = KeyframeChange(kf.pose, p);
  }
  BBA_CUDA(h, cudaMemcpyAsync(d.d_kfs, d.h_kfs, sizeof(KfDevice) * count, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemcpyAsync(d.d_changes, d.h_changes, sizeof(KfChange) * count, cudaMemcpyHostToDevice, s));
  if (bba_status st = MarkStaging(h, s)) return st;
  BBA_CUDA(h, cudaMemsetAsync(d.d_counts, 0, sizeof(unsigned int) * 2, s));
  bba::DeformArgs a;
  if (bba_status st = BuildGeometryArgs(h, &a.geo, s, GeoOrder::kSpatial)) return st;
  a.geo.kfs = d.d_kfs;
  a.geo.kf_list = h->geo.d_all_list;
  a.geo.kf_count = count;
  a.changes = d.d_changes;
  a.counts = d.d_counts;
  BBA_LAUNCH(h, h->launches, LaunchDeformSurfels, a, h->sm_count, s);
  if (bba_status st = ExchangeGeometry(h, s)) return st;
  h->pose.order_stale = true;   // the positions moved
  if (!moved && !unobserved) return BBA_OK;
  BBA_CUDA(h, cudaMemcpyAsync(d.h_counts, d.d_counts, sizeof(unsigned int) * 2, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  uint32_t counts[2] = {d.h_counts[0], d.h_counts[1]};
  if (h->cfg.world_size > 1)   // every rank counted its own shard
    for (uint32_t& c : counts)
      if (bba_status st = SumOverRanks(h, c, s, &c)) return st;
  if (moved) *moved = counts[0];
  if (unobserved) *unobserved = counts[1];
  return BBA_OK;
}

// ---- keyframe pose graph (bba_optimize_pose_graph, DESIGN §3.14) ----
// What the pose graph stages for K keyframes and C constraints: terms (a prior per keyframe, the constraints, the chain), ints
// (held flags, row offsets, two ints per row entry, CSR offsets and columns) and doubles (the terms' blocks, the CSR blocks, b, the
// couplings and the solver's work).  A row holds its prior and one entry per end of a constraint or chain edge.
struct PoseGraphSizes {
  size_t terms, ints, doubles;
};
PoseGraphSizes PoseGraphCapacity(size_t K, size_t C) {
  const size_t terms = 2 * K + C, entries = 3 * K + 2 * C, nnz = 3 * K + 2 * C;
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
  BBA_CUDA(h, g.d_doubles.Reserve(need.doubles, alloc.doubles));
  BBA_CUDA(h, g.h_poses.Reserve(7 * M));
  BBA_CUDA(h, g.d_poses.Reserve(14 * M));
  BBA_CUDA(h, g.d_state.Reserve(1));
  BBA_CUDA(h, g.h_state.Reserve(1));
  return BBA_OK;
}

int FindRoot(std::vector<int>& parent, int k) {
  while (parent[k] != k) k = parent[k] = parent[parent[k]];
  return k;
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
  if (K < 2 && h->pose_prior_count == 0) return BBA_OK;
  const std::vector<PoseConstraint>& cons = h->pose_constraints;
  if (bba_status st = ReservePoseGraph(h, cons.size())) return st;
  auto& g = h->graph;
  const bool chain = o->use_odometry_chain != 0;
  const int max_iterations = o->max_iterations > 0 ? o->max_iterations : 20;   // pose_graph_optimizer.cc kMaxIterations

  // the terms: priors, constraints by id, then the chain at the poses the call starts from
  float* poses = g.h_poses;
  for (int k = 0; k < K; ++k) PoseToArray(h->keyframes[k].pose, poses + 7 * k);
  std::vector<int> prior_term(K, -1);
  int T = 0;
  auto add = [&](int a, int b, const float* z, const float* info) {
    PoseGraphTerm& t = g.h_terms[T++];
    t.a = a;
    t.b = b;
    std::memcpy(t.z, z, sizeof(t.z));
    std::memcpy(t.info, info, sizeof(t.info));
  };
  for (int k = 0; k < K; ++k) {
    const PosePrior& p = h->pose_priors[k];
    if (!p.has) continue;
    prior_term[k] = T;
    add(k, -1, p.pose, p.info);
  }
  const int first_constraint = T;
  for (const PoseConstraint& c : cons) add(c.c.keyframe_a, c.c.keyframe_b, c.c.a_T_b, c.c.information);
  const int first_chain = T;
  if (chain)
    for (int k = 0; k + 1 < K; ++k) {
      double qa[4], ta[3], qb[4], tb[3], q[4], t[3];
      LoadPoseD(poses + 7 * k, qa, ta);
      LoadPoseD(poses + 7 * (k + 1), qb, tb);
      Se3BetweenD(qa, ta, qb, tb, q, t);   // T_k^-1 T_{k+1}
      float z[7];
      for (int j = 0; j < 4; ++j) z[j] = static_cast<float>(q[j]);
      for (int j = 0; j < 3; ++j) z[4 + j] = static_cast<float>(t[j]);
      add(k, k + 1, z, o->odometry_information);
    }

  // the held keyframes: the gauge, the untouched ones, and the lowest id of every component without the gauge or a prior
  std::vector<int> parent(K), lowest(K, -1);
  std::vector<char> touched(K, 0), anchored(K, 0);
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
    if (prior_term[k] >= 0) touched[k] = 1;
    if (prior_term[k] >= 0 || k == gauge) anchored[root] = 1;
  }
  int* held = g.h_ints;
  int held_count = 0;
  for (int k = 0; k < K; ++k) {
    const int root = FindRoot(parent, k);
    held[k] = (k == gauge || !touched[k] || (!anchored[root] && lowest[root] == k)) ? 1 : 0;
    held_count += held[k];
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
    entries += (prior_term[k] >= 0) + binary;
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
  a.max_linear = 6 * (K - held_count);
  for (int round = 0; round <= max_iterations; ++round) {
    a.round = round;
    BBA_LAUNCH(h, h->launches, LaunchPoseGraphRound, a, s);
  }
  BBA_CUDA(h, cudaMemcpyAsync(g.h_state, g.d_state, sizeof(PoseGraphState), cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaMemcpyAsync(poses, g.d_poses, sizeof(float) * 7 * K, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  for (int k = 0; k < K; ++k)
    if (!held[k]) h->keyframes[k].pose = PoseFromArray(poses + 7 * k);
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

}  // namespace
}  // namespace bba

using namespace bba;

extern "C" {

bba_status bba_update_surfel_activation(bba_handle h, void* stream) {
  return GeometryPass(h, /*activation=*/true, static_cast<cudaStream_t>(stream));
}

bba_status bba_optimize_geometry_iteration(bba_handle h, void* stream) {
  return GeometryPass(h, /*activation=*/false, static_cast<cudaStream_t>(stream));
}

bba_status bba_deform_surfels(bba_handle h, int count, const float* original_keyframe_T_global, uint32_t* moved, uint32_t* unobserved,
                              void* stream) {
  return DeformSurfels(h, count, original_keyframe_T_global, moved, unobserved, static_cast<cudaStream_t>(stream));
}

bba_status bba_optimize_pose_graph(bba_handle h, const bba_pose_graph_options* options, bba_pose_graph_result* result, void* stream) {
  return OptimizePoseGraph(h, options, result, static_cast<cudaStream_t>(stream));
}

bba_status bba_optimize_intrinsics(bba_handle h, int optimize_depth, int optimize_color, void* stream) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (!optimize_depth && !optimize_color) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "nothing to optimise");   // kernel_opt_intrinsics.cc:54
  if (bba_status st = CheckSurfels(h)) return st;
  if (bba_status st = CheckCollective(h)) return st;
  return OptimizeIntrinsics(h, optimize_depth != 0, optimize_color != 0, static_cast<cudaStream_t>(stream));
}

bba_status bba_debug_intrinsics_coeffs(bba_handle h, int optimize_depth, int optimize_color, double* sums, float* cells, void* stream) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (!sums || !cells) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_intrinsics_coeffs: null argument");
  if (!optimize_depth && !optimize_color) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "nothing to optimise");
  if (bba_status st = CheckSurfels(h)) return st;
  if (bba_status st = CheckCollective(h)) return st;
  const size_t P = static_cast<size_t>(h->cf_w) * h->cf_h;
  std::memset(sums, 0, sizeof(double) * bba::kIntrinsicsSums);
  std::memset(cells, 0, sizeof(float) * 8 * P);
  if (h->surfels_size == 0 || h->keyframes.empty()) return BBA_OK;   // (the step does nothing then)
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  IntrinsicsEquations eq;
  if (bba_status st = AccumulateIntrinsics(h, optimize_depth != 0, optimize_color != 0, s, &eq)) return st;
  BBA_CUDA(h, cudaMemcpyAsync(sums, h->geo.d_intr_sums, sizeof(double) * bba::kIntrinsicsSums, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaMemcpyAsync(cells, eq.cell_B, sizeof(float) * 8 * P, cudaMemcpyDeviceToHost, s));   // B, D, b2, obs are contiguous
  BBA_CUDA(h, cudaStreamSynchronize(s));
  return BBA_OK;
}

}  // extern "C"

namespace bba {
namespace {

// bba_bundle_adjust
bba_status BundleAdjust(bba_handle h, const bba_ba_options* o, bba_ba_result* res, void* stream) {
  std::memset(res, 0, sizeof(*res));
  if (bba_status st = CheckSurfels(h)) return st;
  // (do_surfel_updates with more than one rank: creation / merging / compaction run REPLICATED -- they are deterministic and
  // every rank holds the whole surfel buffer -- while the geometry and pose steps stay sharded; see PeerFence)
  if (o->use_pcg && h->deterministic)
    return Fail(h, BBA_ERR_UNSUPPORTED, "bba_bundle_adjust: use_pcg is not available in the deterministic mode (bba_set_deterministic)");
  if (o->use_pcg) return BundleAdjustPCG(h, o, res, static_cast<cudaStream_t>(stream));   // direct_ba.cc:436-457
  // direct_ba.cc:427-434
  const bool opt_depth_intr = o->optimize_depth_intrinsics && h->cfg.use_depth_residuals;
  const bool opt_color_intr = o->optimize_color_intrinsics && h->cfg.use_descriptor_residuals;
  if (bba_status st = CheckCollective(h)) return st;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int K = static_cast<int>(h->keyframes.size());
  const uint64_t launches_before = h->launches;
  const auto t_start = std::chrono::steady_clock::now();

  // the caller may have moved the surfels since the last call (through the device view): sort them again at the first pose step
  h->pose.order_stale = true;
  const int fixed_ba_iteration_count = h->ba_iteration_count;
  if (bba_status st = BeginBundleAdjust(h, o, res, s)) return st;
  std::vector<int> keyframes_with_new_surfels;

  const bool fixed_window = o->active_keyframe_window_start > 0 || o->active_keyframe_window_end > 0;   // :330-331
  const bool whole_window = !(o->active_keyframe_window_start != 0 || o->active_keyframe_window_end != K - 1);

  BBA_CUDA(h, cudaMemsetAsync(h->active, 0, h->surfels_size, s));   // :338

  for (int iteration = 0; iteration < o->max_iterations; ++iteration) {
    if (o->progress_function && !o->progress_function(o->progress_user, iteration)) break;
    ++res->iterations_done;
    if (fixed_window) {   // :354-372
      for (int k = 0; k < K; ++k)
        h->keyframes[k].activation =
            (k >= o->active_keyframe_window_start && k <= o->active_keyframe_window_end) ? BBA_KF_ACTIVE : BBA_KF_INACTIVE;
      DetermineCovisibleActiveKeyframes(h);
    }

    BBA_TRACE("iteration start");
    // --- surfel creation (:399-430)
    const uint32_t old_surfels_size = h->surfels_size;
    if (bba_status st = CreateInLoopSurfels(h, o, fixed_ba_iteration_count, s, res, &keyframes_with_new_surfels)) return st;
    if (!keyframes_with_new_surfels.empty()) h->pose.order_stale = true;

    BBA_TRACE("creation done");
    if (bba_status st = UploadKeyframes(h, s)) return st;
    BBA_TRACE("keyframes uploaded");
    const bool has_new = o->optimize_geometry && h->surfels_size > old_surfels_size;
    bba::GeometryArgs g;
    if (bba_status st = BuildGeometryArgs(h, &g, s, has_new ? GeoOrder::kCaller : GeoOrder::kByPairs)) return st;

    BBA_TRACE("after creation + upload");
    // --- surfel activation (:432-456) fused with the normal update of the geometry step (:466-485)
    BBA_CUDA(h, cudaEventRecord(h->ev[0], s));
    if (has_new)   // new surfels are active (:435-441); only the old ones are re-evaluated below
      BBA_CUDA(h, cudaMemsetAsync(h->active + old_surfels_size, bba::kSurfelActiveFlag, h->surfels_size - old_surfels_size, s));
    if (!whole_window) BBA_CUDA(h, cudaMemsetAsync(h->active, bba::kSurfelActiveFlag, old_surfels_size, s));
    if (h->surfels_size > 0) {
      if (whole_window && has_new) {
        bba::GeometryArgs g_old = g, g_new = g;   // (begin / end are LOCAL indices of this rank's shard)
        g_old.end = LocalCountBelow(old_surfels_size, h->cfg.rank, h->cfg.world_size);
        g_new.begin = g_old.end;
        BBA_LAUNCH(h, h->launches, LaunchActivationAndNormals, g_old, h->sm_count, true, true, s);
        BBA_LAUNCH(h, h->launches, LaunchActivationAndNormals, g_new, h->sm_count, false, true, s);
      } else if (whole_window) {
        BBA_LAUNCH(h, h->launches, LaunchActivationAndNormals, g, h->sm_count, true, o->optimize_geometry != 0, s);
      } else if (o->optimize_geometry) {
        BBA_LAUNCH(h, h->launches, LaunchActivationAndNormals, g, h->sm_count, false, true, s);
      }
    }
    BBA_CUDA(h, cudaEventRecord(h->ev[1], s));
    if (o->optimize_geometry && h->surfels_size > 0) BBA_LAUNCH(h, h->launches, LaunchPositionAndDescriptor, g, h->sm_count, s);
    if (bba_status st = ExchangeGeometry(h, s)) return st;   // multi-GPU: all-gather of the updated surfel shards
    BBA_CUDA(h, cudaEventRecord(h->ev[2], s));
    if (bba_status st = MarkStaging(h, s)) return st;

    BBA_TRACE("after geometry");
    // --- surfel merge + compaction (:489-541) for the keyframes that received new surfels
    if (o->do_surfel_updates && !keyframes_with_new_surfels.empty()) {
      uint32_t merged = 0;
      if (bba_status st = MergeAndCompact(h, keyframes_with_new_surfels, s, &merged)) return st;
      res->surfels_merged += merged;
      h->pose.order_stale = true;
    }

    BBA_TRACE("before pose step");
    // --- pose optimisation (:543-577): all non-inactive keyframes at once
    int num_converged = 0;
    if (o->optimize_poses) {
      std::vector<int> ids;
      std::vector<Pose> init;
      for (int k = 0; k < K; ++k) {
        if (h->keyframes[k].activation == BBA_KF_INACTIVE) {
          ++num_converged;
          continue;
        }
        ids.push_back(k);
        init.push_back(h->keyframes[k].pose);
      }
      if (bba_status st = RunPoseStep(h, ids, init, 30, s)) return st;
      res->depth_residual_count = 0;
      res->descriptor_residual_count = 0;
      res->cost = 0;
      for (int k : ids) {
        Keyframe& kf = h->keyframes[k];
        const Pose est = PoseFromArray(h->pose.h_pose_est + 7 * k);
        float lg[6];
        bba::Log(bba::Compose(bba::Inverse(kf.pose), est), lg);   // :562-563
        const bool moved = !bba::IsScale1PoseEstimationConverged(lg);
        kf.pose = est;
        if (moved) {
          kf.activation = BBA_KF_ACTIVE;
        } else {
          kf.activation = BBA_KF_INACTIVE;
          ++num_converged;
        }
        res->pose_iterations_total += h->pose.h_iterations[k];
        const double* fs = h->pose.h_first_stats + 8 * k;
        res->depth_residual_count += static_cast<uint64_t>(fs[0] + 0.5);
        res->descriptor_residual_count += 2 * static_cast<uint64_t>(fs[1] + 0.5);
        res->cost += fs[2] + fs[3];
      }
    } else {
      BBA_CUDA(h, cudaStreamSynchronize(s));
    }
    if (bba_status st = Publish(h, s, false)) return st;   // every pose of this step at once
    BBA_CUDA(h, cudaEventRecord(h->ev[3], s));
    // --- intrinsics optimisation (:584-624)
    if (opt_depth_intr || opt_color_intr) {
      if (bba_status st = OptimizeIntrinsics(h, opt_depth_intr, opt_color_intr, s)) return st;
      BBA_CUDA(h, cudaEventRecord(h->ev[4], s));
      BBA_CUDA(h, cudaEventSynchronize(h->ev[4]));
      cudaEventElapsedTime(&res->ms_intrinsics_optimization, h->ev[3], h->ev[4]);
    }
    BBA_CUDA(h, cudaEventSynchronize(h->ev[3]));
    cudaEventElapsedTime(&res->ms_surfel_activation, h->ev[0], h->ev[1]);
    cudaEventElapsedTime(&res->ms_geometry_optimization, h->ev[1], h->ev[2]);
    cudaEventElapsedTime(&res->ms_pose_optimization, h->ev[2], h->ev[3]);
    if (h->profiling) {
      h->profile.activation_normals_ms += res->ms_surfel_activation;
      h->profile.position_descriptor_ms += res->ms_geometry_optimization;
      h->profile.geometry_launches += (o->optimize_geometry ? 2 : 1);
    }

    if (StopIterating(o, iteration, num_converged, K, t_start, res)) break;   // :693-709
    DetermineCovisibleActiveKeyframes(h);   // :711-717
    if (bba_status st = Publish(h, s, false)) return st;
  }
  BBA_TRACE("iterations done");
  return EndBundleAdjust(h, o, launches_before, res, s);
}

}  // namespace
}  // namespace bba

extern "C" bba_status bba_bundle_adjust(bba_handle h, const bba_ba_options* o, bba_ba_result* res, void* stream) {
  if (!h || !o || !res) return BBA_ERR_INVALID_ARGUMENT;
  const bba_status st = bba::BundleAdjust(h, o, res, static_cast<cudaStream_t>(stream));
  // whatever the call changed of the published state, also on an early return (poses and cameras are published where they
  // change; this covers the activations and the keyframe state of a failed call)
  bba::Publish(h, static_cast<cudaStream_t>(stream), false);
  return st;
}

extern "C" {

bba_status bba_perform_end_tasks(bba_handle h, int do_surfel_updates, uint32_t* deleted, uint32_t* surfels_size, void* stream) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckSurfels(h)) return st;
  uint32_t d = 0;
  if (bba_status st = PerformEndTasks(h, static_cast<cudaStream_t>(stream), &d, do_surfel_updates != 0)) return st;
  if (deleted) *deleted = d;
  if (surfels_size) *surfels_size = h->surfels_size;
  return BBA_OK;
}

bba_status bba_create_surfels_for_keyframe(bba_handle h, int id, int filter_new_surfels, uint32_t* created, void* stream) {
  CHECK_KF(h, id);
  if (bba_status st = CheckSurfels(h)) return st;
  uint32_t c = 0;
  if (bba_status st = CreateSurfelsForKeyframe(h, id, filter_new_surfels != 0, static_cast<cudaStream_t>(stream), &c)) return st;
  if (created) *created = c;
  return BBA_OK;
}

bba_status bba_merge_surfels_for_keyframe(bba_handle h, int id, uint32_t* deleted, void* stream) {
  CHECK_KF(h, id);
  if (bba_status st = CheckSurfels(h)) return st;
  uint32_t d = 0;
  if (bba_status st = MergeSurfelsForKeyframe(h, id, static_cast<cudaStream_t>(stream), &d)) return st;
  if (deleted) *deleted = d;
  return BBA_OK;
}

bba_status bba_compact_surfels(bba_handle h, uint32_t free_count, int with_active_flags, uint32_t* surfels_size, void* stream) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckSurfels(h)) return st;
  if (free_count > h->surfels_size) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "free_count exceeds surfels_size");
  if (bba_status st = CompactSurfels(h, free_count, with_active_flags != 0, static_cast<cudaStream_t>(stream))) return st;
  if (surfels_size) *surfels_size = h->surfels_size;
  return BBA_OK;
}

bba_status bba_pcg_debug(bba_handle h, const bba_ba_options* o, int step, int apply, uint32_t* unknown_count, bba_pcg_probe* out,
                         void* stream) {
  if (!h || !o || !unknown_count || step < 0) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckSurfels(h)) return st;
  const int K = static_cast<int>(h->keyframes.size());
  if (K == 0) return Fail(h, BBA_ERR_STATE, "no keyframes");
  if (o->pcg_gauge_keyframe < 0 || o->pcg_gauge_keyframe >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "pcg_gauge_keyframe out of range");
  if (h->cfg.world_size > 1) return Fail(h, BBA_ERR_UNSUPPORTED, "bba_pcg_debug runs on one rank");
  if (h->deterministic) return Fail(h, BBA_ERR_UNSUPPORTED, "bba_pcg_debug: the PCG solver is not available in the deterministic mode");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PcgLayout L;
  if (bba_status st = MakePcgLayout(h, o, &L)) return st;
  *unknown_count = L.unknown_count;
  if (!out || L.unknown_count == 0) return BBA_OK;
  const uint32_t U = L.unknown_count;
  auto copy = [&](float* dst, const float* src) -> bba_status {
    if (dst) BBA_CUDA(h, cudaMemcpyAsync(dst, src, sizeof(float) * U, cudaMemcpyDeviceToHost, s));
    return BBA_OK;
  };
  // the scalar slots of alpha_n / beta_n of step `step` (BundleAdjustPCG swaps them at every step after the first)
  auto scalars = [&](int slot, double* dst) -> bba_status {
    BBA_CUDA(h, cudaMemcpyAsync(h->pcg.h_scalars, h->pcg.d_scalars, sizeof(double) * 4, cudaMemcpyDeviceToHost, s));
    BBA_CUDA(h, cudaStreamSynchronize(s));
    *dst = h->pcg.h_scalars[slot];
    return BBA_OK;
  };
  if (bba_status st = UploadKeyframes(h, s)) return st;
  const bba::PcgArgs a = MakePcgArgs(h, L, o->pcg_gauge_keyframe);
  int an = 0, bn = 2;
  if (bba_status st = PcgInit(h, L, a, an, s)) return st;
  for (int k = 0;; ++k) {
    if (k > 0) std::swap(an, bn);
    if (bba_status st = PcgStep1(h, L, a, s)) return st;
    if (k == step) break;
    if (bba_status st = PcgStep2(h, L, an, bn, s)) return st;
    if (bba_status st = PcgStep3(h, L, an, bn, s)) return st;
  }
  float *r = h->pcg.d_vec[0], *M = h->pcg.d_vec[1], *delta = h->pcg.d_vec[2], *g = h->pcg.d_vec[3], *p = h->pcg.d_vec[4];
  bba_status st = BBA_OK;
  if ((st = copy(out->r, r)) || (st = copy(out->M, M)) || (st = copy(out->p, p)) || (st = copy(out->g, g)) || (st = copy(out->delta, delta)) ||
      (st = scalars(an, &out->alpha_n)) || (st = scalars(1, &out->alpha_d)))
    return st;
  if ((st = PcgStep2(h, L, an, bn, s)) || (st = copy(out->r_step2, r)) || (st = copy(out->delta_step2, delta)) || (st = copy(out->z, g)) ||
      (st = scalars(bn, &out->beta_n)))
    return st;
  if ((st = PcgStep3(h, L, an, bn, s)) || (st = copy(out->p_step3, p)) || (st = copy(out->g_step3, g)) || (st = scalars(1, &out->alpha_d_step3)))
    return st;
  if (apply) {
    int num_converged = 0;
    if ((st = PcgApplyDelta(h, L, o->pcg_gauge_keyframe, s, &num_converged))) return st;
  }
  BBA_CUDA(h, cudaStreamSynchronize(s));
  return MarkStaging(h, s);
}

}  // extern "C"
