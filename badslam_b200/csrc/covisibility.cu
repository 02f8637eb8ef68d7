// covisibility.cu -- the co-visibility measurements in libbadba_b200 (host side): the whole-replica walk that
// bba_measure_keyframe_covisibility (DESIGN.md §3.19), bba_measure_frame_overlap (§3.20) and bba_estimate_keyframe_exposures
// (§3.21, exposure.cu) run their bit-row launches on, and the first two calls with their entry points.
#include <cmath>
#include <cstring>

#include "handle.hpp"

namespace bba {

bba_status ReserveReplicaWalk(bba_handle h, size_t rows, ReplicaWalk* w) {
  uint32_t chunk = h->covis.chunk;
  if (chunk == 0) {   // whole 256-surfel geometry tiles; the budget counts every row held
    const uint64_t fit = kCovisibilityBitsBudget * 8 / rows;
    chunk = static_cast<uint32_t>(std::max<uint64_t>(256, std::min<uint64_t>(fit, 0xffffff00ull) / 256 * 256));
  }
  w->rows = rows;
  w->chunk = std::max<uint32_t>(1, std::min(chunk, h->surfels_size));
  BBA_CUDA(h, h->covis.d_bits.Reserve(rows * ((w->chunk + 31u) / 32u)));
  return MakeAllKeyframeList(h);
}

bba_status WalkReplica(bba_handle h, const ReplicaWalk& w, const KfDevice* kfs, const int* list, int count, cudaStream_t s,
                       const std::function<bba_status(const GeometryArgs& g, uint32_t words)>& launch) {
  const uint32_t n = h->surfels_size;
  if (n == 0) return BBA_OK;
  // Every rank walks its whole replica (begin 0, end n, one shard), in the spatial order unless the geometry launches keep the
  // caller's (peer stores): the counts and sums are integers, so they do not depend on the order.
  const bool sort = !PeerStores(h);
  if (bba_status st = EnsureSpatialOrder(h, sort, /*rebuild=*/false, s)) return st;
  GeometryArgs g{};
  if (bba_status st = SetGeometryFields(h, sort, kfs, list, count, &g)) return st;
  g.shard_rank = 0;
  g.shard_world = 1;
  g.peers = PeerSet{};
  for (uint32_t begin = 0; begin < n; begin += w.chunk) {
    g.begin = begin;
    g.end = begin + std::min(w.chunk, n - begin);
    const uint32_t words = (g.end - g.begin + 31u) / 32u;
    BBA_CUDA(h, cudaMemsetAsync(h->covis.d_bits, 0, sizeof(uint32_t) * w.rows * words, s));
    if (bba_status st = launch(g, words)) return st;
  }
  return BBA_OK;
}

namespace {

// bba_measure_keyframe_covisibility.  Every argument is checked before anything is enqueued; nothing on the handle changes but the
// spatial order, which is rebuilt when stale (a function of the positions alone).
bba_status MeasureKeyframeCovisibility(bba_handle h, int count, const int* ids, int keyframe_count, uint32_t* out, cudaStream_t s) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_measure_keyframe_covisibility: ";
  const int K = static_cast<int>(h->keyframes.size());
  if (!out) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null out_counts");
  if (count == 0 || count < -1) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad count");
  if (count > 0 && !ids) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null keyframe_ids");
  if (keyframe_count != K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "keyframe_count is not the handle's keyframe count");
  for (int i = 0; i < count; ++i)
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "unknown keyframe id");
  const int rows = count < 0 ? K : count;
  const uint32_t n = h->surfels_size;
  if (K == 0 || n == 0) {
    std::fill(out, out + static_cast<size_t>(rows) * K, 0u);
    return BBA_OK;
  }
  if (bba_status st = CheckSurfels(h)) return st;
  auto& c = h->covis;
  ReplicaWalk w;
  if (bba_status st = ReserveReplicaWalk(h, K, &w)) return st;
  BBA_CUDA(h, c.d_counts.Reserve(static_cast<size_t>(rows) * K));
  if (count > 0) BBA_CUDA(h, c.d_rows.Reserve(count));
  if (bba_status st = UploadKeyframes(h, s)) return st;   // the current poses
  if (count > 0) BBA_CUDA(h, cudaMemcpyAsync(c.d_rows, ids, sizeof(int) * count, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemsetAsync(c.d_counts, 0, sizeof(uint32_t) * rows * K, s));
  CovisibilityGramArgs q{c.d_bits, 0, count > 0 ? c.d_rows.get() : h->geo.d_all_list.get(), rows, K, c.d_counts};
  if (bba_status st = WalkReplica(h, w, h->d_kfs, h->geo.d_all_list, K, s, [&](const GeometryArgs& g, uint32_t words) {
        const CovisibilityBitsArgs a{g, c.d_bits, words};
        BBA_LAUNCH(h, h->launches, LaunchCovisibilityBits, a, h->sm_count, s);
        q.words = words;
        BBA_LAUNCH(h, h->launches, LaunchCovisibilityGram, q, h->sm_count, s);
        return BBA_OK;
      }))
    return st;
  BBA_CUDA(h, cudaMemcpyAsync(out, c.d_counts, sizeof(uint32_t) * rows * K, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  return BBA_OK;
}

// A frame of bba_measure_frame_overlap as the kernels read it: u16 depth and normals rows of the depth width, 2-byte aligned.
bool OverlapFrameOk(bba_handle h, const bba_frame_buffers& f) {
  const size_t row = static_cast<size_t>(h->cfg.depth_width) * 2;
  return f.depth && f.normals && f.depth_pitch >= row && f.normals_pitch >= row && f.depth_pitch <= 0xffffffffull &&
         f.normals_pitch <= 0xffffffffull && !(f.depth_pitch & 1u) && !(f.normals_pitch & 1u) &&
         !(reinterpret_cast<uintptr_t>(f.depth) & 1u) && !(reinterpret_cast<uintptr_t>(f.normals) & 1u);
}

// bba_measure_frame_overlap (DESIGN §3.20).  Every argument is checked before anything is enqueued; nothing on the handle changes
// but the spatial order, which is rebuilt when stale.  The frames' records get rows after the keyframes' in the covisibility bit
// rows (rows K .. K + n - 1, or 0 .. n - 1 without the keyframes' side), so that the keyframe Gram gives shared and, on its
// diagonal, observed_surfels; the frames' cell rows then feed the seed count.
bba_status MeasureFrameOverlap(bba_handle h, int frame_count, const bba_frame_buffers* frames, int count, const bba_frame_overlap_query* queries,
                               int keyframe_count, uint32_t* shared, bba_frame_overlap* out, cudaStream_t s) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_measure_frame_overlap: ";
  const int K = static_cast<int>(h->keyframes.size());
  if (!frames || !queries || !out) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  if (count < 1 || frame_count < 1) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count and frame_count must be at least 1");
  if (keyframe_count != K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "keyframe_count is not the handle's keyframe count");
  for (int f = 0; f < frame_count; ++f)
    if (!OverlapFrameOk(h, frames[f])) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null, misaligned or too narrow frame image");
  for (int i = 0; i < count; ++i) {
    const bba_frame_overlap_query& q = queries[i];
    const std::string which = " in query " + std::to_string(i);
    if (q.frame < 0 || q.frame >= frame_count) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "frame index out of range" + which);
    for (int j = 0; j < 7; ++j)
      if (!std::isfinite(q.global_T_frame[j])) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "non-finite pose" + which);
    const float* p = q.global_T_frame;
    if (p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3] < 1e-12f) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "zero quaternion" + which);
    if (!(q.min_depth > 0.f && q.min_depth <= q.max_depth && std::isfinite(q.max_depth)))
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "depth range must be 0 < min_depth <= max_depth" + which);
  }
  const uint32_t n_surfels = h->surfels_size;
  if (n_surfels > 0)
    if (bba_status st = CheckSurfels(h)) return st;

  const int n = count;
  const bool with_kfs = shared && K > 0;           // the keyframes' bit rows and the full Gram
  const int kf_rows = with_kfs ? K : 0;
  const int cols = kf_rows + n;
  const uint32_t cells = static_cast<uint32_t>(h->cf_w) * h->cf_h;
  const uint32_t cell_words = (cells + 31u) / 32u;
  auto& o = h->overlap;
  // the frusta of the keyframes and queries (AddKeyframeCommon's) and the CSR of the queries' co-visible keyframes
  std::vector<Frustum> kf_frusta(K);
  for (int k = 0; k < K; ++k) {
    const Keyframe& kf = h->keyframes[k];
    MakeFrustum(&kf_frusta[k], h->depth_K, h->cfg.depth_width, h->cfg.depth_height, kf.min_depth, kf.max_depth, kf.pose);
  }
  std::vector<std::vector<int>> covis(n);
  size_t covis_total = 0;
  for (int i = 0; i < n; ++i) {
    Frustum fq;
    MakeFrustum(&fq, h->depth_K, h->cfg.depth_width, h->cfg.depth_height, queries[i].min_depth, queries[i].max_depth,
                PoseFromArray(queries[i].global_T_frame));
    for (int k = 0; k < K; ++k)
      if (FrustaIntersect(fq, kf_frusta[k])) covis[i].push_back(k);
    covis_total += covis[i].size();
  }
  const size_t ints = 2 * static_cast<size_t>(n) + n + 1;   // [frame list 0 .. n-1 | Gram rows | covis offsets]
  const size_t count_words = 3 * static_cast<size_t>(n) + static_cast<size_t>(n) * cols;   // [n][3] seed counts, then [n][cols]
  BBA_CUDA(h, o.d_frames.Reserve(n));
  BBA_CUDA(h, o.h_frames.Reserve(n));
  BBA_CUDA(h, o.d_ints.Reserve(ints));
  BBA_CUDA(h, o.h_ints.Reserve(ints));
  BBA_CUDA(h, o.d_covis.Reserve(std::max<size_t>(covis_total, 1)));
  BBA_CUDA(h, o.h_covis.Reserve(std::max<size_t>(covis_total, 1)));
  BBA_CUDA(h, o.d_cells.Reserve(static_cast<size_t>(n) * cell_words));
  BBA_CUDA(h, o.d_counts.Reserve(count_words));
  BBA_CUDA(h, o.h_counts.Reserve(count_words));
  ReplicaWalk w;
  if (bba_status st = ReserveReplicaWalk(h, cols, &w)) return st;

  // staging: the frame records (UploadKeyframes' records at the query poses), the int lists and the co-visible keyframes
  int* list = o.h_ints;
  int* rows = list + n;
  int* offsets = rows + n;
  size_t e = 0;
  for (int i = 0; i < n; ++i) {
    const bba_frame_overlap_query& q = queries[i];
    const bba_frame_buffers& f = frames[q.frame];
    const Pose pose = PoseFromArray(q.global_T_frame);
    KfDevice& d = o.h_frames[i];
    std::memset(&d, 0, sizeof(d));
    ToMatrix3x4(Inverse(pose), d.T);
    d.depth = f.depth;
    d.normals = f.normals;
    d.depth_pitch = static_cast<uint32_t>(f.depth_pitch);
    d.normals_pitch = static_cast<uint32_t>(f.normals_pitch);
    list[i] = i;
    rows[i] = kf_rows + i;
    offsets[i] = static_cast<int>(e);
    for (int k : covis[i]) o.h_covis[e++] = MakeCovisEntry(h->keyframes[k], pose);   // CreateSurfelsForKeyframe's entries
  }
  offsets[n] = static_cast<int>(e);
  BBA_CUDA(h, cudaMemcpyAsync(o.d_frames, o.h_frames, sizeof(KfDevice) * n, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemcpyAsync(o.d_ints, o.h_ints, sizeof(int) * ints, cudaMemcpyHostToDevice, s));
  if (e) BBA_CUDA(h, cudaMemcpyAsync(o.d_covis, o.h_covis, sizeof(CovisEntry) * e, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemsetAsync(o.d_cells, 0, sizeof(uint32_t) * n * cell_words, s));
  BBA_CUDA(h, cudaMemsetAsync(o.d_counts, 0, sizeof(uint32_t) * count_words, s));

  // the walk: per chunk, the keyframes' bit rows (with shared), the frames' bit rows and cell rows, and the Gram
  if (n_surfels > 0 && with_kfs)
    if (bba_status st = UploadKeyframes(h, s)) return st;   // the current poses
  CovisibilityGramArgs q{h->covis.d_bits, 0, o.d_ints.get() + n, n, cols, o.d_counts.get() + 3 * static_cast<size_t>(n)};
  if (bba_status st = WalkReplica(h, w, o.d_frames, o.d_ints, n, s, [&](const GeometryArgs& g, uint32_t words) {
        if (with_kfs) {
          CovisibilityBitsArgs kb{g, h->covis.d_bits, words};
          kb.geo.kfs = h->d_kfs;
          kb.geo.kf_list = h->geo.d_all_list;
          kb.geo.kf_count = K;
          BBA_LAUNCH(h, h->launches, LaunchCovisibilityBits, kb, h->sm_count, s);
        }
        const CovisibilityBitsArgs fb{g, h->covis.d_bits.get() + static_cast<size_t>(kf_rows) * words, words, o.d_cells, cell_words};
        BBA_LAUNCH(h, h->launches, LaunchCovisibilityBits, fb, h->sm_count, s);
        q.words = words;
        BBA_LAUNCH(h, h->launches, LaunchCovisibilityGram, q, h->sm_count, s);
        return BBA_OK;
      }))
    return st;

  // the seed count, with the minimum observation count of the handle with the frame added
  FrameSeedArgs sa;
  sa.cam = MakeCamera(h);
  sa.frames = o.d_frames;
  sa.frame_count = n;
  sa.cells = cells;
  sa.covered = o.d_cells;
  sa.cell_words = cell_words;
  sa.covis = o.d_covis;
  sa.covis_offsets = o.d_ints.get() + 2 * static_cast<size_t>(n);
  sa.min_observation_count = MinObservationCount(h, h->keyframes.size() + 1);
  sa.counts = o.d_counts;
  BBA_LAUNCH(h, h->launches, LaunchFrameSeedCount, sa, s);
  BBA_CUDA(h, cudaMemcpyAsync(o.h_counts, o.d_counts, sizeof(uint32_t) * count_words, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  const uint32_t* seeds = o.h_counts;
  const uint32_t* gram = seeds + 3 * static_cast<size_t>(n);
  for (int i = 0; i < n; ++i) {
    const uint32_t* row = gram + static_cast<size_t>(i) * cols;
    out[i].observed_surfels = row[kf_rows + i];
    out[i].valid_cells = seeds[3 * i];
    out[i].uncovered_cells = seeds[3 * i + 1];
    out[i].new_surfels = seeds[3 * i + 2];
    if (with_kfs) std::copy(row, row + K, shared + static_cast<size_t>(i) * K);
  }
  return BBA_OK;
}

}  // namespace
}  // namespace bba

using namespace bba;

extern "C" {

bba_status bba_measure_keyframe_covisibility(bba_handle h, int count, const int* keyframe_ids, int keyframe_count, uint32_t* out_counts,
                                             void* stream) {
  return MeasureKeyframeCovisibility(h, count, keyframe_ids, keyframe_count, out_counts, static_cast<cudaStream_t>(stream));
}

bba_status bba_measure_frame_overlap(bba_handle h, int frame_count, const bba_frame_buffers* frames, int count,
                                     const bba_frame_overlap_query* queries, int keyframe_count, uint32_t* shared,
                                     bba_frame_overlap* out, void* stream) {
  return MeasureFrameOverlap(h, frame_count, frames, count, queries, keyframe_count, shared, out, static_cast<cudaStream_t>(stream));
}

bba_status bba_debug_set_covisibility_chunk(bba_handle h, uint32_t surfels) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  h->covis.chunk = surfels;
  return BBA_OK;
}

}  // extern "C"
