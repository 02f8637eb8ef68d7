// place_index.cu -- the randomized-fern keyframe index (DESIGN.md §3.18; Glocker et al., TVCG 2015): bba_index_keyframes (BA
// side), bba_query_place_index and bba_get_place_index_codes (front end), bba_host_place_ferns, and the two kernels.
//
// The rule, owned here and restated by tests/place_index_oracle.py:
//  - ferns: F (a multiple of 8 in [8, 2048]) ferns drawn from splitmix64 with kPlaceFernSeed, six draws per fern in the order
//    cx % 80, cy % 60, t_r, t_g, t_b (% 256), min_raw + draw % (max_raw - min_raw + 1);
//  - cells: cell (cx, cy) of a W x H image is x in [cx W / 80, (cx + 1) W / 80), y in [cy H / 60, (cy + 1) H / 60), on the depth
//    and the colour image separately;
//  - code: fern f's nibble (word f / 8, bit 4 (f % 8)) has bit c = sum of channel c > t_c * n over its colour cell (c = r, g, b:
//    bytes 0..2 of the uchar4 image) and bit 3 = sum of raw d > t_d * n_v over the cell's valid depth pixels, in u64;
//  - difference: the number of ferns whose nibbles differ.
// Every step is integer arithmetic, so the codes and the matches are the same bits in every mode, on every rank and every run.
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "handle.hpp"

namespace bba {
namespace {

constexpr uint64_t kPlaceFernSeed = 0x5EED0F3E4B5A11CEull;   // tests/place_index_oracle.py FERN_SEED
constexpr int kGridW = 80, kGridH = 60;
constexpr int kMaxFerns = 2048;
constexpr int kDefaultFerns = 512;
constexpr float kDefaultMinDepth = 0.5f;
constexpr float kDefaultMaxDepth = 3.0f;   // BadSlamConfig's max_depth cutoff of the preprocessing
constexpr int kMaxMatches = 64;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
// Cells of at most this many pixels keep the u32 sums of raw depth (< 2^15 per pixel) exact.
constexpr int64_t kMaxCellPixels = 1 << 16;

// splitmix64: draw i (0-based) of the stream seeded with `seed`.  The generator is counter-based, so a fern's draws need no
// earlier state and the device can compute the table itself.
__host__ __device__ __forceinline__ uint64_t SplitMix64(uint64_t seed, uint64_t i) {
  uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

struct Fern {
  int cx, cy;
  int t[4];   // r, g, b thresholds, raw depth threshold
};

__host__ __device__ __forceinline__ Fern MakeFern(int f, int min_raw, int max_raw) {
  const uint64_t i = 6ull * static_cast<uint64_t>(f);
  Fern r;
  r.cx = static_cast<int>(SplitMix64(kPlaceFernSeed, i) % kGridW);
  r.cy = static_cast<int>(SplitMix64(kPlaceFernSeed, i + 1) % kGridH);
  for (int c = 0; c < 3; ++c) r.t[c] = static_cast<int>(SplitMix64(kPlaceFernSeed, i + 2 + c) % 256);
  r.t[3] = min_raw + static_cast<int>(SplitMix64(kPlaceFernSeed, i + 5) % static_cast<uint64_t>(max_raw - min_raw + 1));
  return r;
}

struct EncodeArgs {
  const PlaceImage* images;   // [gridDim.x]
  int dw, dh, cw, ch;         // depth and colour image sizes
  int num_ferns, min_raw, max_raw;
};

// One CTA per image.  The fern table is computed into shared memory; then each warp takes ferns f = warp, warp + 8, ...: its
// lanes stride over the fern's colour cell and depth cell, sum in u32 and reduce with __reduce_add_sync; lane 0 compares in u64
// and stores the nibble.  The nibbles are packed into the code row at the end.
__global__ void __launch_bounds__(kThreads) PlaceEncodeKernel(EncodeArgs a) {
  __shared__ int3 ferns[kMaxFerns];   // (cx | cy << 8, t_r | t_g << 8 | t_b << 16, t_d)
  __shared__ uint8_t nibbles[kMaxFerns];
  const PlaceImage im = a.images[blockIdx.x];
  for (int f = threadIdx.x; f < a.num_ferns; f += kThreads) {
    const Fern r = MakeFern(f, a.min_raw, a.max_raw);
    ferns[f] = make_int3(r.cx | (r.cy << 8), r.t[0] | (r.t[1] << 8) | (r.t[2] << 16), r.t[3]);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int f = warp; f < a.num_ferns; f += kWarps) {
    const int3 packed = ferns[f];
    Fern fern;
    fern.cx = packed.x & 0xff;
    fern.cy = packed.x >> 8;
    fern.t[0] = packed.y & 0xff;
    fern.t[1] = (packed.y >> 8) & 0xff;
    fern.t[2] = packed.y >> 16;
    fern.t[3] = packed.z;
    // colour cell
    const int cx0 = fern.cx * a.cw / kGridW, cx1 = (fern.cx + 1) * a.cw / kGridW;
    const int cy0 = fern.cy * a.ch / kGridH, cy1 = (fern.cy + 1) * a.ch / kGridH;
    const int cbw = cx1 - cx0, cn = cbw * (cy1 - cy0);
    uint32_t sr = 0, sg = 0, sb = 0;
    for (int i = lane; i < cn; i += 32) {
      const int x = cx0 + i % cbw, y = cy0 + i / cbw;
      const uchar4 p = *reinterpret_cast<const uchar4*>(im.rgba + static_cast<size_t>(y) * im.rgba_pitch + 4 * static_cast<size_t>(x));
      sr += p.x;
      sg += p.y;
      sb += p.z;
    }
    // depth cell
    const int dx0 = fern.cx * a.dw / kGridW, dx1 = (fern.cx + 1) * a.dw / kGridW;
    const int dy0 = fern.cy * a.dh / kGridH, dy1 = (fern.cy + 1) * a.dh / kGridH;
    const int dbw = dx1 - dx0, dn = dbw * (dy1 - dy0);
    uint32_t sd = 0, nv = 0;
    for (int i = lane; i < dn; i += 32) {
      const int x = dx0 + i % dbw, y = dy0 + i / dbw;
      const uint16_t d = LoadPixelU16(im.depth, im.depth_pitch, x, y);
      if (!(d & kInvalidDepthBit)) {
        sd += d;
        ++nv;
      }
    }
    sr = __reduce_add_sync(0xffffffffu, sr);
    sg = __reduce_add_sync(0xffffffffu, sg);
    sb = __reduce_add_sync(0xffffffffu, sb);
    sd = __reduce_add_sync(0xffffffffu, sd);
    nv = __reduce_add_sync(0xffffffffu, nv);
    if (lane == 0) {
      const uint64_t n = static_cast<uint64_t>(cn);
      uint32_t code = 0;
      code |= (static_cast<uint64_t>(sr) > static_cast<uint64_t>(fern.t[0]) * n) ? 1u : 0u;
      code |= (static_cast<uint64_t>(sg) > static_cast<uint64_t>(fern.t[1]) * n) ? 2u : 0u;
      code |= (static_cast<uint64_t>(sb) > static_cast<uint64_t>(fern.t[2]) * n) ? 4u : 0u;
      code |= (static_cast<uint64_t>(sd) > static_cast<uint64_t>(fern.t[3]) * nv) ? 8u : 0u;
      nibbles[f] = static_cast<uint8_t>(code);
    }
  }
  __syncthreads();
  for (int w = threadIdx.x; w < a.num_ferns / 8; w += kThreads) {
    uint32_t word = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) word |= static_cast<uint32_t>(nibbles[8 * w + i]) << (4 * i);
    im.code[w] = word;
  }
}

LaunchResult LaunchPlaceEncode(const EncodeArgs& a, int images, cudaStream_t s) {
  LaunchResult r;
  PlaceEncodeKernel<<<images, kThreads, 0, s>>>(a);
  r.kernels = 1;
  return r;
}

struct MatchArgs {
  const PlaceQueryRecord* queries;   // [gridDim.x]
  const uint32_t* table;             // the code table of the snapshot's slot, kPlaceRowWords words per keyframe
  const uint8_t* indexed;            // [published keyframes]
  int words, num_ferns, max_matches;
  int* matches;                      // [queries][2 * max_matches + 1]: ids, differences, count
};

// D(query, row): the number of differing nibbles, over the row's `words` words (lanes take words), summed over the warp.
__device__ __forceinline__ int Difference(const uint32_t* query, const uint32_t* row, int words, int lane) {
  int d = 0;
  for (int w = lane; w < words; w += 32) {
    uint32_t x = query[w] ^ __ldg(row + w);
    x = (x | (x >> 1) | (x >> 2) | (x >> 3)) & 0x11111111u;
    d += __popc(x);
  }
  return static_cast<int>(__reduce_add_sync(0xffffffffu, static_cast<uint32_t>(d)));
}

// Whether keyframe k is a candidate of the query.
__device__ __forceinline__ bool Candidate(const MatchArgs& a, const PlaceQueryRecord& q, int k) {
  return k <= q.last && k != q.exclude && a.indexed[k];
}

// One CTA per query.  The query code is staged in shared memory.  Candidates are visited in blocks of 256 consecutive ids, 32 per
// warp, one row per warp step.  Pass 1 builds the histogram of D over [0, F]; warp 0 finds the cut c, the smallest D at which
// the cumulative count reaches m = min(max_matches, candidates), and `need`, how many of the ties at c are taken.  Pass 2 takes
// every candidate with D < c and the `need` smallest ids with D = c (ranked by a ballot within a warp and the warps' tie counts
// in id order), and the final order (D, id) is each selected entry's rank among the selected.  Nothing depends on the grid or
// on the scheduling.
__global__ void __launch_bounds__(kThreads) PlaceMatchKernel(MatchArgs a) {
  __shared__ uint32_t query[kPlaceRowWords];
  __shared__ int hist[kMaxFerns + 1];
  __shared__ int warp_ties[kWarps];
  __shared__ int sel_id[kMaxMatches], sel_d[kMaxMatches];
  __shared__ int sel_n, cut, need, take, ties_before;
  const PlaceQueryRecord q = a.queries[blockIdx.x];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int w = threadIdx.x; w < a.words; w += kThreads) query[w] = q.code[w];
  for (int d = threadIdx.x; d <= a.num_ferns; d += kThreads) hist[d] = 0;
  if (threadIdx.x == 0) sel_n = ties_before = 0;
  __syncthreads();

  // pass 1: the histogram
  for (int base = q.first + 32 * warp; base <= q.last; base += kThreads) {
    for (int j = 0; j < 32; ++j) {
      const int k = base + j;
      if (!Candidate(a, q, k)) continue;   // (uniform over the warp)
      const int d = Difference(query, a.table + static_cast<size_t>(k) * kPlaceRowWords, a.words, lane);
      if (lane == 0) atomicAdd(&hist[d], 1);
    }
  }
  __syncthreads();

  // the cut
  if (warp == 0) {
    int total = 0;
    for (int b = 0; b <= a.num_ferns; b += 32) total += __reduce_add_sync(0xffffffffu, b + lane <= a.num_ferns ? hist[b + lane] : 0);
    const int m = min(a.max_matches, total);
    int c = a.num_ferns + 1, below = 0, running = 0;
    for (int b = 0; m > 0 && b <= a.num_ferns; b += 32) {
      const int v = b + lane <= a.num_ferns ? hist[b + lane] : 0;
      int inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      const unsigned reached = __ballot_sync(0xffffffffu, running + inc >= m);
      if (reached) {
        const int l = __ffs(reached) - 1;
        c = b + l;
        below = running + __shfl_sync(0xffffffffu, inc - v, l);
        break;
      }
      running += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) {
      cut = c;
      need = m - below;
      take = m;
    }
  }
  __syncthreads();

  // pass 2: the selection
  for (int block = q.first; take > 0 && block <= q.last; block += kThreads) {
    const int base = block + 32 * warp;
    int mine = -1;   // lane j: D of keyframe base + j, or -1 when it is not a candidate
    for (int j = 0; j < 32; ++j) {
      const int k = base + j;
      if (!Candidate(a, q, k)) continue;
      const int d = Difference(query, a.table + static_cast<size_t>(k) * kPlaceRowWords, a.words, lane);
      if (lane == j) mine = d;
    }
    const bool tie = mine >= 0 && mine == cut;
    const unsigned ties = __ballot_sync(0xffffffffu, tie);
    if (lane == 0) warp_ties[warp] = __popc(ties);
    __syncthreads();
    int rank = ties_before + __popc(ties & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) rank += warp_ties[w];
    if ((mine >= 0 && mine < cut) || (tie && rank < need)) {
      const int slot = atomicAdd(&sel_n, 1);
      sel_id[slot] = base + lane;
      sel_d[slot] = mine;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 0; w < kWarps; ++w) ties_before += warp_ties[w];
      if (sel_n == take) take = 0;   // all found: stop
    }
    __syncthreads();
  }

  // the order (D, id)
  int* out = a.matches + static_cast<size_t>(blockIdx.x) * (2 * a.max_matches + 1);
  const int n = sel_n;
  for (int t = threadIdx.x; t < a.max_matches; t += kThreads) {
    if (t < n) {
      int rank = 0;
      for (int j = 0; j < n; ++j) rank += sel_d[j] < sel_d[t] || (sel_d[j] == sel_d[t] && sel_id[j] < sel_id[t]);
      out[rank] = sel_id[t];
      out[a.max_matches + rank] = sel_d[t];
    } else {
      out[t] = -1;
      out[a.max_matches + t] = -1;
    }
  }
  if (threadIdx.x == 0) out[2 * a.max_matches] = n;
}

LaunchResult LaunchPlaceMatch(const MatchArgs& a, int queries, cudaStream_t s) {
  LaunchResult r;
  PlaceMatchKernel<<<queries, kThreads, 0, s>>>(a);
  r.kernels = 1;
  return r;
}

// The options resolved (defaults for values <= 0) and checked; *out receives the fern count and the raw depth range.
bba_status ResolveOptions(bba_handle h, const char* fn, const bba_place_index_options& o, PlaceIndexState* out) {
  const std::string name(fn);
  const int F = o.num_ferns > 0 ? o.num_ferns : kDefaultFerns;
  if (F % 8 != 0 || F < 8 || F > kMaxFerns) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": num_ferns must be a multiple of 8 in [8, 2048]");
  if (!std::isfinite(o.min_depth) || !std::isfinite(o.max_depth)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": non-finite depth range");
  const double min_m = o.min_depth > 0.f ? o.min_depth : kDefaultMinDepth;
  const double max_m = o.max_depth > 0.f ? o.max_depth : kDefaultMaxDepth;
  const double scale = static_cast<double>(h->cfg.raw_to_float_depth);
  const long long min_raw = std::llround(min_m / scale), max_raw = std::llround(max_m / scale);
  if (!(min_raw > 0 && min_raw <= max_raw && max_raw <= 0x7fff))
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": the depth range must give 0 < min_raw <= max_raw <= 0x7fff in raw units");
  out->num_ferns = F;
  out->min_raw = static_cast<int>(min_raw);
  out->max_raw = static_cast<int>(max_raw);
  return BBA_OK;
}

// The image sizes the encoding supports: at least one pixel per cell, and cells small enough for exact u32 sums.
bba_status CheckImageSizes(bba_handle h, const char* fn) {
  const auto cell_pixels = [](int w, int hh) {
    return static_cast<int64_t>((w + kGridW - 1) / kGridW) * ((hh + kGridH - 1) / kGridH);
  };
  const bba_config& c = h->cfg;
  if (c.depth_width < kGridW || c.depth_height < kGridH || c.color_width < kGridW || c.color_height < kGridH)
    return Fail(h, BBA_ERR_UNSUPPORTED, std::string(fn) + ": the place index needs depth and colour images of at least 80 x 60");
  if (cell_pixels(c.depth_width, c.depth_height) > kMaxCellPixels || cell_pixels(c.color_width, c.color_height) > kMaxCellPixels)
    return Fail(h, BBA_ERR_UNSUPPORTED, std::string(fn) + ": images too large for the place index's cells");
  return BBA_OK;
}

EncodeArgs MakeEncodeArgs(bba_handle h, const PlaceImage* images, const PlaceIndexState& st) {
  EncodeArgs a{};
  a.images = images;
  a.dw = h->cfg.depth_width;
  a.dh = h->cfg.depth_height;
  a.cw = h->cfg.color_width;
  a.ch = h->cfg.color_height;
  a.num_ferns = st.num_ferns;
  a.min_raw = st.min_raw;
  a.max_raw = st.max_raw;
  return a;
}

bba_status IndexKeyframes(bba_handle h, const bba_place_index_options* o, int count, const int* ids, cudaStream_t s) {
  const char* fn = "bba_index_keyframes";
  const std::string name(fn);
  if (!ids) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": null keyframe_ids");
  if (count < 1) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": count must be at least 1");
  if (bba_status st = CheckImageSizes(h, fn)) return st;
  auto& P = h->place;
  PlaceIndexState opts = P.state;
  if (o || P.state.num_ferns == 0) {
    const bba_place_index_options defaults{0, 0.f, 0.f};
    if (bba_status st = ResolveOptions(h, fn, o ? *o : defaults, &opts)) return st;
  }
  const int K = static_cast<int>(h->keyframes.size());
  for (int i = 0; i < count; ++i)
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": no such keyframe " + std::to_string(ids[i]));

  const int max_kf = h->cfg.max_keyframes;
  if (P.state.num_ferns == 0) {   // the first index: the live table and both slots
    BBA_CUDA(h, P.codes.Reserve(static_cast<size_t>(max_kf) * kPlaceRowWords));
    for (auto& slot : h->fe.place_codes) BBA_CUDA(h, slot.Reserve(static_cast<size_t>(max_kf) * kPlaceRowWords));
  }
  BBA_CUDA(h, P.h_images.Reserve(count));
  BBA_CUDA(h, P.d_images.Reserve(count));
  if (bba_status st = WaitStaging(h)) return st;   // (the pinned records of the previous call were uploaded)
  for (int i = 0; i < count; ++i) {
    const Keyframe& kf = h->keyframes[ids[i]];
    PlaceImage& im = P.h_images[i];
    im.depth = kf.depth;
    im.depth_pitch = static_cast<uint32_t>(kf.depth_pitch);
    im.rgba = kf.rgba;
    im.rgba_pitch = static_cast<uint32_t>(kf.rgba_pitch);
    im.code = P.codes + static_cast<size_t>(ids[i]) * kPlaceRowWords;
  }
  BBA_CUDA(h, cudaMemcpyAsync(P.d_images, P.h_images, sizeof(PlaceImage) * count, cudaMemcpyHostToDevice, s));
  if (bba_status st = MarkStaging(h, s)) return st;
  if (opts.num_ferns != P.state.num_ferns || opts.min_raw != P.state.min_raw || opts.max_raw != P.state.max_raw) {
    P.state.num_ferns = opts.num_ferns;   // new options: every keyframe loses its code
    P.state.min_raw = opts.min_raw;
    P.state.max_raw = opts.max_raw;
    P.state.indexed.assign(max_kf, 0);
  }
  BBA_LAUNCH(h, h->launches, LaunchPlaceEncode, MakeEncodeArgs(h, P.d_images, P.state), count, s);
  for (int i = 0; i < count; ++i) P.state.indexed[ids[i]] = 1;
  return Publish(h, s, true);
}

// A frame's images as the encoder reads them: u16 depth and uchar4 colour loads need 2- and 4-byte aligned rows.
bool FrameImageOk(bba_handle h, const bba_frame_buffers& f) {
  return f.depth && f.color_rgba && f.depth_pitch >= static_cast<size_t>(h->cfg.depth_width) * 2 &&
         f.color_pitch >= static_cast<size_t>(h->cfg.color_width) * 4 && f.depth_pitch <= 0xffffffffull && f.color_pitch <= 0xffffffffull &&
         !(f.depth_pitch & 1u) && !(reinterpret_cast<uintptr_t>(f.depth) & 1u) && !(f.color_pitch & 3u) &&
         !(reinterpret_cast<uintptr_t>(f.color_rgba) & 3u);
}

bba_status QueryPlaceIndex(bba_handle h, int frame_count, const bba_frame_buffers* frames, int count, const bba_place_query* queries,
                           int max_matches, int* match_ids, int* match_differences, int* match_counts, cudaStream_t s) {
  const char* fn = "bba_query_place_index";
  const std::string name(fn);
  if (!queries || !match_ids || !match_differences || !match_counts) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": null argument");
  if (count < 1) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": count must be at least 1");
  if (frame_count < 0 || (frame_count > 0 && !frames)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": bad frames");
  if (max_matches < 1 || max_matches > kMaxMatches) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": max_matches must be in 1..64");
  if (bba_status st = CheckImageSizes(h, fn)) return st;
  int max_id = -1;
  std::vector<int> frame_row(frame_count, -1);   // frame -> row of the frame codes, in first-use order
  std::vector<int> used_frames;
  for (int i = 0; i < count; ++i) {
    const bba_place_query& q = queries[i];
    const std::string which = " in query " + std::to_string(i);
    if (q.keyframe_id >= 0) {
      max_id = std::max(max_id, q.keyframe_id);
    } else if (q.keyframe_id == -1) {
      if (q.frame < 0 || q.frame >= frame_count) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": frame index out of range" + which);
      if (!FrameImageOk(h, frames[q.frame]))
        return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": null, misaligned or too narrow frame image" + which);
      if (frame_row[q.frame] < 0) {
        frame_row[q.frame] = static_cast<int>(used_frames.size());
        used_frames.push_back(q.frame);
      }
    } else {
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": keyframe_id must be >= -1" + which);
    }
  }

  std::lock_guard<std::mutex> call(h->fe.call);
  FrontEndCall view(h);
  PlaceIndexState st;
  std::vector<int> query_kfs;
  for (int i = 0; i < count; ++i)
    if (queries[i].keyframe_id >= 0) query_kfs.push_back(queries[i].keyframe_id);
  if (bba_status e = view.Snapshot(s, -1, fn, max_id, nullptr, &st, &query_kfs)) return e;   // (refuses before claiming)
  const int K = view.keyframe_count;
  const int n_frames = static_cast<int>(used_frames.size());
  const int stride = 2 * max_matches + 1;

  auto& Q = h->fe.place_query;
  BBA_CUDA(h, Q.h_queries.Reserve(count));
  BBA_CUDA(h, Q.d_queries.Reserve(count));
  BBA_CUDA(h, Q.h_indexed.Reserve(std::max(K, 1)));
  BBA_CUDA(h, Q.d_indexed.Reserve(std::max(K, 1)));
  BBA_CUDA(h, Q.d_matches.Reserve(static_cast<size_t>(count) * stride));
  BBA_CUDA(h, Q.h_matches.Reserve(static_cast<size_t>(count) * stride));
  if (n_frames > 0) {
    BBA_CUDA(h, Q.h_images.Reserve(n_frames));
    BBA_CUDA(h, Q.d_images.Reserve(n_frames));
    BBA_CUDA(h, Q.d_frame_codes.Reserve(static_cast<size_t>(n_frames) * kPlaceRowWords));
  }
  for (int i = 0; i < count; ++i) {
    const bba_place_query& q = queries[i];
    PlaceQueryRecord& r = Q.h_queries[i];
    r.code = q.keyframe_id >= 0 ? view.place_codes + static_cast<size_t>(q.keyframe_id) * kPlaceRowWords
                                : Q.d_frame_codes + static_cast<size_t>(frame_row[q.frame]) * kPlaceRowWords;
    r.first = std::min(std::max(q.first_keyframe, 0), K);   // within [0, K], so that the kernel's id arithmetic cannot overflow
    r.last = std::max(std::min(q.last_keyframe, K - 1), -1);
    r.exclude = q.keyframe_id;
    r.pad = 0;
  }
  std::copy(st.indexed.begin(), st.indexed.begin() + K, Q.h_indexed.get());
  for (int i = 0; i < n_frames; ++i) {
    const bba_frame_buffers& f = frames[used_frames[i]];
    PlaceImage& im = Q.h_images[i];
    im.depth = f.depth;
    im.depth_pitch = static_cast<uint32_t>(f.depth_pitch);
    im.rgba = f.color_rgba;
    im.rgba_pitch = static_cast<uint32_t>(f.color_pitch);
    im.code = Q.d_frame_codes + static_cast<size_t>(i) * kPlaceRowWords;
  }
  BBA_CUDA(h, cudaMemcpyAsync(Q.d_queries, Q.h_queries, sizeof(PlaceQueryRecord) * count, cudaMemcpyHostToDevice, s));
  if (K > 0) BBA_CUDA(h, cudaMemcpyAsync(Q.d_indexed, Q.h_indexed, K, cudaMemcpyHostToDevice, s));
  if (n_frames > 0) {
    BBA_CUDA(h, cudaMemcpyAsync(Q.d_images, Q.h_images, sizeof(PlaceImage) * n_frames, cudaMemcpyHostToDevice, s));
    BBA_LAUNCH(h, h->front_end_launches, LaunchPlaceEncode, MakeEncodeArgs(h, Q.d_images, st), n_frames, s);
  }
  MatchArgs a{};
  a.queries = Q.d_queries;
  a.table = view.place_codes;
  a.indexed = Q.d_indexed;
  a.words = st.num_ferns / 8;
  a.num_ferns = st.num_ferns;
  a.max_matches = max_matches;
  a.matches = Q.d_matches;
  BBA_LAUNCH(h, h->front_end_launches, LaunchPlaceMatch, a, count, s);
  if (bba_status e = view.ReleaseSlot()) return e;   // (the match kernel was the last reader of the slot)
  BBA_CUDA(h, cudaMemcpyAsync(Q.h_matches, Q.d_matches, sizeof(int) * count * stride, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  for (int i = 0; i < count; ++i) {
    const int* m = Q.h_matches + static_cast<size_t>(i) * stride;
    std::memcpy(match_ids + static_cast<size_t>(i) * max_matches, m, sizeof(int) * max_matches);
    std::memcpy(match_differences + static_cast<size_t>(i) * max_matches, m + max_matches, sizeof(int) * max_matches);
    match_counts[i] = m[2 * max_matches];
  }
  return BBA_OK;
}

bba_status GetPlaceIndexCodes(bba_handle h, int count, const int* ids, int words_per_code, uint32_t* out, cudaStream_t s) {
  const char* fn = "bba_get_place_index_codes";
  const std::string name(fn);
  if (!ids || !out) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": null argument");
  if (count < 1) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": count must be at least 1");
  int max_id = -1;
  for (int i = 0; i < count; ++i) {
    if (ids[i] < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": no such keyframe");
    max_id = std::max(max_id, ids[i]);
  }
  std::lock_guard<std::mutex> call(h->fe.call);
  FrontEndCall view(h);
  PlaceIndexState st;
  const auto words_ok = [&](int num_ferns) { return num_ferns == 0 || words_per_code == num_ferns / 8; };
  {
    std::lock_guard<std::mutex> lock(h->fe.mu);
    if (!words_ok(h->fe.place.num_ferns)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": words_per_code is not num_ferns / 8");
  }
  const std::vector<int> id_list(ids, ids + count);
  if (bba_status e = view.Snapshot(s, -1, fn, max_id, nullptr, &st, &id_list)) return e;   // (refuses before claiming)
  if (!words_ok(st.num_ferns))   // (the options changed since the check above)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": words_per_code is not num_ferns / 8");
  const size_t words = st.num_ferns / 8;
  for (int i = 0; i < count; ++i)
    BBA_CUDA(h, cudaMemcpyAsync(out + i * words, view.place_codes + static_cast<size_t>(ids[i]) * kPlaceRowWords, sizeof(uint32_t) * words,
                                cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  return view.ReleaseSlot(/*record=*/false);   // (the reads are complete)
}

}  // namespace
}  // namespace bba

using namespace bba;

extern "C" {

bba_status bba_index_keyframes(bba_handle h, const bba_place_index_options* options, int count, const int* keyframe_ids, void* stream) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  return IndexKeyframes(h, options, count, keyframe_ids, static_cast<cudaStream_t>(stream));
}

bba_status bba_query_place_index(bba_handle h, int frame_count, const bba_frame_buffers* frames, int count, const bba_place_query* queries,
                                 int max_matches, int* match_ids, int* match_differences, int* match_counts, void* stream) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  return QueryPlaceIndex(h, frame_count, frames, count, queries, max_matches, match_ids, match_differences, match_counts,
                         static_cast<cudaStream_t>(stream));
}

bba_status bba_get_place_index_codes(bba_handle h, int count, const int* keyframe_ids, int words_per_code, uint32_t* out, void* stream) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  return GetPlaceIndexCodes(h, count, keyframe_ids, words_per_code, out, static_cast<cudaStream_t>(stream));
}

bba_status bba_get_place_index_options(bba_handle h, int* num_ferns, int* min_raw, int* max_raw) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  PlaceIndexState st;
  {
    std::lock_guard<std::mutex> lock(h->fe.mu);
    st.num_ferns = h->fe.place.num_ferns;
    st.min_raw = h->fe.place.min_raw;
    st.max_raw = h->fe.place.max_raw;
  }
  if (num_ferns) *num_ferns = st.num_ferns;
  if (min_raw) *min_raw = st.min_raw;
  if (max_raw) *max_raw = st.max_raw;
  return BBA_OK;
}

int bba_host_place_ferns(int num_ferns, int min_raw, int max_raw, int32_t* cells, int32_t* thresholds) {
  if (num_ferns % 8 != 0 || num_ferns < 8 || num_ferns > kMaxFerns || !(min_raw > 0 && min_raw <= max_raw && max_raw <= 0x7fff) ||
      !cells || !thresholds)
    return BBA_ERR_INVALID_ARGUMENT;
  for (int f = 0; f < num_ferns; ++f) {
    const Fern r = MakeFern(f, min_raw, max_raw);
    cells[2 * f] = r.cx;
    cells[2 * f + 1] = r.cy;
    for (int c = 0; c < 4; ++c) thresholds[4 * f + c] = r.t[c];
  }
  return BBA_OK;
}

}  // extern "C"
