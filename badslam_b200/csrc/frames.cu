// frames.cu -- the frame side of libbadba_b200 (host side): image-pair odometry (buffers, pyramids, the persistent tracking
// kernel's launch and its entry points) and keyframe preprocessing (bba_preprocess_frame, bba_preprocess_raw_frame).  These are
// the front-end calls of include/badba.h: they read the published view of the handle (FrontEndCall), never its live state.
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <utility>

#include "handle.hpp"
#include "preprocess_tile.cuh"

namespace bba {
namespace {

// ---- image-pair odometry (bba_track_frame_pairwise) --------------------------------------------------------------------
// A u8 plane in pitched device memory as a texture with the sampler state of CUDABuffer::CreateTextureObject as the reference
// calls it for the pyramid colour planes (pairwise_frame_tracking.cc:57-79).
bba_status MakePitchedU8Texture(bba_handle h, const PitchedBuffer& plane, int w, int ht, Texture* out) {
  cudaResourceDesc res;
  std::memset(&res, 0, sizeof(res));
  res.resType = cudaResourceTypePitch2D;
  res.res.pitch2D.devPtr = plane.get();
  res.res.pitch2D.desc = cudaCreateChannelDesc(8, 0, 0, 0, cudaChannelFormatKindUnsigned);
  res.res.pitch2D.width = w;
  res.res.pitch2D.height = ht;
  res.res.pitch2D.pitchInBytes = plane.pitch();
  const cudaTextureDesc tex = LinearTextureDesc();
  BBA_CUDA(h, cudaCreateTextureObject(&out->tex.r, &res, &tex, nullptr));
  return BBA_OK;
}

// The level sizes of an odometry pyramid (pairwise_frame_tracking.cc:51-53: int scale_width = depth_width / pow(2, scale)), or
// false when a level would be empty.
bool OdometryLevelSizes(bba_handle h, int num_scales, int* w, int* ht) {
  for (int s = 0; s < num_scales; ++s) {
    w[s] = static_cast<int>(h->cfg.depth_width / std::pow(2, s));
    ht[s] = static_cast<int>(h->cfg.depth_height / std::pow(2, s));
    if (w[s] < 1 || ht[s] < 1) return false;
  }
  return true;
}

// PairwiseFrameTrackingBuffers + CreatePairwiseTrackingInputBuffersAndTextures (pairwise_frame_tracking.cc:39-151), once per
// pyramid of the pool: at least `images` pyramids of at least num_scales levels.  More levels than allocated free the pool first.
// (CheckOdometryCall has checked that every level of num_scales is non-empty.)
bba_status EnsureOdometry(bba_handle h, int num_scales, int images) {
  auto& o = h->odo;
  if (o.num_scales < num_scales) {
    o.pool.clear();
    o.num_scales = num_scales;
    OdometryLevelSizes(h, num_scales, o.w, o.h);
  }
  const int cw = h->cfg.color_width, ch = h->cfg.color_height;
  while (static_cast<int>(o.pool.size()) < images) {
    auto p = std::make_unique<bba_context::Pyramid>();
    BBA_CUDA(h, p->gradmag.Allocate(cw, ch));
    if (bba_status st = MakePitchedU8Texture(h, p->gradmag, cw, ch, &p->gradmag_tex)) return st;
    for (int s = 0; s < o.num_scales; ++s) {
      bba::odom::Image& im = p->image[s];
      BBA_CUDA(h, p->depth[s].Allocate(sizeof(float) * o.w[s], o.h[s]));
      im.depth = p->depth[s].get<float>();
      im.depth_pitch = static_cast<uint32_t>(p->depth[s].pitch() / sizeof(float));
      if (s >= 1) {   // level 0 uses the caller's normal images
        BBA_CUDA(h, p->normals[s].Allocate(sizeof(uint16_t) * o.w[s], o.h[s]));
        im.normals = p->normals[s].get<uint16_t>();
        im.normals_pitch = static_cast<uint32_t>(p->normals[s].pitch());
      }
      BBA_CUDA(h, p->color[s].Allocate(o.w[s], o.h[s]));
      im.color = p->color[s].get();
      im.color_pitch = static_cast<uint32_t>(p->color[s].pitch());
      if (bba_status st = MakePitchedU8Texture(h, p->color[s], o.w[s], o.h[s], &p->color_tex[s])) return st;
      im.color_tex = p->color_tex[s].tex;
    }
    o.pool.push_back(std::move(p));
  }
  BBA_CUDA(h, o.h_images.Reserve(images));
  BBA_CUDA(h, o.d_images.Reserve(images));
  return BBA_OK;
}

// The camera model of one pyramid level: PinholeCamera4f::Scaled (libvis camera.h:1696-1705, 1086-1097: all four parameters
// times the factor, width = factor * width + 0.5) through the builders of surfel_projection.h:42-124.
bba::odom::LevelCamera MakeLevelCamera(bba_handle h, const CameraView& v, int scale, int level_w, int level_h) {
  bba::odom::LevelCamera c;
  const float scaling_factor = static_cast<float>(std::pow(2, scale));
  const float df = static_cast<float>(1.f / scaling_factor);   // depth_camera.Scaled(1.f / scaling_factor)
  const float cf = static_cast<float>((h->cfg.depth_width == h->cfg.color_width) ? (1.f / scaling_factor) : (2.f / scaling_factor));
  const float dK[4] = {v.depth_K[0] * df, v.depth_K[1] * df, v.depth_K[2] * df, v.depth_K[3] * df};
  const float cK[4] = {v.color_K[0] * cf, v.color_K[1] * cf, v.color_K[2] * cf, v.color_K[3] * cf};
  c.w = level_w; c.h = level_h;
  c.fx = dK[0]; c.fy = dK[1]; c.cx = dK[2]; c.cy = dK[3];
  c.fx_inv = 1.0f / dK[0];
  c.fy_inv = 1.0f / dK[1];
  c.cx_inv = -(dK[2] - 0.5f) * c.fx_inv;
  c.cy_inv = -(dK[3] - 0.5f) * c.fy_inv;
  c.d2c_fx = cK[0] / dK[0];
  c.d2c_cx = -1 * cK[0] * dK[2] / dK[0] + cK[2];
  c.d2c_fy = cK[1] / dK[1];
  c.d2c_cy = -1 * cK[1] * dK[3] / dK[1] + cK[3];
  c.cw = static_cast<int>(static_cast<double>(cf) * h->cfg.color_width + 0.5f);
  c.ch = static_cast<int>(static_cast<double>(cf) * h->cfg.color_height + 0.5f);
  c.cfx = cK[0]; c.cfy = cK[1];
  return c;
}

// One image of a chunk: its preprocessed depth and normals and its luma texture.
struct ChunkImage {
  const uint16_t* depth;
  size_t depth_pitch;
  const uint16_t* normals;
  size_t normals_pitch;
  cudaTextureObject_t luma;
};

// Fills the pyramids of a chunk's images (stages 1-3 of odometry.cuh: one launch per stage and level for all of them) for the
// given options, with the cameras and the cfactor of the call's snapshot, and uploads the image table the tracking kernel reads.
// images[0, n_base) are base images, the rest tracked ones.
bba_status BuildOdometryPyramids(bba_handle h, const bba_odometry_options& o, const FrontEndCall& view, const std::vector<ChunkImage>& images,
                                 int n_base, cudaStream_t s) {
  namespace od = bba::odom;
  auto& st = h->odo;
  const int S = o.num_scales, n = static_cast<int>(images.size());
  if (bba_status e = EnsureOdometry(h, S, n)) return e;
  for (int i = 0; i < n; ++i) {
    const ChunkImage& src = images[i];
    const bba_context::Pyramid& p = *st.pool[i];
    od::PyramidImage& im = st.h_images[i];
    im.luma_tex = src.luma;
    im.gradmag = p.gradmag.get();
    im.gradmag_pitch = static_cast<uint32_t>(p.gradmag.pitch());
    im.gradmag_tex = p.gradmag_tex.tex;
    im.raw_depth = src.depth; im.raw_depth_pitch = static_cast<uint32_t>(src.depth_pitch);
    im.raw_normals = src.normals; im.raw_normals_pitch = static_cast<uint32_t>(src.normals_pitch);
    im.tracked = i >= n_base ? 1 : 0;
    for (int l = 0; l < od::kMaxScales; ++l) im.level[l] = l < S ? p.image[l] : od::Image{};
    // level 0 normals are the image's own buffer
    im.level[0].normals = const_cast<uint16_t*>(src.normals); im.level[0].normals_pitch = static_cast<uint32_t>(src.normals_pitch);
  }
  BBA_CUDA(h, cudaMemcpyAsync(st.d_images, st.h_images, sizeof(od::PyramidImage) * n, cudaMemcpyHostToDevice, s));

  od::BrightnessArgs br{};
  br.images = st.d_images;
  br.count = n;
  br.w = h->cfg.color_width; br.h = h->cfg.color_height;
  br.use_gradmag = o.use_gradmag;
  BBA_LAUNCH(h, h->front_end_launches, od::LaunchBrightness, br, s);

  const bba::CameraParams cam = MakeCamera(h, view.cams, view.cfactor);
  od::Level0Args l0{};
  l0.images = st.d_images;
  l0.count = n;
  l0.skip_level0 = o.use_pyramid_level_0 ? 0 : 1;
  l0.w = st.w[0]; l0.h = st.h[0];
  l0.out_w = l0.skip_level0 ? st.w[1] : st.w[0];
  l0.out_h = l0.skip_level0 ? st.h[1] : st.h[0];
  l0.d2c_fx = cam.d2c_fx; l0.d2c_fy = cam.d2c_fy; l0.d2c_cx = cam.d2c_cx; l0.d2c_cy = cam.d2c_cy;
  l0.cw = cam.cw; l0.ch = cam.ch;
  l0.a = cam.a; l0.raw_to_float = cam.raw_to_float; l0.cfactor = cam.cfactor; l0.cf_w = cam.cf_w; l0.cell = cam.cell;
  l0.downsample_color = h->cfg.depth_width == h->cfg.color_width;
  BBA_LAUNCH(h, h->front_end_launches, od::LaunchLevel0, l0, s);

  for (int l = 1; l < S; ++l) {
    // pairwise_frame_tracking.cc:325-347: the tracked images from level 2 on (level 1 too when level 0 is in use), the bases always
    od::DownsampleArgs d{};
    d.images = st.d_images;
    d.count = (l >= 2 || o.use_pyramid_level_0) ? n : n_base;
    d.level = l;
    d.w = st.w[l]; d.h = st.h[l];
    d.in_w = st.w[l - 1]; d.in_h = st.h[l - 1];
    BBA_LAUNCH(h, h->front_end_launches, od::LaunchDownsample, d, s);
  }
  for (int l = 0; l < S; ++l) st.cam[l] = MakeLevelCamera(h, view.cams, l, st.w[l], st.h[l]);
  st.last_num_scales = S;
  st.last_first_scale = o.use_pyramid_level_0 ? 0 : 1;
  return BBA_OK;
}

// Runs the tracking kernel over `entries` (indices into the image table of the last BuildOdometryPyramids) and copies their
// results to h->odo.h_result; debug_scale >= 0 runs the parity hook on entries[0].  Synchronises s.
bba_status LaunchOdometryKernel(bba_handle h, const CameraView& cams, int num_scales, int first_scale, int max_iterations, int use_gradmag,
                                int test_different, int debug_scale, const std::vector<bba::odom::TrackEntry>& entries, cudaStream_t s) {
  namespace od = bba::odom;
  auto& st = h->odo;
  const int count = static_cast<int>(entries.size());
  od::TrackArgs a{};
  for (int l = 0; l < num_scales; ++l) a.cam[l] = st.cam[l];
  a.images = st.d_images;
  a.count = count;
  a.virtual_grid = od::TrackGrid(st.cam[first_scale], h->sm_count);
  a.group_size = od::TrackGroupSize(count, a.virtual_grid, h->sm_count);
  const int groups = od::TrackGroups(count, a.group_size, h->sm_count);
  a.num_scales = num_scales;
  a.first_scale = first_scale;
  a.max_iterations = max_iterations;
  a.use_depth = cams.use_depth;
  a.use_desc = cams.use_desc;
  a.use_gradmag = use_gradmag;
  a.test_different_initial_estimates = test_different;
  a.debug_scale = debug_scale;
  a.baseline_fx = h->cfg.baseline_fx;
  BBA_CUDA(h, st.h_entries.Reserve(count));
  BBA_CUDA(h, st.d_entries.Reserve(count));
  BBA_CUDA(h, st.d_acc.Reserve(static_cast<size_t>(groups) * 3 * 32));
  BBA_CUDA(h, st.d_control.Reserve(od::TrackControlWords(groups)));
  BBA_CUDA(h, st.d_result.Reserve(count));
  BBA_CUDA(h, st.h_result.Reserve(count));
  a.partials = nullptr;
  if (cams.deterministic) {   // the snapshot's mode: fixed-order sums of per-virtual-CTA partials
    BBA_CUDA(h, st.d_partials.Reserve(static_cast<size_t>(groups) * 3 * 32 * a.virtual_grid));
    a.partials = st.d_partials;
  }
  std::copy(entries.begin(), entries.end(), st.h_entries.get());
  a.entries = st.d_entries;
  a.acc = st.d_acc;
  a.control = st.d_control;
  a.result = st.d_result;
  BBA_CUDA(h, cudaMemcpyAsync(st.d_entries, st.h_entries, sizeof(od::TrackEntry) * count, cudaMemcpyHostToDevice, s));
  BBA_CUDA(h, cudaMemsetAsync(st.d_acc, 0, sizeof(double) * 3 * 32 * groups, s));
  BBA_CUDA(h, cudaMemsetAsync(st.d_control, 0, sizeof(unsigned int) * od::TrackControlWords(groups), s));
  BBA_CUDA(h, cudaMemsetAsync(st.d_result, 0, sizeof(od::TrackResult) * count, s));
  BBA_LAUNCH(h, h->front_end_launches, od::LaunchTrack, a, groups, s);
  BBA_CUDA(h, cudaMemcpyAsync(st.h_result, st.d_result, sizeof(od::TrackResult) * count, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  for (int i = 0; i < count; ++i)
    if (st.h_result[i].barrier_timeout) return Fail(h, BBA_ERR_CUDA, "odometry kernel: group barrier timed out");
  // the parity hooks work on the last entry's pyramids
  const od::TrackEntry& last = entries.back();
  st.last_entry = last;
  for (int l = 0; l < num_scales; ++l) {
    st.last_level[0][l] = st.h_images[last.base].level[l];
    st.last_level[1][l] = st.h_images[last.tracked].level[l];
  }
  return BBA_OK;
}

}  // namespace

// The option checks of every odometry call (fn prefixes the messages): num_scales, the depth / colour pyramid combination and the
// level sizes.
bba_status CheckOdometryOptions(bba_handle h, const char* fn, const bba_odometry_options& o) {
  const std::string name(fn);
  if (o.num_scales < 1 || o.num_scales > bba::odom::kMaxScales || (!o.use_pyramid_level_0 && o.num_scales < 2))
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": num_scales must be 1..8 (>= 2 without pyramid level 0)");
  // pairwise_frame_tracking.cc:300-306 (LOG(FATAL) in the reference)
  if (!o.use_pyramid_level_0 && h->cfg.depth_width != h->cfg.color_width && h->cfg.depth_width != 2 * h->cfg.color_width)
    return Fail(h, BBA_ERR_UNSUPPORTED, "The chosen depth / color pyramid level combination is not supported here.");
  int w[bba::odom::kMaxScales], ht[bba::odom::kMaxScales];
  if (!OdometryLevelSizes(h, o.num_scales, w, ht))
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": too many pyramid levels for this image size");
  return BBA_OK;
}

namespace {

// The argument checks of every odometry call (h is not null; fn prefixes the messages): the arrays, the frame buffers, the
// entries' frame indices, the options, the depth / colour pyramid combination and the level sizes.  The keyframe ids are checked
// against the published keyframes in the snapshot, so that a failed check enqueues nothing.
bba_status CheckOdometryCall(bba_handle h, const char* fn, const bba_odometry_options* o, int frame_count, const bba_frame_buffers* frames,
                             int count, const bba_odometry_entry* entries, const float* out) {
  const std::string name(fn);
  if (!o || !frames || !entries || !out) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": null argument");
  if (count < 1 || frame_count < 1) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": count and frame_count must be at least 1");
  for (int f = 0; f < frame_count; ++f) {
    const bba_frame_buffers& b = frames[f];
    if (!b.depth || !b.normals || !b.color_rgba) return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": null frame buffer");
    if (!FramePitchesOk(h, b.depth_pitch, b.normals_pitch, b.color_pitch) || ((b.depth_pitch | b.normals_pitch) & 1u))
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": bad frame buffer pitch");
  }
  for (int i = 0; i < count; ++i) {
    const bba_odometry_entry& e = entries[i];
    if (e.tracked_frame < 0 || e.tracked_frame >= frame_count || e.base_keyframe_id < -1 ||
        (e.base_keyframe_id < 0 && (e.base_frame < 0 || e.base_frame >= frame_count)))
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": frame index out of range in entry " + std::to_string(i));
  }
  return CheckOdometryOptions(h, fn, *o);
}

void CopyOdometryResult(const bba::odom::TrackResult& r, int num_scales, uint32_t launches, bba_odometry_result* result) {
  for (int i = 0; i < 8; ++i) {
    result->iterations[i] = r.iterations[i];
    result->chose_initial[i] = i < num_scales ? r.chose_initial[i] : -1;
  }
  result->residual_count = r.residual_count;
  result->residual_sum = r.residual_sum;
  result->passes = r.passes;
  result->kernel_launches = launches;
}

// Stage 0 of bba_preprocess_raw_frame (validated by the caller), or nullptr for bba_preprocess_frame.
struct RawStage {
  int median_iterations, depth_level, raw_w, raw_h, color_level;
};

// bba_preprocess_frame and bba_preprocess_raw_frame after their own checks; `fn` prefixes the error messages.
bba_status PreprocessFrame(bba_handle h, const char* fn, const bba_preprocess_options* o,
                           const uint16_t* device_raw_depth, size_t raw_depth_pitch,
                           const uint8_t* device_rgb, size_t rgb_pitch,
                           uint16_t* device_depth, size_t depth_pitch,
                           uint16_t* device_normals, size_t normals_pitch,
                           uint16_t* device_radius, size_t radius_pitch,
                           uint8_t* device_color_rgba, size_t color_pitch,
                           float* min_depth, float* max_depth, void* stream, const RawStage* raw_stage) {
  const std::string name(fn);
  if (!h || !o || !device_raw_depth || !device_depth || !device_normals || !device_radius) return h ? Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": null argument") : BBA_ERR_INVALID_ARGUMENT;
  if ((device_rgb == nullptr) != (device_color_rgba == nullptr))
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": rgb input and rgba output go together");
  if ((raw_depth_pitch | depth_pitch | normals_pitch | radius_pitch) & 1u)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": u16 image pitches must be even");
  if (device_color_rgba && ((color_pitch & 3u) || (reinterpret_cast<uintptr_t>(device_color_rgba) & 3u)))
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": the rgba image must be 4-byte aligned");
  if (device_depth == device_raw_depth)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": in-place filtering is not possible (tiles read their neighbours' raw depth)");
  // BilateralFilteringAndDepthCutoffCUDA (cuda_depth_processing.cu:100-128)
  const int radius = static_cast<int>(o->bilateral_filter_radius_factor * o->bilateral_filter_sigma_xy + 0.5f);
  if (radius < 0 || radius > bba::pre::kMaxFilterRadius)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": bilateral filter radius outside [0, 16]");
  if (!(o->bilateral_filter_sigma_xy > 0.f) || !(o->bilateral_filter_sigma_inv_depth > 0.f) || !(o->max_depth > 0.f))
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, name + ": sigma_xy, sigma_inv_depth and max_depth must be positive");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  std::lock_guard<std::mutex> call(h->fe.call);
  BBA_CUDA(h, h->pre.d_min_max.Reserve(2));
  BBA_CUDA(h, h->pre.h_min_max.Reserve(2));
  FrontEndCall view(h);
  if (bba_status st = view.Snapshot(s, -1, fn)) return st;
  const bba::CameraParams cam = MakeCamera(h, view.cams, view.cfactor);
  bba::pre::FrameArgs f{};
  f.w = cam.w; f.h = cam.h;
  f.fx_inv = cam.fx_inv; f.fy_inv = cam.fy_inv; f.cx_inv = cam.cx_inv; f.cy_inv = cam.cy_inv;
  f.raw_to_float = cam.raw_to_float; f.a = cam.a;
  f.cell = cam.cell; f.cf_w = cam.cf_w; f.cfactor = cam.cfactor;
  f.denom_xy = 2.0f * o->bilateral_filter_sigma_xy * o->bilateral_filter_sigma_xy;
  f.denom_value = 2.0f * o->bilateral_filter_sigma_inv_depth * o->bilateral_filter_sigma_inv_depth;
  f.radius = radius;
  f.radius_squared = radius * radius;
  const float max_raw = o->max_depth / cam.raw_to_float;   // bad_slam.cc:703 (float -> u16 at the call)
  f.max_depth = max_raw >= 65535.f ? static_cast<uint16_t>(65535) : static_cast<uint16_t>(max_raw);
  f.raw_depth = device_raw_depth; f.raw_pitch = static_cast<uint32_t>(raw_depth_pitch);
  f.out_depth = device_depth; f.out_depth_pitch = static_cast<uint32_t>(depth_pitch);
  f.out_normals = device_normals; f.out_normals_pitch = static_cast<uint32_t>(normals_pitch);
  f.out_radius = device_radius; f.out_radius_pitch = static_cast<uint32_t>(radius_pitch);
  f.min_max = h->pre.d_min_max;
  f.cw = cam.cw; f.ch = cam.ch;
  f.rgb = device_rgb; f.rgb_pitch = static_cast<uint32_t>(rgb_pitch);
  f.rgba = device_color_rgba; f.rgba_pitch = static_cast<uint32_t>(color_pitch);
  f.tiles_x = (f.w + bba::pre::kTile - 1) / bba::pre::kTile;
  f.tiles_y = (f.h + bba::pre::kTile - 1) / bba::pre::kTile;
  if (raw_stage) {
    f.median_iterations = raw_stage->median_iterations;
    f.depth_level = raw_stage->depth_level;
    f.raw_w = raw_stage->raw_w; f.raw_h = raw_stage->raw_h;
    f.color_level = raw_stage->color_level;
    BBA_LAUNCH(h, h->front_end_launches, LaunchPreprocessRawFrame, f, s);
  } else {
    BBA_LAUNCH(h, h->front_end_launches, LaunchPreprocessFrame, f, s);
  }
  if (bba_status st = view.ReleaseSlot()) return st;
  if (min_depth || max_depth) {   // ComputeMinMaxDepthCUDA returns host values and synchronises (cuda_depth_processing.cu:452-463)
    BBA_CUDA(h, cudaMemcpyAsync(h->pre.h_min_max, h->pre.d_min_max, 2 * sizeof(float), cudaMemcpyDeviceToHost, s));
    BBA_CUDA(h, cudaStreamSynchronize(s));
    if (min_depth) *min_depth = h->pre.h_min_max[0];
    if (max_depth) *max_depth = h->pre.h_min_max[1];
  }
  return BBA_OK;
}

}  // namespace

bba_status TrackPairsOnSnapshot(bba_handle h, const bba_odometry_options& o, FrontEndCall& view, const std::vector<KeyframeView>& kfs,
                                int frame_count, const bba_frame_buffers* frames, int count, const bba_odometry_entry* entries,
                                const int* tracked_keyframe_ids, bool release_slot, float* out, bba_odometry_result* results,
                                cudaStream_t s) {
  namespace od = bba::odom;
  const int max_it = o.max_iterations_per_scale > 0 ? o.max_iterations_per_scale : 30;
  std::vector<cudaTextureObject_t> luma(frame_count);   // the luma textures of the current chunk's frames
  for (int begin = 0; begin < count; begin += BBA_ODOMETRY_CHUNK_ENTRIES) {
    const int n = std::min(BBA_ODOMETRY_CHUNK_ENTRIES, count - begin);
    const uint64_t chunk_before = h->front_end_launches;
    // the chunk's distinct images: bases (keyframe or frame), then tracked ones (frame or keyframe); and the frames among them,
    // which need luma
    std::map<int, int> base_of_kf, base_of_frame, tracked_of_frame, tracked_of_kf;
    std::vector<int> luma_frames;
    std::vector<od::TrackEntry> track(n);
    std::vector<std::pair<int, int>> base_images;   // (keyframe id, -1) or (-1, frame)
    for (int i = 0; i < n; ++i) {
      const bba_odometry_entry& e = entries[begin + i];
      std::map<int, int>& of = e.base_keyframe_id >= 0 ? base_of_kf : base_of_frame;
      const int key = e.base_keyframe_id >= 0 ? e.base_keyframe_id : e.base_frame;
      auto it = of.emplace(key, static_cast<int>(base_images.size()));
      if (it.second) base_images.emplace_back(e.base_keyframe_id >= 0 ? key : -1, e.base_keyframe_id >= 0 ? -1 : key);
      if (e.base_keyframe_id < 0) luma_frames.push_back(e.base_frame);
      track[i].base = it.first->second;
    }
    const int n_base = static_cast<int>(base_images.size());
    std::vector<std::pair<int, int>> tracked_images;   // (keyframe id, -1) or (-1, frame)
    for (int i = 0; i < n; ++i) {
      const bba_odometry_entry& e = entries[begin + i];
      const int tracked_kf = tracked_keyframe_ids ? tracked_keyframe_ids[begin + i] : -1;
      std::map<int, int>& of = tracked_kf >= 0 ? tracked_of_kf : tracked_of_frame;
      const int key = tracked_kf >= 0 ? tracked_kf : e.tracked_frame;
      auto it = of.emplace(key, n_base + static_cast<int>(tracked_images.size()));
      if (it.second) tracked_images.emplace_back(tracked_kf >= 0 ? key : -1, tracked_kf >= 0 ? -1 : key);
      if (tracked_kf < 0) luma_frames.push_back(e.tracked_frame);
      track[i].tracked = it.first->second;
      std::memcpy(track[i].init1, e.base_T_frame_initial_1, sizeof(float) * 7);
      std::memcpy(track[i].init2, o.test_different_initial_estimates ? e.base_T_frame_initial_2 : e.base_T_frame_initial_1, sizeof(float) * 7);
    }
    if (!luma_frames.empty())   // (a chunk of keyframes only has every luma texture already)
      if (bba_status st = MakeFrameLumaTextures(h, /*front_end=*/true, frames, luma_frames, &h->fe.frames, luma.data(), s)) return st;
    std::vector<ChunkImage> images;
    for (const auto* list : {&base_images, &tracked_images})
      for (const auto& b : *list) {
        if (b.first >= 0) {
          const KeyframeView& k = kfs[b.first];
          images.push_back(ChunkImage{k.depth, k.depth_pitch, k.normals, k.normals_pitch, k.tex});
        } else {
          const bba_frame_buffers& f = frames[b.second];
          images.push_back(ChunkImage{f.depth, f.depth_pitch, f.normals, f.normals_pitch, luma[b.second]});
        }
      }
    if (bba_status st = BuildOdometryPyramids(h, o, view, images, n_base, s)) return st;
    if (release_slot && begin + n >= count)
      if (bba_status st = view.ReleaseSlot()) return st;   // (the last level-0 launch was the last reader of the cfactor)
    if (bba_status st = LaunchOdometryKernel(h, view.cams, o.num_scales, o.use_pyramid_level_0 ? 0 : 1, max_it, o.use_gradmag ? 1 : 0,
                                             o.test_different_initial_estimates ? 1 : 0, -1, track, s))
      return st;
    const uint32_t chunk_launches = static_cast<uint32_t>(h->front_end_launches - chunk_before);
    for (int i = 0; i < n; ++i) {
      const od::TrackResult& r = h->odo.h_result[i];
      std::memcpy(out + 7 * static_cast<size_t>(begin + i), r.base_T_frame, sizeof(float) * 7);
      if (results) CopyOdometryResult(r, o.num_scales, chunk_launches, &results[begin + i]);
    }
  }
  return BBA_OK;
}

namespace {

// The odometry of bba_track_frames_pairwise and of its one-entry forms after CheckOdometryCall: chunks of at most
// BBA_ODOMETRY_CHUNK_ENTRIES entries, each with one luma launch for its distinct frames, one pyramid per distinct (image, role)
// and one tracking launch.
bba_status TrackFramesPairwise(bba_handle h, const char* fn, const bba_odometry_options& o, int frame_count, const bba_frame_buffers* frames,
                               int count, const bba_odometry_entry* entries, float* out, bba_odometry_result* results,
                               uint32_t* kernel_launches, cudaStream_t s) {
  int max_kf = -1;
  for (int i = 0; i < count; ++i) max_kf = std::max(max_kf, entries[i].base_keyframe_id);
  std::lock_guard<std::mutex> call(h->fe.call);
  const uint64_t launches_before = h->front_end_launches;
  FrontEndCall view(h);
  std::vector<KeyframeView> kfs;
  if (bba_status st = view.Snapshot(s, -1, fn, max_kf, &kfs)) return st;
  if (bba_status st = TrackPairsOnSnapshot(h, o, view, kfs, frame_count, frames, count, entries, nullptr, /*release_slot=*/true, out,
                                           results, s))
    return st;
  if (kernel_launches) *kernel_launches = static_cast<uint32_t>(h->front_end_launches - launches_before);
  return BBA_OK;
}

// bba_track_frame_pairwise and bba_track_frame_pairwise_to_frame (h is not null): the one-entry call on `frames`, the tracked frame
// last, against keyframe base_keyframe_id or, with -1, against frames[0].  Beside the entry's checks it refuses what an entry
// cannot express: a null init1, and a null init2 with test_different_initial_estimates.
bba_status TrackFramePair(bba_handle h, const char* fn, const bba_odometry_options* o, int base_keyframe_id, int frame_count,
                          const bba_frame_buffers* frames, const float* init1, const float* init2, float* out, bba_odometry_result* result,
                          void* stream) {
  if (!init1) return Fail(h, BBA_ERR_INVALID_ARGUMENT, std::string(fn) + ": null argument");
  bba_odometry_entry entry{};
  entry.base_keyframe_id = base_keyframe_id;
  entry.base_frame = 0;
  entry.tracked_frame = frame_count - 1;
  std::memcpy(entry.base_T_frame_initial_1, init1, sizeof(float) * 7);
  std::memcpy(entry.base_T_frame_initial_2, init2 ? init2 : init1, sizeof(float) * 7);
  if (bba_status st = CheckOdometryCall(h, fn, o, frame_count, frames, 1, &entry, out)) return st;
  if (o->test_different_initial_estimates && !init2)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, std::string(fn) + ": test_different_initial_estimates needs the second estimate");
  return TrackFramesPairwise(h, fn, *o, frame_count, frames, 1, &entry, out, result, nullptr, static_cast<cudaStream_t>(stream));
}

}  // namespace
}  // namespace bba

using namespace bba;

extern "C" {

bba_status bba_track_frame_pairwise(bba_handle h, const bba_odometry_options* o, int base_keyframe_id,
                                    const uint16_t* device_depth, size_t depth_pitch, const uint16_t* device_normals, size_t normals_pitch,
                                    const uint8_t* device_color_rgba, size_t color_pitch, const float init1[7], const float init2[7],
                                    float out[7], bba_odometry_result* result, void* stream) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  // (-1 would mean a frame base in an entry)
  if (base_keyframe_id < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_track_frame_pairwise: no such keyframe");
  const bba_frame_buffers frame{device_depth, depth_pitch, device_normals, normals_pitch, device_color_rgba, color_pitch};
  return TrackFramePair(h, "bba_track_frame_pairwise", o, base_keyframe_id, 1, &frame, init1, init2, out, result, stream);
}

bba_status bba_track_frame_pairwise_to_frame(bba_handle h, const bba_odometry_options* o,
                                             const uint16_t* base_depth, size_t base_depth_pitch,
                                             const uint16_t* base_normals, size_t base_normals_pitch,
                                             const uint8_t* base_color_rgba, size_t base_color_pitch,
                                             const uint16_t* device_depth, size_t depth_pitch, const uint16_t* device_normals,
                                             size_t normals_pitch, const uint8_t* device_color_rgba, size_t color_pitch,
                                             const float init1[7], const float init2[7], float out[7], bba_odometry_result* result,
                                             void* stream) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const bba_frame_buffers frames[2] = {{base_depth, base_depth_pitch, base_normals, base_normals_pitch, base_color_rgba, base_color_pitch},
                                       {device_depth, depth_pitch, device_normals, normals_pitch, device_color_rgba, color_pitch}};
  return TrackFramePair(h, "bba_track_frame_pairwise_to_frame", o, -1, 2, frames, init1, init2, out, result, stream);
}

bba_status bba_track_frames_pairwise(bba_handle h, const bba_odometry_options* o, int frame_count, const bba_frame_buffers* frames,
                                     int count, const bba_odometry_entry* entries, float* base_T_frame_estimate,
                                     bba_odometry_result* results, uint32_t* kernel_launches, void* stream) {
  FrontEndScope front_end;
  const char* fn = "bba_track_frames_pairwise";
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckOdometryCall(h, fn, o, frame_count, frames, count, entries, base_T_frame_estimate)) return st;
  return TrackFramesPairwise(h, fn, *o, frame_count, frames, count, entries, base_T_frame_estimate, results, kernel_launches,
                             static_cast<cudaStream_t>(stream));
}

bba_status bba_odometry_get_level(bba_handle h, int which, int scale, float* host_depth, uint16_t* host_normals, uint8_t* host_color,
                                  int* width, int* height, void* stream) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> call(h->fe.call);
  auto& st = h->odo;
  if (which < 0 || which > 1 || scale < 0 || scale >= st.last_num_scales || (which == 1 && scale < st.last_first_scale))
    return Fail(h, BBA_ERR_STATE, "bba_odometry_get_level: this level was not built by the last bba_track_frame_pairwise call");
  const bba::odom::Image& im = st.last_level[which][scale];
  const int w = st.w[scale], ht = st.h[scale];
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (host_depth) BBA_CUDA(h, cudaMemcpy2DAsync(host_depth, sizeof(float) * w, im.depth, sizeof(float) * im.depth_pitch, sizeof(float) * w, ht, cudaMemcpyDeviceToHost, s));
  if (host_normals) BBA_CUDA(h, cudaMemcpy2DAsync(host_normals, sizeof(uint16_t) * w, im.normals, im.normals_pitch, sizeof(uint16_t) * w, ht, cudaMemcpyDeviceToHost, s));
  if (host_color) BBA_CUDA(h, cudaMemcpy2DAsync(host_color, w, im.color, im.color_pitch, w, ht, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  if (width) *width = w;
  if (height) *height = ht;
  return BBA_OK;
}

bba_status bba_odometry_debug_coeffs(bba_handle h, int scale, int use_gradmag, const float pose_a[7], const float pose_b[7], float H[21],
                                     float b[6], uint32_t* residual_count, float* residual_sum, uint32_t counts[2], float costs[2], void* stream) {
  FrontEndScope front_end;
  if (!h || !pose_a) return BBA_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> call(h->fe.call);
  auto& st = h->odo;
  if (scale < st.last_first_scale || scale >= st.last_num_scales)
    return Fail(h, BBA_ERR_STATE, "bba_odometry_debug_coeffs: this level was not built by the last bba_track_frame_pairwise call");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  FrontEndCall view(h);   // (the residual types; the pyramids hold the cameras of the tracking call)
  if (bba_status s2 = view.Snapshot(s, -1, "bba_odometry_debug_coeffs")) return s2;
  if (bba_status s2 = view.ReleaseSlot(/*record=*/false)) return s2;   // (the cfactor is not read)
  bba::odom::TrackEntry entry = st.last_entry;
  std::memcpy(entry.init1, pose_a, sizeof(float) * 7);
  std::memcpy(entry.init2, pose_b ? pose_b : pose_a, sizeof(float) * 7);
  if (bba_status s2 = LaunchOdometryKernel(h, view.cams, st.last_num_scales, st.last_first_scale, 1, use_gradmag ? 1 : 0, 0, scale, {entry}, s))
    return s2;
  const double* d = st.h_result[0].debug;
  if (H) for (int i = 0; i < 21; ++i) H[i] = static_cast<float>(d[i]);
  if (b) for (int i = 0; i < 6; ++i) b[i] = static_cast<float>(d[21 + i]);
  if (residual_count) *residual_count = static_cast<uint32_t>(d[27] + 0.5);
  if (residual_sum) *residual_sum = static_cast<float>(d[28]);
  if (counts) { counts[0] = static_cast<uint32_t>(d[32] + 0.5); counts[1] = static_cast<uint32_t>(d[34] + 0.5); }
  if (costs) { costs[0] = static_cast<float>(d[33]); costs[1] = static_cast<float>(d[35]); }
  return BBA_OK;
}

bba_status bba_preprocess_frame(bba_handle h, const bba_preprocess_options* o,
                                const uint16_t* device_raw_depth, size_t raw_depth_pitch,
                                const uint8_t* device_rgb, size_t rgb_pitch,
                                uint16_t* device_depth, size_t depth_pitch,
                                uint16_t* device_normals, size_t normals_pitch,
                                uint16_t* device_radius, size_t radius_pitch,
                                uint8_t* device_color_rgba, size_t color_pitch,
                                float* min_depth, float* max_depth, void* stream) {
  FrontEndScope front_end;
  return PreprocessFrame(h, "bba_preprocess_frame", o, device_raw_depth, raw_depth_pitch, device_rgb, rgb_pitch, device_depth,
                         depth_pitch, device_normals, normals_pitch, device_radius, radius_pitch, device_color_rgba, color_pitch,
                         min_depth, max_depth, stream, nullptr);
}

bba_status bba_preprocess_raw_frame(bba_handle h, const bba_raw_frame_options* o,
                                    const uint16_t* device_raw_depth, size_t raw_depth_pitch,
                                    int raw_depth_width, int raw_depth_height,
                                    const uint8_t* device_rgb, size_t rgb_pitch, int rgb_width, int rgb_height,
                                    uint16_t* device_depth, size_t depth_pitch,
                                    uint16_t* device_normals, size_t normals_pitch,
                                    uint16_t* device_radius, size_t radius_pitch,
                                    uint8_t* device_color_rgba, size_t color_pitch,
                                    float* min_depth, float* max_depth, void* stream) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (!o) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_preprocess_raw_frame: null argument");
  const int n = o->median_filter_and_densify_iterations, ld = o->pyramid_level_for_depth, lc = o->pyramid_level_for_color;
  if (n < 0 || ld < 0 || lc < 0)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_preprocess_raw_frame: iteration counts and pyramid levels must not be negative");
  if (n > bba::pre::kMaxMedianIterations)
    return Fail(h, BBA_ERR_UNSUPPORTED, "bba_preprocess_raw_frame: at most 8 median filter and densify iterations are supported");
  if (ld > bba::pre::kMaxPyramidLevel || lc > bba::pre::kMaxPyramidLevel)
    return Fail(h, BBA_ERR_UNSUPPORTED, "bba_preprocess_raw_frame: pyramid levels above 3 are not supported");
  if (n > 0 && ld > 0)   // bad_slam.cc:671-673
    return Fail(h, BBA_ERR_UNSUPPORTED, "bba_preprocess_raw_frame: Simultaneous downscaling and median filtering of depth maps is not implemented.");
  const int w = h->cfg.depth_width, hh = h->cfg.depth_height, cw = h->cfg.color_width, ch = h->cfg.color_height;
  // Camera::Scaled(2^-L) (camera.h:1696-1704): int(factor * W + 0.5)
  const auto scaled = [](int size, int level) { return static_cast<int>(static_cast<double>(size) / (1 << level) + 0.5f); };
  if (raw_depth_width <= 0 || raw_depth_height <= 0 || scaled(raw_depth_width, ld) != w || scaled(raw_depth_height, ld) != hh)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_preprocess_raw_frame: the depth camera is " + std::to_string(w) + "x" +
                std::to_string(hh) + ", not the raw depth's " + std::to_string(raw_depth_width) + "x" +
                std::to_string(raw_depth_height) + " scaled to pyramid level " + std::to_string(ld));
  if (raw_depth_width > (w << ld) || raw_depth_height > (hh << ld))
    return Fail(h, BBA_ERR_UNSUPPORTED, "bba_preprocess_raw_frame: raw depth sizes above depth camera size x 2^level give boxes "
                "of more than 2^level pixels per axis, which the median selection does not hold");
  if (device_rgb && (rgb_width != (cw << lc) || rgb_height != (ch << lc)))
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_preprocess_raw_frame: the rgb image must be the colour camera's size x 2^" +
                std::to_string(lc) + " (" + std::to_string(cw << lc) + "x" + std::to_string(ch << lc) + ", even at every level), not " +
                std::to_string(rgb_width) + "x" + std::to_string(rgb_height));
  const RawStage raw_stage{n, ld, raw_depth_width, raw_depth_height, lc};
  return PreprocessFrame(h, "bba_preprocess_raw_frame", &o->base, device_raw_depth, raw_depth_pitch, device_rgb, rgb_pitch,
                         device_depth, depth_pitch, device_normals, normals_pitch, device_radius, radius_pitch, device_color_rgba,
                         color_pitch, min_depth, max_depth, stream, (n | ld | lc) ? &raw_stage : nullptr);
}

}  // extern "C"
