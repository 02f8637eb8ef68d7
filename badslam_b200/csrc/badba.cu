// badba.cu -- C ABI (include/badba.h) of libbadba_b200: the handle, surfel and keyframe setters / getters, keyframe upload,
// luma textures, intrinsics / cfactor / residual-type accessors, profiling and the device-free bba_host_* entry points.
//
// Host-side structure mirrors the reference's DirectBA (direct_ba.{h,cc}, direct_ba_alternating.cc) but the
// schedule is GPU-first: per outer BA iteration the device runs
//     1 launch   activation + normals      (reference: 1 + K_active + 1 + K + 1 launches)
//     1 launch   position + descriptors    (reference: 1 + K + 1 launches)
//     <=30 x 2   pose accumulate + solve for ALL keyframes at once (reference: K x n_GN x {2 clears, kernel,
//                2 D2H copies, stream sync}, kernel_opt_pose.cc:67-96)
// and the host synchronises ONCE per outer iteration to read back the poses.
#include <cmath>
#include <cstring>

#include "handle.hpp"

namespace bba {

void SetError(bba_handle h, const std::string& msg) {
  std::lock_guard<std::mutex> lock(h->error_mu);
  h->errors[std::this_thread::get_id()] = msg;
}

thread_local int FrontEndScope::depth_ = 0;

bba_status Fail(bba_handle h, bba_status s, const std::string& msg) {
  if (h) SetError(h, msg);
  if (h && h->xchg.group && !FrontEndScope::active()) PoisonLocalGroup(h->xchg.group);
  return s;
}

Pose PoseFromArray(const float p[7]) {
  Pose r;
  r.q[0] = p[0]; r.q[1] = p[1]; r.q[2] = p[2]; r.q[3] = p[3];
  r.t[0] = p[4]; r.t[1] = p[5]; r.t[2] = p[6];
  return r;
}
void PoseToArray(const Pose& r, float p[7]) {
  p[0] = r.q[0]; p[1] = r.q[1]; p[2] = r.q[2]; p[3] = r.q[3];
  p[4] = r.t[0]; p[5] = r.t[1]; p[6] = r.t[2];
}

namespace {
CameraView LiveCameraView(bba_handle h) {
  CameraView v;
  std::memcpy(v.depth_K, h->depth_K, sizeof(v.depth_K));
  std::memcpy(v.color_K, h->color_K, sizeof(v.color_K));
  v.depth_a = h->depth_a;
  v.use_depth = h->cfg.use_depth_residuals;
  v.use_desc = h->cfg.use_descriptor_residuals;
  v.deterministic = h->deterministic ? 1 : 0;
  return v;
}
}  // namespace

CameraParams MakeCamera(bba_handle h, const CameraView& v, const float* cfactor) {
  CameraParams c;
  c.w = h->cfg.depth_width; c.h = h->cfg.depth_height; c.cw = h->cfg.color_width; c.ch = h->cfg.color_height;
  // surfel_projection.h:42-67
  c.fx = v.depth_K[0]; c.fy = v.depth_K[1]; c.cx = v.depth_K[2]; c.cy = v.depth_K[3];
  c.fx_inv = 1.0f / c.fx;
  c.fy_inv = 1.0f / c.fy;
  c.cx_inv = -(c.cx - 0.5f) * c.fx_inv;
  c.cy_inv = -(c.cy - 0.5f) * c.fy_inv;
  c.cfx = v.color_K[0]; c.cfy = v.color_K[1]; c.ccx = v.color_K[2]; c.ccy = v.color_K[3];
  // surfel_projection.h:105-124
  c.d2c_fx = c.cfx / c.fx;
  c.d2c_cx = -1 * c.cfx * c.cx / c.fx + c.ccx;
  c.d2c_fy = c.cfy / c.fy;
  c.d2c_cy = -1 * c.cfy * c.cy / c.fy + c.ccy;
  c.a = v.depth_a;
  c.raw_to_float = h->cfg.raw_to_float_depth;
  c.baseline_fx = h->cfg.baseline_fx;
  c.cell = h->cfg.sparse_surfel_cell_size;
  c.cf_w = h->cf_w;
  c.cell_magic = c.cell > 1 ? static_cast<unsigned int>((0x100000000ull + c.cell - 1) / c.cell) : 0u;
  c.cfactor = const_cast<float*>(cfactor);
  c.use_depth = v.use_depth;
  c.use_desc = v.use_desc;
  return c;
}

CameraParams MakeCamera(bba_handle h) { return MakeCamera(h, LiveCameraView(h), h->d_cfactor); }

bba_status Publish(bba_handle h, cudaStream_t s, bool cfactor) {
  auto& f = h->fe;
  int next = -1;
  if (cfactor) {
    {   // the slot that is not current, once no front-end call claims it (claims last a few launches, never a synchronise)
      std::unique_lock<std::mutex> lock(f.mu);
      next = 1 - f.current;
      f.slot_free.wait(lock, [&] { return f.readers[next] == 0; });
    }
    BBA_CUDA(h, cudaStreamWaitEvent(s, f.readers_done[next], 0));
    BBA_CUDA(h, cudaMemcpyAsync(f.cfactor[next], h->d_cfactor, sizeof(float) * h->cf_w * h->cf_h, cudaMemcpyDeviceToDevice, s));
    BBA_CUDA(h, cudaEventRecord(f.published[next], s));
  }
  std::vector<KeyframeView> kfs(h->keyframes.size());
  for (size_t k = 0; k < kfs.size(); ++k) {
    const Keyframe& kf = h->keyframes[k];
    KeyframeView& v = kfs[k];
    v.depth = kf.depth; v.depth_pitch = kf.depth_pitch;
    v.normals = kf.normals; v.normals_pitch = kf.normals_pitch;
    v.tex = kf.tex;
    v.pose = kf.pose;
    v.min_depth = kf.min_depth; v.max_depth = kf.max_depth;
    v.activation = kf.activation;
    v.prior = h->pose_priors[k];
  }
  const CameraView cams = LiveCameraView(h);
  std::vector<PoseConstraint> constraints = h->pose_constraints;
  std::lock_guard<std::mutex> lock(f.mu);
  f.cams = cams;
  f.kfs.swap(kfs);
  f.constraints.swap(constraints);
  if (cfactor) f.current = next;
  return BBA_OK;
}

bba_status FrontEndCall::Snapshot(cudaStream_t s, int kf_id, const char* fn, int max_kf_id, std::vector<KeyframeView>* all_kfs) {
  auto& f = h_->fe;
  {
    std::lock_guard<std::mutex> lock(f.mu);
    if (std::max(kf_id, max_kf_id) >= static_cast<int>(f.kfs.size())) return Fail(h_, BBA_ERR_INVALID_ARGUMENT, std::string(fn) + ": no such keyframe");
    if (kf_id >= 0) base = f.kfs[kf_id];
    if (all_kfs) *all_kfs = f.kfs;
    cams = f.cams;
    slot_ = f.current;
    ++f.readers[slot_];
  }
  s_ = s;
  cfactor = f.cfactor[slot_];
  BBA_CUDA(h_, cudaStreamWaitEvent(s, f.published[slot_], 0));
  return BBA_OK;
}

bba_status FrontEndCall::ReleaseSlot(bool record) {
  if (slot_ < 0) return BBA_OK;
  auto& f = h_->fe;
  cudaError_t e = cudaSuccess;
  if (record) {   // the event then covers this call's reads and those of every earlier claim of the slot
    e = cudaStreamWaitEvent(s_, f.readers_done[slot_], 0);
    if (e == cudaSuccess) e = cudaEventRecord(f.readers_done[slot_], s_);
  }
  {
    std::lock_guard<std::mutex> lock(f.mu);
    --f.readers[slot_];
  }
  f.slot_free.notify_all();
  slot_ = -1;
  if (e != cudaSuccess) return Fail(h_, BBA_ERR_CUDA, std::string("front-end cfactor release: ") + cudaGetErrorString(e));
  return BBA_OK;
}

bba_status WaitStaging(bba_handle h) {
  if (h->staging.pending) {
    BBA_CUDA(h, cudaEventSynchronize(h->staging.event));
    h->staging.pending = false;
  }
  return BBA_OK;
}
bba_status MarkStaging(bba_handle h, cudaStream_t s) {
  BBA_CUDA(h, cudaEventRecord(h->staging.event, s));
  h->staging.pending = true;
  return BBA_OK;
}

void FillKfDevice(const Keyframe& kf, const Pose& global_T_frame, KfDevice* d) {
  ToMatrix3x4(Inverse(global_T_frame), d->T);
  d->depth = kf.depth;
  d->normals = kf.normals;
  d->tex = kf.tex;
  d->depth_pitch = static_cast<uint32_t>(kf.depth_pitch);
  d->normals_pitch = static_cast<uint32_t>(kf.normals_pitch);
  d->activation = kf.activation;
  d->pad = 0;
}

// Uploads every keyframe's parameters (pose, pointers, activation).  K x 96 bytes.
bba_status UploadKeyframes(bba_handle h, cudaStream_t s) {
  const int K = static_cast<int>(h->keyframes.size());
  if (K == 0) return BBA_OK;
  if (bba_status st = WaitStaging(h)) return st;
  for (int k = 0; k < K; ++k) FillKfDevice(h->keyframes[k], h->keyframes[k].pose, h->staging.h_kfs + k);
  BBA_CUDA(h, cudaMemcpyAsync(h->d_kfs, h->staging.h_kfs, sizeof(KfDevice) * K, cudaMemcpyHostToDevice, s));
  return MarkStaging(h, s);
}

bba_status CheckSurfels(bba_handle h) {
  if (!h->surfels || !h->active) return Fail(h, BBA_ERR_STATE, "surfel buffer / active flags not set");
  return BBA_OK;
}

bool FramePitchesOk(bba_handle h, size_t depth_pitch, size_t normals_pitch, size_t color_pitch) {
  return depth_pitch >= static_cast<size_t>(h->cfg.depth_width) * 2 && normals_pitch >= static_cast<size_t>(h->cfg.depth_width) * 2 &&
         color_pitch >= static_cast<size_t>(h->cfg.color_width) * 4 && depth_pitch <= 0xffffffffull && normals_pitch <= 0xffffffffull;
}

cudaTextureDesc LinearTextureDesc() {
  cudaTextureDesc tex;
  std::memset(&tex, 0, sizeof(tex));
  tex.addressMode[0] = cudaAddressModeClamp;
  tex.addressMode[1] = cudaAddressModeClamp;
  tex.filterMode = cudaFilterModeLinear;
  tex.readMode = cudaReadModeNormalizedFloat;
  tex.normalizedCoords = 0;
  return tex;
}

// Each luma plane (the .w channel of a uchar4 image) as a gather-enabled CUDA array (block-linear: 2-D locality for the sample
// footprints) + a texture with the reference's sampling state (keyframe.cc:67-73).  The arrays and textures of *out[i] are
// created when null and refilled otherwise.  A staging is shared by every upload of one side of the handle, and calls may arrive
// on different streams (the reference's tracking thread and BA thread use their own, bad_slam.cc:73-78,1197-1200): one image
// makes s wait until the previous user's copies have consumed the planes; more images rewrite the pinned source table on the
// host, so the host waits.
bba_status MakeLumaTextures(bba_handle h, bool front_end, int n, const LumaSource* sources, Texture* const* out, cudaStream_t s) {
  const int cw = h->cfg.color_width, ch = h->cfg.color_height;
  LumaStaging& staging = front_end ? h->fe.luma : h->staging.luma;
  if (!staging.free) BBA_CUDA(h, cudaEventCreateWithFlags(&staging.free.r, cudaEventDisableTiming));
  else if (n > 1) BBA_CUDA(h, cudaEventSynchronize(staging.free));
  else BBA_CUDA(h, cudaStreamWaitEvent(s, staging.free, 0));
  if (staging.planes < n) {
    staging.planes = 0;
    BBA_CUDA(h, staging.plane.Allocate(cw, static_cast<size_t>(ch) * n));
    staging.planes = n;
  }
  if (n > 1) {
    BBA_CUDA(h, staging.table.Reserve(n - 1));
    BBA_CUDA(h, staging.table_upload.Reserve(n - 1));
    std::copy(sources + 1, sources + n, staging.table_upload.get());
    BBA_CUDA(h, cudaMemcpyAsync(staging.table, staging.table_upload, sizeof(LumaSource) * (n - 1), cudaMemcpyHostToDevice, s));
  }
  for (int i = 0; i < n; ++i) {
    Texture& luma = *out[i];
    if (!luma.array) {
      const cudaChannelFormatDesc desc = cudaCreateChannelDesc(8, 0, 0, 0, cudaChannelFormatKindUnsigned);
      BBA_CUDA(h, cudaMallocArray(&luma.array.r, &desc, cw, ch, cudaArrayTextureGather));
    }
    if (!luma.tex) {
      cudaResourceDesc res;
      std::memset(&res, 0, sizeof(res));
      res.resType = cudaResourceTypeArray;
      res.res.array.array = luma.array;
      const cudaTextureDesc tex = LinearTextureDesc();
      BBA_CUDA(h, cudaCreateTextureObject(&luma.tex.r, &res, &tex, nullptr));
    }
  }
  const size_t pitch = staging.plane.pitch();
  BBA_LAUNCH(h, front_end ? h->front_end_launches : h->launches, LaunchExtractLuma, sources[0], staging.table.get(), n,
             staging.plane.get(), pitch, cw, ch, s);
  for (int i = 0; i < n; ++i)
    BBA_CUDA(h, cudaMemcpy2DToArrayAsync(out[i]->array, 0, 0, staging.plane.get() + static_cast<size_t>(i) * ch * pitch, pitch, cw,
                                         ch, cudaMemcpyDeviceToDevice, s));
  BBA_CUDA(h, cudaEventRecord(staging.free, s));
  return BBA_OK;
}

bba_status MakeFrameLumaTextures(bba_handle h, bool front_end, const bba_frame_buffers* frames, const std::vector<int>& uses,
                                 std::vector<Texture>* pool, cudaTextureObject_t* luma, cudaStream_t s) {
  std::map<int, int> slot_of_frame;
  std::vector<LumaSource> sources;
  for (int f : uses)
    if (slot_of_frame.emplace(f, static_cast<int>(sources.size())).second) sources.push_back(LumaSource{frames[f].color_rgba, frames[f].color_pitch});
  const int n = static_cast<int>(sources.size());
  if (static_cast<int>(pool->size()) < n) pool->resize(n);
  std::vector<Texture*> textures(n);
  for (int i = 0; i < n; ++i) textures[i] = &(*pool)[i];
  if (bba_status st = MakeLumaTextures(h, front_end, n, sources.data(), textures.data(), s)) return st;
  for (const auto& [f, slot] : slot_of_frame) luma[f] = (*pool)[slot].tex;
  return BBA_OK;
}

namespace {

bba_status AddKeyframeCommon(bba_handle h, Keyframe&& kf, const uint8_t* device_rgba, size_t color_pitch, const float pose[7],
                             float min_depth, float max_depth, cudaStream_t s, int* out_id) {
  if (static_cast<int>(h->keyframes.size()) >= h->cfg.max_keyframes) return Fail(h, BBA_ERR_STATE, "max_keyframes exceeded");
  const LumaSource source{device_rgba, color_pitch};
  Texture* const luma = &kf.luma;
  if (bba_status st = MakeLumaTextures(h, /*front_end=*/false, 1, &source, &luma, s)) return st;
  kf.tex = kf.luma.tex;
  kf.pose = PoseFromArray(pose);
  kf.activation = BBA_KF_ACTIVE;   // keyframe.cc:75
  kf.min_depth = min_depth;
  kf.max_depth = max_depth;
  MakeFrustum(&kf.frustum, h->depth_K, h->cfg.depth_width, h->cfg.depth_height, min_depth, max_depth, kf.pose);
  const int id = static_cast<int>(h->keyframes.size());
  // DetermineNewKeyframeCoVisibility, direct_ba.cc:231-249
  for (int k = 0; k < id; ++k) {
    Keyframe& other = h->keyframes[k];
    Frustum other_frustum;
    MakeFrustum(&other_frustum, h->depth_K, h->cfg.depth_width, h->cfg.depth_height, other.min_depth, other.max_depth, other.pose);
    if (FrustaIntersect(kf.frustum, other_frustum)) {
      kf.covis.push_back(k);
      other.covis.push_back(id);
      if (other.activation == BBA_KF_INACTIVE) other.activation = BBA_KF_COVISIBLE_ACTIVE;
    }
  }
  h->keyframes.push_back(std::move(kf));
  if (out_id) *out_id = id;
  return Publish(h, s, false);
}

}  // namespace
}  // namespace bba

using namespace bba;

extern "C" {

int bba_abi_version(void) { return BBA_ABI_VERSION; }

const char* bba_last_error(bba_handle h) {
  if (!h) return "null handle";
  std::lock_guard<std::mutex> lock(h->error_mu);
  return h->errors[std::this_thread::get_id()].c_str();   // (map nodes stay put: valid until this thread's next failure)
}

bba_status bba_create(const bba_config* cfg, bba_handle* out) {
  if (!cfg || !out) return BBA_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  if (cfg->depth_width <= 0 || cfg->depth_height <= 0 || cfg->color_width <= 0 || cfg->color_height <= 0 ||
      cfg->sparse_surfel_cell_size <= 0 || cfg->max_keyframes <= 0 || cfg->world_size <= 0 || cfg->rank < 0 ||
      cfg->rank >= cfg->world_size || (!cfg->use_depth_residuals && !cfg->use_descriptor_residuals))
    return BBA_ERR_INVALID_ARGUMENT;
  int device_count = 0;
  if (cudaGetDeviceCount(&device_count) != cudaSuccess || device_count == 0) {
    cudaGetLastError();
    return BBA_ERR_NO_DEVICE;   // no CPU fallback exists, by design
  }
  bba_handle h = new bba_context();
  h->cfg = *cfg;
  std::memcpy(h->depth_K, cfg->depth_intrinsics, sizeof(h->depth_K));
  std::memcpy(h->color_K, cfg->color_intrinsics, sizeof(h->color_K));
  h->cf_w = (cfg->depth_width - 1) / cfg->sparse_surfel_cell_size + 1;    // direct_ba.cc:110-113
  h->cf_h = (cfg->depth_height - 1) / cfg->sparse_surfel_cell_size + 1;
  auto fail = [&](const char* what, cudaError_t e) {
    std::fprintf(stderr, "bba_create: %s: %s\n", what, cudaGetErrorString(e));
    bba_destroy(h);
    return BBA_ERR_CUDA;
  };
#define CREATE_TRY(expr)                           \
  do {                                             \
    cudaError_t e__ = (expr);                      \
    if (e__ != cudaSuccess) return fail(#expr, e__); \
  } while (0)
  CREATE_TRY(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CREATE_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  h->sm_count = prop.multiProcessorCount;
  CREATE_TRY(bba::SetPoseAccumulateSmemLimits());
  const size_t K = static_cast<size_t>(cfg->max_keyframes);
  auto& p = h->pose;
  CREATE_TRY(h->d_cfactor.Reserve(static_cast<size_t>(h->cf_w) * h->cf_h));
  CREATE_TRY(cudaMemset(h->d_cfactor, 0, sizeof(float) * h->cf_w * h->cf_h));
  CREATE_TRY(h->d_kfs.Reserve(K));
  h->pose_priors.assign(K, bba::PosePrior{});
  CREATE_TRY(p.d_work_records.Reserve(K));
  CREATE_TRY(p.d_pose_est.Reserve(7 * K));
  CREATE_TRY(p.d_acc.Reserve(bba::kPoseAccSize * K));
  CREATE_TRY(cudaMemset(p.d_acc, 0, sizeof(double) * bba::kPoseAccSize * K));
  CREATE_TRY(p.d_stage_counts.Reserve(2 * K));
  CREATE_TRY(cudaMemset(p.d_stage_counts, 0, sizeof(unsigned long long) * 2 * K));
  CREATE_TRY(p.d_work[0].Reserve(K));
  CREATE_TRY(p.d_work[1].Reserve(K));
  CREATE_TRY(p.d_count.Reserve(2));
  CREATE_TRY(p.d_iterations.Reserve(K));
  CREATE_TRY(p.d_converged.Reserve(K));
  CREATE_TRY(p.d_first_stats.Reserve(8 * K));
  CREATE_TRY(cudaMemset(p.d_first_stats, 0, sizeof(double) * 8 * K));
  CREATE_TRY(h->geo.d_list.Reserve(K));
  CREATE_TRY(h->geo.d_queue.Reserve(1));
  CREATE_TRY(h->xchg.d_pose_pack.Reserve(bba::kPoseSlot * K));
  CREATE_TRY(h->xchg.h_pose_pack.Reserve(bba::kPoseSlot * K));
  CREATE_TRY(h->xchg.d_local_ids.Reserve(K));
  CREATE_TRY(p.d_queue.Reserve(1));
  CREATE_TRY(cudaMemset(p.d_queue, 0, sizeof(unsigned int)));
  CREATE_TRY(p.d_totals.Reserve(8));
  CREATE_TRY(cudaMemset(p.d_totals, 0, sizeof(unsigned long long) * 8));
  CREATE_TRY(p.flag.Reserve(4));
  p.flag[0] = p.flag[1] = p.flag[2] = p.flag[3] = 0;
  p.h_flag = p.flag;
  CREATE_TRY(cudaHostGetDevicePointer(&p.d_flag, p.flag.get(), 0));
  CREATE_TRY(p.h_totals.Reserve(8));
  std::memset(&h->profile, 0, sizeof(h->profile));
  for (auto& e : h->prof_ev) CREATE_TRY(cudaEventCreate(&e.r));
  CREATE_TRY(h->staging.h_kfs.Reserve(K));
  CREATE_TRY(p.h_pose_est.Reserve(7 * K));
  CREATE_TRY(p.h_work.Reserve(K + 2));
  CREATE_TRY(h->geo.h_list.Reserve(K));
  CREATE_TRY(p.h_iterations.Reserve(K));
  CREATE_TRY(p.h_converged.Reserve(K));
  CREATE_TRY(p.h_first_stats.Reserve(8 * K));
  CREATE_TRY(cudaEventCreateWithFlags(&h->staging.event.r, cudaEventDisableTiming));
  for (auto& e : h->ev) CREATE_TRY(cudaEventCreate(&e.r));
  for (int i = 0; i < 2; ++i) {   // both cfactor slots start as the zero cfactor; slot 0 is current
    CREATE_TRY(h->fe.cfactor[i].Reserve(static_cast<size_t>(h->cf_w) * h->cf_h));
    CREATE_TRY(cudaMemset(h->fe.cfactor[i], 0, sizeof(float) * h->cf_w * h->cf_h));
    CREATE_TRY(cudaEventCreateWithFlags(&h->fe.published[i].r, cudaEventDisableTiming));
    CREATE_TRY(cudaEventCreateWithFlags(&h->fe.readers_done[i].r, cudaEventDisableTiming));
  }
#undef CREATE_TRY
  h->keyframes.reserve(K);
  Publish(h, nullptr, false);   // (host state only: cannot fail)
  *out = h;
  return BBA_OK;
}

void bba_destroy(bba_handle h) {
  if (!h) return;
  cudaDeviceSynchronize();
  UnmapPeers(h);
  delete h;
}

bba_status bba_set_surfels(bba_handle h, float* device_surfels, size_t pitch_bytes, uint32_t surfels_size) {
  if (h && (device_surfels != h->surfels || pitch_bytes != h->surfel_pitch_bytes)) UnmapPeers(h);
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (!device_surfels || pitch_bytes % 16 != 0 || (reinterpret_cast<uintptr_t>(device_surfels) & 15) != 0 ||
      pitch_bytes < static_cast<size_t>((surfels_size + 3) / 4) * 16 || surfels_size > h->cfg.max_surfel_count)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT,
                "surfel buffer must be 16-byte aligned with a row pitch that is a multiple of 16 bytes and holds surfels_size floats");
  h->surfels = device_surfels;
  h->surfel_pitch_bytes = pitch_bytes;
  h->surfels_size = surfels_size;
  h->pose.order_stale = true;
  return BBA_OK;
}

bba_status bba_set_active_flags(bba_handle h, uint8_t* device_flags) {
  if (h && device_flags != h->active) UnmapPeers(h);
  if (!h || !device_flags) return BBA_ERR_INVALID_ARGUMENT;
  h->active = device_flags;
  return BBA_OK;
}

bba_status bba_set_surfels_host(bba_handle h, const float* host_surfels, size_t pitch_bytes, uint32_t surfels_size, void* stream) {
  if (!h || !host_surfels) return BBA_ERR_INVALID_ARGUMENT;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t pitch = (static_cast<size_t>(h->cfg.max_surfel_count) * 4 + 511) / 512 * 512;
  BBA_CUDA(h, h->owned_surfels.Reserve(pitch / sizeof(float) * bba::kSurfelRowCount));
  if (!h->owned_active) {
    BBA_CUDA(h, h->owned_active.Reserve(h->cfg.max_surfel_count));
    BBA_CUDA(h, cudaMemsetAsync(h->owned_active, 0, h->cfg.max_surfel_count, s));
  }
  h->owned_surfel_pitch = pitch;
  if (surfels_size > h->cfg.max_surfel_count || pitch_bytes < static_cast<size_t>(surfels_size) * 4)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "surfels_size exceeds max_surfel_count or the host pitch");
  // only the 8 data rows are inputs (kSurfelDataAttributeCount, kernels.cuh:89); rows 8-16 are scratch
  BBA_CUDA(h, cudaMemcpy2DAsync(h->owned_surfels, h->owned_surfel_pitch, host_surfels, pitch_bytes,
                                static_cast<size_t>(surfels_size) * 4, 8, cudaMemcpyHostToDevice, s));
  if (bba_status st = bba_set_surfels(h, h->owned_surfels, h->owned_surfel_pitch, surfels_size)) return st;
  return bba_set_active_flags(h, h->owned_active);
}

bba_status bba_get_surfels_host(bba_handle h, float* host_surfels, size_t pitch_bytes, int rows, void* stream) {
  if (!h || !host_surfels || rows < 1 || rows > bba::kSurfelRowCount) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckSurfels(h)) return st;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  BBA_CUDA(h, cudaMemcpy2DAsync(host_surfels, pitch_bytes, h->surfels, h->surfel_pitch_bytes,
                                static_cast<size_t>(h->surfels_size) * 4, rows, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  return BBA_OK;
}

bba_status bba_get_active_flags_host(bba_handle h, uint8_t* host_flags, void* stream) {
  if (!h || !host_flags) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckSurfels(h)) return st;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  BBA_CUDA(h, cudaMemcpyAsync(host_flags, h->active, h->surfels_size, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  return BBA_OK;
}

bba_status bba_get_surfels_device(bba_handle h, float** device_surfels, size_t* pitch_bytes, uint32_t* surfels_size) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (device_surfels) *device_surfels = h->surfels;
  if (pitch_bytes) *pitch_bytes = h->surfel_pitch_bytes;
  if (surfels_size) *surfels_size = h->surfels_size;
  return BBA_OK;
}

bba_status bba_add_keyframe(bba_handle h, const uint16_t* device_depth, size_t depth_pitch, const uint16_t* device_normals,
                            size_t normals_pitch, const uint16_t* device_radius, size_t radius_pitch,
                            const uint8_t* device_color_rgba, size_t color_pitch, const float global_T_frame[7], float min_depth,
                            float max_depth, void* stream, int* out_keyframe_id) {
  if (!h || !device_depth || !device_normals || !device_color_rgba || !global_T_frame) return BBA_ERR_INVALID_ARGUMENT;
  if (!FramePitchesOk(h, depth_pitch, normals_pitch, color_pitch)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "keyframe buffer pitch too small");
  Keyframe kf;
  kf.depth = device_depth; kf.depth_pitch = depth_pitch;
  kf.normals = device_normals; kf.normals_pitch = normals_pitch;
  kf.radius = device_radius; kf.radius_pitch = radius_pitch;
  kf.rgba = device_color_rgba; kf.rgba_pitch = color_pitch;
  return AddKeyframeCommon(h, std::move(kf), device_color_rgba, color_pitch, global_T_frame, min_depth, max_depth,
                           static_cast<cudaStream_t>(stream), out_keyframe_id);
}

bba_status bba_add_keyframe_host(bba_handle h, const uint16_t* host_depth, const uint16_t* host_normals, const uint16_t* host_radius,
                                 const uint8_t* host_color_rgba, const float global_T_frame[7], float min_depth, float max_depth,
                                 void* stream, int* out_keyframe_id) {
  if (!h || !host_depth || !host_normals || !host_color_rgba || !global_T_frame) return BBA_ERR_INVALID_ARGUMENT;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int w = h->cfg.depth_width, hh = h->cfg.depth_height, cw = h->cfg.color_width, ch = h->cfg.color_height;
  Keyframe kf;   // (frees its copies on every error return)
  size_t pitch = 0;
  const uint16_t* srcs[3] = {host_depth, host_normals, host_radius};
  for (int i = 0; i < 3; ++i) {
    if (!srcs[i]) continue;
    BBA_CUDA(h, kf.owned[i].Allocate(static_cast<size_t>(w) * 2, hh));
    pitch = kf.owned[i].pitch();
    BBA_CUDA(h, cudaMemcpy2DAsync(kf.owned[i].get(), pitch, srcs[i], static_cast<size_t>(w) * 2, static_cast<size_t>(w) * 2, hh,
                                  cudaMemcpyHostToDevice, s));
  }
  kf.depth = kf.owned[0].get<uint16_t>(); kf.depth_pitch = pitch;
  kf.normals = kf.owned[1].get<uint16_t>(); kf.normals_pitch = pitch;
  kf.radius = kf.owned[2].get<uint16_t>(); kf.radius_pitch = pitch;
  // the colour image: the luma plane is derived from it; the copy is kept for the colours of surfels created later
  BBA_CUDA(h, kf.owned_rgba.Allocate(static_cast<size_t>(cw) * 4, ch));
  const uint8_t* rgba = kf.owned_rgba.get();
  const size_t rgba_pitch = kf.owned_rgba.pitch();
  BBA_CUDA(h, cudaMemcpy2DAsync(kf.owned_rgba.get(), rgba_pitch, host_color_rgba, static_cast<size_t>(cw) * 4, static_cast<size_t>(cw) * 4, ch,
                                cudaMemcpyHostToDevice, s));
  kf.rgba = rgba;
  kf.rgba_pitch = rgba_pitch;
  return AddKeyframeCommon(h, std::move(kf), rgba, rgba_pitch, global_T_frame, min_depth, max_depth, s, out_keyframe_id);
}

bba_status bba_update_keyframe_host(bba_handle h, int id, const uint16_t* host_depth, const uint16_t* host_normals,
                                    const uint16_t* host_radius, const uint8_t* host_color_rgba, void* stream) {
  CHECK_KF(h, id);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Keyframe& kf = h->keyframes[id];
  const int w = h->cfg.depth_width, hh = h->cfg.depth_height, cw = h->cfg.color_width, ch = h->cfg.color_height;
  // The library can only write into buffers it owns (keyframes added with bba_add_keyframe_host); caller-owned
  // device buffers are updated by the caller.
  const uint16_t* srcs[3] = {host_depth, host_normals, host_radius};
  const size_t pitches[3] = {kf.depth_pitch, kf.normals_pitch, kf.radius_pitch};
  for (int i = 0; i < 3; ++i) {
    if (!srcs[i]) continue;
    if (!kf.owned[i]) return Fail(h, BBA_ERR_STATE, "keyframe buffers are caller-owned; update them directly");
    BBA_CUDA(h, cudaMemcpy2DAsync(kf.owned[i].get(), pitches[i], srcs[i], static_cast<size_t>(w) * 2, static_cast<size_t>(w) * 2, hh,
                                  cudaMemcpyHostToDevice, s));
  }
  if (host_color_rgba) {
    PitchedBuffer* dst = &kf.owned_rgba;
    if (!*dst) {   // caller-owned colour image: only the library's luma array is refreshed, through a staging image
      dst = &h->staging.color;
      if (!*dst) BBA_CUDA(h, dst->Allocate(static_cast<size_t>(cw) * 4, ch));
    }
    BBA_CUDA(h, cudaMemcpy2DAsync(dst->get(), dst->pitch(), host_color_rgba, static_cast<size_t>(cw) * 4,
                                  static_cast<size_t>(cw) * 4, ch, cudaMemcpyHostToDevice, s));
    const LumaSource source{dst->get(), dst->pitch()};
    Texture* const luma = &kf.luma;
    if (bba_status st = MakeLumaTextures(h, /*front_end=*/false, 1, &source, &luma, s)) return st;
  }
  return Publish(h, s, false);
}

// ---- host-side building blocks, callable without a device (the CPU test-suite checks them against the oracle) ----
void bba_host_se3_exp(const float a[6], float out[7]) { PoseToArray(bba::Exp(a), out); }
void bba_host_se3_log(const float T[7], float out[6]) { bba::Log(PoseFromArray(T), out); }
void bba_host_se3_compose(const float A[7], const float B[7], float out[7]) { PoseToArray(bba::Compose(PoseFromArray(A), PoseFromArray(B)), out); }
void bba_host_se3_inverse(const float A[7], float out[7]) { PoseToArray(bba::Inverse(PoseFromArray(A)), out); }
int bba_host_pose_update_converged(const float x[6]) { return bba::IsScale1PoseEstimationConverged(x) ? 1 : 0; }
int bba_host_solve_ldlt(int n, const double* upper, const double* b, double* x) {
  if (!upper || !b || !x) return 0;
  if (n == 4) bba::SolveLDLT<4>(upper, b, x);
  else if (n == 5) bba::SolveLDLT<5>(upper, b, x);
  else if (n == 6) bba::SolveLDLT<6>(upper, b, x);
  else return 0;
  return 1;
}
void bba_host_pose_prior_terms(const float prior[7], const float pose[7], const float info[21], double H[21], double b[6], double* cost) {
  if (!prior || !pose || !info || !H || !b || !cost) return;
  bba::PosePriorTerms(prior, pose, info, H, b, cost);
}
void bba_host_pose_constraint_terms(const float a_T_b[7], const float pose_a[7], const float pose_b[7], const float info[21], double H[78],
                                    double b[12], double* cost) {
  if (!a_T_b || !pose_a || !pose_b || !info || !H || !b || !cost) return;
  double r[6];
  bba::PoseConstraintTerms(a_T_b, pose_a, pose_b, info, r, H, b, cost);
}
int bba_host_frusta_intersect(const float depth_intrinsics[4], int width, int height, const float global_T_frame_a[7], float min_depth_a,
                              float max_depth_a, const float global_T_frame_b[7], float min_depth_b, float max_depth_b) {
  Frustum a, b;
  MakeFrustum(&a, depth_intrinsics, width, height, min_depth_a, max_depth_a, PoseFromArray(global_T_frame_a));
  MakeFrustum(&b, depth_intrinsics, width, height, min_depth_b, max_depth_b, PoseFromArray(global_T_frame_b));
  return FrustaIntersect(a, b) ? 1 : 0;
}

// Constant-motion model of the odometry front end.  The stored transforms and their inverses are two lists that are updated side
// by side (never re-derived from each other), like base_kf_tr_frame_ / frame_tr_base_kf_ of the reference; products associate
// left to right like its `a * b * c`.
namespace {
const float kIdentityPose[7] = {0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f};
void CopyPose(const float* src, float* dst) { for (int i = 0; i < 7; ++i) dst[i] = src[i]; }
}  // namespace

void bba_host_motion_model_clear(bba_motion_model* m, const float last_kf_frame_T_global[7], const float global_T_frame[7]) {   // bad_slam.cc:542-565
  if (!m) return;
  m->count = 1;
  if (!last_kf_frame_T_global || !global_T_frame) {
    CopyPose(kIdentityPose, m->base_kf_tr_frame[0]);
    CopyPose(kIdentityPose, m->frame_tr_base_kf[0]);
    return;
  }
  const Pose rel = bba::Compose(PoseFromArray(last_kf_frame_T_global), PoseFromArray(global_T_frame));
  PoseToArray(rel, m->base_kf_tr_frame[0]);
  PoseToArray(bba::Inverse(rel), m->frame_tr_base_kf[0]);
}

int bba_host_motion_model_predict(const bba_motion_model* m, int use_motion_model, float e1[7], float e2[7]) {   // bad_slam.cc:767-827
  if (!m || !e1 || !e2 || m->count < 1 || m->count > 3) return 0;
  const int n = m->count;
  const Pose last = PoseFromArray(m->base_kf_tr_frame[n - 1]);
  if (!use_motion_model) {
    PoseToArray(last, e1);
    PoseToArray(last, e2);
    return 1;
  }
  // the motion of the last step applied once more
  Pose first = last;
  if (n >= 2) first = bba::Compose(bba::Compose(last, PoseFromArray(m->frame_tr_base_kf[n - 2])), last);
  PoseToArray(first, e1);
  // the motion of the step before, applied twice to the frame before the last: an outlier in the last frame does not enter
  if (n >= 3) {
    const Pose step = bba::Compose(PoseFromArray(m->frame_tr_base_kf[n - 3]), PoseFromArray(m->base_kf_tr_frame[n - 2]));
    PoseToArray(bba::Compose(bba::Compose(PoseFromArray(m->base_kf_tr_frame[n - 2]), step), step), e2);
  } else {
    PoseToArray(first, e2);
  }
  return 1;
}

void bba_host_motion_model_push(bba_motion_model* m, const float estimate[7]) {   // bad_slam.cc:949-954
  if (!m || !estimate) return;
  if (m->count < 0 || m->count > 3) m->count = 0;
  if (m->count == 3) {
    for (int i = 0; i < 2; ++i) {
      CopyPose(m->base_kf_tr_frame[i + 1], m->base_kf_tr_frame[i]);
      CopyPose(m->frame_tr_base_kf[i + 1], m->frame_tr_base_kf[i]);
    }
    m->count = 2;
  }
  CopyPose(estimate, m->base_kf_tr_frame[m->count]);
  PoseToArray(bba::Inverse(PoseFromArray(estimate)), m->frame_tr_base_kf[m->count]);
  ++m->count;
}

void bba_host_motion_model_rebase(bba_motion_model* m) {   // bad_slam.cc:1057-1068
  if (!m) return;
  if (m->count < 0 || m->count > 3) m->count = 0;
  const int n = m->count;
  if (n == 0) {
    m->count = 1;
  } else {
    const Pose last = PoseFromArray(m->base_kf_tr_frame[n - 1]);
    const Pose last_inv = PoseFromArray(m->frame_tr_base_kf[n - 1]);
    for (int i = 0; i + 1 < n; ++i) {
      PoseToArray(bba::Compose(PoseFromArray(m->frame_tr_base_kf[i]), last), m->frame_tr_base_kf[i]);
      PoseToArray(bba::Compose(last_inv, PoseFromArray(m->base_kf_tr_frame[i])), m->base_kf_tr_frame[i]);
    }
  }
  CopyPose(kIdentityPose, m->base_kf_tr_frame[m->count - 1]);
  CopyPose(kIdentityPose, m->frame_tr_base_kf[m->count - 1]);
}

// Trajectory deformation after a BA call.  Statement by statement trajectory_deformation.cc:45-130 on arrays: keyframes are never
// null here (no deletion), so the reference's skipping of null entries has nothing to skip.  A frame's frame_T_global is the
// inverse of its global_T_frame, as ImageFrame::SetGlobalTFrame stores it (libvis image_frame.h:84-88).
int bba_host_deform_trajectory(int keyframe_count, const int* keyframe_frame_index, const float* original_keyframe_T_global,
                               const float* keyframe_global_T_frame, int start_frame, int end_frame, float* frame_global_T_frame) {
  if (keyframe_count < 1 || !keyframe_frame_index || !original_keyframe_T_global || !keyframe_global_T_frame ||
      !frame_global_T_frame || start_frame < 0 || start_frame > end_frame || keyframe_frame_index[0] < 0)
    return BBA_ERR_INVALID_ARGUMENT;
  for (int k = 1; k < keyframe_count; ++k)
    if (keyframe_frame_index[k] <= keyframe_frame_index[k - 1]) return BBA_ERR_INVALID_ARGUMENT;
  const int K = keyframe_count;
  const int* kf_frame = keyframe_frame_index;
  auto original = [&](int k) { return PoseFromArray(original_keyframe_T_global + 7 * k); };
  auto kf_global_T_frame = [&](int k) { return PoseFromArray(keyframe_global_T_frame + 7 * k); };
  int prev = 0, next = 0;
  for (int frame = start_frame; frame <= end_frame; ++frame) {
    while (next < K && kf_frame[next] <= frame) prev = next++;
    if (kf_frame[prev] == frame) continue;   // a keyframe
    float* pose = frame_global_T_frame + 7 * static_cast<size_t>(frame);
    const Pose global_T_other = PoseFromArray(pose);
    Pose new_global_T_other;
    if (next >= K || kf_frame[prev] > frame) {   // extrapolate at the end / at the start
      new_global_T_other = bba::Compose(kf_global_T_frame(prev), bba::Compose(original(prev), global_T_other));
    } else {   // interpolate
      const Pose other_T_global = bba::Inverse(global_T_other);
      const Pose from_prev = bba::Compose(other_T_global, bba::Compose(kf_global_T_frame(prev), bba::Compose(original(prev), global_T_other)));
      const Pose from_next = bba::Compose(other_T_global, bba::Compose(kf_global_T_frame(next), bba::Compose(original(next), global_T_other)));
      const float factor = static_cast<float>(frame - kf_frame[prev]) * 1.0f / static_cast<float>(kf_frame[next] - kf_frame[prev]);
      Pose interpolated;
      for (int i = 0; i < 3; ++i) interpolated.t[i] = (1 - factor) * from_prev.t[i] + factor * from_next.t[i];
      bba::QuatSlerp(from_prev.q, factor, from_next.q, interpolated.q);
      bba::QuatNormalize(interpolated.q);
      new_global_T_other = bba::Compose(global_T_other, interpolated);
    }
    PoseToArray(new_global_T_other, pose);
  }
  return BBA_OK;
}

void bba_host_exact_sum(const float* values, size_t n, double* out) {
  if (!out) return;
  long long w[kExactWords] = {};
  ExactSum sum{};
  for (size_t i = 0; i < n; ++i) {
    int word;
    long long lo, hi;
    unsigned long long flag;
    if (bba::ExactSplit(values[i], &word, &lo, &hi, &flag)) {
      w[word] += lo;
      w[word + 1] += hi;
    } else {
      sum.flags |= flag;
    }
    // (the words stay exact for any n: carried before any of them could reach 2^62)
    if ((i & 0x3fffffffull) == 0x3fffffffull) bba::ExactCarry(w);
  }
  for (int i = 0; i < kExactWords; ++i) sum.w[i] = static_cast<unsigned long long>(w[i]);
  *out = bba::ExactFinalize(sum);
}

// The readers below are front-end calls: they read the published state (identical to the live state between BA-side calls).
int bba_keyframe_count(bba_handle h) {
  if (!h) return 0;
  std::lock_guard<std::mutex> lock(h->fe.mu);
  return static_cast<int>(h->fe.kfs.size());
}

bba_status bba_set_keyframe_pose(bba_handle h, int id, const float p[7]) {
  CHECK_KF(h, id);
  h->keyframes[id].pose = PoseFromArray(p);
  return Publish(h, nullptr, false);
}
bba_status bba_get_keyframe_pose(bba_handle h, int id, float p[7]) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lock(h->fe.mu);
  if (id < 0 || id >= static_cast<int>(h->fe.kfs.size())) {
    lock.unlock();
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bad keyframe id");
  }
  PoseToArray(h->fe.kfs[id].pose, p);
  return BBA_OK;
}
bba_status bba_set_keyframe_activation(bba_handle h, int id, int activation) {
  CHECK_KF(h, id);
  if (activation < 0 || activation > 2) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bad activation");
  h->keyframes[id].activation = activation;
  return Publish(h, nullptr, false);
}
bba_status bba_get_keyframe_activation(bba_handle h, int id, int* activation) {
  FrontEndScope front_end;
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lock(h->fe.mu);
  if (id < 0 || id >= static_cast<int>(h->fe.kfs.size())) {
    lock.unlock();
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bad keyframe id");
  }
  *activation = h->fe.kfs[id].activation;
  return BBA_OK;
}
bba_status bba_set_keyframe_states(bba_handle h, int count, const float* poses, const int* activation) {
  if (!h || count < 0 || count > static_cast<int>(h->keyframes.size())) return BBA_ERR_INVALID_ARGUMENT;
  bba_status st = BBA_OK;
  for (int k = 0; k < count && !st; ++k) {
    if (poses) h->keyframes[k].pose = PoseFromArray(poses + 7 * k);
    if (activation) {
      if (activation[k] < 0 || activation[k] > 2) st = Fail(h, BBA_ERR_INVALID_ARGUMENT, "bad activation");
      else h->keyframes[k].activation = activation[k];
    }
  }
  Publish(h, nullptr, false);   // (also what was set before a bad activation)
  return st;
}
bba_status bba_get_keyframe_states(bba_handle h, int count, float* poses, int* activation) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lock(h->fe.mu);
  if (count < 0 || count > static_cast<int>(h->fe.kfs.size())) return BBA_ERR_INVALID_ARGUMENT;
  for (int k = 0; k < count; ++k) {
    if (poses) PoseToArray(h->fe.kfs[k].pose, poses + 7 * k);
    if (activation) activation[k] = h->fe.kfs[k].activation;
  }
  return BBA_OK;
}
// ---- soft pose priors ----
namespace {
// Counts the priors and publishes the records.
bba_status CommitPosePriors(bba_handle h) {
  int count = 0;
  for (const PosePrior& p : h->pose_priors) count += p.has ? 1 : 0;
  h->pose_prior_count = count;
  return Publish(h, nullptr, false);
}

bool PoseRecordFinite(const float* pose, const float* info) {
  bool finite = true;
  for (int j = 0; j < 7; ++j) finite = finite && std::isfinite(pose[j]);
  for (int j = 0; j < 21; ++j) finite = finite && std::isfinite(info[j]);
  return finite;
}
}  // namespace

bba_status bba_set_keyframe_pose_priors(bba_handle h, int count, const int* ids, const float* poses, const float* information) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_set_keyframe_pose_priors: ";
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < 0");
  if (count > 0 && (!ids || !poses || !information)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  const int K = static_cast<int>(h->keyframes.size());
  for (int i = 0; i < count; ++i) {
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad keyframe id");
    const float* p = poses + 7 * static_cast<size_t>(i);
    const float* info = information + 21 * static_cast<size_t>(i);
    if (!PoseRecordFinite(p, info)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "non-finite pose or information");
    if (p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3] < 1e-12f) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "zero quaternion");
    if (!InformationPsd(info)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "information matrix is not positive semi-definite");
  }
  if (count > 0)
    if (bba_status st = ReservePoseTerms(h, h->pose_constraints.size())) return st;
  for (int i = 0; i < count; ++i) {
    PosePrior& r = h->pose_priors[ids[i]];
    std::memcpy(r.pose, poses + 7 * static_cast<size_t>(i), sizeof(r.pose));
    std::memcpy(r.info, information + 21 * static_cast<size_t>(i), sizeof(r.info));
    r.has = 1;
  }
  return CommitPosePriors(h);
}

bba_status bba_clear_keyframe_pose_priors(bba_handle h, int count, const int* ids) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_clear_keyframe_pose_priors: ";
  const int K = static_cast<int>(h->keyframes.size());
  if (count == -1) {
    std::fill(h->pose_priors.begin(), h->pose_priors.end(), PosePrior{});
    return CommitPosePriors(h);
  }
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < -1");
  if (count > 0 && !ids) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  for (int i = 0; i < count; ++i)
    if (ids[i] < 0 || ids[i] >= K) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad keyframe id");
  for (int i = 0; i < count; ++i) h->pose_priors[ids[i]] = PosePrior{};
  return CommitPosePriors(h);
}

bba_status bba_get_keyframe_pose_prior(bba_handle h, int id, float pose[7], float information[21], int* has_prior) {
  FrontEndScope front_end;
  if (!h || !has_prior) return BBA_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lock(h->fe.mu);
  if (id < 0 || id >= static_cast<int>(h->fe.kfs.size())) {
    lock.unlock();
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bad keyframe id");
  }
  const PosePrior& p = h->fe.kfs[id].prior;
  *has_prior = p.has;
  if (pose) std::memcpy(pose, p.pose, sizeof(p.pose));
  if (information) std::memcpy(information, p.info, sizeof(p.info));
  return BBA_OK;
}

// ---- soft relative pose constraints ----
bba_status bba_add_keyframe_pose_constraints(bba_handle h, int count, const bba_pose_constraint* constraints, int* out_ids) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_add_keyframe_pose_constraints: ";
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < 0");
  if (count > 0 && !constraints) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  const int K = static_cast<int>(h->keyframes.size());
  for (int i = 0; i < count; ++i) {
    const bba_pose_constraint& c = constraints[i];
    if (c.keyframe_a < 0 || c.keyframe_a >= K || c.keyframe_b < 0 || c.keyframe_b >= K)
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "bad keyframe id");
    if (c.keyframe_a == c.keyframe_b) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "keyframe_a == keyframe_b");
    if (!PoseRecordFinite(c.a_T_b, c.information)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "non-finite pose or information");
    const float* q = c.a_T_b;
    if (q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3] < 1e-12f) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "zero quaternion");
    if (!InformationPsd(c.information)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "information matrix is not positive semi-definite");
  }
  if (count == 0) return BBA_OK;
  if (bba_status st = ReservePoseTerms(h, h->pose_constraints.size() + count)) return st;
  for (int i = 0; i < count; ++i) {
    PoseConstraint r{};
    r.id = h->next_pose_constraint_id++;
    r.c = constraints[i];
    double info_a[21];
    PoseConstraintInformationA(r.c.a_T_b, r.c.information, info_a);
    for (int j = 0; j < 21; ++j) r.info_a[j] = static_cast<float>(info_a[j]);
    h->pose_constraints.push_back(r);
    if (out_ids) out_ids[i] = r.id;
  }
  return Publish(h, nullptr, false);
}

bba_status bba_remove_keyframe_pose_constraints(bba_handle h, int count, const int* ids) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  const std::string fn = "bba_remove_keyframe_pose_constraints: ";
  auto& cons = h->pose_constraints;
  if (count == -1) {
    cons.clear();
    return Publish(h, nullptr, false);
  }
  if (count < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "count < -1");
  if (count > 0 && !ids) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "null argument");
  std::vector<char> drop(cons.size(), 0);
  for (int i = 0; i < count; ++i) {
    // ids increase along the list
    auto it = std::lower_bound(cons.begin(), cons.end(), ids[i], [](const PoseConstraint& c, int id) { return c.id < id; });
    if (it == cons.end() || it->id != ids[i]) return Fail(h, BBA_ERR_INVALID_ARGUMENT, fn + "unknown constraint id");
    drop[it - cons.begin()] = 1;
  }
  size_t n = 0;
  for (size_t i = 0; i < cons.size(); ++i)
    if (!drop[i]) cons[n++] = cons[i];
  cons.resize(n);
  return Publish(h, nullptr, false);
}

bba_status bba_get_keyframe_pose_constraints(bba_handle h, int capacity, int* ids, bba_pose_constraint* out, int* count) {
  FrontEndScope front_end;
  if (!h || !count) return BBA_ERR_INVALID_ARGUMENT;
  if (capacity < 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_get_keyframe_pose_constraints: capacity < 0");
  std::lock_guard<std::mutex> lock(h->fe.mu);
  const std::vector<PoseConstraint>& cons = h->fe.constraints;
  *count = static_cast<int>(cons.size());
  const int n = std::min(capacity, *count);
  for (int i = 0; i < n; ++i) {
    if (ids) ids[i] = cons[i].id;
    if (out) out[i] = cons[i].c;
  }
  return BBA_OK;
}

bba_status bba_get_covisibility(bba_handle h, int id, uint8_t* out_row) {
  CHECK_KF(h, id);
  std::memset(out_row, 0, h->keyframes.size());
  for (int o : h->keyframes[id].covis) out_row[o] = 1;
  return BBA_OK;
}

bba_status bba_set_intrinsics(bba_handle h, const float d[4], const float c[4], float a) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (d) std::memcpy(h->depth_K, d, sizeof(h->depth_K));
  if (c) std::memcpy(h->color_K, c, sizeof(h->color_K));
  h->depth_a = a;
  return Publish(h, nullptr, false);
}
bba_status bba_set_residual_types(bba_handle h, int use_depth_residuals, int use_descriptor_residuals) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (!use_depth_residuals && !use_descriptor_residuals)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_set_residual_types: at least one residual type must stay enabled");
  h->cfg.use_depth_residuals = use_depth_residuals != 0;
  h->cfg.use_descriptor_residuals = use_descriptor_residuals != 0;
  return Publish(h, nullptr, false);
}
bba_status bba_get_residual_types(bba_handle h, int* use_depth_residuals, int* use_descriptor_residuals) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lock(h->fe.mu);
  if (use_depth_residuals) *use_depth_residuals = h->fe.cams.use_depth;
  if (use_descriptor_residuals) *use_descriptor_residuals = h->fe.cams.use_desc;
  return BBA_OK;
}
bba_status bba_get_intrinsics(bba_handle h, float d[4], float c[4], float* a) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lock(h->fe.mu);
  if (d) std::memcpy(d, h->fe.cams.depth_K, sizeof(h->fe.cams.depth_K));
  if (c) std::memcpy(c, h->fe.cams.color_K, sizeof(h->fe.cams.color_K));
  if (a) *a = h->fe.cams.depth_a;
  return BBA_OK;
}
bba_status bba_cfactor_size(bba_handle h, int* w, int* hh) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (w) *w = h->cf_w;
  if (hh) *hh = h->cf_h;
  return BBA_OK;
}
bba_status bba_set_cfactor_host(bba_handle h, const float* host, void* stream) {
  if (!h || !host) return BBA_ERR_INVALID_ARGUMENT;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  BBA_CUDA(h, cudaMemcpyAsync(h->d_cfactor, host, sizeof(float) * h->cf_w * h->cf_h, cudaMemcpyHostToDevice, s));
  if (bba_status st = Publish(h, s, true)) return st;
  BBA_CUDA(h, cudaStreamSynchronize(s));
  return BBA_OK;
}
bba_status bba_get_cfactor_host(bba_handle h, float* host, void* stream) {
  FrontEndScope front_end;
  if (!h || !host) return BBA_ERR_INVALID_ARGUMENT;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  FrontEndCall view(h);
  if (bba_status st = view.Snapshot(s, -1, "bba_get_cfactor_host")) return st;
  BBA_CUDA(h, cudaMemcpyAsync(host, view.cfactor, sizeof(float) * h->cf_w * h->cf_h, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  return view.ReleaseSlot(/*record=*/false);   // (the read is complete)
}

uint32_t bba_surfels_size(bba_handle h) { return h ? h->surfels_size : 0; }

bba_status bba_get_ba_iteration_counts(bba_handle h, int* ba_iteration_count, int* last_ba_iteration_count) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (ba_iteration_count) *ba_iteration_count = h->ba_iteration_count;
  if (last_ba_iteration_count) *last_ba_iteration_count = h->last_ba_iteration_count;
  return BBA_OK;
}
bba_status bba_set_ba_iteration_counts(bba_handle h, int ba_iteration_count, int last_ba_iteration_count) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  h->ba_iteration_count = ba_iteration_count;
  h->last_ba_iteration_count = last_ba_iteration_count;
  return BBA_OK;
}

uint64_t bba_kernel_launch_count(bba_handle h) { return h ? h->launches + h->front_end_launches : 0; }

bba_status bba_set_deterministic(bba_handle h, int on) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (on && h->cfg.world_size > 1)
    return Fail(h, BBA_ERR_UNSUPPORTED, "bba_set_deterministic: the deterministic mode runs on one rank (world_size 1)");
  if (on && !h->deterministic) {
    // the exact sums of the pose kernel and of the intrinsics step, zero from here on (every user clears what it consumed)
    const uint32_t P = static_cast<uint32_t>(h->cf_w) * h->cf_h;
    const size_t pose = static_cast<size_t>(kPoseAccSize) * h->cfg.max_keyframes;
    const size_t intr = static_cast<size_t>(7) * P + kIntrinsicsSums;
    BBA_CUDA(h, h->pose.d_exact.Reserve(pose));
    BBA_CUDA(h, h->geo.d_intr_exact.Reserve(intr));
    BBA_CUDA(h, cudaMemset(h->pose.d_exact, 0, sizeof(ExactSum) * pose));
    BBA_CUDA(h, cudaMemset(h->geo.d_intr_exact, 0, sizeof(ExactSum) * intr));
  }
  h->deterministic = on != 0;
  return Publish(h, nullptr, false);
}

bba_status bba_get_deterministic(bba_handle h, int* on) {
  if (!h || !on) return BBA_ERR_INVALID_ARGUMENT;
  std::lock_guard<std::mutex> lock(h->fe.mu);
  *on = h->fe.cams.deterministic;
  return BBA_OK;
}

bba_status bba_debug_exact_sum(bba_handle h, const float* device_values, uint64_t n, double* out, void* stream) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (!out || (n && !device_values)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_exact_sum: null argument");
  if (n >= (1ull << 31)) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_exact_sum: an exact sum holds fewer than 2^31 values");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DeviceBuffer<ExactSum> sum;
  DeviceBuffer<double> d_out;
  BBA_CUDA(h, sum.Reserve(1));
  BBA_CUDA(h, d_out.Reserve(1));
  BBA_CUDA(h, cudaMemsetAsync(sum, 0, sizeof(ExactSum), s));
  BBA_LAUNCH(h, h->launches, LaunchExactSumDebug, device_values, n, sum, d_out, h->sm_count, s);
  BBA_CUDA(h, cudaMemcpyAsync(out, d_out, sizeof(double), cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  return BBA_OK;
}

bba_status bba_set_profiling(bba_handle h, int enable) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  h->profiling = enable < 0 ? 0 : (enable > 2 ? 2 : enable);
  return BBA_OK;
}

bba_status bba_get_profile(bba_handle h, bba_profile* out, int reset) {
  if (!h || !out) return BBA_ERR_INVALID_ARGUMENT;
  *out = h->profile;
  if (reset) std::memset(&h->profile, 0, sizeof(h->profile));
  return BBA_OK;
}

}  // extern "C"
