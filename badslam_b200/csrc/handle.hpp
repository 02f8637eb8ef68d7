// handle.hpp -- the library handle (bba_context) and what the host units of libbadba_b200 share: the owners of device / pinned
// memory, events and textures, the keyframe record, error reporting and the helpers that more than one unit calls.
//
// Host units: badba.cu (handle, setters / getters, keyframes, textures, bba_host_*), pose_step.cu (spatial order, pose step),
// bundle_adjust.cu (BA schemes, intrinsics, PCG, surfel lifecycle, pose graph), multi_gpu.cu (sharding, exchange, peer replicas),
// frames.cu (odometry, preprocessing).  None of them contains a kernel.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/badba.h"
#include "host_math.hpp"
#include "kernels.cuh"
#include "odometry.cuh"

namespace bba {

// ---- owners ------------------------------------------------------------------------------------------------------------------
// One CUDA resource (a pointer, event, array or texture object) that Free releases when its owner is destroyed or assigned to.
template <class R, auto Free>
struct Owned {
  R r{};
  Owned() = default;
  Owned(Owned&& o) noexcept : r(o.r) { o.r = R{}; }
  Owned& operator=(Owned&& o) noexcept {
    Owned old(std::move(*this));
    r = o.r;
    o.r = R{};
    return *this;
  }
  ~Owned() {
    if (r) Free(r);
  }
  operator R() const { return r; }
};

// `count` elements of T from Alloc, released by Free.  Reserve(need, alloc) grows on demand: nothing happens when the buffer
// exists and holds `need` elements; otherwise the old buffer is freed first and max(need, alloc) elements are allocated (alloc:
// headroom for later growth).  Pointer and capacity change together, after the allocation succeeded; a failed call leaves no
// buffer.
template <class T, cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
class Buffer {
 public:
  cudaError_t Reserve(size_t need, size_t alloc = 0) {
    if (p_.r && need <= count_) return cudaSuccess;
    p_ = {};
    count_ = 0;
    void* p = nullptr;
    if (cudaError_t e = Alloc(&p, sizeof(T) * std::max(need, alloc))) return e;
    p_.r = static_cast<T*>(p);
    count_ = std::max(need, alloc);
    return cudaSuccess;
  }
  T* get() const { return p_.r; }
  operator T*() const { return p_.r; }
  T* operator->() const { return p_.r; }

 private:
  Owned<T*, Free> p_;
  size_t count_ = 0;
};

inline cudaError_t MappedAlloc(void** p, size_t bytes) { return cudaHostAlloc(p, bytes, cudaHostAllocMapped); }
template <class T> using DeviceBuffer = Buffer<T, cudaMalloc, cudaFree>;
template <class T> using PinnedBuffer = Buffer<T, cudaMallocHost, cudaFreeHost>;
template <class T> using MappedBuffer = Buffer<T, MappedAlloc, cudaFreeHost>;   // pinned host memory the device can address

// A pitched 2-D device image; Allocate (re)allocates it, and a failed call leaves no image.
class PitchedBuffer {
 public:
  cudaError_t Allocate(size_t width_bytes, size_t height) {
    p_ = {};
    pitch_ = 0;
    void* p = nullptr;
    size_t pitch = 0;
    if (cudaError_t e = cudaMallocPitch(&p, &pitch, width_bytes, height)) return e;
    p_.r = p;
    pitch_ = pitch;
    return cudaSuccess;
  }
  template <class T = uint8_t> T* get() const { return static_cast<T*>(p_.r); }
  size_t pitch() const { return pitch_; }
  explicit operator bool() const { return p_.r != nullptr; }

 private:
  Owned<void*, cudaFree> p_;
  size_t pitch_ = 0;
};

using Event = Owned<cudaEvent_t, cudaEventDestroy>;

// A texture object and, when the texture reads a CUDA array, that array (released after the texture).
struct Texture {
  Owned<cudaArray_t, cudaFreeArray> array;
  Owned<cudaTextureObject_t, cudaDestroyTextureObject> tex;
};

// ---- keyframes ---------------------------------------------------------------------------------------------------------------
struct Keyframe {
  // what the kernels read: the caller's buffers, or the owned copies below
  const uint16_t* depth = nullptr;
  const uint16_t* normals = nullptr;
  const uint16_t* radius = nullptr;
  size_t depth_pitch = 0, normals_pitch = 0, radius_pitch = 0;
  cudaTextureObject_t tex = 0;     // luma.tex, or a texture the entry borrows
  const uint8_t* rgba = nullptr;   // uchar4 colour image (caller-owned, or owned_rgba): surfel colours at creation
  size_t rgba_pitch = 0;
  PitchedBuffer owned[3];          // depth / normals / radius copies made by bba_add_keyframe_host
  PitchedBuffer owned_rgba;
  Texture luma;                    // library-owned u8 CUDA array (the .w channel of the colour image) + its texture
  int last_active_in_ba_iteration = -1;   // keyframe.cc:47-48
  int last_covis_in_ba_iteration = -1;
  Pose pose;                 // global_T_frame
  int activation = BBA_KF_ACTIVE;
  float min_depth = 0.f, max_depth = 0.f;
  Frustum frustum;
  std::vector<int> covis;
};

// ---- the front end's view (badba.h "Conventions"; DESIGN.md "Front end beside a running BA") -----------------------------------
// What front-end calls read of a keyframe: copied from its Keyframe record whenever the BA side publishes.
struct KeyframeView {
  const uint16_t* depth = nullptr;
  const uint16_t* normals = nullptr;
  size_t depth_pitch = 0, normals_pitch = 0;
  cudaTextureObject_t tex = 0;
  Pose pose;
  float min_depth = 0.f, max_depth = 0.f;
  int activation = BBA_KF_ACTIVE;
  PosePrior prior{};
};

// A soft relative pose constraint as the handle keeps it: its id, the caller's record, and the information of the equivalent
// prior on keyframe_a (host_math.hpp PoseConstraintInformationA).
struct PoseConstraint {
  int id;
  bba_pose_constraint c;
  float info_a[21];
};

// The cameras, the depth deformation parameter a, the residual types and the deterministic mode as the BA side published them last.
struct CameraView {
  float depth_K[4] = {}, color_K[4] = {};
  float depth_a = 0.f;
  int use_depth = 1, use_desc = 1;
  int deterministic = 0;
};

// The u8 planes that luma extraction writes before the copies into CUDA arrays (stacked, `planes` colour images high), the
// source table of the images after the first (pinned upload copy + device table) and the event after which the next user may
// overwrite them (MakeLumaTextures).
struct LumaStaging {
  PitchedBuffer plane;
  int planes = 0;
  PinnedBuffer<LumaSource> table_upload;
  DeviceBuffer<LumaSource> table;
  Event free;
};

}  // namespace bba

struct bba_context {
  bba_config cfg;
  float depth_K[4], color_K[4];
  float depth_a = 0.f;
  int cf_w = 0, cf_h = 0;
  int sm_count = 132;
  // bba_last_error: the message of the last failed call per calling thread
  std::mutex error_mu;
  std::map<std::thread::id, std::string> errors;

  float* surfels = nullptr;
  size_t surfel_pitch_bytes = 0;
  uint32_t surfels_size = 0;
  uint8_t* active = nullptr;
  bba::DeviceBuffer<float> owned_surfels;   // bba_set_surfels_host
  size_t owned_surfel_pitch = 0;
  bba::DeviceBuffer<uint8_t> owned_active;

  bba::DeviceBuffer<float> d_cfactor;
  std::vector<bba::Keyframe> keyframes;
  bba::DeviceBuffer<bba::KfDevice> d_kfs;   // [max_kf] the keyframes' parameters as the kernels read them
  // soft pose priors by keyframe id (bba_set_keyframe_pose_priors) and how many keyframes have one; with no prior and no
  // constraint the pose solve and the PCG solver run without pose terms
  std::vector<bba::PosePrior> pose_priors;   // [max_kf]
  int pose_prior_count = 0;
  // soft relative pose constraints (bba_add_keyframe_pose_constraints) in id order, and the id the next one gets
  std::vector<bba::PoseConstraint> pose_constraints;
  int next_pose_constraint_id = 0;

  // staging: pinned records and the shared planes of the keyframe / frame uploads
  struct Staging {
    bba::PinnedBuffer<bba::KfDevice> h_kfs;
    bba::Event event;      // recorded after the last upload from the pinned staging buffers
    bool pending = false;
    bba::LumaStaging luma;      // luma staging of the BA side: keyframes and bba_estimate_frame_poses_for_frames
    bba::PitchedBuffer color;   // uchar4 staging image for bba_update_keyframe_host
  } staging;

  // Luma of the frames that are not keyframes (bba_estimate_frame_poses_for_frames, pose_step.cu): one array + texture per
  // distinct frame of a chunk, created on first use; the pool is trimmed to the free keyframe slots at the start of a call.
  std::vector<bba::Texture> frame_luma;

  // pose step (pose_step.cu) and the spatial order of the surfels
  struct PoseStep {
    bba::DeviceBuffer<bba::KfDevice> d_work_records;   // [max_kf] the pose kernel's work list as contiguous records
    bba::DeviceBuffer<float> d_pose_est;
    bba::DeviceBuffer<double> d_acc;
    bba::DeviceBuffer<bba::ExactSum> d_exact;   // deterministic mode: [max_kf][32], the pose kernel's sums instead of d_acc
    bba::DeviceBuffer<unsigned long long> d_stage_counts;
    bba::DeviceBuffer<int> d_work[2];
    bba::DeviceBuffer<int> d_count;   // 2 ints
    bba::DeviceBuffer<int> d_iterations;
    bba::DeviceBuffer<int> d_converged;
    bba::DeviceBuffer<double> d_first_stats;
    bba::DeviceBuffer<unsigned long long> d_totals;   // [8]
    bba::DeviceBuffer<unsigned int> d_queue;          // work-item counter of the pose kernel
    bba::MappedBuffer<int> flag;         // 4 ints
    volatile int* h_flag = nullptr;      // flag: {iterations completed, work items left}
    int* d_flag = nullptr;               // device alias of h_flag
    bba::PinnedBuffer<float> h_pose_est;
    bba::PinnedBuffer<int> h_work;   // max_kf + 2
    bba::PinnedBuffer<int> h_iterations;
    bba::PinnedBuffer<int> h_converged;
    bba::PinnedBuffer<double> h_first_stats;
    bba::PinnedBuffer<unsigned long long> h_totals;
    // the soft pose terms of the keyframes in the step (StagePoseTerms): CSR offsets [max_kf + 1] and records, staged at the
    // start of every pose step; reserved by the calls that add priors or constraints
    bba::PinnedBuffer<int> h_term_offsets;
    bba::DeviceBuffer<int> d_term_offsets;
    bba::PinnedBuffer<bba::PoseTerm> h_terms;
    bba::DeviceBuffer<bba::PoseTerm> d_terms;
    // Spatial order of the surfels (bba::LaunchSpatialOrder) and the pose step's stream in that order (bba::LaunchPoseStream); the
    // geometry step's stream (bba::LaunchGeometryStream) shares the buffer.
    // The order is rebuilt at the start of every BA call, after an in-loop change of the surfel set, and whenever the surfel
    // count differs from the one it was built for; in between it may lag behind the positions, which costs culling, never
    // correctness.
    struct Order {
      bba::DeviceBuffer<uint32_t> words;       // keys in / out, index, perm, 8 bound words
      bba::DeviceBuffer<unsigned char> temp;   // CUB scratch
      bba::DeviceBuffer<float> stream;         // [kPoseStreamRows][capacity], rebuilt at the start of a pose step / geometry launch
      bba::DeviceBuffer<float> boxes;          // [capacity / kSpatialChunk][8]
      bba::SpatialOrderBuffers view{};
      uint32_t capacity = 0;                   // also the stream's pitch
    } order;
    uint32_t order_n = 0;
    bool order_stale = true;
    int group = 0;   // keyframes per work item of the pose kernel (bba_debug_set_pose_group); 0: the launcher's choice
  } pose;

  // geometry step and intrinsics step (bundle_adjust.cu)
  struct Geometry {
    bba::DeviceBuffer<int> d_list;
    bba::PinnedBuffer<int> h_list;
    bba::DeviceBuffer<unsigned int> d_queue;        // work-item counter of the geometry kernels
    bba::DeviceBuffer<unsigned int> d_tile_epoch;   // per-tile group epochs of the geometry kernels
    const uint32_t* perm = nullptr;   // the order of the last geometry launches (pose.order's perm or null), for ExchangeGeometry
    // intrinsics step: [head 64 | B 5P | D P | b2 P | obs P | x1 8] floats + 34 fp64 sums
    bba::DeviceBuffer<float> d_intr;
    bba::DeviceBuffer<double> d_intr_sums;
    bba::DeviceBuffer<bba::ExactSum> d_intr_exact;   // deterministic mode: [7 P] per-cell sums (B rows, D, b2) + kIntrinsicsSums
    bba::DeviceBuffer<int> d_all_list;   // 0 .. max_kf-1
    bba::PinnedBuffer<double> h_intr_sums;
    bba::PinnedBuffer<float> h_intr_x1;   // 8 floats
  } geo;

  // surfel deformation (bba_deform_surfels): the keyframe records at the caller's original poses, the keyframes' pose changes and
  // the two counters
  struct Deform {
    bba::PinnedBuffer<bba::KfDevice> h_kfs;
    bba::DeviceBuffer<bba::KfDevice> d_kfs;
    bba::PinnedBuffer<bba::KfChange> h_changes;
    bba::DeviceBuffer<bba::KfChange> d_changes;
    bba::DeviceBuffer<unsigned int> d_counts;   // [2] moved, unobserved
    bba::PinnedBuffer<unsigned int> h_counts;
  } deform;

  // keyframe pose graph (bba_optimize_pose_graph): the terms, the held flags, the row lists and the block-CSR structure (one pinned
  // staging buffer of ints and its device copy), the fp32 poses and the state; the terms' blocks, H, b, M and the solver's work in
  // one fp64 buffer.  Sized for max_keyframes and the constraints, with room to double the constraints (ReservePoseGraph).
  struct PoseGraph {
    bba::PinnedBuffer<bba::PoseGraphTerm> h_terms;
    bba::DeviceBuffer<bba::PoseGraphTerm> d_terms;
    bba::PinnedBuffer<int> h_ints;
    bba::DeviceBuffer<int> d_ints;
    bba::PinnedBuffer<float> h_poses;        // [max_kf][7]
    bba::DeviceBuffer<float> d_poses;        // [2][max_kf][7]: the poses, then the poses before the last step
    bba::DeviceBuffer<double> d_doubles;
    bba::DeviceBuffer<bba::PoseGraphState> d_state;
    bba::PinnedBuffer<bba::PoseGraphState> h_state;
  } graph;

  // in-loop surfel lifecycle (creation / merge / compaction) and the end tasks
  struct Lifecycle {
    bba::DeviceBuffer<unsigned int> d_sup;         // [3][cells]
    bba::DeviceBuffer<unsigned int> d_cell_bits;   // [cells]
    bba::DeviceBuffer<unsigned int> d_flags;       // [w * h]
    bba::DeviceBuffer<unsigned int> d_scan_out;    // [w * h]
    bba::DeviceBuffer<unsigned int> d_scan_sums;   // block sums of the creation's and the compaction's scan
    bba::DeviceBuffer<bba::CovisEntry> d_covis;    // [max_keyframes]
    bba::PinnedBuffer<bba::CovisEntry> h_covis;
    bba::DeviceBuffer<bba::KfRadius> d_kf_radius;  // [max_keyframes]
    bba::PinnedBuffer<bba::KfRadius> h_kf_radius;
    bba::DeviceBuffer<unsigned int> d_deleted_count;
    bba::PinnedBuffer<unsigned int> h_count;       // a created or deleted count on its way to the host
  } life;
  int last_ba_iteration_count = -1;   // direct_ba.cc:126

  // PCG solver: r, M, delta, g, p
  struct Pcg {
    bba::DeviceBuffer<float> d_vec[5];
    bba::DeviceBuffer<double> d_scalars;   // [0] / [2] alpha_n, beta_n (roles swap), [1] alpha_d
    bba::PinnedBuffer<double> h_scalars;
    bba::PinnedBuffer<float> h_delta;      // pose part (6 * max_keyframes) + 16
    // the pose-block terms (priors, constraints) at the poses of the current outer iteration (StagePcgPoseTerms)
    bba::PinnedBuffer<bba::PcgPoseBlock> h_pose_blocks;
    bba::DeviceBuffer<bba::PcgPoseBlock> d_pose_blocks;
    bba::PinnedBuffer<bba::PcgPoseTerm> h_pose_terms;
    bba::DeviceBuffer<bba::PcgPoseTerm> d_pose_terms;
    int pose_blocks = 0;
  } pcg;

  // multi-GPU exchange (multi_gpu.cu)
  struct Exchange {
    bba_collective_fn collective = nullptr;
    void* collective_user = nullptr;
    // The local group this handle is a member of (local_group.cu), and the reason its last exchange failed: a local group's
    // collective returns nothing, so it leaves the reason here for Collective.
    bba_local_group group = nullptr;
    std::string exchange_error;
    bba::DeviceBuffer<float> d_exchange;    // [world][rows][shard_len] floats, rows <= kShardRows (ExchangeShards)
    bba::DeviceBuffer<float> d_pose_pack;   // [max_kf][kPoseSlot] floats
    bba::PinnedBuffer<float> h_pose_pack;
    bba::DeviceBuffer<int> d_local_ids;     // [max_kf]
    bba::DeviceBuffer<float> d_count_xchg;  // [2] this rank's count for the sum all-reduce (SumOverRanks)
    bba::PinnedBuffer<float> h_count_xchg;
    bba::DeviceBuffer<float> d_barrier;
    // NVLink peer replicas (bba_peer_import)
    bba::PeerSet peers{};                       // count == 0: not mapped
    void* peer_bases[2 * bba::kMaxPeers] = {};  // what cudaIpcOpenMemHandle returned (closed on unmap)
    int peer_base_count = 0;
    // With mapped peers: set by every REPLICATED whole-buffer pass (surfel creation / merge / compaction / end tasks), cleared
    // by the next collective.  The geometry kernels store into the other ranks' replicas; a rank must not start them while a
    // slower rank is still reading or rewriting its whole replica in such a pass (PeerFence).
    bool replicated_pass_pending = false;
  } xchg;

  // image-pair odometry (bba_track_frame_pairwise, bba_track_frames_pairwise), lazily allocated: a pool of pyramids, one per
  // distinct image and role of a chunk (the intensity / gradient-magnitude plane, colour-sized, and the depth / normal / colour
  // levels), the chunk's image and entry tables, accumulators + barriers + results of the persistent kernel
  struct Pyramid {
    bba::PitchedBuffer gradmag;
    bba::Texture gradmag_tex;
    bba::PitchedBuffer depth[bba::odom::kMaxScales], normals[bba::odom::kMaxScales], color[bba::odom::kMaxScales];
    bba::Texture color_tex[bba::odom::kMaxScales];
    bba::odom::Image image[bba::odom::kMaxScales] = {};   // views of the planes above
  };
  struct Odometry {
    int num_scales = 0;          // levels allocated in every pyramid of the pool
    int last_num_scales = 0;     // levels filled by the last call (parity hooks)
    int last_first_scale = 0;
    std::vector<std::unique_ptr<Pyramid>> pool;
    int w[bba::odom::kMaxScales] = {}, h[bba::odom::kMaxScales] = {};
    // The last chunk's tables as the kernels read them; the parity hooks work on its last entry.
    bba::odom::LevelCamera cam[bba::odom::kMaxScales] = {};
    bba::odom::Image last_level[2][bba::odom::kMaxScales] = {};   // [0 base | 1 tracked][scale] of the last entry
    bba::odom::TrackEntry last_entry{};
    bba::PinnedBuffer<bba::odom::PyramidImage> h_images;
    bba::DeviceBuffer<bba::odom::PyramidImage> d_images;
    bba::PinnedBuffer<bba::odom::TrackEntry> h_entries;
    bba::DeviceBuffer<bba::odom::TrackEntry> d_entries;
    bba::DeviceBuffer<double> d_acc;             // [groups][3][32]
    bba::DeviceBuffer<double> d_partials;        // deterministic mode: [groups][3][virtual grid][32] (TrackArgs::partials)
    bba::DeviceBuffer<unsigned int> d_control;   // TrackArgs::control
    bba::DeviceBuffer<bba::odom::TrackResult> d_result;   // [entries of a chunk]
    bba::PinnedBuffer<bba::odom::TrackResult> h_result;
  } odo;

  // keyframe preprocessing (bba_preprocess_frame)
  struct Preprocess {
    bba::DeviceBuffer<float> d_min_max;
    bba::PinnedBuffer<float> h_min_max;
  } pre;

  // The state front-end calls read (Publish writes it; FrontEndCall takes a snapshot), and the buffers only they use.  Front-end
  // calls never touch the live state above, which the BA side changes while it runs.
  struct FrontEnd {
    std::mutex mu;                       // guards the published fields below; never held across a launch or a synchronise
    std::condition_variable slot_free;   // a cfactor slot lost its last reader
    bba::CameraView cams;
    std::vector<bba::KeyframeView> kfs;
    std::vector<bba::PoseConstraint> constraints;   // the soft relative pose constraints, in id order
    // Two device copies of the cfactor.  Publish copies d_cfactor into the slot that is not current, on the BA side's stream,
    // after that slot's readers are done, records `published` and makes the slot current; a front-end call claims the
    // current slot, makes its stream wait on `published` and records `readers_done` after its last read.
    bba::DeviceBuffer<float> cfactor[2];
    bba::Event published[2];
    bba::Event readers_done[2];
    int current = 0;
    int readers[2] = {0, 0};   // claims between FrontEndCall::Snapshot and ReleaseSlot
    std::mutex call;           // serialises the front-end calls that use the buffers below and odo / pre
    bba::LumaStaging luma;
    std::vector<bba::Texture> frames;   // luma of the distinct frames of an odometry chunk, grown on demand
  } fe;

  // kernels launched by BA-side calls and by front-end calls (bba_kernel_launch_count: the sum); two counters so that the
  // launches a BA call reports are its own while the front end runs beside it
  std::atomic<uint64_t> launches{0};
  std::atomic<uint64_t> front_end_launches{0};
  int ba_iteration_count = 0;
  // predicted cost of one pose step per keyframe (Gauss-Newton iterations x per-evaluation cost of the last step it took
  // part in); 0 = unknown.  Identical on every rank; drives the keyframe -> rank assignment of the pose step.
  std::vector<float> kf_cost;

  // deterministic mode (bba_set_deterministic): exact or fixed-order sums on the pose, intrinsics and odometry paths
  bool deterministic = false;

  // profiling (bba_set_profiling)
  int profiling = 0;   // 0 off, 1 event timing, 2 event timing + byte-model counters in every iteration
  bba_profile profile;
  bba::Event prof_ev[64];
  bba::Event ev[6];
};

namespace bba {

// Sets the calling thread's bba_last_error message and returns s.  A failure of a BA-side call on a member of a local group
// poisons the group, so that the other ranks' exchanges return instead of waiting for this rank (FrontEndScope).
bba_status Fail(bba_handle h, bba_status s, const std::string& msg);
// Sets the calling thread's bba_last_error message.
void SetError(bba_handle h, const std::string& msg);

// Marks the calling thread as inside a front-end call (badba.h "Conventions") while it lives: its failures concern that call
// only and leave the handle's local group in service.
class FrontEndScope {
 public:
  FrontEndScope() { ++depth_; }
  ~FrontEndScope() { --depth_; }
  FrontEndScope(const FrontEndScope&) = delete;
  FrontEndScope& operator=(const FrontEndScope&) = delete;
  static bool active() { return depth_ > 0; }

 private:
  static thread_local int depth_;
};

// local_group.cu
void PoisonLocalGroup(bba_local_group g);

#define BBA_CUDA(h, expr)                                                                                  \
  do {                                                                                                      \
    cudaError_t e__ = (expr);                                                                               \
    if (e__ != cudaSuccess)                                                                                 \
      return Fail(h, BBA_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__));                    \
  } while (0)

// Calls launcher(...), adds the kernels it enqueued to `counter` (h->launches or h->front_end_launches) and fails when the
// launcher or the runtime's last error reports an error.  Never synchronises: a fault while a kernel runs surfaces later.
#define BBA_LAUNCH(h, counter, launcher, ...)                                                                \
  do {                                                                                                      \
    const ::bba::LaunchResult r__ = launcher(__VA_ARGS__);                                                  \
    (counter) += r__.kernels;                                                                               \
    const cudaError_t last__ = cudaGetLastError();                                                          \
    const cudaError_t e__ = r__.error != cudaSuccess ? r__.error : last__;                                  \
    if (e__ != cudaSuccess) return Fail(h, BBA_ERR_CUDA, std::string(#launcher) + ": " + cudaGetErrorString(e__)); \
  } while (0)

// BADBA_TRACE=1: stage markers on stderr (debugging aid for host-side faults)
#define BBA_TRACE(msg)                                                                   \
  do {                                                                                   \
    static const bool on__ = std::getenv("BADBA_TRACE") != nullptr;                      \
    if (on__) { std::fprintf(stderr, "[badba] %s:%d %s\n", __func__, __LINE__, msg); std::fflush(stderr); } \
  } while (0)

#define CHECK_KF(h, id)                                                                   \
  if (!(h)) return BBA_ERR_INVALID_ARGUMENT;                                              \
  if ((id) < 0 || (id) >= static_cast<int>((h)->keyframes.size())) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bad keyframe id")

// badba.cu
Pose PoseFromArray(const float p[7]);
void PoseToArray(const Pose& r, float p[7]);
// The camera of the BA side's live state, or of a published view with the cfactor slot it claimed.
CameraParams MakeCamera(bba_handle h);
CameraParams MakeCamera(bba_handle h, const CameraView& v, const float* cfactor);
// Publishes the cameras, residual types and keyframe records for the front end and, with `cfactor`, a copy of d_cfactor
// enqueued on s (BA side only; after every change of that state).
bba_status Publish(bba_handle h, cudaStream_t s, bool cfactor);

// The snapshot a front-end call reads instead of the live state.  Snapshot copies the published cameras (and the record of
// keyframe `kf_id` when >= 0) under fe.mu and claims the current cfactor slot: s waits for its publication.  ReleaseSlot
// drops the claim after the call's last read of the slot: with `record`, s first waits for the slot's previous readers and
// then records "readers done" (without, the caller has synchronised s).  The destructor releases a claim still held.
class FrontEndCall {
 public:
  explicit FrontEndCall(bba_handle h) : h_(h) {}
  ~FrontEndCall() { ReleaseSlot(); }
  FrontEndCall(const FrontEndCall&) = delete;
  FrontEndCall& operator=(const FrontEndCall&) = delete;
  // (max_kf_id: fails unless every keyframe id up to it is published; all_kfs: receives every published keyframe record)
  bba_status Snapshot(cudaStream_t s, int kf_id, const char* fn, int max_kf_id = -1, std::vector<KeyframeView>* all_kfs = nullptr);
  bba_status ReleaseSlot(bool record = true);
  CameraView cams;
  KeyframeView base;
  const float* cfactor = nullptr;

 private:
  bba_handle h_;
  cudaStream_t s_ = nullptr;
  int slot_ = -1;
};

bba_status WaitStaging(bba_handle h);
bba_status MarkStaging(bba_handle h, cudaStream_t s);
void FillKfDevice(const Keyframe& kf, const Pose& global_T_frame, KfDevice* d);
bba_status UploadKeyframes(bba_handle h, cudaStream_t s);
bba_status CheckSurfels(bba_handle h);
// Whether the depth / normal / colour pitches of a frame hold rows of the configured image sizes (and fit kernel arguments).
bool FramePitchesOk(bba_handle h, size_t depth_pitch, size_t normals_pitch, size_t color_pitch);
// Clamp addressing, linear filtering, normalised float reads and unnormalised coordinates (keyframe.cc:67-73, and
// CUDABuffer::CreateTextureObject as pairwise_frame_tracking.cc:57-79 calls it).
cudaTextureDesc LinearTextureDesc();
// The surfel buffer's pitch in floats, as the kernels take it.
inline uint32_t SurfelPitch(bba_handle h) { return static_cast<uint32_t>(h->surfel_pitch_bytes / sizeof(float)); }
// The camera, the surfel buffer, its pitch in floats and the surfel count in kernel arguments.
template <class Args> void SetSurfelFields(bba_handle h, Args* a) {
  a->cam = MakeCamera(h);
  a->surfels = h->surfels;
  a->pitch = SurfelPitch(h);
  a->n = h->surfels_size;
}
// The luma textures of n >= 1 colour images in device memory (sources[i] -> *out[i]): one extraction launch and one copy per
// image into its array.  front_end: through fe.luma, counted as front-end launches; otherwise through staging.luma.
bba_status MakeLumaTextures(bba_handle h, bool front_end, int n, const LumaSource* sources, Texture* const* out, cudaStream_t s);
// The luma textures of the frames `uses` names (indices into frames, repeats allowed) in one MakeLumaTextures call: the distinct
// frames in first-use order get (*pool)[0], (*pool)[1], ..., and luma[f] becomes frame f's texture.  The pool grows when it holds
// fewer textures than there are distinct frames.
bba_status MakeFrameLumaTextures(bba_handle h, bool front_end, const bba_frame_buffers* frames, const std::vector<int>& uses,
                                 std::vector<Texture>* pool, cudaTextureObject_t* luma, cudaStream_t s);

// pose_step.cu
// The surfel count from which a launch over n keyframes puts the surfels into spatial order: sorting costs ~0.1 ms of launches
// plus the sort itself, more than the culling it buys on small work (PreparePoseAccumulate).
constexpr uint64_t kSpatialOrderMinPairs = 16u << 20;   // (surfel, keyframe) pairs per launch
bba_status EnsureSpatialOrder(bba_handle h, bool sort, bool rebuild, cudaStream_t s);
bba_status RunPoseStep(bba_handle h, const std::vector<int>& ids, const std::vector<Pose>& init, int max_iterations, cudaStream_t s);
// Reserves the staging buffers of the soft pose terms (pose step and PCG) for a prior on every keyframe and `constraints`
// constraints, with room to double the constraints before the next allocation.  The calls that add priors or constraints make
// it before they change anything; the staging repeats it, a no-op unless an earlier reservation failed.
bba_status ReservePoseTerms(bba_handle h, size_t constraints);
// The soft relative pose constraints that touch each of the first K keyframes, in id order: indices into
// h->pose_constraints, adj[off[k] .. off[k + 1]).
void ConstraintAdjacency(bba_handle h, int K, std::vector<int>* off, std::vector<int>* adj);

// multi_gpu.cu
void ShardSurfels(uint32_t n, int rank, int world, uint32_t* local_cap, uint32_t* shard_len);
uint32_t LocalCountBelow(uint32_t global_end, int rank, int world);
void AssignKeyframes(bba_handle h, const std::vector<int>& ids, std::vector<int>* owner);
bba_status CheckCollective(bba_handle h);
// Runs the registered exchange (bba_set_collective or a local group) on `buffer`; fails with BBA_ERR_STATE when a local
// group's exchange did not complete (its group is poisoned).
bba_status Collective(bba_handle h, int op, void* buffer, size_t count, cudaStream_t s);
// The sum of every rank's `count` in *total, through one sum all-reduce (a barrier) and a synchronise of s.
bba_status SumOverRanks(bba_handle h, uint32_t count, cudaStream_t s, uint32_t* total);
// Whether the kernels store their shard's surfel rows into every rank's replica (bba_peer_import) instead of an exchange.
bool PeerStores(bba_handle h);
// The peer replicas kernel arguments get: empty unless PeerStores.
PeerSet KernelPeers(bba_handle h);
bba_status PeerFence(bba_handle h, cudaStream_t s);
bba_status ExchangeShards(bba_handle h, const ShardRows& rows, const uint32_t* perm, cudaStream_t s);
bba_status ExchangeGeometry(bba_handle h, cudaStream_t s);
void UnmapPeers(bba_handle h);

// The range of this rank's surfel shard (all surfels on one GPU) in kernel arguments.
template <class Args> void SetShardFields(bba_handle h, Args* a) {
  a->begin = 0;
  a->shard_rank = static_cast<uint32_t>(h->cfg.rank);
  a->shard_world = static_cast<uint32_t>(h->cfg.world_size);
  ShardSurfels(h->surfels_size, h->cfg.rank, h->cfg.world_size, &a->end, nullptr);
}

}  // namespace bba
