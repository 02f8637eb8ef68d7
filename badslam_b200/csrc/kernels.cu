// kernels.cu -- hand-written sm_90a kernels of the direct-BA hot path.
//
//  * PoseAccumulateKernel: ONE persistent launch evaluates the pose normal equations of a whole LIST of
//    keyframes (the reference launches AccumulatePoseEstimationCoeffsCUDAKernel once per keyframe and
//    Gauss-Newton iteration, kernel_opt_pose.cc:74-88).  Surfel tiles are staged into shared memory by the
//    TMA engine (cp.async.bulk + mbarrier, double-buffered); each warp owns (tile, keyframe) work items,
//    keeps the 21 H + 6 b + 5 bookkeeping sums in registers across the whole tile, and reduces them with a
//    31-shuffle transposed butterfly followed by one fp64 RED per lane (the reference does 27 block-wide CUB
//    reductions + atomics per residual type per 256 surfels, gauss_newton.cuh:59-92).  The PRE instantiations split the CTA
//    into producer warps (association) and consumer warps (sums, reduction), see PoseAccumulateKernel.
//  * ActivationNormalsKernel / PositionDescriptorKernel: surfel-major geometry step.  One thread owns one
//    surfel, loops over all non-inactive keyframes with the accumulators in registers and applies the update
//    in the same kernel -- the reference's reset / K x accumulate / update launch chain with 16-72 bytes of
//    read-modify-write per associated pair (kernel_opt_geometry.cc:114-199) becomes one pass with none.
//  * GeometryPassKernel: both of them in one tile-major launch, for the iterations without new surfels.
//
// Built with -use_fast_math like the reference (applications/badslam/CMakeLists.txt:74-75).
#include "persistent.cuh"

#include <cuda.h>

#include <algorithm>

namespace bba {

// ------------------------------------------------------------------------------------------------
// mbarrier / bulk-copy (TMA) primitives, raw PTX.

__device__ __forceinline__ uint32_t SmemAddr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void MbarInit(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(SmemAddr(bar)), "r"(count));
}
__device__ __forceinline__ void FenceBarrierInit() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void MbarArriveExpectTx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(SmemAddr(bar)), "r"(bytes) : "memory");
}
// (MbarArrive / MbarWait / MbarTest take the barrier's shared-memory address, SmemAddr, so that a loop can keep it in a register.)
__device__ __forceinline__ void MbarArrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void MbarWait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra.uni WAIT_DONE;\n"
      "bra.uni WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
// Non-blocking form of MbarWait: has the phase of the given parity completed?
__device__ __forceinline__ bool MbarTest(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}
// 1-D bulk copy global -> shared, completion signalled on an mbarrier (TMA engine; SASS UBLKCP).
__device__ __forceinline__ void BulkCopyG2S(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(SmemAddr(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(SmemAddr(bar))
               : "memory");
}

// ------------------------------------------------------------------------------------------------

// A texture handle that is the same in every lane, said in a way ptxas can see (a shuffle from lane 0): without it every
// TEX / TLD4 is wrapped in a per-lane "waterfall" loop (R2UR + predicated fetch + BRA.U.ANY, ~8 extra instructions per fetch).
// Must be called by all 32 lanes.
__device__ __forceinline__ cudaTextureObject_t UniformTexture(cudaTextureObject_t tex) {
  const unsigned long long t = tex;
  const unsigned lo = __shfl_sync(0xffffffffu, static_cast<unsigned>(t), 0);
  const unsigned hi = __shfl_sync(0xffffffffu, static_cast<unsigned>(t >> 32), 0);
  return (static_cast<unsigned long long>(hi) << 32) | lo;
}

constexpr int kPoseMinCtas = 2;      // resident CTAs per SM the register allocation is tuned for
constexpr int kPoseChunkShift = 8;   // log2 of the surfels one warp evaluates per (keyframe) sub-item
constexpr int kPoseThreads = 256;
constexpr int kPoseUnroll = 1;       // surfels of a chunk evaluated concurrently per lane
constexpr int kPoseStagedRows = 7;   // x y z normal radius^2 d1 d2
constexpr int kPoseStagedRowsPre = 14;   // x y z d1 d2 + the 9 frame rows (normal, tangent point 1, tangent point 2)
static_assert(kPoseStagedRowsPre == kPoseStreamRows, "the PRE instantiations stage every row of the pose stream");

// Does the axis-aligned box {min x y z, -, max x y z, -} lie surely outside the view of the keyframe with frame_T_global T, i.e.
// would ProjectIntoImage reject every position in it?  The box is culled when its 8 corners all lie beyond one plane: z = 0 or one
// of the four image borders moved out by a pixel.  Each plane test is f(p) < -e A(p) with f linear in the camera-frame point
// (e.g. fx x + (cx + 1) z for the left border) and A(p) the same sum over absolute terms (A >= the size of every intermediate in
// fp32); f + e A is convex, so the test holding at the corners holds everywhere in the box.  With e = 1e-5, some 80 fp32 ulps,
// it absorbs the rounding of this test and of the kernel's own transform, so that the kernel's fp32 z is <= 0 or its pixel
// coordinate at least about a pixel beyond the border: culling drops no pair that the kernel would have found in the image.
// Non-finite boxes compare false and are never culled.
// PlanesOutside: the planes (bit 0 z = 0, bits 1-4 the borders) that the point (px, py, pz) lies beyond.
__device__ __forceinline__ unsigned PlanesOutside(const CameraParams& cam, const float* __restrict__ T, float px, float py, float pz) {
  float v[3], a[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    v[r] = T[4 * r] * px + T[4 * r + 1] * py + T[4 * r + 2] * pz + T[4 * r + 3];
    a[r] = fabsf(T[4 * r] * px) + fabsf(T[4 * r + 1] * py) + fabsf(T[4 * r + 2] * pz) + fabsf(T[4 * r + 3]);
  }
  constexpr float e = 1e-5f;
  const float l_x = cam.cx + 1.f, r_x = cam.cx - static_cast<float>(cam.w) - 1.f;
  const float l_y = cam.cy + 1.f, r_y = cam.cy - static_cast<float>(cam.h) - 1.f;
  unsigned out = (v[2] < -e * a[2]) ? 1u : 0u;
  out |= (cam.fx * v[0] + l_x * v[2] < -e * (cam.fx * a[0] + fabsf(l_x) * a[2])) ? 2u : 0u;
  out |= (cam.fx * v[0] + r_x * v[2] > e * (cam.fx * a[0] + fabsf(r_x) * a[2])) ? 4u : 0u;
  out |= (cam.fy * v[1] + l_y * v[2] < -e * (cam.fy * a[1] + fabsf(l_y) * a[2])) ? 8u : 0u;
  out |= (cam.fy * v[1] + r_y * v[2] > e * (cam.fy * a[1] + fabsf(r_y) * a[2])) ? 16u : 0u;
  if (!(cam.fx > 0.f && cam.fy > 0.f)) out &= 1u;   // the border planes assume a camera that does not mirror the image
  return out;
}
// The test spread over a warp: each lane passes one corner (lane L corner L & 7, so that the warp covers all 8); must be called
// by all 32 lanes.
__device__ __forceinline__ bool CornersOutsideView(const CameraParams& cam, const float* __restrict__ T, float px, float py, float pz) {
  return __reduce_and_sync(0xffffffffu, PlanesOutside(cam, T, px, py, pz)) != 0u;
}
// The test within one lane, over all 8 corners of the box {lo x y z} - {hi x y z}: the same per-corner expressions, so the same
// decision as CornersOutsideView on the box's corners.
__device__ __forceinline__ bool BoxOutsideViewLane(const CameraParams& cam, const float* __restrict__ T, const float (&lo)[3],
                                                   const float (&hi)[3]) {
  unsigned out = 0x1fu;
#pragma unroll 1   // unrolled, the eight corners in flight cost the geometry kernels up to 18 registers and an SM's 4th CTA
  for (int c = 0; c < 8; ++c) out &= PlanesOutside(cam, T, (c & 1) ? hi[0] : lo[0], (c & 2) ? hi[1] : lo[1], (c & 4) ? hi[2] : lo[2]);
  return out != 0u;
}
// The same for the box {min x y z, -, max x y z, -}.
__device__ __forceinline__ bool BoxOutsideView(const CameraParams& cam, const float* __restrict__ T, const float* box, int lane) {
  const int c = lane & 7;
  return CornersOutsideView(cam, T, box[(c & 1) ? 4 : 0], box[(c & 2) ? 5 : 1], box[(c & 4) ? 6 : 2]);
}

// Warp-specialised PRE instantiations: two producer warpgroups (association, no accumulators) and one consumer warpgroup (all the
// per-pair maths after the association, the normal-equation sums and the reductions).  Consumer warp c serves producer warps c and
// c + 4 with one accumulator set each.  setmaxnreg moves registers from the producers to the consumers; the three must fit the
// 80 registers per thread that 2 CTAs of 384 threads are launched with: 256 * 72 + 128 * 96 = 384 * 80.
constexpr int kPoseProducerWarps = 8;
constexpr int kPoseConsumerWarps = 4;
constexpr int kPoseWsThreads = 32 * (kPoseProducerWarps + kPoseConsumerWarps);
constexpr int kPoseProducerRegs = 72;
constexpr int kPoseConsumerRegs = 96;
static_assert(kPoseProducerWarps * kPoseProducerRegs + kPoseConsumerWarps * kPoseConsumerRegs ==
                  (kPoseProducerWarps + kPoseConsumerWarps) * 80, "register split");
// A slot holds one 32-surfel step of a producer: lane L's record at position L, whether or not lane L associated.  A record is 15
// floats in four float4 chunks -- {lp.x lp.y lp.z ln.x} {ln.y ln.z d nx} {ny r1 r2 gx1} {gy1 gx2 gy2 -} -- stored chunk-major
// ([chunk][lane]) so that each of the four 16-byte stores and loads of a warp covers 512 contiguous bytes without a bank conflict.
// Each producer owns a ring of two slots with a full / empty mbarrier pair per slot.
constexpr int kPoseRecChunks = 4;
constexpr int kPoseRingSlots = 2;
constexpr int kPoseSlotChunks = kPoseRecChunks * 32;
constexpr size_t kPoseRingBytes = sizeof(float4) * kPoseSlotChunks * kPoseRingSlots * kPoseProducerWarps;

template <int N>
__device__ __forceinline__ void SetMaxRegsDec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void SetMaxRegsInc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N)); }

// The normal-equation sums of one associated pair (kernel_opt_pose.cu:88-142).  photo: the descriptor residuals count.
template <bool STATS>
__device__ __forceinline__ void AccumulatePair(const CameraParams& cam, const Assoc& r, const DescEval& e, bool photo,
                                               float (&acc)[kPoseAccSize]) {
  acc[27] += 1.f;
  if (cam.use_depth) {
    float inv_stddev;
    Vec3 up;
    const float raw = DepthResidual(cam, r, &inv_stddev, &up);
    float J[6];
    DepthPoseJacobian(r, inv_stddev, up, J);
    AccumulateHb(acc, J, raw, DepthWeight(raw));
    if (STATS) acc[29] += DepthCost(raw);
  }
  if (cam.use_desc && photo) {
    acc[28] += 1.f;
    float J[6];
    DescPoseJacobian(cam, r.lp, e.gx1, e.gy1, J);
    AccumulateHb(acc, J, e.r1, DescWeight(e.r1));
    DescPoseJacobian(cam, r.lp, e.gx2, e.gy2, J);
    AccumulateHb(acc, J, e.r2, DescWeight(e.r2));
    if (STATS) {
      acc[30] += DescCost(e.r1);
      acc[31] += DescCost(e.r2);
    }
  }
}

// The same from a pair's record (the four chunks of a slot position, kPoseRecChunks).
template <bool STATS>
__device__ __forceinline__ void AccumulateRecord(const CameraParams& cam, const float4 (&q)[kPoseRecChunks], bool photo,
                                                 float (&acc)[kPoseAccSize]) {
  Assoc r;
  r.lp = V3(q[0].x, q[0].y, q[0].z);
  r.ln = V3(q[0].w, q[1].x, q[1].y);
  r.d = q[1].z;
  r.nx = q[1].w;
  r.ny = q[2].x;
  DescEval e;
  e.r1 = q[2].y;
  e.r2 = q[2].z;
  e.gx1 = q[2].w;
  e.gy1 = q[3].x;
  e.gx2 = q[3].y;
  e.gy2 = q[3].z;
  AccumulatePair<STATS>(cam, r, e, photo, acc);
}

// Where a sub-item's warp total of slot `lane` goes: one fp64 atomic into acc, or (DET, the deterministic mode) a deposit into the
// slot's exact sum, whose value does not depend on the order in which the sub-items finish.  A keyframe's slot receives one deposit
// per sub-item, at most chunks per tile x tiles = ceil(n / 128) <= 2^25 for any surfel count below 2^32: far below the 2^31 deposits
// an ExactSum holds.
template <bool DET>
__device__ __forceinline__ void StorePoseTotal(const PoseAccumulateArgs& args, int kf, int lane, float total) {
  if constexpr (DET) ExactDeposit(args.exact + static_cast<size_t>(kf) * kPoseAccSize + lane, total);
  else atomicAdd(args.acc + static_cast<size_t>(kf) * kPoseAccSize + lane, static_cast<double>(total));
}

// Work decomposition.  A work ITEM is (group of <= args.group keyframes from the work list) x (tile of TILE surfels); items are
// handed out through a global counter in GROUP-MAJOR order, so at any moment all resident CTAs read the images of the
// same one or two groups of keyframes while surfel tiles stream through shared memory via TMA (once per group: the larger the
// group, the fewer passes over the surfels).  Inside an item the warps steal SUB-ITEMS (keyframe, 256- or 128-surfel chunk) from
// a shared-memory counter, which evens out the very different cost of culled vs. associated chunks.  The group decides only
// which sub-items share a staged tile, never what a sub-item computes.
// STATS: also produce the residual costs and the stage counters of the byte model (the reference computes its
// residual count / cost only in debug mode, kernel_opt_pose.cu:312-320,373-381).
// PRE: the surfels are read from the pose stream in spatial order (LaunchPoseStream: positions, descriptors and the per-surfel
// frames -- unpacked normal, tangent points -- instead of the packed normal and the radius), a sub-item whose chunk box lies outside
// its keyframe's view (BoxOutsideView) is skipped without projecting a surfel, and the CTA is warp-specialised: the producer warps run the item loop below up to the association and hand each associated pair to
// their consumer warp as a record.  Without PRE every warp accumulates its own pairs (26 of 32 lanes busy on average) and
// holds the 32 sums in registers throughout.
// Every 32-surfel step with an associated lane fills one slot, lane L's record at position L (no packing: on the sorted stream
// ~94 % of a visible chunk's lanes are in the image); lane L of the consumer sums the record of every slot of the sub-item whose
// associated-lane mask has bit L, i.e. its surfels j = L (mod 32), with fresh sums, and reduces once at the sub-item's last slot.
// The fp32 partials therefore depend on the sub-item alone, never on timing, and are the same with and without STATS.
// DET: the warp totals go to exact sums (StorePoseTotal); with the partials fixed by the sub-item, the result is then the same bits
// in every run.
template <int TILE, bool STATS, bool PRE, bool DET>
__global__ void __launch_bounds__(PRE ? kPoseWsThreads : kPoseThreads, kPoseMinCtas)
    PoseAccumulateKernel(const __grid_constant__ PoseAccumulateArgs args) {
  constexpr int kRows = PRE ? kPoseStagedRowsPre : kPoseStagedRows;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* stage_base = reinterpret_cast<float*>(smem_raw);   // [2][kRows][TILE]
  float4* rings = reinterpret_cast<float4*>(stage_base + 2 * kRows * TILE);   // PRE: [producer][slot][kPoseSlotChunks]
  // [2][G] the work group's keyframe records, staged with the tile
  KfDevice* s_kf = reinterpret_cast<KfDevice*>(rings + (PRE ? kPoseRingBytes / sizeof(float4) : 0));
  __shared__ __align__(16) float s_box[2][PRE ? TILE / kSpatialChunk : 1][8];   // PRE: the tile's chunk boxes, staged with it
  __shared__ __align__(8) uint64_t full_bar[2];
  __shared__ unsigned int s_item[2];
  __shared__ int s_sub[2];
  // PRE: step handoff, per producer and slot: full / empty barriers (32 arrivals each: every lane releases its own accesses) and
  // the slot header {associated-lane mask, photometric-lane mask, last step of its sub-item, keyframe id; keyframe id -1: the
  // producer has finished}
  __shared__ __align__(8) uint64_t batch_full[PRE ? kPoseProducerWarps : 1][kPoseRingSlots];
  __shared__ __align__(8) uint64_t batch_empty[PRE ? kPoseProducerWarps : 1][kPoseRingSlots];
  __shared__ int4 batch_hdr[PRE ? kPoseProducerWarps : 1][kPoseRingSlots];

  const int n_work = __ldg(args.work_count);
  if (n_work <= 0) return;

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const uint32_t n_tiles = (args.n + TILE - 1) / TILE;
  const int G = args.group;
  const uint32_t n_groups = (n_work + G - 1) / G;
  const uint32_t n_items = n_groups * n_tiles;
  // 256-surfel chunks (one warp-level reduction per 8 steps); 128-surfel ones when the work list holds fewer than 4 keyframes,
  // so that every warp of the CTA still finds a sub-item (the tail of a Gauss-Newton loop)
  constexpr int kTileShift = (TILE == 1024) ? 10 : (TILE == 512) ? 9 : 8;

  const CameraParams& cam = args.cam;
  constexpr int kRowIds[kPoseStagedRows] = {kRowX, kRowY, kRowZ, kRowNormal, kRowRadiusSq, kRowD1, kRowD2};

  auto issue_tile = [&](uint32_t item, int s) {
    const uint32_t group = item / n_tiles, tile = item - group * n_tiles;
    const uint32_t base = tile * TILE;
    const uint32_t cnt = min(static_cast<uint32_t>(TILE), args.n - base);
    const uint32_t bytes = ((cnt * 4u + 15u) / 16u) * 16u;
    const uint32_t kf_bytes = static_cast<uint32_t>(sizeof(KfDevice)) * min(G, n_work - static_cast<int>(group) * G);
    // PRE: the boxes of the tile's chunks come with it (32 bytes each)
    const uint32_t box_bytes = PRE ? (cnt + kSpatialChunk - 1) / kSpatialChunk * 8 * sizeof(float) : 0u;
    MbarArriveExpectTx(&full_bar[s], bytes * kRows + kf_bytes + box_bytes);
    BulkCopyG2S(s_kf + s * G, args.work_records + static_cast<size_t>(group) * G, kf_bytes, &full_bar[s]);
    if (PRE) {
      BulkCopyG2S(&s_box[s][0][0], args.boxes + static_cast<size_t>(base / kSpatialChunk) * 8, box_bytes, &full_bar[s]);
#pragma unroll
      for (int r = 0; r < kPoseStreamRows; ++r)
        BulkCopyG2S(stage_base + (s * kRows + r) * TILE, args.stream + static_cast<size_t>(r) * args.stream_pitch + base, bytes,
                    &full_bar[s]);
    } else {
#pragma unroll
      for (int r = 0; r < kPoseStagedRows; ++r) {
        BulkCopyG2S(stage_base + (s * kRows + r) * TILE,
                    args.surfels + static_cast<size_t>(kRowIds[r]) * args.pitch + base, bytes, &full_bar[s]);
      }
    }
  };

  // No CTA-wide barrier in the item loop: a warp that has run out of sub-items of stage s moves on to stage s ^ 1 at once.
  // The LAST warp to leave a stage (shared-memory counter) re-arms it: claims the next item, resets the sub-item counter and
  // starts the TMA copies; everybody else finds the stage ready through its mbarrier phase.  When the queue is exhausted the
  // stage gets a sentinel item and a plain arrive, so that the waiting warps wake up and leave.
  __shared__ int s_done[2];
  constexpr int kWarps = PRE ? kPoseProducerWarps : kPoseThreads / 32;   // the warps that run the item loop
  auto arm_stage = [&](int s) {   // one thread
    s_sub[s] = 0;
    s_done[s] = 0;
    const unsigned int item = atomicAdd(args.queue, 1u);
    s_item[s] = item;
    if (item < n_items) issue_tile(item, s);
    else MbarArrive(SmemAddr(&full_bar[s]));
  };
  if (tid == 0) {
    MbarInit(&full_bar[0], 1);
    MbarInit(&full_bar[1], 1);
    if (PRE) {
      for (int p = 0; p < kPoseProducerWarps; ++p)
        for (int b = 0; b < kPoseRingSlots; ++b) {
          MbarInit(&batch_full[p][b], 32);
          MbarInit(&batch_empty[p][b], 32);
        }
    }
    FenceBarrierInit();
    arm_stage(0);
    arm_stage(1);
  }
  __syncthreads();

  // Step handoff.  Use number u of a producer's ring is slot u & 1 in phase (u >> 1) & 1; a slot starts out empty.
  uint32_t batch_seq = 0;   // producer: the ring use that the next step goes to
  bool pending = false;     // producer: use batch_seq - 1 holds the sub-item's latest step and is not yet handed over
  if constexpr (PRE) {
    if (warp >= kPoseProducerWarps) {
      SetMaxRegsInc<kPoseConsumerRegs>();
      const int c = warp - kPoseProducerWarps;
      float acc0[kPoseAccSize], acc1[kPoseAccSize];
#pragma unroll
      for (int i = 0; i < kPoseAccSize; ++i) acc0[i] = acc1[i] = 0.f;
      uint32_t seq0 = 0, seq1 = 0;
      bool done0 = false, done1 = false;
      // Takes the next step of producer p if it is ready; false if not.  The slot is released as soon as its records are in
      // registers.
      auto consume = [&](int p, uint32_t& seq, bool& done, float (&acc)[kPoseAccSize]) {
        const int b = seq & 1;
        if (!__all_sync(0xffffffffu, MbarTest(SmemAddr(&batch_full[p][b]), (seq >> 1) & 1))) return false;
        const int4 h = batch_hdr[p][b];
        if (h.w < 0) {
          done = true;
          return true;
        }
        const float4* rec = rings + (p * kPoseRingSlots + b) * kPoseSlotChunks + lane;
        float4 q[kPoseRecChunks];
#pragma unroll
        for (int c = 0; c < kPoseRecChunks; ++c) q[c] = rec[c * 32];
        MbarArrive(SmemAddr(&batch_empty[p][b]));
        ++seq;
        const unsigned bit = 1u << lane;
        if (static_cast<unsigned>(h.x) & bit) AccumulateRecord<STATS>(args.cam, q, (static_cast<unsigned>(h.y) & bit) != 0u, acc);
        if (h.z) {
          StorePoseTotal<DET>(args, h.w, lane, WarpTransposeReduce(acc, lane));
#pragma unroll
          for (int i = 0; i < kPoseAccSize; ++i) acc[i] = 0.f;
        }
        return true;
      };
      while (!(done0 && done1)) {
        bool progress = false;
        if (!done0) progress |= consume(c, seq0, done0, acc0);
        if (!done1) progress |= consume(c + kPoseConsumerWarps, seq1, done1, acc1);
        if (!progress) __nanosleep(32);
      }
      return;
    }
    SetMaxRegsDec<kPoseProducerRegs>();
  }
  // PRE producers: the ring, and the barriers of its slot 0 (slot 1's follow at + 8 bytes)
  float4* my_ring = rings + warp * kPoseRingSlots * kPoseSlotChunks;
  const uint32_t my_full = SmemAddr(&batch_full[PRE ? warp : 0][0]), my_empty = SmemAddr(&batch_empty[PRE ? warp : 0][0]);
  auto acquire_slot = [&](uint32_t u) { MbarWait(my_empty + 8 * (u & 1), ((u >> 1) & 1) ^ 1); };
  auto commit_slot = [&](uint32_t u) { MbarArrive(my_full + 8 * (u & 1)); };

  for (uint32_t it = 0;; ++it) {
    const int s = it & 1;
    MbarWait(SmemAddr(&full_bar[s]), (it >> 1) & 1);
    const unsigned int item = *reinterpret_cast<volatile unsigned int*>(&s_item[s]);
    if (item >= n_items) break;

    // staged rows: x y z normal radius^2 d1 d2, or (PRE) x y z d1 d2 + 9 frame rows
    const float* sx = stage_base + (s * kRows + 0) * TILE;
    const float* sy = sx + TILE;
    const float* sz = sy + TILE;
    const float* sn = sz + TILE;                 // !PRE: packed normal
    const float* sr = sn + TILE;                 // !PRE: radius^2
    const float* sd1 = PRE ? sz + TILE : sr + TILE;
    const float* sd2 = sd1 + TILE;
    const float* sf = sd2 + TILE;                // PRE: nx ny nz q1x q1y q1z q2x q2y q2z
    const uint32_t group = item / n_tiles;
    const uint32_t tile = item - group * n_tiles;
    const uint32_t base = tile * TILE;
    const uint32_t cnt = min(static_cast<uint32_t>(TILE), args.n - base);
    const int kfs_in_group = min(G, n_work - static_cast<int>(group) * G);
    // One chunk size per launch: sizing per item from its group's keyframe count cost more in the extra warp reductions of the
    // smaller chunks than the idle warps of the few short groups save (on the project's first GPU, not on the H100).
    const int wanted_shift = n_work >= 4 ? kPoseChunkShift : 7;
    const int chunk_shift = wanted_shift < kTileShift ? wanted_shift : kTileShift;
    const uint32_t chunk_len = 1u << chunk_shift;
    const int chunks_per_tile = TILE >> chunk_shift;
    const int n_sub = kfs_in_group * chunks_per_tile;

    for (;;) {
      int sub = 0;
      if (lane == 0) sub = atomicAdd(&s_sub[s], 1);
      sub = __shfl_sync(0xffffffffu, sub, 0);
      if (sub >= n_sub) break;
      const int kf_local = sub / chunks_per_tile;
      const uint32_t j0 = static_cast<uint32_t>(sub - kf_local * chunks_per_tile) << chunk_shift;
      if (j0 >= cnt) continue;
      const uint32_t j1 = min(cnt, j0 + chunk_len);
      KfRegs K;
      const int kf = LoadKfShared(s_kf + s * G + kf_local, &K);
      if (PRE && BoxOutsideView(cam, K.T, s_box[s][PRE ? j0 / kSpatialChunk : 0], lane)) continue;   // no pair in the image
      K.tex = UniformTexture(K.tex);

      float acc[kPoseAccSize];
#pragma unroll
      for (int i = 0; i < kPoseAccSize; ++i) acc[i] = 0.f;
      unsigned touched = 0;
      unsigned n_inimg = 0, n_depthok = 0;

#pragma unroll kPoseUnroll
      for (uint32_t j = j0 + lane; j < j0 + (j1 - j0 + 31u) / 32u * 32u; j += 32) {
        int st = 0;
        Assoc r;
        Vec3 gp, nrm;
        DescEval e;
        bool photo = false;
        if (j < j1) {
          gp = V3(sx[j], sy[j], sz[j]);
          if (ProjectIntoImage(cam, K.T, gp, &r)) {
            // Not EvalPair: through it the variants without precomputed frames sum H and b that differ in the last bits.
            // Put every gather of the pair in flight before the first dependent use: the pixel's depth / normal /
            // cfactor, and -- speculatively, ~99 % of in-image pairs end up associated -- the six texture fetches of
            // the descriptor residual.  The association tests below then wait for the slowest load once.
            const PixelLoads l = LoadPixel(cam, K.depth, K.depth_pitch, K.normals, K.normals_pitch, r);
            nrm = PRE ? V3(sf[j], sf[TILE + j], sf[2 * TILE + j]) : UnpackNormal(__float_as_uint(sn[j]));
            if (cam.use_desc) {
              float ccx, ccy;
              photo = DepthToColor(cam, r.pxf, r.pyf, &ccx, &ccy);
              float t1x, t1y, t2x, t2y;
              if (PRE) {
                ProjectTangentPoints(cam, K.T, V3(sf[3 * TILE + j], sf[4 * TILE + j], sf[5 * TILE + j]),
                                     V3(sf[6 * TILE + j], sf[7 * TILE + j], sf[8 * TILE + j]), &t1x, &t1y, &t2x, &t2y);
              } else {
                TangentProjections(cam, K.T, gp, nrm, sr[j], &t1x, &t1y, &t2x, &t2y);
              }
              EvalDescriptor(K.tex, ccx, ccy, t1x, t1y, t2x, t2y, sd1[j], sd2[j], &e);
            }
            st = Associate(cam, K.T, nrm, l, &r);
          }
        }
        if (STATS) {
          // per-lane counts (one predicated add each), summed over the warp once per chunk below
          n_inimg += st >= 1;
          n_depthok += st >= 2;
        }
        const unsigned assoc_mask = __ballot_sync(0xffffffffu, st == 3);
        if (assoc_mask == 0) continue;
        if constexpr (PRE) {
          // The step goes to a slot of its own.  The previous one is handed over only now that it is known not to be the
          // sub-item's last (its header says whether it is).
          const unsigned photo_mask = __ballot_sync(0xffffffffu, st == 3 && photo);
          if (pending) commit_slot(batch_seq - 1);
          acquire_slot(batch_seq);
          float4* rec = my_ring + (batch_seq & 1) * kPoseSlotChunks + lane;
          if (st == 3) {
            rec[0 * 32] = make_float4(r.lp.x, r.lp.y, r.lp.z, r.ln.x);
            rec[1 * 32] = make_float4(r.ln.y, r.ln.z, r.d, r.nx);
            rec[2 * 32] = make_float4(r.ny, e.r1, e.r2, e.gx1);
            rec[3 * 32] = make_float4(e.gy1, e.gx2, e.gy2, 0.f);
          }
          if (lane == 0) batch_hdr[warp][batch_seq & 1] = make_int4(static_cast<int>(assoc_mask), static_cast<int>(photo_mask), 0, kf);
          ++batch_seq;
          pending = true;
        } else {
          touched |= assoc_mask;
          if (st == 3) AccumulatePair<STATS>(cam, r, e, photo, acc);
        }
      }

      if (PRE && pending) {   // the sub-item's last slot, also when its last steps had no associated lane
        if (lane == 0) batch_hdr[warp][(batch_seq - 1) & 1].z = 1;
        commit_slot(batch_seq - 1);
        pending = false;
      } else if (!PRE && touched) {
        StorePoseTotal<DET>(args, kf, lane, WarpTransposeReduce(acc, lane));
      }
      if (STATS) {
        n_inimg = __reduce_add_sync(0xffffffffu, n_inimg);
        n_depthok = __reduce_add_sync(0xffffffffu, n_depthok);
      }
      if (STATS && lane == 0 && n_inimg) {
        atomicAdd(args.stage_counts + 2 * kf, static_cast<unsigned long long>(n_inimg));
        if (n_depthok) atomicAdd(args.stage_counts + 2 * kf + 1, static_cast<unsigned long long>(n_depthok));
      }
    }
    __syncwarp();
    if (lane == 0) {
      __threadfence_block();   // this warp's reads of stage s are complete before the stage can be handed back
      if (atomicAdd(&s_done[s], 1) == kWarps - 1) {
        __threadfence_block();
        arm_stage(s);
      }
    }
  }
  if (PRE) {   // no more slots from this producer
    acquire_slot(batch_seq);
    if (lane == 0) batch_hdr[warp][batch_seq & 1] = make_int4(0, 0, 0, -1);
    commit_slot(batch_seq);
  }
}

// work_records[i] = kfs[work_list[i]] with pad = the keyframe id: makes the records of a work group contiguous.
__global__ void __launch_bounds__(128) PackWorkRecordsKernel(const KfDevice* __restrict__ kfs, const int* __restrict__ work_list,
                                                             const int* __restrict__ work_count, KfDevice* __restrict__ records) {
  const int n = __ldg(work_count);
  constexpr int kWords = sizeof(KfDevice) / 16;   // 6 x 16 bytes per record
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n * kWords; i += gridDim.x * blockDim.x) {
    const int rec = i / kWords, w = i - rec * kWords;
    const int kf = __ldg(work_list + rec);
    uint4 v = __ldg(reinterpret_cast<const uint4*>(kfs + kf) + w);
    if (w == kWords - 1) v.y = static_cast<unsigned int>(kf);   // KfDevice::pad
    reinterpret_cast<uint4*>(records + rec)[w] = v;
  }
}

// Dynamic shared memory of the pose kernel: two stages of surfel rows, (PRE) the producers' rings, and the two stages' group records.
static constexpr size_t PoseSmemBytes(int tile, bool pre, int group) {
  return static_cast<size_t>(2) * (pre ? kPoseStagedRowsPre : kPoseStagedRows) * tile * sizeof(float) + (pre ? kPoseRingBytes : 0) +
         static_cast<size_t>(2) * group * sizeof(KfDevice);
}

template <int TILE, bool PRE>
static cudaError_t SetPoseSmemLimit() {
  const int smem = static_cast<int>(PoseSmemBytes(TILE, PRE, kPoseMaxGroup));
  for (const void* k : {reinterpret_cast<const void*>(PoseAccumulateKernel<TILE, false, PRE, false>),
                        reinterpret_cast<const void*>(PoseAccumulateKernel<TILE, true, PRE, false>),
                        reinterpret_cast<const void*>(PoseAccumulateKernel<TILE, false, PRE, true>),
                        reinterpret_cast<const void*>(PoseAccumulateKernel<TILE, true, PRE, true>)})
    if (const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)) return e;
  return cudaSuccess;
}

cudaError_t SetPoseAccumulateSmemLimits() {
  for (cudaError_t e : {SetPoseSmemLimit<256, true>(), SetPoseSmemLimit<512, true>(), SetPoseSmemLimit<256, false>(),
                        SetPoseSmemLimit<512, false>(), SetPoseSmemLimit<1024, false>()})
    if (e != cudaSuccess) return e;
  return cudaSuccess;
}

template <int TILE, bool STATS, bool PRE>
static void LaunchPoseAccumulateT(const PoseAccumulateArgs& args, int sm_count, cudaStream_t stream) {
  const size_t smem = PoseSmemBytes(TILE, PRE, args.group);
  const dim3 grid(kPoseMinCtas * sm_count), block(PRE ? kPoseWsThreads : kPoseThreads);   // persistent
  if (args.exact) PoseAccumulateKernel<TILE, STATS, PRE, true><<<grid, block, smem, stream>>>(args);
  else PoseAccumulateKernel<TILE, STATS, PRE, false><<<grid, block, smem, stream>>>(args);
}

template <bool STATS>
static void LaunchPoseAccumulateS(const PoseAccumulateArgs& args, int sm_count, int variant, cudaStream_t stream) {
  // Tile size: as large as possible (one group of TMA transactions per item), but small enough that a keyframe group still
  // yields several items per resident CTA.  With the precomputed frames 14 rows are staged: 512 surfels x 2 stages = 56 KB per
  // CTA (two CTAs per SM), the same footprint as 1024 surfels of the 7-row variant.
  if (variant == kPoseVariantAuto) {
    const uint64_t slots = static_cast<uint64_t>(kPoseMinCtas * sm_count) * 4;
    if (args.stream != nullptr) variant = args.n >= slots * 512 ? kPoseVariant512Pre : kPoseVariant256Pre;
    else variant = args.n >= slots * 1024 ? kPoseVariant1024 : args.n >= slots * 512 ? kPoseVariant512 : kPoseVariant256;
  }
  switch (variant) {
    case kPoseVariant256Pre: LaunchPoseAccumulateT<256, STATS, true>(args, sm_count, stream); break;
    case kPoseVariant512Pre: LaunchPoseAccumulateT<512, STATS, true>(args, sm_count, stream); break;
    case kPoseVariant256: LaunchPoseAccumulateT<256, STATS, false>(args, sm_count, stream); break;
    case kPoseVariant512: LaunchPoseAccumulateT<512, STATS, false>(args, sm_count, stream); break;
    case kPoseVariant1024: LaunchPoseAccumulateT<1024, STATS, false>(args, sm_count, stream); break;
  }
}

LaunchResult LaunchPoseAccumulate(const PoseAccumulateArgs& args, int sm_count, bool with_stats, int max_work, cudaStream_t stream,
                                  int variant) {
  // (max_work = 0: a rank of a multi-GPU job whose share of the pose step's work list is empty -- no launch at all, a grid of
  // zero blocks is an invalid configuration)
  if (args.n == 0 || max_work <= 0) return {};
  PackWorkRecordsKernel<<<(max_work * 6 + 127) / 128, 128, 0, stream>>>(args.kfs, args.work_list, args.work_count, args.work_records);
  // Keyframes per work item.  Every item stages its tile's stream rows once for the whole group, so that one pass over the
  // keyframes reads the stream n_work / group times.  In spatial order the tiles that the resident CTAs work on at one time are a
  // compact region, a patch of each keyframe's image, so a group of 32 keyframes still gathers from a small part of L2: on cfg3 one
  // 200-keyframe launch without stats took 6.90 ms at 32, 6.84 at 24, 7.14 at 16 and 7.48 at 8 (DESIGN §7.1).  In the caller's
  // order a tile is a band across a whole image and larger groups did not pay (cfg2).
  PoseAccumulateArgs a = args;
  if (a.group == 0) a.group = a.stream && a.stream_sorted ? 32 : 8;
  if (with_stats) LaunchPoseAccumulateS<true>(a, sm_count, variant, stream);
  else LaunchPoseAccumulateS<false>(a, sm_count, variant, stream);
  return {2};
}

// ------------------------------------------------------------------------------------------------
// Geometry step.  One thread owns one surfel and keeps its accumulators in registers while it walks over a GROUP of
// keyframes; work items (keyframe group, 256-surfel tile) are handed out group-major through a global counter so that
// all resident CTAs gather from the same <= 32 keyframes' images at a time (L2-resident) -- the surfel-major variant
// that looped over all K keyframes per thread re-read the images from HBM ~40 times.
// Surfels are visited in stream order (GeometryArgs): their inputs come from the geometry stream the launcher gathers first, in
// spatial order when the handle's order is current.  Between groups the partial sums of a surfel are parked in the scratch rows
// 8..16 of the surfel buffer (the rows the reference uses for exactly this purpose, kernels.cuh:78-86) at its stream position,
// so that they stay coalesced; a per-tile epoch word orders (group g, tile t) after (group g-1, tile t) (ClaimItem, RetireItem).
// Work items are owned by warps: there is no CTA-wide barrier in these kernels.  With K <= 32 there is a single group and no
// scratch traffic at all.

constexpr int kGeoThreads = 256;
// Keyframes per work item.  A group's images (1.5 MB per keyframe at 640x480) are what all resident warps gather from at one
// time; between groups a surfel's partial sums are parked in the scratch rows.  32 keeps a group's images (48 MB) around the size
// of the H100's L2; with the warp-box culling most (warp, keyframe) steps cost a box test only, so fewer groups -- less parked-sum
// traffic -- beat 16: on cfg3 the two geometry stages took 8.70 instead of 9.31 ms (one H100 80GB HBM3, 700 W limit).
constexpr int kGeoGroup = 32;

// The <= kGeoGroup keyframe records of a work item, copied once per item into the warp's own shared-memory slice (coalesced
// 16-byte loads; the per-keyframe reads in the pair loop are then conflict-free broadcasts with a fixed ~25-cycle latency
// instead of a chain of dependent L1 accesses: keyframe id -> record row 2 -> rows 0, 1 -> image pointers).
// Staging all records of the launch once per CTA instead did not pay on the project's first GPU with these group items; the
// tile-major GeometryPassKernel, whose items span every keyframe, does stage them so.
__device__ __forceinline__ void StageGroupRecords(const KfDevice* __restrict__ kfs, const int* __restrict__ kf_list, int count,
                                                  KfDevice* dst, int lane) {
  constexpr int kWords = sizeof(KfDevice) / 16;
  __syncwarp();   // the previous item's readers are done
  const int my_kf = lane < count ? __ldg(kf_list + lane) : 0;
#pragma unroll
  for (int w = 0; w < (kGeoGroup * kWords + 31) / 32; ++w) {
    const int idx = w * 32 + lane, rec = idx / kWords, part = idx - rec * kWords;
    const int kf = __shfl_sync(0xffffffffu, my_kf, rec & 31);
    if (rec < count) {
      uint4 v = __ldg(reinterpret_cast<const uint4*>(kfs + kf) + part);
      reinterpret_cast<uint4*>(dst + rec)[part] = v;
    }
  }
  __syncwarp();
}

// The box {lo} - {hi} over the finite coordinates of the lanes with `in` (per axis, like the pose stream's chunk boxes), in every
// lane.  Without such a lane the box is NaN, which is never culled.  Must be called by all 32 lanes.
__device__ __forceinline__ void WarpBox(const Vec3& p, bool in, float (&lo)[3], float (&hi)[3]) {
  const float c[3] = {p.x, p.y, p.z};
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) {
    const bool f = in && isfinite(c[ax]);
    lo[ax] = FromOrderedBits(__reduce_min_sync(0xffffffffu, f ? OrderedBits(c[ax]) : 0xffffffffu));
    hi[ax] = FromOrderedBits(__reduce_max_sync(0xffffffffu, f ? OrderedBits(c[ax]) : 0u));
  }
}

static_assert(kGeoGroup <= 32, "one lane per keyframe of a group");
// The keyframes of a group of n_kf records whose view the box {lo} - {hi} may reach, as a mask (bit j: record j): lane j tests
// record j (BoxOutsideViewLane), one ballot collects them.  ACTIVE_ONLY: only the kActive keyframes (activation 0).  Must be
// called by all 32 lanes.
template <bool ACTIVE_ONLY>
__device__ __forceinline__ unsigned VisibleKeyframes(const CameraParams& cam, const KfDevice* recs, int n_kf, const float (&lo)[3],
                                                     const float (&hi)[3], int lane) {
  bool visible = false;
  if (lane < n_kf) {
    KfRegs K;
    LoadKfShared(recs + lane, &K);
    visible = (!ACTIVE_ONLY || K.activation == 0) && !BoxOutsideViewLane(cam, K.T, lo, hi);
  }
  return __ballot_sync(0xffffffffu, visible);
}

// Pops the lowest set bit of the warp-uniform mask *m and returns its index; -1 when *m is empty.
__device__ __forceinline__ int PopLowest(unsigned* m) {
  if (*m == 0u) return -1;
  const int j = __ffs(*m) - 1;
  *m &= *m - 1u;
  return j;
}

// A result row of caller index i, stored into every replica.
__device__ __forceinline__ void StoreSurfelRow(const GeometryArgs& a, int row, uint32_t i, float v) {
  StoreReplicas(a.surfels, a.peers.surfels, a.peers.count, static_cast<size_t>(row) * a.pitch + i, v);
}

// The stream position s of the lane's surfel in sub-step `sub` of a work item's tile, and whether it is one of the launch's surfels.
__device__ __forceinline__ bool GeoStreamPosition(const GeometryArgs& a, uint32_t tile, uint32_t sub, int lane, uint32_t* s) {
  const uint32_t li = a.begin + (tile << a.tile_shift) + sub * 32 + lane;
  *s = SurfelShardToGlobal(li, a.shard_rank, a.shard_world);
  return li < a.end && *s < a.n;
}
// The caller index of the surfel at stream position s.
__device__ __forceinline__ uint32_t GeoResultIndex(const GeometryArgs& a, uint32_t s) { return a.perm ? __ldg(a.perm + s) : s; }
// The N partial sums a surfel parks in the scratch rows 8 .. 8 + N - 1 between keyframe groups, at its stream position.
template <int N>
__device__ __forceinline__ void LoadParkedSums(const GeometryArgs& a, uint32_t s, float (&v)[N]) {
#pragma unroll
  for (int r = 0; r < N; ++r) v[r] = __ldcg(a.surfels + (kRowAccum0 + r) * static_cast<size_t>(a.pitch) + s);
}
template <int N>
__device__ __forceinline__ void StoreParkedSums(const GeometryArgs& a, uint32_t s, const float (&v)[N]) {
#pragma unroll
  for (int r = 0; r < N; ++r) __stcg(a.surfels + (kRowAccum0 + r) * static_cast<size_t>(a.pitch) + s, v[r]);
}

// An associated pair's term of a surfel's normal sums n (x y z, count), kernel_opt_geometry.cu:545-553: global_R_frame * the
// keyframe pixel's normal, global_R_frame = R(frame_T_global)^T.
__device__ __forceinline__ void AddPairNormal(const float* __restrict__ T, const Assoc& r, float (&n)[4]) {
  const Vec3 ln = U16ToImageSpaceNormal(r.kf_normal);
  n[0] += T[0] * ln.x + T[4] * ln.y + T[8] * ln.z;
  n[1] += T[1] * ln.x + T[5] * ln.y + T[9] * ln.z;
  n[2] += T[2] * ln.x + T[6] * ln.y + T[10] * ln.z;
  n[3] += 1.f;
}
// The new packed normal from the sums, count >= 1 (kernel_opt_geometry.cu:577-597: the mean is packed without re-normalisation).
__device__ __forceinline__ uint32_t PackedMeanNormal(const float (&n)[4]) {
  const float inv = 1.f / n[3];
  return PackNormal(V3(inv * n[0], inv * n[1], inv * n[2]));
}

// A surfel's 3x3 normal equations over (t along the normal, d1, d2): H00 H01 H02 H11 H22 | b0 b1 b2.  H12 is never accumulated, by
// the reference either (kernel_opt_geometry.cu:216-227).
struct PositionSums {
  float H00 = 0.f, H01 = 0.f, H02 = 0.f, H11 = 0.f, H22 = 0.f, b0 = 0.f, b1 = 0.f, b2 = 0.f;
};
// One associated pair's terms.
template <bool USE_DEPTH, bool USE_DESC>
__device__ __forceinline__ void AccumulatePosition(const CameraParams& cam, const Assoc& r, const DescEval& e, bool photo, PositionSums& q) {
  if (USE_DEPTH) {
    float inv_stddev;
    Vec3 up;
    const float raw = DepthResidual(cam, r, &inv_stddev, &up);
    const float jac = -inv_stddev;   // kernel_opt_geometry.cu:138
    const float w = DepthWeight(raw);
    if (USE_DESC) {
      q.H00 += w * jac * jac;
      q.b0 += w * raw * jac;
    } else {
      // kernel_opt_geometry.cu:452-456
      const float wj = w * jac;
      q.H00 += wj * jac;
      q.b0 += wj * raw;
    }
  }
  if (USE_DESC && photo) {
    // kernel_opt_geometry.cu:176-181.  PcgAccumulateKernel has its own copy: it scales the gradients by cfx / cfy first,
    // here term1 / term2 carry them, and the two orders round differently.
    const float term1 = -cam.cfx * (r.ln.x * r.lp.z - r.ln.z * r.lp.x);
    const float term2 = -cam.cfy * (r.ln.y * r.lp.z - r.ln.z * r.lp.y);
    const float term3 = 1.f / (r.lp.z * r.lp.z);
    const float j1 = -(e.gx1 * term1 + e.gy1 * term2) * term3;
    const float j2 = -(e.gx2 * term1 + e.gy2 * term2) * term3;
    constexpr float jd = -1.f;
    const float w1 = DescWeight(e.r1), wr1 = w1 * e.r1;
    const float w2 = DescWeight(e.r2), wr2 = w2 * e.r2;
    q.H00 += w1 * j1 * j1 + w2 * j2 * j2;
    q.H01 += w1 * j1 * jd;
    q.H11 += w1 * jd * jd;
    q.b0 += wr1 * j1 + wr2 * j2;
    q.b1 += wr1 * jd;
    q.H02 += w2 * j2 * jd;
    q.H22 += w2 * jd * jd;
    q.b2 += wr2 * jd;
  }
}
// The solve and the stores into caller index i: the surfel moves along its normal nrm from gp; with descriptors d1 / d2 change too.
template <bool USE_DESC>
__device__ __forceinline__ void UpdatePosition(const GeometryArgs& a, uint32_t i, const Vec3& gp, const Vec3& nrm, float d1, float d2,
                                               const PositionSums& q) {
  if (!USE_DESC) {
    // UpdateSurfelPositionCUDAKernel, kernel_opt_geometry.cu:487-507
    if (q.H00 > 1e-6f) {
      const float t = -1.f * q.b0 / q.H00;
      StoreSurfelRow(a, kRowX, i, gp.x + t * nrm.x);
      StoreSurfelRow(a, kRowY, i, gp.y + t * nrm.y);
      StoreSurfelRow(a, kRowZ, i, gp.z + t * nrm.z);
    }
  } else {
    // UpdateSurfelPositionAndDescriptorCUDAKernel, kernel_opt_geometry.cu:273-361 (in-place Cholesky)
    constexpr float kEpsilon = 1e-6f;
    constexpr float H12 = 0.f;
    const float L00 = sqrtf(q.H00 + kEpsilon);
    const float L01 = q.H01 / L00;
    const float L11 = sqrtf((q.H11 + kEpsilon) - L01 * L01);
    const float L02 = q.H02 / L00;
    const float L12 = (H12 - L02 * L01) / L11;
    const float L22 = sqrtf((q.H22 + kEpsilon) - L02 * L02 - L12 * L12);
    const float y0 = q.b0 / L00;
    const float y1 = (q.b1 - L01 * y0) / L11;
    const float y2 = (q.b2 - L02 * y0 - L12 * y1) / L22;
    const float x2 = y2 / L22;
    const float x1 = (y1 - L12 * x2) / L11;
    const float x0 = (y0 - L02 * x2 - L01 * x1) / L00;
    if (x0 != 0) {
      StoreSurfelRow(a, kRowX, i, gp.x - x0 * nrm.x);
      StoreSurfelRow(a, kRowY, i, gp.y - x0 * nrm.y);
      StoreSurfelRow(a, kRowZ, i, gp.z - x0 * nrm.z);
    }
    if (x1 != 0) StoreSurfelRow(a, kRowD1, i, fmaxf(-180.f, fminf(180.f, d1 - x1)));
    if (x2 != 0) StoreSurfelRow(a, kRowD2, i, fmaxf(-180.f, fminf(180.f, d2 - x2)));
  }
}

// Both geometry kernels walk a work item's tile in sub-steps of 32 stream positions, one surfel per lane, with the keyframe loop
// executed by the whole warp.  In spatial order a sub-step's surfels are a compact cluster: the box of the lanes that still have
// pairs to evaluate is tested against the views of all keyframes of the group at once, one keyframe per lane (VisibleKeyframes,
// the pose kernel's plane tests), and the warp walks only the keyframes that some of them may project into.  The box test rejects
// only pairs that ProjectIntoImage rejects, so every surfel still sums exactly the pairs it summed before, in keyframe order.
template <bool DETERMINE, bool NORMALS>
__global__ void __launch_bounds__(kGeoThreads) ActivationNormalsKernel(const __grid_constant__ GeometryArgs a) {
  extern __shared__ __align__(16) unsigned char geo_smem[];   // one kGeoGroup-record slice per warp
  KfDevice* s_kfs = reinterpret_cast<KfDevice*>(geo_smem);
  const uint32_t tile_len = 1u << a.tile_shift;
  const uint32_t n_tiles = (a.end - a.begin + tile_len - 1) >> a.tile_shift;
  const uint32_t n_groups = (a.kf_count + kGeoGroup - 1) / kGeoGroup;
  const uint32_t n_items = n_groups * n_tiles;
  const size_t P = a.pitch, F = a.stream_pitch;
  const int lane = threadIdx.x & 31;
  uint32_t group, tile;
  while (ClaimItem(a.queue, n_tiles, n_items, a.tile_epoch, &group, &tile)) {
    const bool first = group == 0, last = group + 1 == n_groups;
    const int j_begin = group * kGeoGroup, j_end = min(a.kf_count, static_cast<int>(group + 1) * kGeoGroup);
    const int n_kf = j_end - j_begin;
    KfDevice* recs = s_kfs + (threadIdx.x >> 5) * kGeoGroup;
    StageGroupRecords(a.kfs, a.kf_list + j_begin, n_kf, recs, lane);
    for (uint32_t sub = 0; sub < tile_len / 32; ++sub) {
      uint32_t s;
      const bool in_range = GeoStreamPosition(a, tile, sub, lane, &s);
      const uint32_t flags = in_range ? __float_as_uint(a.stream[(kGeoStreamRows - 1) * F + s]) : 0u;
      const bool live = in_range && (DETERMINE || (flags & kSurfelActiveFlag));   // normals are updated for active surfels only
      if (__ballot_sync(0xffffffffu, live) == 0) continue;
      bool act = !DETERMINE;
      float ns[4] = {0.f, 0.f, 0.f, 0.f};   // normal sums
      if (!first && live) {
        if (NORMALS) LoadParkedSums(a, s, ns);
        if (DETERMINE) act = __ldcg(a.surfels + (kRowAccum0 + 4) * P + s) != 0.f;
      }
      // activation alone stops at the first association with an active keyframe
      const bool walk = live && (NORMALS || !act);
      if (__ballot_sync(0xffffffffu, walk) != 0) {
        Vec3 gp = V3(0.f, 0.f, 0.f), nrm = V3(0.f, 0.f, 1.f);
        if (walk) {
          gp = V3(a.stream[0 * F + s], a.stream[1 * F + s], a.stream[2 * F + s]);
          nrm = UnpackNormal(__float_as_uint(a.stream[3 * F + s]));
        }
        float lo[3], hi[3];
        WarpBox(gp, walk, lo, hi);
        // activation only looks at kActive keyframes
        unsigned vis = VisibleKeyframes<!NORMALS>(a.cam, recs, n_kf, lo, hi, lane);
        // One pair's association and sums.
        auto accumulate = [&](const KfRegs& K, const PixelLoads& l, Assoc& r) {
          if (Associate(a.cam, K.T, nrm, l, &r) != 3) return;
          if (K.activation == 0) act = true;
          if (NORMALS) AddPairNormal(K.T, r, ns);
        };
        // The sums run in keyframe order (the summation order -- and with it the result -- is the reference's: one thread,
        // ascending keyframes).
        for (int j = PopLowest(&vis); j >= 0; j = PopLowest(&vis)) {
          KfRegs K;
          LoadKfShared(recs + j, &K);
          Assoc r;
          // Not ProjectAssociate: through it the cfg3 activation + normals stage took 3.34-3.39 instead of 3.22-3.25 ms (H100 80GB HBM3, 700 W)
          if (walk && (NORMALS || !act) && ProjectIntoImage(a.cam, K.T, gp, &r))
            accumulate(K, LoadPixel(a.cam, K.depth, K.depth_pitch, K.normals, K.normals_pitch, r), r);
          if (!NORMALS && __all_sync(0xffffffffu, !walk || act)) break;
        }
      }
      if (!live) continue;
      if (!last) {
        if (NORMALS) StoreParkedSums(a, s, ns);
        if (DETERMINE) __stcg(a.surfels + (kRowAccum0 + 4) * P + s, act ? 1.f : 0.f);
      } else {
        const uint32_t i = GeoResultIndex(a, s);
        // SetSurfelInactive + DetermineActiveSurfels (kernel_surfel_activation.cu:38-79)
        if (DETERMINE) StoreReplicas(a.active, a.peers.active, a.peers.count, i, act ? kSurfelActiveFlag : static_cast<uint8_t>(flags & ~kSurfelActiveFlag));
        if (NORMALS && act && ns[3] >= 1.f) StoreSurfelRow(a, kRowNormal, i, __uint_as_float(PackedMeanNormal(ns)));
      }
    }
    RetireItem(a.tile_epoch, group, tile);
  }
}

template <bool USE_DEPTH, bool USE_DESC>
__global__ void __launch_bounds__(kGeoThreads, 3) PositionDescriptorKernel(const __grid_constant__ GeometryArgs a) {
  extern __shared__ __align__(16) unsigned char geo_smem[];
  KfDevice* s_kfs = reinterpret_cast<KfDevice*>(geo_smem);
  const uint32_t tile_len = 1u << a.tile_shift;
  const uint32_t n_tiles = (a.end - a.begin + tile_len - 1) >> a.tile_shift;
  const uint32_t n_groups = (a.kf_count + kGeoGroup - 1) / kGeoGroup;
  const uint32_t n_items = n_groups * n_tiles;
  const size_t P = a.pitch, F = a.stream_pitch;
  const int lane = threadIdx.x & 31;
  uint32_t group, tile;
  while (ClaimItem(a.queue, n_tiles, n_items, a.tile_epoch, &group, &tile)) {
    const bool first = group == 0, last = group + 1 == n_groups;
    const int j_begin = group * kGeoGroup, j_end = min(a.kf_count, static_cast<int>(group + 1) * kGeoGroup);
    KfDevice* recs = s_kfs + (threadIdx.x >> 5) * kGeoGroup;
    StageGroupRecords(a.kfs, a.kf_list + j_begin, j_end - j_begin, recs, lane);
    for (uint32_t sub = 0; sub < tile_len / 32; ++sub) {
      const uint32_t li = a.begin + (tile << a.tile_shift) + sub * 32 + lane;
      const uint32_t s = SurfelShardToGlobal(li, a.shard_rank, a.shard_world);
      // The keyframe loop below is executed by the whole warp (a lane without a live surfel just skips every pair): the
      // per-keyframe record -- in particular the texture handle -- is then provably warp-uniform, see UniformTexture().
      const bool live = li < a.end && s < a.n && (__float_as_uint(a.stream[(kGeoStreamRows - 1) * F + s]) & kSurfelActiveFlag);
      if (__ballot_sync(0xffffffffu, live) == 0) continue;
      Vec3 gp = V3(0.f, 0.f, 0.f), nrm = V3(0.f, 0.f, 1.f);
      float radius_sq = 0.f, d1 = 0.f, d2 = 0.f;
      if (live) {
        gp = V3(a.stream[0 * F + s], a.stream[1 * F + s], a.stream[2 * F + s]);
        nrm = UnpackNormal(__float_as_uint(a.stream[3 * F + s]));
        if (USE_DESC) {
          radius_sq = a.stream[4 * F + s];
          d1 = a.stream[5 * F + s];
          d2 = a.stream[6 * F + s];
        }
      }
      PositionSums q;
      if (!first && live) {
        // same row assignment as the reference's accumulators (kernel_opt_geometry.cu:216-227)
        q.H00 = __ldcg(a.surfels + (kRowAccum0 + 0) * P + s);
        q.b0 = __ldcg(a.surfels + (kRowAccum0 + 6) * P + s);
        if (USE_DESC) {
          q.H01 = __ldcg(a.surfels + (kRowAccum0 + 1) * P + s);
          q.H02 = __ldcg(a.surfels + (kRowAccum0 + 2) * P + s);
          q.H11 = __ldcg(a.surfels + (kRowAccum0 + 3) * P + s);
          q.H22 = __ldcg(a.surfels + (kRowAccum0 + 5) * P + s);
          q.b1 = __ldcg(a.surfels + (kRowAccum0 + 7) * P + s);
          q.b2 = __ldcg(a.surfels + (kRowAccum0 + 8) * P + s);
        }
      }
      float lo[3], hi[3];
      WarpBox(gp, live, lo, hi);
      unsigned vis = VisibleKeyframes<false>(a.cam, recs, j_end - j_begin, lo, hi, lane);
      // The visible keyframes in ascending order.
      for (int j = PopLowest(&vis); j >= 0; j = PopLowest(&vis)) {
        KfRegs K;
        LoadKfShared(recs + j, &K);
        K.tex = UniformTexture(K.tex);
        Assoc r;
        if (!live || !ProjectIntoImage(a.cam, K.T, gp, &r)) continue;
        PixelLoads l;
        DescEval e;
        bool photo = false;
        if (EvalPair(a.cam, K, gp, nrm, radius_sq, d1, d2, USE_DESC, &r, &l, &e, &photo) == 3)
          AccumulatePosition<USE_DEPTH, USE_DESC>(a.cam, r, e, photo, q);
      }

      if (!live) continue;
      if (!last) {
        __stcg(a.surfels + (kRowAccum0 + 0) * P + s, q.H00);
        __stcg(a.surfels + (kRowAccum0 + 6) * P + s, q.b0);
        if (USE_DESC) {
          __stcg(a.surfels + (kRowAccum0 + 1) * P + s, q.H01);
          __stcg(a.surfels + (kRowAccum0 + 2) * P + s, q.H02);
          __stcg(a.surfels + (kRowAccum0 + 3) * P + s, q.H11);
          __stcg(a.surfels + (kRowAccum0 + 5) * P + s, q.H22);
          __stcg(a.surfels + (kRowAccum0 + 7) * P + s, q.b1);
          __stcg(a.surfels + (kRowAccum0 + 8) * P + s, q.b2);
        }
        continue;
      }
      UpdatePosition<USE_DESC>(a, GeoResultIndex(a, s), gp, nrm, d1, d2, q);
    }
    RetireItem(a.tile_epoch, group, tile);
  }
}

// ActivationNormalsKernel<DETERMINE, true> and PositionDescriptorKernel in one launch, tile-major: a work item is a surfel tile
// alone, and a warp carries each 32-surfel sub-step through every keyframe twice with all sums in registers, so nothing is parked
// between keyframe groups and no item waits for another.  A surfel's position pass needs only its own new activation and normal.
// Every keyframe record of the launch is staged once per CTA; lane g keeps the visibility word of records 32 g .. 32 g + 31 for
// the sub-step's box (VisibleKeyframes), which both passes walk in ascending keyframe order.  The position pass reuses the mask of
// the activation pass: its box holds every surfel the position pass updates, and the box test rejects only pairs that
// ProjectIntoImage rejects.  Each sum therefore takes the same terms in the same order as in the two group-major kernels, and the
// rows, flags and normals come out bit for bit the same.
template <bool DETERMINE, bool USE_DEPTH, bool USE_DESC>
__global__ void __launch_bounds__(kGeoThreads, 3) GeometryPassKernel(const __grid_constant__ GeometryArgs a) {
  extern __shared__ __align__(16) unsigned char geo_smem[];   // the kf_count records
  KfDevice* recs = reinterpret_cast<KfDevice*>(geo_smem);
  const int n_kf = a.kf_count;
  constexpr int kWords = sizeof(KfDevice) / 16;
  for (int idx = threadIdx.x; idx < n_kf * kWords; idx += blockDim.x) {
    const int rec = idx / kWords, part = idx - rec * kWords;
    reinterpret_cast<uint4*>(recs + rec)[part] = __ldg(reinterpret_cast<const uint4*>(a.kfs + __ldg(a.kf_list + rec)) + part);
  }
  __syncthreads();
  const uint32_t tile_len = 1u << a.tile_shift;
  const uint32_t n_tiles = (a.end - a.begin + tile_len - 1) >> a.tile_shift;
  const int n_words = (n_kf + 31) / 32;
  const size_t F = a.stream_pitch;
  const int lane = threadIdx.x & 31;
  uint32_t unused, tile;
  while (ClaimItem(a.queue, n_tiles, n_tiles, nullptr, &unused, &tile)) {
    for (uint32_t sub = 0; sub < tile_len / 32; ++sub) {
      uint32_t s;
      const bool in_range = GeoStreamPosition(a, tile, sub, lane, &s);
      const uint32_t flags = in_range ? __float_as_uint(a.stream[(kGeoStreamRows - 1) * F + s]) : 0u;
      const bool live = in_range && (DETERMINE || (flags & kSurfelActiveFlag));
      if (__ballot_sync(0xffffffffu, live) == 0) continue;
      Vec3 gp = V3(0.f, 0.f, 0.f);
      uint32_t packed = 0u;   // the packed normal
      if (live) {
        gp = V3(a.stream[0 * F + s], a.stream[1 * F + s], a.stream[2 * F + s]);
        packed = __float_as_uint(a.stream[3 * F + s]);
      }
      float lo[3], hi[3];
      WarpBox(gp, live, lo, hi);
      unsigned vis_word = 0u;   // lane g: records 32 g ..
      for (int g = 0; g < n_words; ++g) {
        const unsigned v = VisibleKeyframes<false>(a.cam, recs + 32 * g, min(32, n_kf - 32 * g), lo, hi, lane);
        if (lane == g) vis_word = v;
      }

      // Activation and normals (ActivationNormalsKernel).
      bool act = !DETERMINE;
      float ns[4] = {0.f, 0.f, 0.f, 0.f};
      {
        const Vec3 nrm = UnpackNormal(packed);
        for (int g = 0; g < n_words; ++g) {
          unsigned vis = __shfl_sync(0xffffffffu, vis_word, g);
          for (int j = PopLowest(&vis); j >= 0; j = PopLowest(&vis)) {
            KfRegs K;
            LoadKfShared(recs + 32 * g + j, &K);
            Assoc r;
            if (live && ProjectIntoImage(a.cam, K.T, gp, &r) &&
                Associate(a.cam, K.T, nrm, LoadPixel(a.cam, K.depth, K.depth_pitch, K.normals, K.normals_pitch, r), &r) == 3) {
              if (K.activation == 0) act = true;
              AddPairNormal(K.T, r, ns);
            }
          }
        }
      }
      uint32_t i = 0;
      if (live) {
        i = GeoResultIndex(a, s);
        if (DETERMINE) StoreReplicas(a.active, a.peers.active, a.peers.count, i, act ? kSurfelActiveFlag : static_cast<uint8_t>(flags & ~kSurfelActiveFlag));
        if (act && ns[3] >= 1.f) {
          packed = PackedMeanNormal(ns);
          StoreSurfelRow(a, kRowNormal, i, __uint_as_float(packed));
        }
      }

      // Position and descriptors (PositionDescriptorKernel) of the surfels that are active now, with their new normal.
      const bool update = live && act;
      if (__ballot_sync(0xffffffffu, update) == 0) continue;
      const Vec3 nrm = UnpackNormal(packed);
      float radius_sq = 0.f, d1 = 0.f, d2 = 0.f;
      if (USE_DESC && update) {
        radius_sq = a.stream[4 * F + s];
        d1 = a.stream[5 * F + s];
        d2 = a.stream[6 * F + s];
      }
      PositionSums q;
      for (int g = 0; g < n_words; ++g) {
        unsigned vis = __shfl_sync(0xffffffffu, vis_word, g);
        for (int j = PopLowest(&vis); j >= 0; j = PopLowest(&vis)) {
          KfRegs K;
          LoadKfShared(recs + 32 * g + j, &K);
          K.tex = UniformTexture(K.tex);
          Assoc r;
          if (!update || !ProjectIntoImage(a.cam, K.T, gp, &r)) continue;
          PixelLoads l;
          DescEval e;
          bool photo = false;
          if (EvalPair(a.cam, K, gp, nrm, radius_sq, d1, d2, USE_DESC, &r, &l, &e, &photo) == 3)
            AccumulatePosition<USE_DEPTH, USE_DESC>(a.cam, r, e, photo, q);
        }
      }
      if (update) UpdatePosition<USE_DESC>(a, i, gp, nrm, d1, d2, q);
    }
  }
}

// The surfel deformation (DESIGN §3.13).  The walk is ActivationNormalsKernel's: the keyframe groups of a tile in ascending order,
// the warp's box culled against the group's views, the sums parked between groups in the scratch rows.  The records carry the
// ORIGINAL poses, so the voters of a surfel are the keyframes it is associated with at those poses, in ascending id; each adds
// D_k p - p and R_k n.  A surfel without a voter takes the keyframe whose original camera centre is nearest.  The per-surfel sums
// run in keyframe order without atomics, so a surfel's result does not depend on the order, the warp, the grouping or the culling.
constexpr int kDeformSums = 8;   // displacement x y z, normal x y z, voters, moved voters
__global__ void __launch_bounds__(kGeoThreads) DeformSurfelsKernel(const __grid_constant__ DeformArgs d) {
  extern __shared__ __align__(16) unsigned char geo_smem[];
  const GeometryArgs& a = d.geo;
  KfDevice* s_kfs = reinterpret_cast<KfDevice*>(geo_smem);
  const uint32_t tile_len = 1u << a.tile_shift;
  const uint32_t n_tiles = (a.end - a.begin + tile_len - 1) >> a.tile_shift;
  const uint32_t n_groups = (a.kf_count + kGeoGroup - 1) / kGeoGroup;
  const uint32_t n_items = n_groups * n_tiles;
  const size_t F = a.stream_pitch;
  const int lane = threadIdx.x & 31;
  // One voter's terms: D p - p and R n.
  auto vote = [&](const KfChange* __restrict__ c, const Vec3& p, const Vec3& n, float (&v)[kDeformSums]) {
    const float* D = c->D;
    const Vec3 q = Transform(D, p);
    v[0] += q.x - p.x;
    v[1] += q.y - p.y;
    v[2] += q.z - p.z;
    const Vec3 rn = Rotate(D, n);
    v[3] += rn.x;
    v[4] += rn.y;
    v[5] += rn.z;
    v[6] += 1.f;
    if (!__ldg(&c->unmoved)) v[7] += 1.f;
  };
  uint32_t group, tile;
  while (ClaimItem(a.queue, n_tiles, n_items, a.tile_epoch, &group, &tile)) {
    const bool first = group == 0, last = group + 1 == n_groups;
    const int j_begin = group * kGeoGroup, j_end = min(a.kf_count, static_cast<int>(group + 1) * kGeoGroup);
    const int n_kf = j_end - j_begin;
    KfDevice* recs = s_kfs + (threadIdx.x >> 5) * kGeoGroup;
    StageGroupRecords(a.kfs, a.kf_list + j_begin, n_kf, recs, lane);
    for (uint32_t sub = 0; sub < tile_len / 32; ++sub) {
      uint32_t s;
      const bool in_range = GeoStreamPosition(a, tile, sub, lane, &s);
      Vec3 gp = V3(0.f, 0.f, 0.f), nrm = V3(0.f, 0.f, 1.f);
      if (in_range) gp = V3(a.stream[0 * F + s], a.stream[1 * F + s], a.stream[2 * F + s]);
      const bool live = in_range && !isnan(gp.x);   // deleted surfels: x = NaN
      if (__ballot_sync(0xffffffffu, live) == 0) continue;
      if (live) nrm = UnpackNormal(__float_as_uint(a.stream[3 * F + s]));
      float v[kDeformSums] = {};
      if (!first && live) LoadParkedSums(a, s, v);
      float lo[3], hi[3];
      WarpBox(gp, live, lo, hi);
      unsigned vis = VisibleKeyframes<false>(a.cam, recs, n_kf, lo, hi, lane);
      for (int j = PopLowest(&vis); j >= 0; j = PopLowest(&vis)) {
        KfRegs K;
        LoadKfShared(recs + j, &K);
        Assoc r;
        if (live && ProjectIntoImage(a.cam, K.T, gp, &r) &&
            Associate(a.cam, K.T, nrm, LoadPixel(a.cam, K.depth, K.depth_pitch, K.normals, K.normals_pitch, r), &r) == 3)
          vote(d.changes + j_begin + j, gp, nrm, v);
      }
      if (live && !last) StoreParkedSums(a, s, v);
      bool unobserved = false, moved = false;
      if (live && last) {
        // Fallback: the keyframe whose original camera centre is nearest, the smaller id on a tie.
        unobserved = v[6] == 0.f;
        if (unobserved) {
          int best = 0;
          float best_d = INFINITY;
          for (int k = 0; k < a.kf_count; ++k) {
            const Vec3 e = gp - V3(__ldg(&d.changes[k].centre[0]), __ldg(&d.changes[k].centre[1]), __ldg(&d.changes[k].centre[2]));
            const float dist = Dot(e, e);
            if (dist < best_d) {
              best_d = dist;
              best = k;
            }
          }
          vote(d.changes + best, gp, nrm, v);
        }
        // A surfel whose voters are all unmoved keeps its bits.
        moved = v[7] != 0.f;
        if (moved) {
          const uint32_t i = GeoResultIndex(a, s);
          StoreSurfelRow(a, kRowX, i, gp.x + __fdiv_rn(v[0], v[6]));
          StoreSurfelRow(a, kRowY, i, gp.y + __fdiv_rn(v[1], v[6]));
          StoreSurfelRow(a, kRowZ, i, gp.z + __fdiv_rn(v[2], v[6]));
          const float len = __fsqrt_rn(v[3] * v[3] + v[4] * v[4] + v[5] * v[5]);
          // (normals that cancel out keep the old one)
          if (len > 0.f)
            StoreSurfelRow(a, kRowNormal, i, __uint_as_float(PackNormal(V3(__fdiv_rn(v[3], len), __fdiv_rn(v[4], len), __fdiv_rn(v[5], len)))));
        }
      }
      if (last) {
        const unsigned moved_lanes = __ballot_sync(0xffffffffu, moved), unobserved_lanes = __ballot_sync(0xffffffffu, unobserved);
        if (lane == 0 && moved_lanes) atomicAdd(d.counts, __popc(moved_lanes));
        if (lane == 0 && unobserved_lanes) atomicAdd(d.counts + 1, __popc(unobserved_lanes));
      }
    }
    RetireItem(a.tile_epoch, group, tile);
  }
}

// Keyframe co-visibility, bit rows (DESIGN §3.19).  The walk is DeformSurfelsKernel's at the current poses, without the sums: for
// every 32-surfel sub-step and visible keyframe j the ballot of the association test is word w = sub-step of row j, stored when
// it is not zero.  Nothing is parked between groups, so the items need no epoch order.  The association test is ProjectAssociate's
// three steps (SupportLevel0Kernel's test), spelled out.  CELLS (the frames of bba_measure_frame_overlap, DESIGN §3.20): every
// associated lane also sets the bit of its pixel's sparse cell in record j's cell row -- the cells surfel creation would find
// supported.
//
// The walk itself is CovisibilityWalk: for every sub-step it calls v.Begin(s, live), then v.Pair(row, w, s, assoc, r) for every
// visible keyframe (row: its position in kf_list, assoc: the lane's association test), then v.End(s, live); the calls are
// warp-uniform.  The exposure walk (ExposureWalkKernel, DESIGN §3.21) is the same walk with another visitor.
template <class Visitor>
__device__ __forceinline__ void CovisibilityWalk(const GeometryArgs& a, Visitor& v) {
  extern __shared__ __align__(16) unsigned char geo_smem[];
  KfDevice* s_kfs = reinterpret_cast<KfDevice*>(geo_smem);
  const uint32_t tile_len = 1u << a.tile_shift;
  const uint32_t n_tiles = (a.end - a.begin + tile_len - 1) >> a.tile_shift;
  const uint32_t n_groups = (a.kf_count + kGeoGroup - 1) / kGeoGroup;
  const uint32_t n_items = n_groups * n_tiles;
  const size_t F = a.stream_pitch;
  const int lane = threadIdx.x & 31;
  uint32_t group, tile;
  while (ClaimItem(a.queue, n_tiles, n_items, nullptr, &group, &tile)) {
    const int j_begin = group * kGeoGroup, j_end = min(a.kf_count, static_cast<int>(group + 1) * kGeoGroup);
    const int n_kf = j_end - j_begin;
    KfDevice* recs = s_kfs + (threadIdx.x >> 5) * kGeoGroup;
    StageGroupRecords(a.kfs, a.kf_list + j_begin, n_kf, recs, lane);
    for (uint32_t sub = 0; sub < tile_len / 32; ++sub) {
      uint32_t s;
      const bool in_range = GeoStreamPosition(a, tile, sub, lane, &s);
      Vec3 gp = V3(0.f, 0.f, 0.f), nrm = V3(0.f, 0.f, 1.f);
      if (in_range) gp = V3(a.stream[0 * F + s], a.stream[1 * F + s], a.stream[2 * F + s]);
      const bool live = in_range && !isnan(gp.x);   // deleted surfels: x = NaN
      if (__ballot_sync(0xffffffffu, live) == 0) continue;
      if (live) nrm = UnpackNormal(__float_as_uint(a.stream[3 * F + s]));
      float lo[3], hi[3];
      WarpBox(gp, live, lo, hi);
      unsigned vis = VisibleKeyframes<false>(a.cam, recs, n_kf, lo, hi, lane);
      const uint32_t w = (tile << (a.tile_shift - 5)) + sub;
      v.Begin(s, live);
      for (int j = PopLowest(&vis); j >= 0; j = PopLowest(&vis)) {
        KfRegs K;
        LoadKfShared(recs + j, &K);
        Assoc r;
        const bool assoc = live && ProjectIntoImage(a.cam, K.T, gp, &r) &&
                           Associate(a.cam, K.T, nrm, LoadPixel(a.cam, K.depth, K.depth_pitch, K.normals, K.normals_pitch, r), &r) == 3;
        v.Pair(j_begin + j, w, s, assoc, r);
      }
      v.End(s, live);
    }
  }
}

template <bool CELLS>
struct CovisibilityVisitor {
  const CovisibilityBitsArgs& c;
  __device__ __forceinline__ void Begin(uint32_t, bool) {}
  __device__ __forceinline__ void End(uint32_t, bool) {}
  __device__ __forceinline__ void Pair(int row, uint32_t w, uint32_t, bool assoc, const Assoc& r) {
    const unsigned word = __ballot_sync(0xffffffffu, assoc);
    if ((threadIdx.x & 31) == 0 && word) c.bits[static_cast<size_t>(row) * c.words + w] = word;
    if (CELLS && assoc) {
      const unsigned int cell = SparseCell(c.geo.cam, r.px, r.py);
      atomicOr(c.cells + static_cast<size_t>(row) * c.cell_words + (cell >> 5), 1u << (cell & 31u));
    }
  }
};

template <bool CELLS>
__global__ void __launch_bounds__(kGeoThreads) CovisibilityBitsKernel(const __grid_constant__ CovisibilityBitsArgs c) {
  CovisibilityVisitor<CELLS> v{c};
  CovisibilityWalk(c.geo, v);
}

// Keyframe exposures (DESIGN §3.21): the observation of a pair and its membership (ExposureWalkArgs), then per RHS
//  false: n and sum of the members, summed over the keyframes of a sub-step in registers and added with one integer atomic
//         per surfel; with bits, the members' ballot words;
//  true:  rhs[row] += n y - sum, reduced over the warp and added with one integer atomic per keyframe and sub-step.
template <bool RHS>
struct ExposureVisitor {
  const ExposureWalkArgs& e;
  uint32_t cnt = 0, tn = 0;   // accumulate: members of the sub-step; the surfel's test count / rhs: n
  long long acc = 0, tsum = 0;   // accumulate: their sum / rhs: sum; the surfel's test sum
  __device__ __forceinline__ void Begin(uint32_t s, bool live) {
    if (!live) return;
    const uint32_t i = s - e.geo.begin;
    if (e.test_n) {
      tn = __ldg(e.test_n + i);
      tsum = __ldg(e.test_sum + i);
    }
    if (RHS) {
      cnt = __ldg(e.n + i);
      acc = __ldg(e.sum + i);
    }
  }
  __device__ __forceinline__ void Pair(int row, uint32_t w, uint32_t, bool assoc, const Assoc& r) {
    int y = 0;
    bool member = false;
    float ccx, ccy;
    if (assoc && DepthToColor(e.geo.cam, r.pxf, r.pyf, &ccx, &ccy)) {
      const ExposureImage im = e.images[row];
      const int v = __ldg(im.rgba + static_cast<size_t>(ccy) * im.pitch + 4 * static_cast<size_t>(ccx) + 3);
      if (v >= e.min_luma && v <= e.max_luma) {
        y = e.log_q16[v];
        member = true;
        if (e.test_n) {
          const long long d = static_cast<long long>(tn) * (y - __ldg(e.test_x + row)) - tsum;
          member = (d < 0 ? -d : d) <= static_cast<long long>(tn) * e.tau;
        }
      }
    }
    if (RHS) {
      long long t = member ? static_cast<long long>(cnt) * y - acc : 0;
      if (__ballot_sync(0xffffffffu, member) == 0) return;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if ((threadIdx.x & 31) == 0 && t) atomicAdd(reinterpret_cast<unsigned long long*>(e.rhs + row), static_cast<unsigned long long>(t));
    } else {
      if (member) {
        ++cnt;
        acc += y - (e.sub_x ? __ldg(e.sub_x + row) : 0);
      }
      if (e.bits) {
        const unsigned word = __ballot_sync(0xffffffffu, member);
        if ((threadIdx.x & 31) == 0 && word) e.bits[static_cast<size_t>(row) * e.words + w] = word;
      }
    }
  }
  __device__ __forceinline__ void End(uint32_t s, bool live) {
    if (RHS || !live || cnt == 0) return;
    const uint32_t i = s - e.geo.begin;
    atomicAdd(e.n + i, cnt);
    atomicAdd(reinterpret_cast<unsigned long long*>(e.sum + i), static_cast<unsigned long long>(acc));
    cnt = 0;
    acc = 0;
  }
};

template <bool RHS>
__global__ void __launch_bounds__(kGeoThreads) ExposureWalkKernel(const __grid_constant__ ExposureWalkArgs e) {
  ExposureVisitor<RHS> v{e};
  CovisibilityWalk(e.geo, v);
}

// Keyframe co-visibility, the counts: counts[i][b] += sum_w popc(bits[rows[i]][w] & bits[b][w]).  A CTA owns a 64 x 64 tile of
// counts and the word range blockIdx.z of every row; it stages 32-word slices of its 64 listed rows and 64 columns in shared
// memory, and thread (tx, ty) sums rows ty + 16 i and columns tx + 16 j (i, j < 4) in registers.  A slice pair in which either side
// is all zero -- most of them: a keyframe sees a compact part of the spatially ordered stream -- is skipped.  The sums go to the
// counts with integer atomics, so the result does not depend on the order in which the CTAs finish.
constexpr int kGramTile = 64, kGramSlice = 32, kGramThreads = 256;
__global__ void __launch_bounds__(kGramThreads) CovisibilityGramKernel(const __grid_constant__ CovisibilityGramArgs a) {
  __shared__ uint32_t s_a[kGramTile][kGramSlice + 1], s_b[kGramTile][kGramSlice + 1];   // (+1: conflict-free column reads)
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int row0 = blockIdx.y * kGramTile, col0 = blockIdx.x * kGramTile;
  const uint32_t per = (a.words + gridDim.z - 1) / gridDim.z;
  const uint32_t w0 = blockIdx.z * per, w1 = min(a.words, w0 + per);
  // staging: thread t loads word t % 32 of tile rows t / 32 + 8 k
  const int load_w = threadIdx.x & 31, load_r = threadIdx.x >> 5;
  const uint32_t* a_row[kGramTile / 8];
  const uint32_t* b_row[kGramTile / 8];
#pragma unroll
  for (int k = 0; k < kGramTile / 8; ++k) {
    const int r = row0 + load_r + 8 * k, b = col0 + load_r + 8 * k;
    a_row[k] = r < a.row_count ? a.bits + static_cast<size_t>(__ldg(a.rows + r)) * a.words : nullptr;
    b_row[k] = b < a.col_count ? a.bits + static_cast<size_t>(b) * a.words : nullptr;
  }
  uint32_t acc[4][4] = {};
  for (uint32_t base = w0; base < w1; base += kGramSlice) {
    const uint32_t w = base + load_w;
    uint32_t any_a = 0u, any_b = 0u;
#pragma unroll
    for (int k = 0; k < kGramTile / 8; ++k) {
      const uint32_t va = w < w1 && a_row[k] ? __ldg(a_row[k] + w) : 0u;
      const uint32_t vb = w < w1 && b_row[k] ? __ldg(b_row[k] + w) : 0u;
      s_a[load_r + 8 * k][load_w] = va;
      s_b[load_r + 8 * k][load_w] = vb;
      any_a |= va;
      any_b |= vb;
    }
    const bool nonzero_a = __syncthreads_or(any_a != 0u);
    const bool nonzero_b = __syncthreads_or(any_b != 0u);
    if (nonzero_a && nonzero_b) {
#pragma unroll 4
      for (int kk = 0; kk < kGramSlice; ++kk) {
        uint32_t x[4], y[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          x[i] = s_a[ty + 16 * i][kk];
          y[i] = s_b[tx + 16 * i][kk];
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] += __popc(x[i] & y[j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = row0 + ty + 16 * i, b = col0 + tx + 16 * j;
      if (acc[i][j] && r < a.row_count && b < a.col_count) atomicAdd(a.counts + static_cast<size_t>(r) * a.col_count + b, acc[i][j]);
    }
}

constexpr size_t kGeoSmemBytes = sizeof(KfDevice) * (kGeoThreads / 32) * kGeoGroup;   // the per-warp record slices

// Everything a geometry launch does before its kernel: the grid (with *a's tile), the counters and the stream gather.
template <typename Kernel>
static LaunchResult PrepareGeo(Kernel kernel, GeometryArgs* a, int sm_count, bool desc_rows, cudaStream_t stream, uint32_t* grid) {
  int per_sm = 0;
  LaunchResult r{1, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kGeoThreads, kGeoSmemBytes)};
  *grid = EpochOrderedGrid(per_sm, sm_count, kGeoThreads, a->end - a->begin, (a->kf_count + kGeoGroup - 1) / kGeoGroup, &a->tile_shift);
  const uint32_t n_tiles = (a->end - a->begin + (1u << a->tile_shift) - 1) >> a->tile_shift;
  r += cudaMemsetAsync(a->queue, 0, sizeof(unsigned int), stream);
  r += cudaMemsetAsync(a->tile_epoch, 0, sizeof(unsigned int) * n_tiles, stream);
  r += LaunchGeometryStream(*a, desc_rows, stream);
  return r;
}

static GeometryArgs& Geo(GeometryArgs& a) { return a; }
template <typename Args> static GeometryArgs& Geo(Args& a) { return a.geo; }

// PrepareGeo, then the kernel on its argument struct a (a GeometryArgs, or a struct with one in .geo).
template <typename Kernel, typename Args>
static LaunchResult LaunchGeo(Kernel kernel, Args a, int sm_count, bool desc_rows, cudaStream_t stream) {
  uint32_t grid;
  const LaunchResult r = PrepareGeo(kernel, &Geo(a), sm_count, desc_rows, stream, &grid);
  kernel<<<grid, kGeoThreads, kGeoSmemBytes, stream>>>(a);
  return r;
}

LaunchResult LaunchDeformSurfels(const DeformArgs& a, int sm_count, cudaStream_t stream) {
  if (a.geo.end <= a.geo.begin || a.geo.kf_count <= 0) return {};
  return LaunchGeo(DeformSurfelsKernel, a, sm_count, false, stream);
}

LaunchResult LaunchCovisibilityBits(const CovisibilityBitsArgs& a, int sm_count, cudaStream_t stream) {
  if (a.geo.end <= a.geo.begin || a.geo.kf_count <= 0) return {};
  if (a.cells) return LaunchGeo(CovisibilityBitsKernel<true>, a, sm_count, false, stream);
  return LaunchGeo(CovisibilityBitsKernel<false>, a, sm_count, false, stream);
}

LaunchResult LaunchExposureWalk(const ExposureWalkArgs& a, int sm_count, cudaStream_t stream) {
  if (a.geo.end <= a.geo.begin || a.geo.kf_count <= 0) return {};
  if (a.rhs) return LaunchGeo(ExposureWalkKernel<true>, a, sm_count, false, stream);
  return LaunchGeo(ExposureWalkKernel<false>, a, sm_count, false, stream);
}

// grid.z splits the words so that the grid holds about four CTAs per SM (one slice at least per CTA).
LaunchResult LaunchCovisibilityGram(const CovisibilityGramArgs& a, int sm_count, cudaStream_t stream) {
  if (a.words == 0 || a.row_count <= 0 || a.col_count <= 0) return {};
  const uint32_t gx = (a.col_count + kGramTile - 1) / kGramTile, gy = (a.row_count + kGramTile - 1) / kGramTile;
  if (gy > 65535) return {0, cudaErrorInvalidValue};
  const uint64_t tiles = static_cast<uint64_t>(gx) * gy, slices = (a.words + kGramSlice - 1) / kGramSlice;
  const uint64_t gz = std::min<uint64_t>({std::max<uint64_t>(1, (4 * static_cast<uint64_t>(sm_count) + tiles - 1) / tiles), slices, 65535});
  CovisibilityGramKernel<<<dim3(gx, gy, static_cast<uint32_t>(gz)), kGramThreads, 0, stream>>>(a);
  return {1};
}

LaunchResult LaunchActivationAndNormals(const GeometryArgs& a, int sm_count, bool determine_activation, bool update_normals,
                                        cudaStream_t stream) {
  if (a.end <= a.begin || (!determine_activation && !update_normals)) return {};
  if (a.kf_count <= 0) {
    // no keyframe to look at: activation clears every flag, normals keep their value
    if (determine_activation) return {0, cudaMemsetAsync(a.active, 0, a.n, stream)};   // (every rank clears its whole replica)
    return {};
  }
  if (determine_activation && update_normals) return LaunchGeo(ActivationNormalsKernel<true, true>, a, sm_count, false, stream);
  if (determine_activation) return LaunchGeo(ActivationNormalsKernel<true, false>, a, sm_count, false, stream);
  return LaunchGeo(ActivationNormalsKernel<false, true>, a, sm_count, false, stream);
}

LaunchResult LaunchPositionAndDescriptor(const GeometryArgs& a, int sm_count, cudaStream_t stream) {
  if (a.end <= a.begin || a.kf_count <= 0) return {};
  if (a.cam.use_desc) {
    if (a.cam.use_depth) return LaunchGeo(PositionDescriptorKernel<true, true>, a, sm_count, true, stream);
    return LaunchGeo(PositionDescriptorKernel<false, true>, a, sm_count, true, stream);
  }
  return LaunchGeo(PositionDescriptorKernel<true, false>, a, sm_count, false, stream);
}

template <bool DETERMINE, bool USE_DEPTH, bool USE_DESC>
static LaunchResult LaunchGeometryPassT(GeometryArgs a, int sm_count, int tile_shift, cudaStream_t stream) {
  const auto kernel = GeometryPassKernel<DETERMINE, USE_DEPTH, USE_DESC>;
  const size_t smem = sizeof(KfDevice) * a.kf_count;
  int per_sm = 0;
  LaunchResult r{1, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kGeoThreads, smem)};
  const uint32_t grid = TileGrid(per_sm, sm_count, a.end - a.begin, tile_shift, &a.tile_shift);
  r += cudaMemsetAsync(a.queue, 0, sizeof(unsigned int), stream);
  kernel<<<grid, kGeoThreads, smem, stream>>>(a);
  return r;
}

template <bool DETERMINE>
static LaunchResult LaunchGeometryPassD(const GeometryArgs& a, int sm_count, int tile_shift, cudaStream_t stream) {
  if (a.cam.use_desc) {
    if (a.cam.use_depth) return LaunchGeometryPassT<DETERMINE, true, true>(a, sm_count, tile_shift, stream);
    return LaunchGeometryPassT<DETERMINE, false, true>(a, sm_count, tile_shift, stream);
  }
  return LaunchGeometryPassT<DETERMINE, true, false>(a, sm_count, tile_shift, stream);
}

LaunchResult LaunchGeometryPass(const GeometryArgs& a, int sm_count, bool determine_activation, int tile_shift, cudaStream_t stream) {
  if (a.end <= a.begin) return {};
  if (!GeometryPassFits(a)) return {0, cudaErrorInvalidValue};
  if (determine_activation) return LaunchGeometryPassD<true>(a, sm_count, tile_shift, stream);
  return LaunchGeometryPassD<false>(a, sm_count, tile_shift, stream);
}

// ------------------------------------------------------------------------------------------------
// Multi-GPU exchange helpers (the collectives themselves run in the host's NCCL communicator).

// Both kernels loop over kShardRows - 1 constant slots, so that rows.ids[r] is read straight from the kernel arguments, and load
// every row before the first store, so that the loads are in flight together.
__global__ void __launch_bounds__(256) PackShardKernel(const float* __restrict__ surfels, uint32_t pitch,
                                                       const uint8_t* __restrict__ active, uint32_t n, ShardRows rows,
                                                       const uint32_t* __restrict__ perm, uint32_t rank, uint32_t world, uint32_t shard_len,
                                                       float* __restrict__ slice) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;   // local index
  if (c >= shard_len) return;
  const uint32_t s = SurfelShardToGlobal(c, rank, world);   // stream position
  const bool in = s < n;
  const uint32_t i = in && perm ? __ldg(perm + s) : s;
  float v[kShardRows];
#pragma unroll
  for (int r = 0; r < kShardRows - 1; ++r) v[r] = in && r < rows.count ? surfels[static_cast<size_t>(rows.ids[r]) * pitch + i] : 0.f;
  v[kShardRows - 1] = in && rows.active ? static_cast<float>(active[i]) : 0.f;
#pragma unroll
  for (int r = 0; r < kShardRows - 1; ++r)
    if (r < rows.count) slice[static_cast<size_t>(r) * shard_len + c] = v[r];
  if (rows.active) slice[static_cast<size_t>(rows.count) * shard_len + c] = v[kShardRows - 1];
}

__global__ void __launch_bounds__(256) UnpackShardsKernel(float* __restrict__ surfels, uint32_t pitch, uint8_t* __restrict__ active,
                                                          uint32_t n, ShardRows rows, const uint32_t* __restrict__ perm, uint32_t shard_len,
                                                          uint32_t world, int skip_rank, const float* __restrict__ buffer) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;   // stream position
  if (s >= n) return;
  const uint32_t granule = s >> kShardGranuleShift;
  const uint32_t rank = granule % world;
  if (static_cast<int>(rank) == skip_rank) return;
  const uint32_t c = ((granule / world) << kShardGranuleShift) | (s & ((1u << kShardGranuleShift) - 1u));
  const uint32_t i = perm ? __ldg(perm + s) : s;
  const float* slice = buffer + static_cast<size_t>(rank) * (rows.count + rows.active) * shard_len;
  float v[kShardRows];
#pragma unroll
  for (int r = 0; r < kShardRows - 1; ++r) v[r] = r < rows.count ? slice[static_cast<size_t>(r) * shard_len + c] : 0.f;
  v[kShardRows - 1] = rows.active ? slice[static_cast<size_t>(rows.count) * shard_len + c] : 0.f;
#pragma unroll
  for (int r = 0; r < kShardRows - 1; ++r)
    if (r < rows.count) surfels[static_cast<size_t>(rows.ids[r]) * pitch + i] = v[r];
  if (rows.active) active[i] = static_cast<uint8_t>(v[kShardRows - 1]);
}

LaunchResult LaunchPackShard(const float* surfels, uint32_t pitch, const uint8_t* active, uint32_t n, ShardRows rows, const uint32_t* perm,
                             uint32_t rank, uint32_t world, uint32_t shard_len, float* slice, cudaStream_t stream) {
  if (shard_len == 0) return {};
  PackShardKernel<<<(shard_len + 255) / 256, 256, 0, stream>>>(surfels, pitch, active, n, rows, perm, rank, world, shard_len, slice);
  return {1};
}

LaunchResult LaunchUnpackShards(float* surfels, uint32_t pitch, uint8_t* active, uint32_t n, ShardRows rows, const uint32_t* perm,
                                uint32_t shard_len, int world, int skip_rank, const float* buffer, cudaStream_t stream) {
  if (n == 0) return {};
  UnpackShardsKernel<<<(n + 255) / 256, 256, 0, stream>>>(surfels, pitch, active, n, rows, perm, shard_len, static_cast<uint32_t>(world),
                                                          skip_rank, buffer);
  return {1};
}

__global__ void PackPoseResultsKernel(const int* __restrict__ ids, int n, const float* __restrict__ pose_est,
                                      const int* __restrict__ iterations, const int* __restrict__ converged,
                                      const double* __restrict__ first_stats, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int kf = ids[i];
  float* o = out + static_cast<size_t>(kf) * kPoseSlot;
  for (int j = 0; j < 7; ++j) o[j] = pose_est[kf * 7 + j];
  o[7] = static_cast<float>(iterations[kf]);
  o[8] = static_cast<float>(converged[kf]);
  for (int j = 0; j < 8; ++j) o[9 + j] = static_cast<float>(first_stats[kf * 8 + j]);
}

LaunchResult LaunchPackPoseResults(const int* ids, int n, const float* pose_est, const int* iterations, const int* converged,
                                   const double* first_stats, float* out, cudaStream_t stream) {
  if (n <= 0) return {};
  PackPoseResultsKernel<<<(n + 127) / 128, 128, 0, stream>>>(ids, n, pose_est, iterations, converged, first_stats, out);
  return {1};
}

// ------------------------------------------------------------------------------------------------
// uchar4 (.w = luma, cuda_image_processing.cu:165-176) -> dense u8 luma planes.  128-bit loads: 4 pixels per thread.
// grid.z = image: image z reads `first` (z = 0) or rest[z - 1] and writes rows [z * h, (z + 1) * h) of the luma planes.

__global__ void __launch_bounds__(256) ExtractLumaKernel(LumaSource first, const LumaSource* __restrict__ rest,
                                                         uint8_t* __restrict__ luma, size_t luma_pitch, int w, int h) {
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int y = blockIdx.y;
  if (x4 >= w || y >= h) return;
  const LumaSource f = blockIdx.z == 0 ? first : rest[blockIdx.z - 1];
  const uint8_t* src = f.rgba + static_cast<size_t>(y) * f.pitch + static_cast<size_t>(x4) * 4;
  uint8_t* dst = luma + (static_cast<size_t>(blockIdx.z) * h + y) * luma_pitch + x4;
  if (f.gain != 1.f) {   // exposure compensation (DESIGN §3.21); v / g correctly rounded, as the host and the tests compute it
    for (int k = 0; k < 4 && x4 + k < w; ++k) dst[k] = static_cast<uint8_t>(fminf(255.f, rintf(__fdiv_rn(src[4 * k + 3], f.gain))));
    return;
  }
  if (x4 + 3 < w &&(reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src));
    const uint32_t packed = (v.x >> 24) | ((v.y >> 24) << 8) | ((v.z >> 24) << 16) | ((v.w >> 24) << 24);
    *reinterpret_cast<uint32_t*>(dst) = packed;
  } else {
    for (int k = 0; k < 4 && x4 + k < w; ++k) dst[k] = src[4 * k + 3];
  }
}

LaunchResult LaunchExtractLuma(LumaSource first, const LumaSource* rest, int images, uint8_t* luma, size_t luma_pitch, int w, int h,
                               cudaStream_t stream) {
  if (images <= 0) return {};
  if (images > 65535) return {0, cudaErrorInvalidValue};   // grid.z
  dim3 block(256);
  dim3 grid((w / 4 + 255) / 256 + 1, h, images);
  ExtractLumaKernel<<<grid, block, 0, stream>>>(first, rest, luma, luma_pitch, w, h);
  return {1};
}

}  // namespace bba
