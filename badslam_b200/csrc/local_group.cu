// local_group.cu -- local groups (bba_local_group_*): the ranks of a multi-GPU bundle adjustment as handles of one process,
// each driven by its own host thread, exchanging through device memory and CUDA events instead of a host collective.
//
// A group installs GroupCollective as every member's bba_collective_fn (user = the member's record).  Both operations run in
// two phases ordered by the host rendezvous (rendezvous.hpp) and by events only -- no kernel ever waits for another rank:
//   phase 1: each rank records `ready` on its stream once its buffer holds its contribution and publishes (buffer, event);
//            every stream waits on every other rank's `ready`, then
//              ALLREDUCE_SUM: one kernel sums the ranks' buffers in rank order 0..N-1 into this rank's scratch;
//              ALLGATHER:     copies of the other ranks' slices out of their buffers into this rank's buffer;
//   phase 2: each rank records `done` (it has finished reading the others' buffers) and publishes it; every stream waits on
//            every other rank's `done` before it overwrites its own buffer (the all-reduce's copy of the scratch back) or
//            returns it to the library for reuse.
// Every rank therefore computes the same fp32 sums in the same order: the replicas stay bit-identical.
//
// The sum kernel is built without -use_fast_math: denormal inputs and results are kept, as a sequential host sum keeps them.
#include <cstring>

#include "handle.hpp"
#include "rendezvous.hpp"

namespace bba {
namespace {

constexpr int kMaxRanks = kMaxPeers + 1;

struct SumArgs {
  const float* src[kMaxRanks];
  float* dst;
  size_t count;
  int ranks;
};

// dst[i] = ((src[0][i] + src[1][i]) + src[2][i]) + ...: 128-bit loads and stores where every pointer is 16-byte aligned, a
// scalar loop over the tail (and over everything otherwise).  The other ranks' buffers are read over NVLink when they live on
// another device.
__global__ void __launch_bounds__(256) LocalGroupSumKernel(SumArgs a, int vec) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t first = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  size_t scalar_begin = 0;
  if (vec) {
    const size_t n4 = a.count / 4;
    for (size_t i = first; i < n4; i += stride) {
      float4 acc = reinterpret_cast<const float4*>(a.src[0])[i];
#pragma unroll
      for (int r = 1; r < kMaxRanks; ++r) {   // (constant indices: the pointers stay in the parameter bank)
        if (r >= a.ranks) break;
        const float4 v = reinterpret_cast<const float4*>(a.src[r])[i];
        acc.x = __fadd_rn(acc.x, v.x);
        acc.y = __fadd_rn(acc.y, v.y);
        acc.z = __fadd_rn(acc.z, v.z);
        acc.w = __fadd_rn(acc.w, v.w);
      }
      reinterpret_cast<float4*>(a.dst)[i] = acc;
    }
    scalar_begin = n4 * 4;
  }
  for (size_t i = scalar_begin + first; i < a.count; i += stride) {
    float acc = a.src[0][i];
#pragma unroll
    for (int r = 1; r < kMaxRanks; ++r) {
      if (r >= a.ranks) break;
      acc = __fadd_rn(acc, a.src[r][i]);
    }
    a.dst[i] = acc;
  }
}

// What a rank publishes in each phase.
struct Slot {
  void* buffer = nullptr;
  cudaEvent_t event = nullptr;
  int op = -1;
  size_t count = 0;
};

}  // namespace
}  // namespace bba

// One rank of a group: the collective's `user`.
struct bba_local_group_member {
  bba_local_group group = nullptr;
  bba_handle h = nullptr;
  int rank = 0;
  int device = 0;
  int sm_count = 0;
  bba::Event ready, done;
  bba::DeviceBuffer<float> scratch;   // the all-reduce's sums, on this rank's device
};

struct bba_local_group_s {
  explicit bba_local_group_s(int n) : count(n), rendezvous(n) {}
  const int count;
  bool peer_stores = false;
  bba_local_group_member members[bba::kMaxPeers + 1];
  bba::Rendezvous<bba::Slot> rendezvous;
};

namespace bba {

void PoisonLocalGroup(bba_local_group g) { g->rendezvous.Poison(); }

namespace {

// One exchange of rank m on stream s; an empty string on success, else the reason (the group is then poisoned).
std::string RunExchange(bba_local_group_member& m, int op, void* buffer, size_t count, cudaStream_t s) {
  bba_local_group g = m.group;
  const int n = g->count;
  Slot all[kMaxRanks];
#define LG_CUDA(expr)                                                              \
  do {                                                                             \
    const cudaError_t e__ = (expr);                                                \
    if (e__ != cudaSuccess) return std::string(#expr) + ": " + cudaGetErrorString(e__); \
  } while (0)
  if (op != BBA_COLLECTIVE_ALLREDUCE_SUM && op != BBA_COLLECTIVE_ALLGATHER) return "unknown collective op";
  // phase 1: contributions ready
  LG_CUDA(cudaEventRecord(m.ready, s));
  if (!g->rendezvous.Exchange(m.rank, Slot{buffer, m.ready, op, count}, all)) return "the local group is poisoned";
  for (int q = 0; q < n; ++q)
    if (all[q].op != op || all[q].count != count)
      return "the ranks of the local group issued different exchanges (op " + std::to_string(all[q].op) + " count " +
             std::to_string(all[q].count) + " on rank " + std::to_string(q) + ", op " + std::to_string(op) + " count " +
             std::to_string(count) + " on rank " + std::to_string(m.rank) + ")";
  for (int q = 0; q < n; ++q)
    if (q != m.rank) LG_CUDA(cudaStreamWaitEvent(s, all[q].event, 0));
  if (op == BBA_COLLECTIVE_ALLREDUCE_SUM) {
    if (count > 0) {
      LG_CUDA(m.scratch.Reserve(count, count + count / 4));
      SumArgs a{};
      bool aligned = (reinterpret_cast<uintptr_t>(m.scratch.get()) & 15) == 0;
      for (int q = 0; q < n; ++q) {
        a.src[q] = static_cast<const float*>(all[q].buffer);
        aligned = aligned && (reinterpret_cast<uintptr_t>(all[q].buffer) & 15) == 0;
      }
      a.dst = m.scratch;
      a.count = count;
      a.ranks = n;
      const size_t work = aligned ? (count + 3) / 4 : count;
      const unsigned int blocks = static_cast<unsigned int>(std::min<size_t>((work + 255) / 256, static_cast<size_t>(4) * m.sm_count));
      LocalGroupSumKernel<<<std::max(blocks, 1u), 256, 0, s>>>(a, aligned ? 1 : 0);
      LG_CUDA(cudaGetLastError());
      ++m.h->launches;
    }
  } else {
    for (int q = 0; q < n; ++q)
      if (q != m.rank && count > 0)
        LG_CUDA(cudaMemcpyAsync(static_cast<char*>(buffer) + q * count, static_cast<const char*>(all[q].buffer) + q * count, count,
                                cudaMemcpyDefault, s));
  }
  // phase 2: every rank has finished reading the others' buffers
  LG_CUDA(cudaEventRecord(m.done, s));
  if (!g->rendezvous.Exchange(m.rank, Slot{buffer, m.done, op, count}, all)) return "the local group is poisoned";
  for (int q = 0; q < n; ++q)
    if (q != m.rank) LG_CUDA(cudaStreamWaitEvent(s, all[q].event, 0));
  if (op == BBA_COLLECTIVE_ALLREDUCE_SUM && count > 0)
    LG_CUDA(cudaMemcpyAsync(buffer, m.scratch, sizeof(float) * count, cudaMemcpyDeviceToDevice, s));
#undef LG_CUDA
  return std::string();
}

void GroupCollective(void* user, int op, void* buffer, size_t count, void* stream) {
  auto& m = *static_cast<bba_local_group_member*>(user);
  std::string why = RunExchange(m, op, buffer, count, static_cast<cudaStream_t>(stream));
  if (!why.empty()) {
    m.group->rendezvous.Poison();
    m.h->xchg.exchange_error = "local group exchange, rank " + std::to_string(m.rank) + ": " + why;
  }
}

bba_status CreateFail(bba_handle h, bba_status s, const std::string& msg) {
  if (h) SetError(h, "bba_local_group_create: " + msg);
  return s;
}

}  // namespace
}  // namespace bba

using namespace bba;

extern "C" {

bba_status bba_local_group_create(const bba_handle* ranks, int count, int peer_stores, bba_local_group* out) {
  if (!ranks || !out || count < 1) return BBA_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  for (int i = 0; i < count; ++i)
    if (!ranks[i]) return BBA_ERR_INVALID_ARGUMENT;
  bba_handle h0 = ranks[0];
  if (count > kMaxRanks) return CreateFail(h0, BBA_ERR_UNSUPPORTED, "more than 9 ranks");
  // every check before anything changes
  for (int i = 0; i < count; ++i) {
    bba_handle h = ranks[i];
    if (h->cfg.world_size != count || h->cfg.rank != i)
      return CreateFail(h, BBA_ERR_INVALID_ARGUMENT, "ranks[i] must be the handle of rank i of a world of `count` ranks");
    if (h->xchg.group) return CreateFail(h, BBA_ERR_STATE, "the handle is already a member of a local group");
    if (h->xchg.peers.count > 0) return CreateFail(h, BBA_ERR_STATE, "the handle has imported peer replicas (bba_peer_unmap first)");
    if (peer_stores) {
      if (bba_status st = CheckSurfels(h)) return st;
      if (h->surfels_size != h0->surfels_size || h->surfel_pitch_bytes != h0->surfel_pitch_bytes)
        return CreateFail(h, BBA_ERR_INVALID_ARGUMENT, "peer_stores: the replicas differ in surfels_size or pitch");
    }
  }
  int caller_device = 0;
  BBA_CUDA(h0, cudaGetDevice(&caller_device));
  for (int i = 0; i < count; ++i)
    for (int j = 0; j < count; ++j) {
      const int di = ranks[i]->cfg.device, dj = ranks[j]->cfg.device;
      int can = 0;
      if (di == dj) continue;
      BBA_CUDA(h0, cudaDeviceCanAccessPeer(&can, di, dj));
      if (!can) return CreateFail(h0, BBA_ERR_UNSUPPORTED, "devices " + std::to_string(di) + " and " + std::to_string(dj) +
                                                          " cannot access each other's memory");
    }
  std::unique_ptr<bba_local_group_s> g(new bba_local_group_s(count));
  g->peer_stores = peer_stores != 0;
  auto setup = [&]() -> bba_status {
    for (int i = 0; i < count; ++i) {
      bba_local_group_member& m = g->members[i];
      m.group = g.get();
      m.h = ranks[i];
      m.rank = i;
      m.device = ranks[i]->cfg.device;
      m.sm_count = ranks[i]->sm_count;
      BBA_CUDA(m.h, cudaSetDevice(m.device));
      // what the caller enqueued before (surfel uploads, flag initialisation) is complete before any rank's exchange or peer
      // store: the members' streams are ordered by the group's events only from here on
      BBA_CUDA(m.h, cudaDeviceSynchronize());
      BBA_CUDA(m.h, cudaEventCreateWithFlags(&m.ready.r, cudaEventDisableTiming));
      BBA_CUDA(m.h, cudaEventCreateWithFlags(&m.done.r, cudaEventDisableTiming));
      // peer access of this rank's device to every other rank's (a property of the process: left enabled at destroy)
      for (int j = 0; j < count; ++j) {
        const int d = ranks[j]->cfg.device;
        if (d == m.device) continue;
        const cudaError_t e = cudaDeviceEnablePeerAccess(d, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) {
          cudaGetLastError();
        } else {
          BBA_CUDA(m.h, e);
        }
      }
    }
    return BBA_OK;
  };
  const bba_status st = setup();
  cudaSetDevice(caller_device);
  if (st != BBA_OK) return st;
  for (int i = 0; i < count; ++i) {
    bba_handle h = ranks[i];
    h->xchg.group = g.get();
    h->xchg.collective = GroupCollective;
    h->xchg.collective_user = &g->members[i];
    if (g->peer_stores && count > 1) {
      PeerSet ps{};
      for (int q = 0; q < count; ++q) {
        if (q == i) continue;
        ps.surfels[ps.count] = ranks[q]->surfels;
        ps.active[ps.count] = ranks[q]->active;
        ++ps.count;
      }
      h->xchg.peers = ps;
      h->xchg.replicated_pass_pending = true;   // the replicas were written outside the group: fence the first peer stores
    }
  }
  *out = g.release();
  return BBA_OK;
}

bba_status bba_local_group_reset(bba_local_group g) {
  if (!g) return BBA_ERR_INVALID_ARGUMENT;
  g->rendezvous.Reset();
  return BBA_OK;
}

bba_status bba_local_group_poison(bba_local_group g) {
  if (!g) return BBA_ERR_INVALID_ARGUMENT;
  g->rendezvous.Poison();
  return BBA_OK;
}

void bba_local_group_destroy(bba_local_group g) {
  if (!g) return;
  int caller_device = 0;
  cudaGetDevice(&caller_device);
  for (int i = 0; i < g->count; ++i) {   // no exchange of the group may still run on a device when its buffers go
    cudaSetDevice(g->members[i].device);
    cudaDeviceSynchronize();
  }
  cudaSetDevice(caller_device);
  for (int i = 0; i < g->count; ++i) {
    bba_handle h = g->members[i].h;
    h->xchg.group = nullptr;
    h->xchg.collective = nullptr;
    h->xchg.collective_user = nullptr;
    if (g->peer_stores) h->xchg.peers = PeerSet{};
  }
  delete g;
}

bba_status bba_debug_collective(bba_handle h, int op, void* device_buffer, size_t count, void* stream) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (op != BBA_COLLECTIVE_ALLREDUCE_SUM && op != BBA_COLLECTIVE_ALLGATHER)
    return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_collective: unknown op");
  if (!device_buffer && count > 0) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_debug_collective: null buffer");
  if (!h->xchg.collective) return Fail(h, BBA_ERR_STATE, "bba_debug_collective: no exchange registered");
  return Collective(h, op, device_buffer, count, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
