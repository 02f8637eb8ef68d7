// multi_gpu.cu -- multi-GPU support of libbadba_b200 (one process per GPU): surfel and keyframe sharding, the exchange of the
// geometry step's results, the barrier in front of peer stores, and the NVLink peer replicas (IPC export / import / unmap).
#include <cstring>

#include "handle.hpp"

namespace bba {
namespace {

// Keyframe -> rank assignment of a pose step.  Without statistics: round-robin over the work list
// (bba_shard_keyframe_owner).  With the statistics of the previous pose step (replicated, hence identical on all ranks):
// longest-processing-time-first onto the least loaded rank, so that the ranks finish their Gauss-Newton loops together.
void BalanceWork(const float* cost, int n, int world, int* owner) {
  double known_sum = 0;
  int known = 0;
  for (int i = 0; i < n; ++i)
    if (cost && cost[i] > 0) { known_sum += cost[i]; ++known; }
  if (known == 0 || world <= 1) {
    for (int i = 0; i < n; ++i) owner[i] = world > 1 ? i % world : 0;
    return;
  }
  const double fallback = known_sum / known;
  std::vector<std::pair<double, int>> order(n);
  for (int i = 0; i < n; ++i) order[i] = {-(cost[i] > 0 ? static_cast<double>(cost[i]) : fallback), i};
  std::sort(order.begin(), order.end());   // descending cost, ties by list position
  std::vector<double> load(world, 0.0);
  for (const auto& e : order) {
    int best = 0;
    for (int r = 1; r < world; ++r)
      if (load[r] < load[best]) best = r;
    owner[e.second] = best;
    load[best] -= e.first;
  }
}

// A barrier across the ranks: a 1-element sum all-reduce (every rank's earlier work on s precedes its contribution).
bba_status Barrier(bba_handle h, cudaStream_t s) {
  auto& x = h->xchg;
  BBA_CUDA(h, x.d_barrier.Reserve(1));
  BBA_CUDA(h, cudaMemsetAsync(x.d_barrier, 0, sizeof(float), s));
  return Collective(h, BBA_COLLECTIVE_ALLREDUCE_SUM, x.d_barrier, 1, s);
}

bba_status AllocationBase(bba_handle h, const void* ptr, void** base) {
  typedef int (*GetRangeFn)(unsigned long long*, size_t*, unsigned long long);
  // (looked up once per process; the initialisation of a local static is thread-safe, so handles of several threads may race here)
  static const GetRangeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &p, cudaEnableDefault, &q) != cudaSuccess) {
      cudaGetLastError();
      p = nullptr;
    }
    return reinterpret_cast<GetRangeFn>(p);
  }();
  if (!fn) return Fail(h, BBA_ERR_CUDA, "cuMemGetAddressRange is not available");
  unsigned long long b = 0;
  size_t size = 0;
  if (fn(&b, &size, reinterpret_cast<unsigned long long>(ptr)) != 0) return Fail(h, BBA_ERR_CUDA, "cuMemGetAddressRange failed");
  *base = reinterpret_cast<void*>(b);
  return BBA_OK;
}

// A member of a local group exchanges through its group: the calls that would replace that are refused, and leave the group
// in service (nothing changed).
bba_status RefuseMember(bba_handle h, const char* fn) {
  SetError(h, std::string(fn) + ": the handle is a member of a local group (bba_local_group_destroy first)");
  return BBA_ERR_STATE;
}

}  // namespace

void AssignKeyframes(bba_handle h, const std::vector<int>& ids, std::vector<int>* owner) {
  std::vector<float> cost(ids.size(), 0.f);
  for (size_t i = 0; i < ids.size(); ++i)
    if (ids[i] < static_cast<int>(h->kf_cost.size())) cost[i] = h->kf_cost[ids[i]];
  BalanceWork(cost.data(), static_cast<int>(ids.size()), h->cfg.world_size, owner->data());
}

// 256-surfel granules dealt round-robin (kernels.cuh SurfelShardToGlobal).  local_cap: size of this rank's local index space
// (a multiple of 256; the last granule may reach past n); shard_len: the same for rank 0 = slice length of the exchange.
void ShardSurfels(uint32_t n, int rank, int world, uint32_t* local_cap, uint32_t* shard_len) {
  const uint32_t granules = (n + 255u) / 256u;
  const uint32_t w = static_cast<uint32_t>(std::max(world, 1)), r = static_cast<uint32_t>(rank);
  const uint32_t mine = granules > r ? (granules - r + w - 1) / w : 0;
  if (local_cap) *local_cap = (world <= 1) ? n : mine * 256u;
  if (shard_len) *shard_len = ((granules + w - 1) / w) * 256u;
}

// Number of this rank's LOCAL surfel indices whose global index is below `global_end` (local -> global is monotonic).
uint32_t LocalCountBelow(uint32_t global_end, int rank, int world) {
  if (world <= 1) return global_end;
  const uint32_t full = global_end >> 8, rest = global_end & 255u;   // granules completely below, surfels of the next one
  const uint32_t w = static_cast<uint32_t>(world), r = static_cast<uint32_t>(rank);
  uint32_t mine = full > r ? (full - r + w - 1) / w : 0;
  uint32_t n = mine * 256u;
  if (full % w == r) n += rest;
  return n;
}

bba_status CheckCollective(bba_handle h) {
  if (h->cfg.world_size > 1 && !h->xchg.collective)
    return Fail(h, BBA_ERR_STATE, "world_size > 1 but no collective registered (bba_set_collective)");
  return BBA_OK;
}

bba_status Collective(bba_handle h, int op, void* buffer, size_t count, cudaStream_t s) {
  auto& x = h->xchg;
  x.exchange_error.clear();
  x.collective(x.collective_user, op, buffer, count, s);
  if (!x.exchange_error.empty()) return Fail(h, BBA_ERR_STATE, x.exchange_error);
  return BBA_OK;
}

// The count travels as two exactly representable floats (its low 12 bits, the rest), so that the float sum stays exact.
bba_status SumOverRanks(bba_handle h, uint32_t count, cudaStream_t s, uint32_t* total) {
  auto& x = h->xchg;
  BBA_CUDA(h, x.d_count_xchg.Reserve(2));
  BBA_CUDA(h, x.h_count_xchg.Reserve(2));
  x.h_count_xchg[0] = static_cast<float>(count & 0xfffu);
  x.h_count_xchg[1] = static_cast<float>(count >> 12);
  BBA_CUDA(h, cudaMemcpyAsync(x.d_count_xchg, x.h_count_xchg, sizeof(float) * 2, cudaMemcpyHostToDevice, s));
  if (bba_status st = Collective(h, BBA_COLLECTIVE_ALLREDUCE_SUM, x.d_count_xchg, 2, s)) return st;
  BBA_CUDA(h, cudaMemcpyAsync(x.h_count_xchg, x.d_count_xchg, sizeof(float) * 2, cudaMemcpyDeviceToHost, s));
  BBA_CUDA(h, cudaStreamSynchronize(s));
  *total = static_cast<uint32_t>(x.h_count_xchg[0] + 0.5f) + (static_cast<uint32_t>(x.h_count_xchg[1] + 0.5f) << 12);
  return BBA_OK;
}

bool PeerStores(bba_handle h) { return h->cfg.world_size > 1 && h->xchg.peers.count == h->cfg.world_size - 1; }
PeerSet KernelPeers(bba_handle h) { return PeerStores(h) ? h->xchg.peers : PeerSet{}; }

// Every rank has updated `rows` of its own surfel shard only (granules of stream positions, surfel perm[s] at position s; perm
// null: the caller's order): each rank packs them into its slice of the exchange buffer, one all-gather, and every rank unpacks
// the other ranks' slices.  The buffer grows to room for kShardRows rows of max_surfel_count surfels (or more).
bba_status ExchangeShards(bba_handle h, const ShardRows& rows, const uint32_t* perm, cudaStream_t s) {
  auto& x = h->xchg;
  const int world = h->cfg.world_size, rank = h->cfg.rank;
  uint32_t shard_len, max_len;
  ShardSurfels(h->surfels_size, rank, world, nullptr, &shard_len);
  ShardSurfels(std::max(h->cfg.max_surfel_count, h->surfels_size), 0, world, nullptr, &max_len);
  const size_t slice_floats = static_cast<size_t>(rows.count + rows.active) * shard_len;
  BBA_CUDA(h, x.d_exchange.Reserve(world * slice_floats, static_cast<size_t>(world) * kShardRows * max_len));
  BBA_LAUNCH(h, h->launches, LaunchPackShard, h->surfels, SurfelPitch(h), h->active, h->surfels_size, rows, perm, rank, world,
             shard_len, x.d_exchange + slice_floats * rank, s);
  if (bba_status st = Collective(h, BBA_COLLECTIVE_ALLGATHER, x.d_exchange, slice_floats * sizeof(float), s)) return st;
  BBA_LAUNCH(h, h->launches, LaunchUnpackShards, h->surfels, SurfelPitch(h), h->active, h->surfels_size, rows, perm, shard_len,
             world, rank, x.d_exchange, s);
  return BBA_OK;
}

// After the geometry step every rank has updated only its own surfel shard (granules of the order the geometry launches used).
bba_status ExchangeGeometry(bba_handle h, cudaStream_t s) {
  if (h->cfg.world_size <= 1 || h->surfels_size == 0) return BBA_OK;
  // the geometry kernels already stored the updated rows into every replica over NVLink: only a barrier is left
  if (PeerStores(h)) return Barrier(h, s);
  return ExchangeShards(h, ShardRows{{kRowX, kRowY, kRowZ, kRowNormal, kRowD1, kRowD2}, 6, 1}, h->geo.perm, s);
}

// A barrier across the ranks in front of kernels that write into the peers' replicas, needed only when a replicated pass ran
// since the last collective.
bba_status PeerFence(bba_handle h, cudaStream_t s) {
  if (h->cfg.world_size <= 1 || !h->xchg.replicated_pass_pending) return BBA_OK;
  h->xchg.replicated_pass_pending = false;
  if (!PeerStores(h)) return BBA_OK;   // exchange through the host's collective: no remote stores
  if (bba_status st = CheckCollective(h)) return st;
  return Barrier(h, s);
}

void UnmapPeers(bba_handle h) {
  auto& x = h->xchg;
  for (int i = 0; i < x.peer_base_count; ++i) cudaIpcCloseMemHandle(x.peer_bases[i]);
  x.peer_base_count = 0;
  x.peers = PeerSet{};
}

}  // namespace bba

using namespace bba;

extern "C" {

bba_status bba_peer_export(bba_handle h, bba_peer_handle* out) {
  if (!h || !out) return BBA_ERR_INVALID_ARGUMENT;
  if (bba_status st = CheckSurfels(h)) return st;
  std::memset(out, 0, sizeof(*out));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "bba_peer_handle layout");
  void* base = nullptr;
  cudaIpcMemHandle_t ipc;
  if (bba_status st = AllocationBase(h, h->surfels, &base)) return st;
  BBA_CUDA(h, cudaIpcGetMemHandle(&ipc, base));
  std::memcpy(out->surfels_ipc, &ipc, 64);
  out->surfels_offset = static_cast<uint64_t>(reinterpret_cast<const char*>(h->surfels) - static_cast<const char*>(base));
  if (bba_status st = AllocationBase(h, h->active, &base)) return st;
  BBA_CUDA(h, cudaIpcGetMemHandle(&ipc, base));
  std::memcpy(out->active_ipc, &ipc, 64);
  out->active_offset = static_cast<uint64_t>(reinterpret_cast<const char*>(h->active) - static_cast<const char*>(base));
  out->pitch_bytes = h->surfel_pitch_bytes;
  out->surfels_size = h->surfels_size;
  out->rank = h->cfg.rank;
  return BBA_OK;
}

bba_status bba_peer_import(bba_handle h, const bba_peer_handle* all, int count) {
  if (!h || !all) return BBA_ERR_INVALID_ARGUMENT;
  if (count != h->cfg.world_size) return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_peer_import: need one handle per rank");
  if (count - 1 > kMaxPeers) return Fail(h, BBA_ERR_UNSUPPORTED, "bba_peer_import: more than 8 ranks");
  if (h->xchg.group) return RefuseMember(h, "bba_peer_import");
  if (bba_status st = CheckSurfels(h)) return st;
  UnmapPeers(h);
  auto& x = h->xchg;
  PeerSet ps{};
  for (int r = 0; r < count; ++r) {
    if (r == h->cfg.rank) continue;
    const bba_peer_handle& ph = all[r];
    if (ph.rank != r || ph.pitch_bytes != h->surfel_pitch_bytes || ph.surfels_size != h->surfels_size) {
      UnmapPeers(h);
      return Fail(h, BBA_ERR_INVALID_ARGUMENT, "bba_peer_import: replica layout differs between ranks");
    }
    cudaIpcMemHandle_t ipc;
    void* base_s = nullptr;
    std::memcpy(&ipc, ph.surfels_ipc, 64);
    cudaError_t e = cudaIpcOpenMemHandle(&base_s, ipc, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      UnmapPeers(h);
      return Fail(h, BBA_ERR_CUDA, std::string("cudaIpcOpenMemHandle(surfels): ") + cudaGetErrorString(e));
    }
    x.peer_bases[x.peer_base_count++] = base_s;
    void* base_a = base_s;
    if (std::memcmp(ph.surfels_ipc, ph.active_ipc, 64) != 0) {
      std::memcpy(&ipc, ph.active_ipc, 64);
      e = cudaIpcOpenMemHandle(&base_a, ipc, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        UnmapPeers(h);
        return Fail(h, BBA_ERR_CUDA, std::string("cudaIpcOpenMemHandle(active): ") + cudaGetErrorString(e));
      }
      x.peer_bases[x.peer_base_count++] = base_a;
    }
    ps.surfels[ps.count] = reinterpret_cast<float*>(static_cast<char*>(base_s) + ph.surfels_offset);
    ps.active[ps.count] = reinterpret_cast<uint8_t*>(static_cast<char*>(base_a) + ph.active_offset);
    ++ps.count;
  }
  x.peers = ps;
  return BBA_OK;
}

int bba_peer_count(bba_handle h) { return h ? h->xchg.peers.count : 0; }

bba_status bba_mark_replica_rewritten(bba_handle h) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  h->xchg.replicated_pass_pending = true;   // -> PeerFence in front of the next kernel with peer stores
  return BBA_OK;
}

bba_status bba_peer_unmap(bba_handle h) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  UnmapPeers(h);
  return BBA_OK;
}

bba_status bba_set_collective(bba_handle h, bba_collective_fn fn, void* user) {
  if (!h) return BBA_ERR_INVALID_ARGUMENT;
  if (h->xchg.group) return RefuseMember(h, "bba_set_collective");
  h->xchg.collective = fn;
  h->xchg.collective_user = user;
  return BBA_OK;
}

int bba_shard_surfel_owner(uint32_t surfel_index, int world_size) {
  return world_size > 1 ? static_cast<int>((surfel_index >> kShardGranuleShift) % static_cast<uint32_t>(world_size)) : 0;
}

uint32_t bba_shard_surfel_local_index(uint32_t surfel_index, int world_size) {
  if (world_size <= 1) return surfel_index;
  const uint32_t g = surfel_index >> kShardGranuleShift;
  return ((g / static_cast<uint32_t>(world_size)) << kShardGranuleShift) | (surfel_index & ((1u << kShardGranuleShift) - 1u));
}

uint32_t bba_shard_slice_length(uint32_t surfels_size, int world_size) {
  uint32_t len = 0;
  ShardSurfels(surfels_size, 0, world_size, nullptr, &len);
  return len;
}

int bba_shard_keyframe_owner(int list_index, int world_size) { return world_size > 1 ? list_index % world_size : 0; }

void bba_balance_keyframes(const float* cost, int count, int world_size, int* owner) {
  if (count > 0 && owner) BalanceWork(cost, count, world_size, owner);
}

}  // extern "C"
