// rendezvous.hpp -- the host barrier of a local group (local_group.cu): the n ranks of one process each publish a slot and
// receive every rank's slot of the same round.  Plain C++ (no CUDA), so that tests/harness/rendezvous_host.cpp can drive it
// with std::threads on a machine without a GPU.
#pragma once

#include <algorithm>
#include <condition_variable>
#include <cstdint>
#include <mutex>
#include <vector>

namespace bba {

// A generation-counted barrier that carries one Slot per rank.  Round g keeps its slots in slots_[g & 1]: a rank that leaves
// round g early can publish its slot of round g + 1 while slower ranks still copy round g's, and it cannot reach round g + 2
// before every rank has arrived at g + 1, i.e. finished copying g.
//
// Poisoned state: once Poison() is called, every rank waiting in a round that has not completed and every later Exchange
// returns false at once, so no thread waits forever for a rank that gave up.  Reset() restores service; it must only be called while no rank is
// inside Exchange.
template <class Slot>
class Rendezvous {
 public:
  explicit Rendezvous(int n) : n_(n) {
    slots_[0].resize(n);
    slots_[1].resize(n);
  }

  // Publishes `mine` as rank's slot of the current round, waits until every rank has published, and copies the round's n
  // slots (indexed by rank) to `all`.  false: the rendezvous is poisoned (nothing was copied).
  bool Exchange(int rank, const Slot& mine, Slot* all) {
    std::unique_lock<std::mutex> lock(mu_);
    if (poisoned_) return false;
    const uint64_t gen = generation_;
    std::vector<Slot>& round = slots_[gen & 1];
    round[rank] = mine;
    if (++arrived_ == n_) {
      arrived_ = 0;
      ++generation_;
      cv_.notify_all();
    } else {
      cv_.wait(lock, [&] { return generation_ != gen || poisoned_; });
      // (a round that completed is delivered to every rank, even when a faster rank has poisoned the group since)
      if (generation_ == gen) return false;
    }
    std::copy(round.begin(), round.end(), all);
    return true;
  }

  void Poison() {
    std::lock_guard<std::mutex> lock(mu_);
    poisoned_ = true;
    cv_.notify_all();
  }

  // Clears the poisoned state and forgets the ranks that had arrived in the round that was abandoned.
  void Reset() {
    std::lock_guard<std::mutex> lock(mu_);
    poisoned_ = false;
    arrived_ = 0;
    ++generation_;
  }

  bool poisoned() {
    std::lock_guard<std::mutex> lock(mu_);
    return poisoned_;
  }

  uint64_t generation() {
    std::lock_guard<std::mutex> lock(mu_);
    return generation_;
  }

 private:
  const int n_;
  std::mutex mu_;
  std::condition_variable cv_;
  uint64_t generation_ = 0;
  int arrived_ = 0;
  bool poisoned_ = false;
  std::vector<Slot> slots_[2];
};

}  // namespace bba
