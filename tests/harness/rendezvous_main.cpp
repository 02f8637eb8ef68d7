// TEST HARNESS (CPU suite only): drives the host rendezvous of a local group (badslam_b200/csrc/rendezvous.hpp) with 2..9
// std::threads, no GPU.  Built and run by tests/test_local_group_rendezvous.py, plain and under sanitizers; it is not part of
// libbadba_b200.so.  Prints one line per scenario and exits non-zero on the first violation.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <thread>
#include <vector>

#include "../../badslam_b200/csrc/rendezvous.hpp"

namespace {

struct Slot {
  int rank = -1;
  long round = -1;
};

std::atomic<int> failures{0};

void Expect(bool ok, const char* what, int n, int rank, long round) {
  if (ok) return;
  if (failures.fetch_add(1) < 10) std::printf("FAIL %s: n %d rank %d round %ld\n", what, n, rank, round);
}

// Every rank runs `rounds` rounds; each round's slots must all carry that round, indexed by rank.
void InOrder(bba::Rendezvous<Slot>& rv, int n, long rounds) {
  std::vector<std::thread> threads;
  for (int r = 0; r < n; ++r)
    threads.emplace_back([&, r] {
      std::vector<Slot> all(n);
      for (long i = 0; i < rounds; ++i) {
        const bool ok = rv.Exchange(r, Slot{r, i}, all.data());
        Expect(ok, "exchange refused", n, r, i);
        for (int q = 0; q < n; ++q) Expect(all[q].rank == q && all[q].round == i, "slot out of order", n, r, i);
      }
    });
  for (auto& t : threads) t.join();
}

// Rank `poisoner` poisons instead of arriving at round `at`: every other rank completes the rounds before it, is released from
// round `at` with false, and every later Exchange returns false at once.
void Poisoned(bba::Rendezvous<Slot>& rv, int n, int poisoner, long at) {
  std::vector<std::thread> threads;
  for (int r = 0; r < n; ++r)
    threads.emplace_back([&, r] {
      std::vector<Slot> all(n);
      for (long i = 0; i < at; ++i) Expect(rv.Exchange(r, Slot{r, i}, all.data()), "exchange before the poison", n, r, i);
      if (r == poisoner) {
        rv.Poison();
        return;
      }
      Expect(!rv.Exchange(r, Slot{r, at}, all.data()), "waiter not released by the poison", n, r, at);
      for (long i = at + 1; i < at + 50; ++i) Expect(!rv.Exchange(r, Slot{r, i}, all.data()), "exchange after the poison", n, r, i);
    });
  for (auto& t : threads) t.join();
  Expect(rv.poisoned(), "poisoned state lost", n, poisoner, at);
}

}  // namespace

int main(int argc, char** argv) {
  const long rounds = argc > 1 ? std::atol(argv[1]) : 5000;
  for (int n = 2; n <= 9; ++n) {
    bba::Rendezvous<Slot> rv(n);
    InOrder(rv, n, rounds);
    Expect(rv.generation() == static_cast<uint64_t>(rounds), "generation count", n, -1, rounds);
    std::printf("n %d: %ld rounds in order\n", n, rounds);
    for (int p = 0; p < n; ++p) {
      const long at = 17 + 3 * p;
      Poisoned(rv, n, p, at);
      rv.Reset();
      Expect(!rv.poisoned(), "reset", n, p, at);
      InOrder(rv, n, 200);   // service restored
    }
    std::printf("n %d: poison from every rank releases every waiter; reset restores service\n", n);
  }
  // a poison while every other rank waits in the same round, from a thread that is not a rank
  {
    const int n = 5;
    bba::Rendezvous<Slot> rv(n);
    std::vector<std::thread> threads;
    for (int r = 0; r < n - 1; ++r)
      threads.emplace_back([&, r] {
        std::vector<Slot> all(n);
        Expect(!rv.Exchange(r, Slot{r, 0}, all.data()), "waiter not released by an outside poison", n, r, 0);
      });
    std::this_thread::sleep_for(std::chrono::milliseconds(20));
    rv.Poison();
    for (auto& t : threads) t.join();
    rv.Reset();
    InOrder(rv, n, 100);
    std::printf("outside poison releases the waiting ranks\n");
  }
  if (failures.load() != 0) {
    std::printf("%d failures\n", failures.load());
    return 1;
  }
  std::printf("all ok\n");
  return 0;
}
