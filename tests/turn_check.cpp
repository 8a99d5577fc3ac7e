// Checks of ltesniffer_b200/csrc/turn.hpp, built and run by test_turn.py: batches numbered by seq pass the four ordered sections of a sharded
// call (exchange, full-table fetch, walk, gather) in seq order, a duplicate or stale seq is refused before it touches any turn, and a batch
// that fails passes every section on.  Exits 0 and prints "ok"; any failed check or a wait past the watchdog exits non-zero.
#include "turn.hpp"
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <thread>
#include <unistd.h>
#include <vector>

#define CHECK(c)                                                                                   \
  do {                                                                                             \
    if (!(c)) {                                                                                    \
      fprintf(stderr, "%s:%d: check failed: %s\n", __FILE__, __LINE__, #c);                        \
      _exit(1);                                                                                    \
    }                                                                                              \
  } while (0)

struct Shard { // the four turns of a sharded rank, and the order in which batches entered each section
  Turn                  turn[4];
  std::vector<uint64_t> log[4];
  // one call of ltephy_decode_subframes_sharded: claim at entry, then the sections in order; fail_at = section index before which it fails
  bool call(uint64_t seq, int fail_at = 4)
  {
    if (!turn[0].claim(seq)) return false;
    TurnGuard g0(turn[0], seq), g1(turn[1], seq), g2(turn[2], seq), g3(turn[3], seq);
    TurnGuard* g[4] = {&g0, &g1, &g2, &g3};
    for (int k = 0; k < 4; k++) {
      if (k == fail_at) return true;
      g[k]->take();
      log[k].push_back(seq);
      std::this_thread::sleep_for(std::chrono::microseconds(200));
      g[k]->pass();
    }
    return true;
  }
  uint64_t next(int k)
  {
    std::lock_guard<std::mutex> lk(turn[k].m);
    return turn[k].next;
  }
};

int main()
{
  std::thread([] { // a turn that is never passed on makes this program fail instead of hang
    std::this_thread::sleep_for(std::chrono::seconds(30));
    fprintf(stderr, "watchdog: a turn was never passed on\n");
    _exit(2);
  }).detach();

  { // a second call with the seq of a call in flight is refused at entry and touches no turn; the owner goes through all four sections
    Shard sh;
    CHECK(sh.turn[0].claim(0));                    // call A, still in phase A
    CHECK(!sh.turn[0].claim(0));                   // call B, same seq: refused
    for (int k = 0; k < 4; k++) CHECK(sh.next(k) == 0);
    {
      TurnGuard g0(sh.turn[0], 0), g1(sh.turn[1], 0), g2(sh.turn[2], 0), g3(sh.turn[3], 0);
      TurnGuard* g[4] = {&g0, &g1, &g2, &g3};
      for (int k = 0; k < 4; k++) g[k]->take(), g[k]->pass();
    }
    for (int k = 0; k < 4; k++) CHECK(sh.next(k) == 1);
    CHECK(!sh.call(0));                            // after its turn: stale
    CHECK(sh.call(1));
    for (int k = 0; k < 4; k++) CHECK(sh.log[k].size() == 1 && sh.log[k][0] == 1 && sh.next(k) == 2);
  }

  { // 8 threads race with the same seq while another thread holds seq 0: exactly one owns seq 1, and every section sees 0 then 1
    Shard                 sh;
    std::atomic<int>      go{0}, won{0};
    std::vector<std::thread> th;
    CHECK(sh.turn[0].claim(0));
    for (int i = 0; i < 8; i++)
      th.emplace_back([&] {
        while (!go.load()) std::this_thread::yield();
        won += sh.call(1);
      });
    go = 1;
    std::this_thread::sleep_for(std::chrono::milliseconds(20));
    {
      TurnGuard g0(sh.turn[0], 0), g1(sh.turn[1], 0), g2(sh.turn[2], 0), g3(sh.turn[3], 0);
      TurnGuard* g[4] = {&g0, &g1, &g2, &g3};
      for (int k = 0; k < 4; k++) g[k]->take(), sh.log[k].push_back(0), g[k]->pass();
    }
    for (auto& t : th) t.join();
    CHECK(won.load() == 1);
    for (int k = 0; k < 4; k++) CHECK(sh.log[k] == std::vector<uint64_t>({0, 1}) && sh.next(k) == 2);
    CHECK(sh.turn[0].claimed.empty());
  }

  { // batches arriving in reverse order enter every section in seq order; batch 2 fails before its first section and batch 4 before the
    // walk, and both still pass every section on
    Shard                    sh;
    std::vector<std::thread> th;
    for (int s = 7; s >= 0; s--) {
      th.emplace_back([&sh, s] { CHECK(sh.call((uint64_t)s, s == 2 ? 0 : s == 4 ? 2 : 4)); });
      std::this_thread::sleep_for(std::chrono::milliseconds(1));
    }
    for (auto& t : th) t.join();
    CHECK(sh.log[0] == std::vector<uint64_t>({0, 1, 3, 4, 5, 6, 7}) && sh.log[1] == sh.log[0]);
    CHECK(sh.log[2] == std::vector<uint64_t>({0, 1, 3, 5, 6, 7}) && sh.log[3] == sh.log[2]);
    for (int k = 0; k < 4; k++) CHECK(sh.next(k) == 8);
  }

  { // LTEPHY_SEQ_NONE: never owned, never refused, takes no part in the order; take() still excludes the other holders
    Turn turn;
    CHECK(turn.claim(LTEPHY_SEQ_NONE) && turn.claim(LTEPHY_SEQ_NONE));
    long                     count = 0;
    std::vector<std::thread> th;
    for (int i = 0; i < 4; i++)
      th.emplace_back([&] {
        for (int j = 0; j < 10000; j++) {
          TurnGuard g(turn, LTEPHY_SEQ_NONE);
          g.take();
          count = count + 1;
        }
      });
    for (auto& t : th) t.join();
    CHECK(count == 40000 && turn.next == 0 && turn.claimed.empty());
  }
  printf("ok\n");
  return 0;
}
