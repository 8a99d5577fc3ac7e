// turn.hpp -- batches entering a section strictly in the order of their sequence numbers 0, 1, 2, ...  The single-GPU decode has one
// turn per search object (its walk), the sharded decode one per ordered section.  Private to libltephy_b200.
#pragma once
#include "../../include/ltephy_search.h"
#include <condition_variable>
#include <cstdint>
#include <mutex>
#include <set>

struct Turn {
  std::mutex              m; // also held by whoever has the turn, for as long as it has it
  std::condition_variable cv;
  uint64_t                next = 0; // the seq whose turn it is
  std::set<uint64_t>      claimed;  // seqs >= next that a call owns
  // Makes the calling batch the one owner of seq.  false: seq's turn has been passed on already (a reused seq, or a restart from 0), so
  // waiting for it would never end, or another call owns seq and this one would run the batch twice.  The caller then refuses seq before it
  // makes a TurnGuard, so the refusal consumes nothing.  LTEPHY_SEQ_NONE takes no part in the order and is never owned.
  bool claim(uint64_t seq)
  {
    std::lock_guard<std::mutex> lk(m);
    return seq == LTEPHY_SEQ_NONE || (seq >= next && claimed.insert(seq).second);
  }
};

// The turn of a batch that owns its seq (Turn::claim, on this turn or on one that every batch takes before it).  It is passed on exactly
// once, on every path out of the guard's scope, an error path included, so a failing batch never leaves the later ones waiting.
struct TurnGuard {
  Turn&                        t;
  const uint64_t               seq;
  std::unique_lock<std::mutex> lk;
  bool                         done = false;
  TurnGuard(Turn& t_, uint64_t s) : t(t_), seq(s), lk(t_.m, std::defer_lock) {}
  ~TurnGuard() { pass(); }
  // Waits for the turn and holds it until pass().  With LTEPHY_SEQ_NONE it only excludes the other holders of the turn.
  void take()
  {
    lk.lock();
    t.cv.wait(lk, [&] { return seq == LTEPHY_SEQ_NONE || t.next == seq; });
  }
  // Hands the turn to seq + 1.  A batch that never took its turn (it failed before, or skips the section) waits for it first.
  void pass()
  {
    if (done) return;
    if (!lk.owns_lock()) take();
    if (seq != LTEPHY_SEQ_NONE) t.next = seq + 1, t.claimed.erase(seq);
    lk.unlock();
    done = true;
    t.cv.notify_all();
  }
};
