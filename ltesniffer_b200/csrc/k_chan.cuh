// k_chan.cuh -- arguments shared by the channeliser kernel (k_chan.cu) and its host code (chan.cu).  Private to libltephy_b200.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#define CHAN_THREADS 256
#define CHAN_MAX_SEGS 16 // 8 carriers x 2 antennas

struct ChanSeg {       // one (carrier, antenna) of a call: outputs m0 .. m0 + count - 1, in tiles of M
  const float2* g;     // [T] taps g[k] at k + H
  const float2* rot;   // [P] r[m mod P]
  float2*       out;   // [count] this antenna's row of the carrier's output
  uint64_t      m0;    // first output index
  uint32_t      count, D, T, P;
  uint32_t      M;     // outputs per tile
  uint32_t      rows;  // rows of the tile's polyphase input in shared memory: M - 1 + ceil(T / D)
  uint32_t      tile0; // first tile of this segment in the grid
  uint32_t      a;     // antenna
};

struct ChanArgs {
  const float2* x;     // [A][lda] samples first .. first + lda - 1
  uint64_t      lda, first;
  uint32_t      nseg, pad;
  ChanSeg       seg[CHAN_MAX_SEGS];
};

// every tile of every segment in one launch: ntiles CTAs of CHAN_THREADS, smem bytes of dynamic shared memory
extern "C" int launch_chan(const ChanArgs& g, uint32_t ntiles, size_t smem, cudaStream_t st);
