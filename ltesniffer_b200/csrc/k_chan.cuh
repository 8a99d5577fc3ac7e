// k_chan.cuh -- arguments shared by the channeliser kernel (k_chan.cu) and its host code (chan.cu).  Private to libltephy_b200.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/ltephy_b200.h"

#define CHAN_THREADS 256
#define CHAN_MAX_SEGS 16 // 8 carriers x 2 antennas

struct ChanSeg {       // one (carrier, antenna) of a call: outputs m0 .. m0 + count - 1, in tiles of L R (an integer carrier: L = 1, M = D)
  const float2* g;     // [L][Kp] phase taps g_phi[k] at [phi][k + Kb]
  const float2* rot;   // [P] r[m mod P]
  float2*       out;   // [count] this antenna's row of the carrier's output
  uint64_t      n0;    // floor(m0 M / L): the capture sample of output m0
  uint64_t      count;
  uint32_t      phi0;  // m0 M mod L
  uint32_t      r0;    // m0 mod P
  uint32_t      L, M, Kp, Ka, P;
  uint32_t      R;     // outputs per phase class in a tile: a tile holds outputs m0 + i0 + c + L r, c < L, r < R
  uint32_t      Q;     // phases of the tile's span in shared memory: position s at row s / Q of phase s mod Q (M at L = 1, else 1)
  uint32_t      rows;  // rows per phase: ceil(longest span / Q)
  uint32_t      tile0; // first tile of this segment in the grid
  uint32_t      a;     // antenna
};

struct ChanArgs {
  const void*    x;     // [A][lda] complex samples first .. first + lda - 1, in the plan's format
  uint64_t       lda, first;
  uint32_t       nseg;  // segments in seg[] (a call of ltephy_chan_run)
  uint32_t       tps;   // tiles per segment of tab (the raster scan)
  const ChanSeg* tab;   // device-resident segments, every one of tps tiles: segment tile / tps; nullptr selects seg[]
  ChanSeg        seg[CHAN_MAX_SEGS];
};

// every tile of every segment in one launch: ntiles CTAs of CHAN_THREADS, smem bytes of dynamic shared memory; fmt is the plan's iq_format.
// g.tab selects the form that takes the segment of a tile from the device table instead of g.seg.
extern "C" int launch_chan(const ChanArgs& g, uint32_t ntiles, size_t smem, uint32_t fmt, cudaStream_t st);

// host (chan.cu), shared with the raster scan (scan.cu)
// geometry of carrier (offset_hz, N) at fs_in under flags; 0, or INVALID_INPUTS with the reason in the last error
int chan_geometry(uint32_t fs_in, int32_t offset_hz, uint32_t N, uint32_t flags, ltephy_chan_poly_t* q);
// its tables (any of hp, g, rot may be nullptr)
int chan_design(uint32_t fs_in, int32_t offset_hz, uint32_t N, uint32_t flags, ltephy_chan_poly_t* out, float* hp, float* g, float* rot);
// the tile shape of a carrier: R, Q and rows of ChanSeg, and the shared memory its tiles take
void chan_tiles(const ltephy_chan_poly_t& q, uint32_t* R, uint32_t* Q, uint32_t* rows, size_t* smem);
// the outputs of a call on capture samples first .. first + n - 1: the first lo, count cnt, and the capture sample the next call must include
void chan_range(const ltephy_chan_poly_t& q, uint64_t first, uint64_t n, uint64_t* lo, uint64_t* cnt, uint64_t* next);
