// k_track.cuh -- arguments shared by the tracker kernels (k_track.cu) and their host code (track.cu).  Private to libltephy_b200.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

struct TrackArgs {
  const void*   x;   // [A][lda] samples of the push in the tracker's iq_format (float2, short2 or char2)
  uint64_t      lda;
  uint32_t      N, A;
  const float2* rep; // [N] replica of the tracked PSS
  float         ep;  // its energy
};

struct TrackWin {   // metric positions t0 .. t0 + cnt - 1 (relative to x), written to m[w * stride ...]
  uint64_t t0;
  uint32_t cnt, pad;
};

// fmt: the iq_format of g.x
// T1: m[w][i] = metric at win[w].t0 + i, in lteo_track's order
extern "C" int launch_track_metric(const TrackArgs& g, uint32_t fmt, const TrackWin* win, uint32_t nwin, uint32_t maxcnt, uint32_t stride, float* m,
                                   cudaStream_t st);
// T2: c[(h * A + a) * 2 + half] = the correlation of antenna a at pos[h] over k < N / 2 (half 0) or k >= N / 2 (half 1)
extern "C" int launch_track_sums(const TrackArgs& g, uint32_t fmt, const uint64_t* pos, uint32_t nh, float2* c, cudaStream_t st);
// T3: out[k][a][n] = x[a][start[k] + n] (tabA[k][n >> 7] tabB[k][n & 127]), n < 15 N, always cf32
extern "C" int launch_track_cut(const TrackArgs& g, uint32_t fmt, const uint64_t* start, const float2* tabA, const float2* tabB, uint32_t nsf, float2* out,
                                cudaStream_t st);
