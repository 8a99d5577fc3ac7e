// k_sync.cuh -- arguments shared by the cell search kernels (k_sync.cu) and their host code (sync.cu).  Private to libltephy_b200.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/ltephy_b200.h"

#define SYNC_BINS 9600 // coarse bins per half-frame: 75 N / D

struct SyncArgs {
  const void*   x;   // [A][lda] samples in the handle's iq_format (float2, short2 or char2)
  uint64_t      lda, L, J; // J: coarse offsets whose window fits, (L - N) / D + 1
  uint32_t      N, D, A, nh; // nh: half-frames with a window start below L - N + 1, (L - N) / HF + 1
  const float2* rep; // [3][N] PSS replicas
  const float2* W;   // [N] exp(-j 2 pi i / N)
  float         ep[3];
};

struct SyncPeak {
  uint32_t bin;   // coarse peak bin
  float    peak;  // folded coarse peak
  float    side;  // largest folded value more than 2 bins away
  uint32_t tau;   // refined timing in [0, HF)
  float    rpeak; // folded stride-1 metric at tau
  float    s_re, s_im; // CFO sum
};

struct SyncSss {
  uint64_t      tau[3];
  uint32_t      h0[3], nH[3], nhmax; // half-frames h0 .. h0 + nH - 1 have both windows inside the capture
  float         rot[3][2];            // exp(-j phi) of the CFO estimate over N + 9 D samples
  const float2* dpss;                 // [3][62] d_u
  const float*  seq;                  // [3][168][2][62] SSS of subframe 0 / 5
};

// host (sync.cu): d_u and the replica of N_ID_2 = u, returns E_p
float sync_pss_replica(uint32_t N, uint32_t u, float2* d, float2* rep);
// host (sync.cu): the cell search of the L samples x[a * lda + i] (device memory, i < L <= max_samples) on h's stream; blocks until out[3] is
// written.  ltephy_cell_search_device is lda = L; the tracker's find state (track.cu) searches a window of its own buffer in place.
// x holds samples in the handle's iq_format.
int sync_run(ltephy_sync_t* h, const void* x, uint64_t lda, uint64_t L, ltephy_cell_t* out);

// fmt: the iq_format of g.x
extern "C" int launch_sync_pss(const SyncArgs& g, uint32_t fmt, float* m, float* fold, SyncPeak* pk, float* rm, float4* c12, float* refined, cudaStream_t st,
                               uint64_t* launches);
extern "C" int launch_sync_sss(const SyncArgs& g, uint32_t fmt, const SyncSss& s, float2* Y, float* sss, cudaStream_t st, uint64_t* launches);
