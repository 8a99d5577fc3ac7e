// k_sync.cuh -- arguments shared by the cell search kernels (k_sync.cu) and their host code (sync.cu).  Private to libltephy_b200.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/ltephy_b200.h"

#define SYNC_BINS 9600 // coarse bins per half-frame: 75 N / D

// A search covers one capture, or a batch of captures of the same length (the raster scan's points): capture p is blockIdx.y of every grid, its
// samples at x + p ps, and each intermediate of one capture is followed by that of the next.
struct SyncArgs {
  const void*   x;   // [points][A][lda] samples in the handle's iq_format (float2, short2 or char2), capture p at x + p ps
  uint64_t      lda, ps, L, J; // J: coarse offsets whose window fits, (L - N) / D + 1
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

struct SyncPt { // the SSS stage's inputs of one capture, decided on the host from its SyncPeak
  uint64_t      tau[3];
  uint32_t      h0[3], nH[3];        // half-frames h0 .. h0 + nH - 1 have both windows inside the capture
  float         rot[3][2];           // exp(-j phi) of the CFO estimate over N + 9 D samples
};

struct SyncSss {
  const SyncPt* pt;                  // [points], device memory
  uint32_t      nhmax;               // the largest nH of every capture and N_ID_2
  const float2* dpss;                // [3][62] d_u
  const float*  seq;                 // [3][168][2][62] SSS of subframe 0 / 5
};

// host (sync.cu): d_u and the replica of N_ID_2 = u, returns E_p
float sync_pss_replica(uint32_t N, uint32_t u, float2* d, float2* rep);
// host (sync.cu): the cell search of the L samples x[a * lda + i] (device memory, i < L <= max_samples) on h's stream; blocks until out[3] is
// written.  ltephy_cell_search_device is lda = L; the tracker's find state (track.cu) searches a window of its own buffer in place.
// x holds samples in the handle's iq_format.
int sync_run(ltephy_sync_t* h, const void* x, uint64_t lda, uint64_t L, ltephy_cell_t* out);
// host (sync.cu): the cell search of np captures at once, capture p at x + p ps (device memory, cf32 or the handle's iq_format), each exactly
// what sync_run gives it; out[3 np].  Two host round trips for the batch.  np <= the handle's points (sync_create_batch).
int sync_run_batch(ltephy_sync_t* h, const void* x, uint64_t lda, uint64_t ps, uint64_t L, uint32_t np, ltephy_cell_t* out);
// host (sync.cu): a search handle whose buffers hold batches of up to points captures, on its own stream
int sync_create_batch(const ltephy_sync_cfg_t* cfg, uint32_t points, ltephy_sync_t** out);
cudaStream_t sync_stream(ltephy_sync_t* h);

// np captures (grid y); fmt: the iq_format of g.x
extern "C" int launch_sync_pss(const SyncArgs& g, uint32_t np, uint32_t fmt, float* m, float* fold, SyncPeak* pk, float* rm, float4* c12, float* refined, cudaStream_t st,
                               uint64_t* launches);
extern "C" int launch_sync_sss(const SyncArgs& g, uint32_t np, uint32_t fmt, const SyncSss& s, float2* Y, float* sss, cudaStream_t st, uint64_t* launches);
