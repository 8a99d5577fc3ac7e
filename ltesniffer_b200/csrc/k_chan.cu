// k_chan.cu -- channeliser kernel (DESIGN.md §2 "channeliser", §4 C1): every (carrier, antenna, tile of outputs) of a call in one launch.
// y[m] = r[m mod P] * sum_{k=-H..H} g[k] x[m D - k], the sum a serial k-ascending chain of separate fp32 products and adds (-fmad=false), as
// lteo_chan_run (oracle/lte_chan_oracle.c) computes it, so the results equal the oracle's bit for bit.
#include "k_chan.cuh"
#include <cstdint>

// One CTA per tile of M outputs.  The taps and the tile's input span [m0 D - H, (m0 + M - 1) D + H] sit in shared memory, the span split into its
// D phases: sample s of the span (s = t D + u for output t and tap u = H - k) lies at row t + u / D of phase u mod D.  For a fixed tap the threads
// of a warp (consecutive t) then read consecutive 8-byte words, and the tap itself is a broadcast.
__global__ void __launch_bounds__(CHAN_THREADS) chan_kernel(const __grid_constant__ ChanArgs g)
{
  extern __shared__ float2 csm[];
  const uint32_t tile = blockIdx.x;
  uint32_t       si   = 0;
  while (si + 1 < g.nseg && tile >= g.seg[si + 1].tile0) si++;
  const ChanSeg& q  = g.seg[si];
  const uint32_t D = q.D, T = q.T, rows = q.rows, i0 = (tile - q.tile0) * q.M;
  const uint32_t Mt = min(q.M, q.count - i0), span = (Mt - 1) * D + T;
  const uint64_t m0   = q.m0 + i0;
  const int64_t  base = (int64_t)(m0 * D) - (int64_t)(T / 2); // capture sample of span position 0
  float2*        gs   = csm;
  float2*        xs   = csm + T;
  for (uint32_t j = threadIdx.x; j < T; j += blockDim.x) gs[j] = q.g[j];
  const float2* xa = g.x + (uint64_t)q.a * g.lda;
  for (uint32_t s = threadIdx.x; s < span; s += blockDim.x) {
    const int64_t i = base + (int64_t)s; // samples before 0 are zero; every other sample of the span lies inside the call
    xs[(s % D) * rows + s / D] = i >= 0 ? xa[(uint64_t)i - g.first] : make_float2(0.0f, 0.0f);
  }
  __syncthreads();
  const uint32_t p0 = (T - 1) % D, r0 = (T - 1) / D, mp = (uint32_t)(m0 % q.P);
  for (uint32_t t = threadIdx.x; t < Mt; t += blockDim.x) {
    float    ar = 0.0f, ai = 0.0f;
    uint32_t p = p0, r = r0 + t; // u = T - 1 - j: phase u mod D, row t + u / D
    for (uint32_t j = 0; j < T; j++) {
      const float2 v = xs[p * rows + r], c = gs[j];
      ar             = ar + (c.x * v.x - c.y * v.y);
      ai             = ai + (c.x * v.y + c.y * v.x);
      if (p == 0) p = D - 1, r--;
      else p--;
    }
    const float2 rr = __ldg(&q.rot[(mp + t) % q.P]);
    q.out[i0 + t]   = make_float2(rr.x * ar - rr.y * ai, rr.x * ai + rr.y * ar);
  }
}

extern "C" int launch_chan(const ChanArgs& g, uint32_t ntiles, size_t smem, cudaStream_t st)
{
  if (!ntiles) return 0;
  if (cudaFuncSetAttribute(chan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
  chan_kernel<<<ntiles, CHAN_THREADS, smem, st>>>(g);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
