// k_chan.cu -- channeliser kernels (DESIGN.md §2 "channeliser", §4 C1): every (carrier, antenna, tile of outputs) of a call in one launch per
// kind of carrier.  Integer carriers: y[m] = r[m mod P] * sum_{k=-H..H} g[k] x[m D - k]; rational carriers: y[m] = r[m mod P] *
// sum_{k=-Kb..Ka} g_phi[k] x[n - k], n = floor(m M / L), phi = m M mod L.  Each sum is a serial k-ascending chain of separate fp32 products and
// adds (-fmad=false), as lteo_chan_run / lteo_chan_run_poly (oracle/) compute it, so the results equal the oracles' bit for bit.  The input is
// converted to cf32 where it is staged into shared memory; sc16 and sc8 scale by a power of two, which is exact.
#include "k_chan.cuh"
#include <cstdint>

__device__ __forceinline__ float2 chan_cf32(float2 v) { return v; }
__device__ __forceinline__ float2 chan_cf32(short2 v) { return make_float2((float)v.x * 0x1p-15f, (float)v.y * 0x1p-15f); }
__device__ __forceinline__ float2 chan_cf32(char2 v) { return make_float2((float)v.x * 0x1p-7f, (float)v.y * 0x1p-7f); }

// One CTA per tile of M outputs.  The taps and the tile's input span [m0 D - H, (m0 + M - 1) D + H] sit in shared memory, the span split into its
// D phases: sample s of the span (s = t D + u for output t and tap u = H - k) lies at row t + u / D of phase u mod D.  For a fixed tap the threads
// of a warp (consecutive t) then read consecutive 8-byte words, and the tap itself is a broadcast.
template <typename X>
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
  const X* xa = static_cast<const X*>(g.x) + (uint64_t)q.a * g.lda;
  for (uint32_t s = threadIdx.x; s < span; s += blockDim.x) {
    const int64_t i = base + (int64_t)s; // samples before 0 are zero; every other sample of the span lies inside the call
    xs[(s % D) * rows + s / D] = i >= 0 ? chan_cf32(xa[(uint64_t)i - g.first]) : make_float2(0.0f, 0.0f);
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

// One CTA per tile of L R outputs m0 + i0 + c + L r (phase class c < L, row r < R).  Every output of class c has the same phase phi, and
// consecutive rows of a class lie M capture samples apart, so thread w = c R + r works on class c: a warp's tap reads are one address (a
// broadcast through L1; the [L][Kp] table, up to 256 KB, stays in global memory and L2) and its input reads stride M through the tile's span
// [n(first) - Ka, n(last) + Kb], staged once in shared memory as cf32.
template <typename X>
__global__ void __launch_bounds__(CHAN_THREADS) chan_poly_kernel(const __grid_constant__ ChanPolyArgs g)
{
  extern __shared__ float2 csm[];
  const uint32_t tile = blockIdx.x;
  uint32_t       si   = 0;
  while (si + 1 < g.nseg && tile >= g.seg[si + 1].tile0) si++;
  const ChanPolySeg& q = g.seg[si];
  const uint32_t     L = q.L, M = q.M, Kp = q.Kp, R = q.R, t = tile - q.tile0;
  const uint64_t     i0 = (uint64_t)t * L * R;
  const uint32_t     Mt = (uint32_t)min((uint64_t)L * R, q.count - i0);
  const uint32_t     span = (q.phi0 + (Mt - 1) * M) / L + Kp;
  const int64_t      base = (int64_t)(q.n0 + (uint64_t)t * R * M) - (int64_t)q.Ka; // capture sample of span position 0
  const X*           xa   = static_cast<const X*>(g.x) + (uint64_t)q.a * g.lda;
  for (uint32_t s = threadIdx.x; s < span; s += blockDim.x) {
    const int64_t i = base + (int64_t)s; // samples before 0 are zero; every other sample of the span lies inside the call
    csm[s] = i >= 0 ? chan_cf32(xa[(uint64_t)i - g.first]) : make_float2(0.0f, 0.0f);
  }
  __syncthreads();
  const uint32_t mp = (uint32_t)((q.r0 + i0) % q.P);
  for (uint32_t w = threadIdx.x; w < L * R; w += blockDim.x) {
    const uint32_t c = w / R, r = w - c * R, o = c + L * r;
    if (o >= Mt) continue;
    const uint32_t u  = q.phi0 + c * M;
    const float2*  gp = q.g + (size_t)(u % L) * Kp;
    const float2*  xp = csm + (u / L + r * M + Kp - 1); // j = k + Kb: sample n - k at span position n - n(first) + Ka - k
    float          ar = 0.0f, ai = 0.0f;
    for (uint32_t j = 0; j < Kp; j++) {
      const float2 v = xp[-(int32_t)j], cc = __ldg(&gp[j]);
      ar             = ar + (cc.x * v.x - cc.y * v.y);
      ai             = ai + (cc.x * v.y + cc.y * v.x);
    }
    const float2 rr = __ldg(&q.rot[(mp + o) % q.P]);
    q.out[i0 + o]   = make_float2(rr.x * ar - rr.y * ai, rr.x * ai + rr.y * ar);
  }
}

template <typename K, typename A>
static int chan_launch(K* k, const A& g, uint32_t ntiles, size_t smem, cudaStream_t st)
{
  if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
  k<<<ntiles, CHAN_THREADS, smem, st>>>(g);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int launch_chan(const ChanArgs& g, uint32_t ntiles, size_t smem, uint32_t fmt, cudaStream_t st)
{
  if (!ntiles) return 0;
  switch (fmt) {
    case 0: return chan_launch(chan_kernel<float2>, g, ntiles, smem, st);
    case 1: return chan_launch(chan_kernel<short2>, g, ntiles, smem, st);
    case 2: return chan_launch(chan_kernel<char2>, g, ntiles, smem, st);
    default: return -1;
  }
}

extern "C" int launch_chan_poly(const ChanPolyArgs& g, uint32_t ntiles, size_t smem, uint32_t fmt, cudaStream_t st)
{
  if (!ntiles) return 0;
  switch (fmt) {
    case 0: return chan_launch(chan_poly_kernel<float2>, g, ntiles, smem, st);
    case 1: return chan_launch(chan_poly_kernel<short2>, g, ntiles, smem, st);
    case 2: return chan_launch(chan_poly_kernel<char2>, g, ntiles, smem, st);
    default: return -1;
  }
}
