// k_chan.cu -- the channeliser kernel (DESIGN.md §2 "channeliser", §4 C1): every (carrier, antenna, tile of outputs) of a call in one launch.
// y[m] = r[m mod P] * sum_{k=-Kb..Ka} g_phi[k] x[n - k], n = floor(m M / L), phi = m M mod L; an integer carrier is L = 1, M = D, Ka = Kb = H.
// Each sum is a serial k-ascending chain of separate fp32 products and adds (-fmad=false), as lteo_chan_run / lteo_chan_run_poly (oracle/)
// compute it, so the results equal the oracles' bit for bit.  The input is converted to cf32 where it is staged into shared memory; sc16 and sc8
// scale by a power of two, which is exact.
#include "dev_common.cuh"
#include "k_chan.cuh"
#include <cstdint>

// The serial k-ascending chain of one output: taps t[0 .. Kp) against span positions s, s - 1, .., s - Kp + 1, position s at row s / Q of phase
// s mod Q of xs.  LDG: the taps are read through L1, else from shared memory.
template <bool LDG>
__device__ __forceinline__ float2 chan_chain(const float2* t, const float2* xs, uint32_t Kp, uint32_t Q, uint32_t rows, uint32_t p, uint32_t row)
{
  float    ar = 0.0f, ai = 0.0f;
  for (uint32_t j = 0; j < Kp; j++) {
    const float2 v = xs[p * rows + row], c = LDG ? __ldg(t++) : *t++;
    ar             = ar + (c.x * v.x - c.y * v.y);
    ai             = ai + (c.x * v.y + c.y * v.x);
    if (p == 0) p = Q - 1, row--;
    else p--;
  }
  return make_float2(ar, ai);
}

// output i of the segment: y = r[m mod P] a, mp = m mod P before the reduction
__device__ __forceinline__ void chan_store(const ChanSeg& q, uint64_t i, uint32_t mp, float2 a)
{
  const float2 rr = __ldg(&q.rot[mp % q.P]);
  q.out[i]        = make_float2(rr.x * a.x - rr.y * a.y, rr.x * a.y + rr.y * a.x);
}

// One CTA per tile of L R outputs m0 + i0 + c + L r (phase class c < L, row r < R).  Every output of class c has the same phase phi, and
// consecutive rows of a class lie M capture samples apart, so thread w = c R + r works on class c.  The tile's span [n(first) - Ka, n(last) + Kb]
// is staged once in shared memory as cf32, split into Q phases: position s at row s / Q of phase s mod Q.  An integer carrier has Q = D, so for
// a fixed tap the threads of a warp (consecutive r) read consecutive 8-byte words; a rational one has Q = 1 and reads words M apart.  At L = 1
// the tile has one phase class: its Kp taps sit in shared memory ahead of the span and the whole CTA reads one tap address per term (a broadcast,
// two taps per 16-byte load).  At L > 1 a warp's tap reads are one address when R >= 32, through L1 (the [L][Kp] table, up to 256 KB, stays in
// global memory and L2).  TAB: the segment of a tile is entry tile / tps of the device table g.tab (the raster scan's thousands of (point, antenna)
// segments, every one of tps tiles), else the one of g.seg whose tiles hold it.
template <typename X, bool TAB>
__global__ void __launch_bounds__(CHAN_THREADS) chan_kernel(const __grid_constant__ ChanArgs g)
{
  extern __shared__ float2 csm[];
  const uint32_t tile = blockIdx.x;
  uint32_t       si   = 0;
  if (TAB) si = tile / g.tps;
  else
    while (si + 1 < g.nseg && tile >= g.seg[si + 1].tile0) si++;
  const ChanSeg& q = TAB ? g.tab[si] : g.seg[si];
  const uint32_t L = q.L, M = q.M, Kp = q.Kp, R = q.R, Q = q.Q, rows = q.rows, t = tile - q.tile0;
  const uint64_t i0   = (uint64_t)t * L * R;
  const uint32_t Mt   = (uint32_t)min((uint64_t)L * R, q.count - i0);
  const uint32_t span = (q.phi0 + (Mt - 1) * M) / L + Kp;
  const int64_t  base = (int64_t)(q.n0 + (uint64_t)t * R * M) - (int64_t)q.Ka; // capture sample of span position 0
  const X*       xa   = static_cast<const X*>(g.x) + (uint64_t)q.a * g.lda;
  float2* const  xs   = csm + (L == 1 ? Kp : 0);
  if (L == 1)
    for (uint32_t j = threadIdx.x; j < Kp; j += blockDim.x) csm[j] = q.g[j];
  // samples before 0 are zero; every other sample of the span lies inside the call
  if (Q == 1)
    for (uint32_t s = threadIdx.x; s < span; s += blockDim.x) {
      const int64_t i = base + (int64_t)s;
      xs[s]           = i >= 0 ? chan_cf32(xa[(uint64_t)i - g.first]) : make_float2(0.0f, 0.0f);
    }
  else
    for (uint32_t s = threadIdx.x; s < span; s += blockDim.x) {
      const int64_t i            = base + (int64_t)s;
      xs[(s % Q) * rows + s / Q] = i >= 0 ? chan_cf32(xa[(uint64_t)i - g.first]) : make_float2(0.0f, 0.0f);
    }
  __syncthreads();
  const uint32_t mp = (uint32_t)((q.r0 + i0) % q.P);
  if (L == 1) { // Q = M: output t reads span positions t Q + Kp - 1 down, from row t + (Kp - 1) / Q of phase (Kp - 1) mod Q
    const uint32_t p1 = (Kp - 1) % Q, r1 = (Kp - 1) / Q;
    for (uint32_t t = threadIdx.x; t < Mt; t += blockDim.x) chan_store(q, i0 + t, mp + t, chan_chain<false>(csm, xs, Kp, Q, rows, p1, r1 + t));
  } else // Q = 1
    for (uint32_t w = threadIdx.x; w < L * R; w += blockDim.x) {
      const uint32_t c = w / R, r = w - c * R, o = c + L * r, u = q.phi0 + c * M;
      if (o < Mt) chan_store(q, i0 + o, mp + o, chan_chain<true>(q.g + (size_t)(u % L) * Kp, xs, Kp, 1, rows, 0, u / L + r * M + Kp - 1));
    }
}

extern "C" int launch_chan(const ChanArgs& g, uint32_t ntiles, size_t smem, uint32_t fmt, cudaStream_t st)
{
  if (!ntiles) return 0;
  const auto k = g.tab ? (fmt == 0 ? chan_kernel<float2, true> : fmt == 1 ? chan_kernel<short2, true> : fmt == 2 ? chan_kernel<char2, true> : nullptr)
                      : (fmt == 0 ? chan_kernel<float2, false> : fmt == 1 ? chan_kernel<short2, false> : fmt == 2 ? chan_kernel<char2, false> : nullptr);
  if (!k || cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
  k<<<ntiles, CHAN_THREADS, smem, st>>>(g);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
