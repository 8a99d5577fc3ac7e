// k_track.cu -- tracker kernels (DESIGN.md §2 "tracking", §4 T1-T3): the stride-1 PSS metric over the measurement window of every half-frame of a
// push, the half-symbol correlations of the CFO sum at the chosen positions, and the cut of every subframe with its carrier-offset rotation.
// Every float sum runs in the order lteo_track (oracle_track/lte_track_oracle.c) restates, built with -fmad=false, so the results equal the
// oracle's bit for bit.
#include "dev_common.cuh"
#include "k_track.cuh"
#include <cstdint>

#define TM_THREADS 256
#define TM_R 4 // positions per thread, TM_THREADS apart: a block covers TM_THREADS * TM_R consecutive positions of one window

// grid (tiles, windows).  The replica and the tile's TM_THREADS * TM_R + N - 1 samples of one antenna sit in shared memory; lane l reads sample
// q + k with consecutive q across the warp, so a warp's reads are consecutive 8-byte words, and the replica tap is a broadcast.
// X, here and below: the sample type of g.x, converted to cf32 where it is loaded.
template <typename X>
__global__ void __launch_bounds__(TM_THREADS) track_metric_kernel(TrackArgs g, const TrackWin* __restrict__ win, uint32_t stride,
                                                                  float* __restrict__ m)
{
  extern __shared__ float2 tsm[];
  const uint32_t N = g.N, T = TM_THREADS * TM_R;
  const TrackWin w = win[blockIdx.y];
  const uint32_t i0 = blockIdx.x * T;
  if (i0 >= w.cnt) return;
  float2*        p  = tsm;
  float2*        xs = tsm + N;
  const uint32_t span = min(T, w.cnt - i0) + N - 1;
  for (uint32_t i = threadIdx.x; i < N; i += blockDim.x) p[i] = g.rep[i];
  float P[TM_R], E[TM_R];
#pragma unroll
  for (int r = 0; r < TM_R; r++) P[r] = E[r] = 0.0f;
  for (uint32_t a = 0; a < g.A; a++) {
    __syncthreads();
    const X* xa = static_cast<const X*>(g.x) + (uint64_t)a * g.lda + w.t0 + i0;
    for (uint32_t i = threadIdx.x; i < T + N - 1; i += blockDim.x) xs[i] = i < span ? chan_cf32(xa[i]) : make_float2(0.0f, 0.0f);
    __syncthreads();
    float cr[TM_R], ci[TM_R], e[TM_R];
#pragma unroll
    for (int r = 0; r < TM_R; r++) cr[r] = ci[r] = e[r] = 0.0f;
    const float2* xq = xs + threadIdx.x;
    for (uint32_t k = 0; k < N; k++) {
      const float2 q = p[k];
#pragma unroll
      for (int r = 0; r < TM_R; r++) {
        const float2 v = xq[r * TM_THREADS + k];
        cr[r]          = cr[r] + (v.x * q.x + v.y * q.y);
        ci[r]          = ci[r] + (v.y * q.x - v.x * q.y);
        e[r]           = e[r] + (v.x * v.x + v.y * v.y);
      }
    }
#pragma unroll
    for (int r = 0; r < TM_R; r++) {
      P[r] = P[r] + (cr[r] * cr[r] + ci[r] * ci[r]);
      E[r] = E[r] + e[r];
    }
  }
#pragma unroll
  for (int r = 0; r < TM_R; r++) {
    const uint32_t i = i0 + threadIdx.x + r * TM_THREADS;
    if (i >= w.cnt) continue;
    const float den = g.ep * E[r];
    m[(uint64_t)blockIdx.y * stride + i] = den == 0.0f ? 0.0f : P[r] / den;
  }
}

// one thread per (half-frame, antenna, half): the N / 2 products of one half in ascending order
template <typename X>
__global__ void track_sums_kernel(TrackArgs g, const uint64_t* __restrict__ pos, uint32_t nh, float2* __restrict__ c)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nh * g.A * 2) return;
  const uint32_t h = t / (g.A * 2), a = (t / 2) % g.A, half = t % 2, k0 = half * (g.N / 2);
  const X*       xa = static_cast<const X*>(g.x) + (uint64_t)a * g.lda + pos[h];
  float          cr = 0.0f, ci = 0.0f;
  for (uint32_t k = k0; k < k0 + g.N / 2; k++) {
    const float2 v = chan_cf32(xa[k]), q = g.rep[k];
    cr             = cr + (v.x * q.x + v.y * q.y);
    ci             = ci + (v.y * q.x - v.x * q.y);
  }
  c[t] = make_float2(cr, ci);
}

// grid (15 N / 256, nsf * A): one sample per thread, both factor tables of the subframe read through the read-only cache
template <typename X>
__global__ void __launch_bounds__(256) track_cut_kernel(TrackArgs g, const uint64_t* __restrict__ start, const float2* __restrict__ tabA,
                                                        const float2* __restrict__ tabB, float2* __restrict__ out)
{
  const uint32_t SF = 15 * g.N, n = blockIdx.x * blockDim.x + threadIdx.x, k = blockIdx.y / g.A, a = blockIdx.y % g.A;
  if (n >= SF) return;
  const float2 A = __ldg(&tabA[(uint64_t)k * (SF / 128) + (n >> 7)]), B = __ldg(&tabB[k * 128 + (n & 127)]);
  const float  rr = A.x * B.x - A.y * B.y, ri = A.x * B.y + A.y * B.x;
  const float2 v  = chan_cf32(static_cast<const X*>(g.x)[(uint64_t)a * g.lda + start[k] + n]);
  out[((uint64_t)k * g.A + a) * SF + n] = make_float2(v.x * rr - v.y * ri, v.x * ri + v.y * rr);
}

extern "C" int launch_track_metric(const TrackArgs& g, uint32_t fmt, const TrackWin* win, uint32_t nwin, uint32_t maxcnt, uint32_t stride, float* m,
                                   cudaStream_t st)
{
  if (!nwin) return 0;
  const uint32_t T    = TM_THREADS * TM_R;
  const size_t   smem = (size_t)(2 * g.N + T - 1) * sizeof(float2);
  return with_iq_type(fmt, [&](auto z) {
    using X = decltype(z);
    if (cudaFuncSetAttribute(track_metric_kernel<X>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
    track_metric_kernel<X><<<dim3((maxcnt + T - 1) / T, nwin), TM_THREADS, smem, st>>>(g, win, stride, m);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
  });
}

extern "C" int launch_track_sums(const TrackArgs& g, uint32_t fmt, const uint64_t* pos, uint32_t nh, float2* c, cudaStream_t st)
{
  if (!nh) return 0;
  const uint32_t nt = nh * g.A * 2;
  with_iq_type(fmt, [&](auto z) {
    track_sums_kernel<decltype(z)><<<(nt + 127) / 128, 128, 0, st>>>(g, pos, nh, c);
    return 0;
  });
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int launch_track_cut(const TrackArgs& g, uint32_t fmt, const uint64_t* start, const float2* tabA, const float2* tabB, uint32_t nsf,
                                float2* out, cudaStream_t st)
{
  if (!nsf) return 0;
  with_iq_type(fmt, [&](auto z) {
    track_cut_kernel<decltype(z)><<<dim3((15 * g.N + 255) / 256, nsf * g.A), 256, 0, st>>>(g, start, tabA, tabB, out);
    return 0;
  });
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
