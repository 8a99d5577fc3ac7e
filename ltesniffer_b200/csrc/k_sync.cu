// k_sync.cu -- cell search kernels (DESIGN.md §2 "cell search", §4): coarse PSS correlation at stride D = N / 128, half-frame fold and peak,
// stride-1 refinement with the CFO sums, 62-bin DFTs of the PSS / SSS symbols and the SSS hypothesis table.  Every float sum runs in the
// order lteo_cell_search (oracle/lte_sync_oracle.c) restates, built with -fmad=false, so the results equal the oracle's bit for bit.
#include "dev_common.cuh"
#include "k_sync.cuh"
#include <cstdint>

#define COARSE_THREADS 256
#define COARSE_R 4 // offsets per thread, 32 apart: lane l of warp w owns local offsets 32 R w + 32 r + l

// Samples of the block's window sit in shared memory at (i / D) * Ds + i % D with Ds = D + 1 for even D, D for odd D.  The lanes of a warp read
// samples D apart, so an even D would put every lane of a half-warp on one bank pair; with the odd stride Ds they all land on different ones.
static __device__ __forceinline__ uint32_t sync_pad_stride(uint32_t D) { return D | 1u; }

// m[u][j] = sum_a |c_ua(jD)|^2 / (E_p[u] sum_a E_a(jD)); each thread keeps 4 offsets x 3 replicas of correlations and the 4 window energies in registers.
// X, here and below: the sample type of g.x, converted to cf32 where it is loaded.
template <typename X>
__global__ void __launch_bounds__(COARSE_THREADS) sync_coarse_kernel(SyncArgs g, float* __restrict__ m)
{
  extern __shared__ float4 sm4[];
  const uint32_t N = g.N, D = g.D, Ds = sync_pad_stride(D), T = COARSE_THREADS * COARSE_R;
  float4*        rA = sm4;                                  // (p0, p1) per tap
  float2*        rB = reinterpret_cast<float2*>(rA + N);    // p2 per tap
  float2*        xs = rB + N;                               // (T + N / D) * Ds samples
  const uint64_t j0 = (uint64_t)blockIdx.x * T, s0 = j0 * D;
  m += (uint64_t)blockIdx.y * 3 * g.J;
  const uint32_t span = T * D + N;
  for (uint32_t i = threadIdx.x; i < N; i += blockDim.x) {
    const float2 a = g.rep[i], b = g.rep[N + i];
    rA[i] = make_float4(a.x, a.y, b.x, b.y);
    rB[i] = g.rep[2 * N + i];
  }
  const uint32_t q0 = (threadIdx.x >> 5) * 32 * COARSE_R + (threadIdx.x & 31);
  float          P[3][COARSE_R], E[COARSE_R];
#pragma unroll
  for (int r = 0; r < COARSE_R; r++) {
    E[r] = 0.0f;
#pragma unroll
    for (int u = 0; u < 3; u++) P[u][r] = 0.0f;
  }
  for (uint32_t a = 0; a < g.A; a++) {
    __syncthreads();
    const X* xa = static_cast<const X*>(g.x) + blockIdx.y * g.ps + (uint64_t)a * g.lda;
    for (uint32_t i = threadIdx.x; i < span; i += blockDim.x) {
      const uint64_t s    = s0 + i;
      xs[(i / D) * Ds + i % D] = s < g.L ? chan_cf32(xa[s]) : make_float2(0.0f, 0.0f);
    }
    __syncthreads();
    float cr[3][COARSE_R], ci[3][COARSE_R], e[COARSE_R];
#pragma unroll
    for (int r = 0; r < COARSE_R; r++) {
      e[r] = 0.0f;
#pragma unroll
      for (int u = 0; u < 3; u++) cr[u][r] = ci[u][r] = 0.0f;
    }
    for (uint32_t qb = 0; qb < N / D; qb++) {
      const float2* xq = xs + (q0 + qb) * Ds;
      for (uint32_t i = 0; i < D; i++) {
        const uint32_t k  = qb * D + i;
        const float4   pa = rA[k];
        const float2   pb = rB[k];
#pragma unroll
        for (int r = 0; r < COARSE_R; r++) {
          const float2 v = xq[r * 32 * Ds + i];
          cr[0][r]       = cr[0][r] + (v.x * pa.x + v.y * pa.y);
          ci[0][r]       = ci[0][r] + (v.y * pa.x - v.x * pa.y);
          cr[1][r]       = cr[1][r] + (v.x * pa.z + v.y * pa.w);
          ci[1][r]       = ci[1][r] + (v.y * pa.z - v.x * pa.w);
          cr[2][r]       = cr[2][r] + (v.x * pb.x + v.y * pb.y);
          ci[2][r]       = ci[2][r] + (v.y * pb.x - v.x * pb.y);
          e[r]           = e[r] + (v.x * v.x + v.y * v.y);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < COARSE_R; r++) {
#pragma unroll
      for (int u = 0; u < 3; u++) P[u][r] = P[u][r] + (cr[u][r] * cr[u][r] + ci[u][r] * ci[u][r]);
      E[r] = E[r] + e[r];
    }
  }
#pragma unroll
  for (int r = 0; r < COARSE_R; r++) {
    const uint64_t j = j0 + q0 + 32 * r;
    if (j >= g.J) continue;
#pragma unroll
    for (int u = 0; u < 3; u++) {
      const float den  = g.ep[u] * E[r];
      m[u * g.J + j]   = den == 0.0f ? 0.0f : P[u][r] / den;
    }
  }
}

// fold[u][b] = (sum over h of m[u][b + 9600 h]) / count, h ascending
__global__ void sync_fold_kernel(SyncArgs g, const float* __restrict__ m, float* __restrict__ fold)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * SYNC_BINS) return;
  const uint32_t u = t / SYNC_BINS, b = t % SYNC_BINS;
  m += (uint64_t)blockIdx.y * 3 * g.J, fold += blockIdx.y * 3 * SYNC_BINS;
  float          sum = 0.0f;
  uint32_t       cnt = 0;
  for (uint64_t j = b; j < g.J; j += SYNC_BINS, cnt++) sum = sum + m[u * g.J + j];
  fold[t] = sum / (float)cnt;
}

// one block of 1024 per N_ID_2: argmax of the fold (ties to the lowest bin), then the largest value more than 2 bins away (circularly)
__global__ void __launch_bounds__(1024) sync_peak_kernel(const float* __restrict__ fold, SyncPeak* __restrict__ pk)
{
  __shared__ float    sv[1024];
  __shared__ uint32_t si[1024];
  const uint32_t      up = blockIdx.y * 3 + blockIdx.x; // (capture, N_ID_2)
  const float*        f  = fold + up * SYNC_BINS;
  float               bv = -1.0f;
  uint32_t            bi = 0xFFFFFFFFu;
  for (uint32_t b = threadIdx.x; b < SYNC_BINS; b += blockDim.x)
    if (f[b] > bv) bv = f[b], bi = b;
  sv[threadIdx.x] = bv, si[threadIdx.x] = bi;
  __syncthreads();
  for (uint32_t off = 512; off; off >>= 1) {
    if (threadIdx.x < off) {
      const float v2 = sv[threadIdx.x + off];
      const uint32_t i2 = si[threadIdx.x + off];
      if (v2 > sv[threadIdx.x] || (v2 == sv[threadIdx.x] && i2 < si[threadIdx.x])) sv[threadIdx.x] = v2, si[threadIdx.x] = i2;
    }
    __syncthreads();
  }
  const uint32_t bp = si[0];
  const float    peak = sv[0];
  __syncthreads();
  float side = 0.0f;
  for (uint32_t b = threadIdx.x; b < SYNC_BINS; b += blockDim.x) {
    const uint32_t d = b > bp ? b - bp : bp - b, dc = d < SYNC_BINS - d ? d : SYNC_BINS - d;
    if (dc > 2 && f[b] > side) side = f[b];
  }
  sv[threadIdx.x] = side;
  __syncthreads();
  for (uint32_t off = 512; off; off >>= 1) {
    if (threadIdx.x < off) sv[threadIdx.x] = fmaxf(sv[threadIdx.x], sv[threadIdx.x + off]);
    __syncthreads();
  }
  if (threadIdx.x == 0) pk[up] = SyncPeak{bp, peak, sv[0], 0, 0.0f, 0.0f, 0.0f};
}

// the metric of one window at stride 1, in lteo_cell_search's sync_metric order
template <typename X>
static __device__ float sync_window_metric(const SyncArgs& g, const X* x, uint64_t t, const float2* __restrict__ p, float ep)
{
  float P = 0.0f, E = 0.0f;
  for (uint32_t a = 0; a < g.A; a++) {
    const X* xa = x + (uint64_t)a * g.lda + t;
    float    cr = 0.0f, ci = 0.0f, e = 0.0f;
    for (uint32_t k = 0; k < g.N; k++) {
      const float2 v = chan_cf32(xa[k]), w = p[k];
      cr             = cr + (v.x * w.x + v.y * w.y);
      ci             = ci + (v.y * w.x - v.x * w.y);
      e              = e + (v.x * v.x + v.y * v.y);
    }
    P = P + (cr * cr + ci * ci);
    E = E + e;
  }
  const float den = ep * E;
  return den == 0.0f ? 0.0f : P / den;
}

// rm[u][h][i]: metric at ((bp D + HF + i - (D - 1)) mod HF) + h HF, for the 2D - 1 offsets i around the coarse peak and every half-frame h
template <typename X>
__global__ void sync_refine_kernel(SyncArgs g, const SyncPeak* __restrict__ pk, float* __restrict__ rm)
{
  const uint32_t NR = 2 * g.D - 1, t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * g.nh * NR) return;
  const uint32_t u = t / (g.nh * NR), h = (t / NR) % g.nh, i = t % NR;
  pk += blockIdx.y * 3, rm += (uint64_t)blockIdx.y * 3 * g.nh * NR;
  const uint64_t HF = 75ull * g.N, tt = ((uint64_t)pk[u].bin * g.D + HF + i - (g.D - 1)) % HF + h * HF;
  const float    ep = u == 0 ? g.ep[0] : u == 1 ? g.ep[1] : g.ep[2]; // no run-time index into the parameters (it would copy them to local memory)
  if (tt + g.N <= g.L) rm[t] = sync_window_metric<X>(g, static_cast<const X*>(g.x) + blockIdx.y * g.ps, tt, g.rep + u * g.N, ep);
}

// one block per N_ID_2: fold the refined metrics, pick the best offset (ties to the lowest), then S = sum_h sum_a c2 conj(c1) at that timing
template <typename X>
__global__ void sync_select_kernel(SyncArgs g, const float* __restrict__ rm, float4* __restrict__ c12, SyncPeak* __restrict__ pk,
                                                          float* __restrict__ refined)
{
  __shared__ float  ref[32];
  __shared__ uint32_t s_tau;
  const uint32_t u = blockIdx.x, NR = 2 * g.D - 1;
  const uint64_t HF = 75ull * g.N;
  rm += (uint64_t)blockIdx.y * 3 * g.nh * NR, c12 += (uint64_t)blockIdx.y * 3 * g.nh * g.A, pk += blockIdx.y * 3, refined += blockIdx.y * 3 * NR;
  const uint32_t bp = pk[u].bin;
  if (threadIdx.x < NR) {
    const uint32_t i  = threadIdx.x;
    const uint64_t t0 = ((uint64_t)bp * g.D + HF + i - (g.D - 1)) % HF;
    float          sum = 0.0f;
    uint32_t       cnt = 0;
    for (uint32_t h = 0; t0 + h * HF + g.N <= g.L; h++, cnt++) sum = sum + rm[(u * g.nh + h) * NR + i];
    ref[i]              = sum / (float)cnt;
    refined[u * NR + i] = ref[i];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t ib = 0;
    for (uint32_t i = 1; i < NR; i++)
      if (ref[i] > ref[ib]) ib = i;
    s_tau       = (uint32_t)(((uint64_t)bp * g.D + HF + ib - (g.D - 1)) % HF);
    pk[u].tau   = s_tau;
    pk[u].rpeak = ref[ib];
  }
  __syncthreads();
  const uint64_t tau = s_tau;
  const float2*  p   = g.rep + u * g.N;
  for (uint32_t w = threadIdx.x; w < g.nh * g.A; w += blockDim.x) {
    const uint32_t h = w / g.A, a = w % g.A;
    const uint64_t t = tau + h * HF;
    if (t + g.N > g.L) continue;
    const X* xa  = static_cast<const X*>(g.x) + blockIdx.y * g.ps + (uint64_t)a * g.lda + t;
    float    c1r = 0.0f, c1i = 0.0f, c2r = 0.0f, c2i = 0.0f;
    for (uint32_t k = 0; k < g.N / 2; k++) {
      const float2 v = chan_cf32(xa[k]), q = p[k];
      c1r            = c1r + (v.x * q.x + v.y * q.y);
      c1i            = c1i + (v.y * q.x - v.x * q.y);
    }
    for (uint32_t k = g.N / 2; k < g.N; k++) {
      const float2 v = chan_cf32(xa[k]), q = p[k];
      c2r            = c2r + (v.x * q.x + v.y * q.y);
      c2i            = c2i + (v.y * q.x - v.x * q.y);
    }
    c12[(u * g.nh + h) * g.A + a] = make_float4(c1r, c1i, c2r, c2i);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float sr = 0.0f, si = 0.0f;
    for (uint32_t h = 0; tau + h * HF + g.N <= g.L; h++)
      for (uint32_t a = 0; a < g.A; a++) {
        const float4 c = c12[(u * g.nh + h) * g.A + a];
        sr             = sr + (c.z * c.x + c.w * c.y);
        si             = si + (c.w * c.x - c.z * c.y);
      }
    pk[u].s_re = sr, pk[u].s_im = si;
  }
}

// Y[u][hs][a][sym][n]: 62-bin DFT of the PSS (sym 0, at tau + h HF) and SSS (sym 1, N + 9D earlier) windows, h = h0[u] + hs, twiddles in shared memory
template <typename X>
__global__ void __launch_bounds__(256) sync_dft_kernel(SyncArgs g, SyncSss s, float2* __restrict__ Y)
{
  extern __shared__ float2 W[];
  for (uint32_t i = threadIdx.x; i < g.N; i += blockDim.x) W[i] = g.W[i];
  __syncthreads();
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x, per_u = s.nhmax * g.A * 2 * 62;
  if (t >= 3 * per_u) return;
  const uint32_t u = t / per_u, n = t % 62, sym = (t / 62) % 2, a = (t / 124) % g.A, hs = (t / (124 * g.A)) % s.nhmax;
  const SyncPt&  q = s.pt[blockIdx.y];
  if (hs >= q.nH[u]) return;
  const uint64_t tp = q.tau[u] + (uint64_t)(q.h0[u] + hs) * 75ull * g.N, t0 = sym ? tp - g.N - 9 * g.D : tp;
  const X*       xa = static_cast<const X*>(g.x) + blockIdx.y * g.ps + (uint64_t)a * g.lda + t0;
  const uint32_t f  = n < 31 ? g.N + n - 31 : n - 30;
  float          yr = 0.0f, yi = 0.0f;
  uint32_t       idx = 0; // (f m) mod N
  for (uint32_t m = 0; m < g.N; m++) {
    const float2 v = chan_cf32(xa[m]), w = W[idx];
    yr             = yr + (v.x * w.x - v.y * w.y);
    yi             = yi + (v.x * w.y + v.y * w.x);
    idx += f;
    if (idx >= g.N) idx -= g.N;
  }
  Y[(uint64_t)blockIdx.y * 3 * per_u + t] = make_float2(yr, yi);
}

// one warp per (N_ID_2, N_ID_1): z[n] = sum_a Y_sss conj(Y_pss conj(d_u) exp(-j phi)) (real part), then for every half-frame the two SSS
// correlations in lteo_det_sum order (lane l: n = l, l + 32, then the halving tree), added to A(N_ID_1, q) with q xor (h mod 2)
__global__ void __launch_bounds__(256) sync_sss_kernel(SyncArgs g, SyncSss s, const float2* __restrict__ Y, float* __restrict__ out)
{
  const uint32_t wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= 3 * 168) return;
  const uint32_t u = wid / 168, n1 = wid % 168, per_u = s.nhmax * g.A * 124;
  const float*   q0 = s.seq + ((u * 168 + n1) * 2 + 0) * 62, *q1 = q0 + 62;
  const SyncPt&  q  = s.pt[blockIdx.y];
  const uint32_t nH = q.nH[u], h0 = q.h0[u];
  const float2*  Yu = Y + (blockIdx.y * 3 + u) * per_u;
  float          A0 = 0.0f, A1 = 0.0f;
  for (uint32_t hs = 0; hs < nH; hs++) {
    float p0 = 0.0f, p1 = 0.0f;
    for (uint32_t n = lane; n < 62; n += 32) {
      const float2 d  = s.dpss[u * 62 + n];
      float        zr = 0.0f;
      for (uint32_t a = 0; a < g.A; a++) {
        const float2* Ya = Yu + (hs * g.A + a) * 124;
        const float2  yp = Ya[n], ys = Ya[62 + n];
        const float   hr = yp.x * d.x + yp.y * d.y, hi = yp.y * d.x - yp.x * d.y;
        const float   rc = __ldg(&q.rot[u][0]), rs = __ldg(&q.rot[u][1]); // loaded where used: hoisted, they spilled
        const float   gr = hr * rc - hi * rs, gi = hr * rs + hi * rc;
        zr               = zr + (ys.x * gr + ys.y * gi);
      }
      p0 = p0 + zr * q0[n];
      p1 = p1 + zr * q1[n];
    }
    for (uint32_t off = 16; off; off >>= 1) {
      p0 = p0 + __shfl_down_sync(0xFFFFFFFFu, p0, off);
      p1 = p1 + __shfl_down_sync(0xFFFFFFFFu, p1, off);
    }
    const uint32_t h = h0 + hs;
    A0               = A0 + ((h & 1) ? p1 : p0);
    A1               = A1 + ((h & 1) ? p0 : p1);
  }
  if (lane == 0) out[((blockIdx.y * 3 + u) * 168 + n1) * 2] = A0, out[((blockIdx.y * 3 + u) * 168 + n1) * 2 + 1] = A1;
}

extern "C" int launch_sync_pss(const SyncArgs& g, uint32_t np, uint32_t fmt, float* m, float* fold, SyncPeak* pk, float* rm, float4* c12, float* refined,
                               cudaStream_t st, uint64_t* launches)
{
  const uint32_t T = COARSE_THREADS * COARSE_R, Ds = g.D | 1u;
  const size_t   smem = (size_t)g.N * 24 + (size_t)(T + g.N / g.D) * Ds * 8;
  return with_iq_type(fmt, [&](auto z) {
    using X = decltype(z);
    if (cudaFuncSetAttribute(sync_coarse_kernel<X>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
    sync_coarse_kernel<X><<<dim3((unsigned)((g.J + T - 1) / T), np), COARSE_THREADS, smem, st>>>(g, m);
    sync_fold_kernel<<<dim3((3 * SYNC_BINS + 255) / 256, np), 256, 0, st>>>(g, m, fold);
    sync_peak_kernel<<<dim3(3, np), 1024, 0, st>>>(fold, pk);
    const uint32_t nr = 3 * g.nh * (2 * g.D - 1);
    sync_refine_kernel<X><<<dim3((nr + 127) / 128, np), 128, 0, st>>>(g, pk, rm);
    sync_select_kernel<X><<<dim3(3, np), 256, 0, st>>>(g, rm, c12, pk, refined);
    *launches += 5;
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
  });
}

extern "C" int launch_sync_sss(const SyncArgs& g, uint32_t np, uint32_t fmt, const SyncSss& s, float2* Y, float* sss, cudaStream_t st, uint64_t* launches)
{
  const uint32_t nt = 3 * s.nhmax * g.A * 124;
  if (nt)
    with_iq_type(fmt, [&](auto z) {
      sync_dft_kernel<decltype(z)><<<dim3((nt + 255) / 256, np), 256, g.N * sizeof(float2), st>>>(g, s, Y);
      return 0;
    });
  sync_sss_kernel<<<dim3((3 * 168 * 32 + 255) / 256, np), 256, 0, st>>>(g, s, Y, sss);
  *launches += nt ? 2 : 1;
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
