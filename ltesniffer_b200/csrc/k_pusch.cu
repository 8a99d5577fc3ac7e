// k_pusch.cu -- K9: PUSCH receive chain, one CTA per UL grant: DMRS least-squares estimate on the two reference symbols (once per grant),
// 3-tap smoothing, noise / RSRP, timing-offset sums, time interpolation (or per-slot estimates under type-1 hopping), zero-forcing
// equalisation, M_sc-point mixed-radix IDFT (transform de-precoding), int16 soft demodulation, descrambling, control-information
// de-multiplexing (CQI / RI symbols taken out, ACK symbols erased) and channel de-interleaving.
// Restates srsran_chest_ul_estimate_pusch + the front half of srsran_pusch_decode as called from PUSCH_Decoder::decode_run
// (reference src/src/UL_Sniffer_PUSCH.cc:250-263) with the configuration of :421-450; the UL OFDM demodulation (srsran_enb_ul_fft, :392)
// is ofdm_rx_kernel in UL mode.  L_prb >= 3 (the 1- and 2-PRB DMRS base sequences are table-defined, 36.211 Tables 5.5.1.2-1/2).
// With NA = 2 receive antennas (DESIGN.md §2 "uplink receive diversity") each antenna is estimated alone and the equaliser combines them as
// eq_port0 does: sum_a conj(h_a) y_a / sum_a |h_a|^2; NA = 1 compiles to the one-antenna arithmetic.
// The IDFT is a Stockham autosort with radices 5.., 3.., 4.., 2 whose butterflies are plain sums in index order, the same expression tree
// as the oracle's, so the soft bits are bit-identical for every 2^a 3^b 5^c size.
#include "dev_common.cuh"
#include "k_launch.cuh"
#include "dev_ul.cuh"
#include "dev_eq.cuh"

// RI / ACK / CQI position of the symbol in row k, column c of the R' = M x 12 channel-interleaver matrix (36.212 5.2.2.7 / 5.2.2.8, normal CP:
// RI in columns {1,4,7,10}, ACK in {2,3,8,9}, both filled from the bottom row upwards in column-set order 0,3,2,1; CQI first in the row-major stream).
// kind 0 data, 1 CQI, 2 RI, 3 ACK over data (erasure), 4 ACK over CQI; dpos = index of the symbol in the UL-SCH stream
__device__ __forceinline__ uint32_t uci_pos(uint32_t M, uint32_t k, uint32_t c, uint32_t qp_ack, uint32_t qp_ri, uint32_t qp_cqi, uint32_t& dpos)
{
  const uint32_t u = M - 1 - k;
  uint32_t       before = qp_ri - min(qp_ri, 4u * (M - k)), kind = 0;
  bool           is_ri = false;
#pragma unroll
  for (uint32_t j = 0; j < 4; j++) {
    const uint32_t col = 1 + 3 * j, i = 4 * u + ((3 * j) & 3);
    if (i < qp_ri) {
      before += col < c;
      is_ri |= col == c;
    }
  }
  dpos = 0;
  if (is_ri) return 2;
  const uint32_t idx = k * 12 + c - before;
  if (idx < qp_cqi)
    kind = 1;
  else
    dpos = idx - qp_cqi;
  const int ja = c == 2 ? 0 : c == 3 ? 1 : c == 8 ? 2 : c == 9 ? 3 : -1;
  if (ja >= 0 && 4 * u + ((3 * (uint32_t)ja) & 3) < qp_ack) kind = kind == 0 ? 3 : 4;
  return kind;
}

template <uint32_t R> __device__ __forceinline__ void idft_butterfly(const float2* __restrict__ W, const float2* __restrict__ src, float2* __restrict__ dst, uint32_t M,
                                                                      uint32_t Ns, uint32_t j)
{
  const uint32_t Q = M / R, k = j % Ns, tstep = k * (M / (Ns * R));
  float2         v[R];
#pragma unroll
  for (uint32_t r = 0; r < R; r++) {
    const float2 x = src[j + r * Q];
    if (r * tstep) {
      const float2 w = W[r * tstep];
      v[r]           = make_float2(x.x * w.x - x.y * w.y, x.x * w.y + x.y * w.x);
    } else
      v[r] = x;
  }
  const uint32_t o0 = (j / Ns) * Ns * R + k;
#pragma unroll
  for (uint32_t q = 0; q < R; q++) {
    float ar = v[0].x, ai = v[0].y;
#pragma unroll
    for (uint32_t r = 1; r < R; r++) {
      const float2 w = W[((r * q) % R) * Q];
      ar             = ar + (v[r].x * w.x - v[r].y * w.y);
      ai             = ai + (v[r].x * w.y + v[r].y * w.x);
    }
    dst[o0 + q * Ns] = make_float2(ar, ai);
  }
}

#define PUSCH_PASS_CAP 2400u // float2 per ping-pong buffer: S = min(12, PUSCH_PASS_CAP / M) data symbols are transformed together

// grid (grants); ulsym [n][NA][14][nsc]
template <uint32_t NA>
__global__ void __launch_bounds__(256) pusch_kernel(const __grid_constant__ DevCell c, const DevUlGrant* __restrict__ grants,
                                                    const float2* __restrict__ ulsym, const float2* __restrict__ dmrs_pool,
                                                    const float2* __restrict__ idft_pool, const uint32_t* __restrict__ seq_pool,
                                                    short* __restrict__ llr_pool, DevUlChest* __restrict__ chest, uint32_t max_M)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const DevUlGrant g = grants[blockIdx.x];
  const uint32_t   M = g.M, tid = threadIdx.x, nt = blockDim.x, nsc = c.nsc;
  float2*          ls = reinterpret_cast<float2*>(smem_raw); // [2][M], one antenna at a time
  float2*          sm = ls + 2 * max_M;                      // [NA][2][M]
  float2*          W  = sm + 2 * NA * max_M;                 // [M]
  float2*          bufA = W + max_M;                         // [S][M]
  float2*          bufB = bufA + PUSCH_PASS_CAP;
  __shared__ float red[NA][2][4];
  const float2*    y  = ulsym + (size_t)g.sf * NA * 14 * nsc; // antenna a at y + a 14 nsc

  for (uint32_t i = tid; i < M; i += nt) W[i] = idft_pool[g.idft_off + i];
  const float f0 = 0.3333f, f1 = 1.0f - 2.0f * 0.3333f, f2 = 0.3333f;
#pragma unroll
  for (uint32_t a = 0; a < NA; a++) {
    const float2* ya  = y + a * 14 * nsc;
    float2*       sma = sm + a * 2 * M;
    if (a) __syncthreads(); // the previous antenna's sums have read ls
    for (uint32_t i = tid; i < 2 * M; i += nt) {
      const uint32_t sl = i / M, n = i % M;
      const float2   v = ya[(7 * sl + 3) * nsc + g.k0[sl] + n], r = dmrs_pool[g.dmrs_off[sl] + n];
      ls[i]            = make_float2(v.x * r.x + v.y * r.y, v.y * r.x - v.x * r.y);
    }
    __syncthreads();
    for (uint32_t i = tid; i < 2 * M; i += nt) {
      const uint32_t sl = i / M, n = i % M;
      float          ar = 0.0f, ai = 0.0f, ws = 0.0f;
      if (n > 0) ar = ar + f0 * ls[sl * M + n - 1].x, ai = ai + f0 * ls[sl * M + n - 1].y, ws = ws + f0;
      ar = ar + f1 * ls[i].x, ai = ai + f1 * ls[i].y, ws = ws + f1;
      if (n + 1 < M) ar = ar + f2 * ls[sl * M + n + 1].x, ai = ai + f2 * ls[sl * M + n + 1].y, ws = ws + f2;
      sma[i] = make_float2(ar / ws, ai / ws);
    }
    __syncthreads();
    const uint32_t warp = tid >> 5, lane = tid & 31;
    if (warp < 2) { // one warp per slot: noise, power and the lag-1 correlation of the LS estimates (timing offset)
      float pn = 0.0f, pp = 0.0f, cr = 0.0f, ci = 0.0f;
      for (uint32_t n = lane; n < M; n += 32) {
        const float2 s = sma[warp * M + n], r = ls[warp * M + n];
        const float  dr = r.x - s.x, di = r.y - s.y;
        pn = pn + (dr * dr + di * di);
        pp = pp + (s.x * s.x + s.y * s.y);
        if (n + 1 < M) {
          const float2 r1 = ls[warp * M + n + 1];
          cr = cr + (r1.x * r.x + r1.y * r.y);
          ci = ci + (r1.y * r.x - r1.x * r.y);
        }
      }
      pn = warp_tree_sum(pn), pp = warp_tree_sum(pp), cr = warp_tree_sum(cr), ci = warp_tree_sum(ci);
      if (lane == 0) red[a][warp][0] = pn, red[a][warp][1] = pp, red[a][warp][2] = cr, red[a][warp][3] = ci;
    }
  }
  __syncthreads();
  if (tid == 0) { // antenna-major, then slot; cr / ci per slot summed over the antennas
    float nsum = 0.0f, psum = 0.0f;
    for (uint32_t a = 0; a < NA; a++) nsum = nsum + red[a][0][0], nsum = nsum + red[a][1][0];
    for (uint32_t a = 0; a < NA; a++) psum = psum + red[a][0][1], psum = psum + red[a][1][1];
    const float ncorr = (1.0f - 2.0f * f1) + (f0 * f0 + f1 * f1 + f2 * f2);
    DevUlChest  o;
    o.noise = (nsum / (float)(2 * M * NA)) / ncorr;
    o.rsrp  = psum / (float)(2 * M * NA);
    o.cr[0] = red[0][0][2], o.ci[0] = red[0][0][3], o.cr[1] = red[0][1][2], o.ci[1] = red[0][1][3];
    for (uint32_t a = 1; a < NA; a++)
      o.cr[0] = o.cr[0] + red[a][0][2], o.ci[0] = o.ci[0] + red[a][0][3], o.cr[1] = o.cr[1] + red[a][1][2], o.ci[1] = o.ci[1] + red[a][1][3];
    chest[blockIdx.x] = o;
  }
  // ---- data symbols, S at a time: equalise, IDFT, demap, descramble, de-multiplex, de-interleave --------------------
  const uint32_t  S = min(12u, PUSCH_PASS_CAP / M);
  const float     scl = 1.0f / sqrtf((float)M);
  const uint32_t* seq = seq_pool + g.scr_off;
  short*          out = llr_pool + g.llr_off;
  const uint32_t  qm  = g.qm;
  const bool      hop = g.k0[0] != g.k0[1];
  for (uint32_t c0 = 0; c0 < 12; c0 += S) {
    const uint32_t ns = min(S, 12 - c0);
    for (uint32_t i = tid; i < ns * M; i += nt) {
      const uint32_t s = i / M, n = i % M, cc = c0 + s, l = cc + (cc >= 3) + (cc >= 9), sl = cc / 6; // data symbols 0,1,2,4,5,6,7,8,9,11,12,13
      const float    t = (float)((int)l - 3) / 7.0f;
      float          nr = 0.0f, ni = 0.0f, den = 0.0f;
#pragma unroll
      for (uint32_t a = 0; a < NA; a++) { // antenna 0's terms start the sums: one antenna is the one-antenna expression
        const float2* sma = sm + a * 2 * M;
        const float2  A = sma[n], B = sma[M + n];
        const float2  h = hop ? sma[sl * M + n] : make_float2(A.x + (B.x - A.x) * t, A.y + (B.y - A.y) * t);
        const float2  v = y[(a * 14 + l) * nsc + g.k0[sl] + n];
        const float   tr = v.x * h.x + v.y * h.y, ti = v.y * h.x - v.x * h.y, td = h.x * h.x + h.y * h.y;
        nr = a ? nr + tr : tr, ni = a ? ni + ti : ti, den = a ? den + td : td;
      }
      bufA[i] = make_float2(eq_div(nr, den), eq_div(ni, den)); // no channel: 0, not NaN
    }
    __syncthreads();
    float2 * src = bufA, *dst = bufB;
    uint32_t Ns  = 1;
    for (uint32_t st = 0; st < g.nrad; st++) {
      const uint32_t R = (g.rad >> (4 * st)) & 15u, Q = M / R;
      for (uint32_t i = tid; i < ns * Q; i += nt) {
        const uint32_t s = i / Q, j = i % Q;
        if (R == 5)
          idft_butterfly<5>(W, src + s * M, dst + s * M, M, Ns, j);
        else if (R == 3)
          idft_butterfly<3>(W, src + s * M, dst + s * M, M, Ns, j);
        else if (R == 4)
          idft_butterfly<4>(W, src + s * M, dst + s * M, M, Ns, j);
        else
          idft_butterfly<2>(W, src + s * M, dst + s * M, M, Ns, j);
      }
      __syncthreads();
      float2* t = src;
      src = dst, dst = t, Ns *= R;
    }
    for (uint32_t i = tid; i < ns * M; i += nt) {
      const uint32_t s = i % ns, k = i / ns, cc = c0 + s; // adjacent threads: adjacent columns of one row -> adjacent soft bits
      uint32_t       dpos;
      const uint32_t kind = uci_pos(M, k, cc, g.qp_ack, g.qp_ri, g.qp_cqi, dpos);
      if (kind != 0 && kind != 3) continue;
      const float2 zz = kind == 3 ? make_float2(0.0f, 0.0f) : src[s * M + k]; // ACK over data: erased, zero soft bits
      soft_bits(zz, scl, qm, seq, (cc * M + k) * qm, out + dpos * qm);
    }
    __syncthreads();
  }
}

extern "C" void launch_pusch(const DevCell& c, const DevUlGrant* grants, uint32_t ngrants, uint32_t max_M, const float2* ulsym, const float2* dmrs_pool,
                             const float2* idft_pool, const uint32_t* seq_pool, short* llr_pool, DevUlChest* chest, cudaStream_t st, uint64_t* launches)
{
  if (!ngrants) return;
  // ls [2][M], sm [A][2][M], W [M] and the two IDFT buffers: 86 KB at M = 1200 with one antenna, 106 KB with two (two CTAs per SM either way)
  const size_t smem = ((size_t)(3 + 2 * c.ul_nof_rx) * max_M + 2 * PUSCH_PASS_CAP) * sizeof(float2);
  const int    cap  = (int)(((3 + 2 * c.ul_nof_rx) * 1200 + 2 * PUSCH_PASS_CAP) * sizeof(float2));
  if (c.ul_nof_rx == 2) {
    cudaFuncSetAttribute(pusch_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap); // per device / context
    pusch_kernel<2><<<ngrants, 256, smem, st>>>(c, grants, ulsym, dmrs_pool, idft_pool, seq_pool, llr_pool, chest, max_M);
  } else {
    cudaFuncSetAttribute(pusch_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap);
    pusch_kernel<1><<<ngrants, 256, smem, st>>>(c, grants, ulsym, dmrs_pool, idft_pool, seq_pool, llr_pool, chest, max_M);
  }
  *launches += 1;
}
