// k_frontend.cu -- sm_90a kernels K1 (OFDM rx), K2 (CRS channel estimate), K3+K4 (PCFICH + PDCCH LLR),
// K10 (per-RB power).  Together they replace srsran_ue_dl_decode_fft_estimate as called from
// DCISearch::search (reference src/src/DCISearch.cc:562) and SubframePower::computePower
// (src/src/SubframePower.cc:18-58).  Compiled with -fmad=false: every float expression is evaluated
// in the order written, which is the order of the CPU oracle, so results are compared bit-for-bit.
#include "dev_common.cuh"
#include "k_launch.cuh"
#include "dev_eq.cuh"

// =================================================================================================
// K1: batched OFDM receive.  One CTA per (symbol, antenna, subframe), fft/8 threads.  The transform is the oracle's radix-2 decimation-in-time
// FFT (bit-reversed input, stages 1..log2 n, same twiddle table, same operation order -> bit-identical output) with three stages fused per
// pass in registers:
//  * pass 1 (stages 1-3) reads its 8 inputs x[t + m n/8] straight from global memory (thread t owns the group whose index is the bit reversal
//    of t, so the bit-reversal permutation costs nothing and every load instruction is one coalesced 256-byte row per warp);
//  * later passes exchange through ONE shared-memory array in the layout i ^ ((i >> 6) & 31): the lanes of a warp differ either in index bits
//    10..6 (pass 1 write, pass 2) or in bits 4..0 (later passes, final read), so every access is bank-conflict free;
//  * twiddles come from per-stage contiguous tables (tw_st[H + pos] = W_{2H}^pos) through the read-only path: coalesced, no staging.
// HBM traffic per antenna-subframe: 30720 cf32 read once, 16800 cf32 written.
// =================================================================================================
__device__ __forceinline__ uint32_t fft_swz(uint32_t i) { return i ^ ((i >> 6) & 31u); }
__device__ __forceinline__ void     fft_bfly(float2& a, float2& b, const float2 w)
{
  const float  tr = w.x * b.x - w.y * b.y;
  const float  ti = w.x * b.y + w.y * b.x;
  const float2 x  = a;
  a               = make_float2(x.x + tr, x.y + ti);
  b               = make_float2(x.x - tr, x.y - ti);
}

template <int G> // G = number of radix-2 stages fused in this pass (1..3), first stage s0 (half block h0 = 2^(s0-1))
__device__ __forceinline__ void fft_pass(float2* work, const float2* __restrict__ tw_st, uint32_t n, uint32_t s0, uint32_t tid, uint32_t nthreads)
{
  constexpr uint32_t GS = 1u << G;        // elements per group
  const uint32_t     h0 = 1u << (s0 - 1), ngroups = n / GS, hi = ngroups / h0;
  for (uint32_t w = tid; w < ngroups; w += nthreads) {
    // small h0: the lanes of a warp take the high index bits (conflict-free with the swizzle), otherwise the low ones
    const uint32_t gid  = h0 < 32 ? (w % hi) * h0 + w / hi : w;
    const uint32_t lo   = gid % h0, base = (gid / h0) * (h0 * GS) + lo;
    float2         v[GS];
#pragma unroll
    for (uint32_t j = 0; j < GS; j++) v[j] = work[fft_swz(base + j * h0)];
#pragma unroll
    for (uint32_t ss = 0; ss < (uint32_t)G; ss++) {
      const uint32_t half = h0 << ss;
#pragma unroll
      for (uint32_t q = 0; q < (1u << ss); q++) { // one twiddle W_{2 half}^{lo + q h0} per q, shared by the butterflies that differ in the bits above ss
        const float2 wv = __ldg(&tw_st[half + lo + q * h0]);
#pragma unroll
        for (uint32_t j = 0; j < GS; j++)
          if (!(j & (1u << ss)) && (j & ((1u << ss) - 1)) == q) fft_bfly(v[j], v[j + (1u << ss)], wv);
      }
    }
#pragma unroll
    for (uint32_t j = 0; j < GS; j++) work[fft_swz(base + j * h0)] = v[j];
  }
}

// R3: the symbol has 3 * 2^k samples (srsRAN's default sampling rates, 1536 at 100 PRB): three power-of-two transforms F_r of x[3 m + r] run
// side by side (thread = (r, t)), then X[k] = (F0[k mod M] + W_N^k F1[k mod M]) + W_N^(2k) F2[k mod M] -- the oracle's expression.
// X: the input's sample type (float2, short2 or char2), converted to cf32 on load, before the rotations.
template <bool UL, bool R3, bool CFO, typename X>
__global__ void __launch_bounds__(256) ofdm_rx_kernel(const __grid_constant__ DevCell c, const X* __restrict__ iq, float2* __restrict__ sym)
{
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t l = blockIdx.x, a = blockIdx.y, sf = blockIdx.z, n = c.fft, M = c.sub, L = c.log2n, q8 = M >> 3;
  const uint32_t nt = R3 ? blockDim.x / 3 : blockDim.x, r = R3 ? threadIdx.x / nt : 0u, tid = R3 ? threadIdx.x % nt : threadIdx.x;
  float2*        work = reinterpret_cast<float2*>(smem_raw) + r * M; // [3][M] or [fft], swizzled
  const uint32_t nant = gridDim.y; // c.nof_rx, or c.ul_nof_rx on the UL carrier
  const X*       src = iq + ((size_t)sf * nant + a) * c.sf_len + c.sym_off[l];
  const float2*  tw_st = c.tw_st;

  // ---- pass 1: stages 1..3 of group g = bitrev(t): A[8 g + j] = x_r[bitrev3(j) M/8 + t], x_r[i] = x[3 i + r] (x[i] for a power-of-two symbol)
  {
    const float2   w1 = __ldg(&tw_st[1]), w20 = __ldg(&tw_st[2]), w21 = __ldg(&tw_st[3]);
    const float2   w40 = __ldg(&tw_st[4]), w41 = __ldg(&tw_st[5]), w42 = __ldg(&tw_st[6]), w43 = __ldg(&tw_st[7]);
    for (uint32_t t = tid; t < q8; t += nt) {
      const uint32_t g = __brev(t) >> (32 - (L - 3));
      float2         v[8];
#pragma unroll
      for (uint32_t j = 0; j < 8; j++) {
        const uint32_t m = ((j & 1u) << 2) | (j & 2u) | (j >> 2), idx = R3 ? 3 * (t + m * q8) + r : t + m * q8;
        float2         x = chan_cf32(src[idx]);
        if (CFO) { // constant frequency-offset correction of the file samples (srsran_cfo_correct in srsran_ue_sync's file mode)
          const float2 rr = __ldg(&(UL ? c.ul_cfo_rot : c.cfo_rot)[c.sym_off[l] + idx]);
          x               = make_float2(x.x * rr.x - x.y * rr.y, x.x * rr.y + x.y * rr.x);
        }
        if (UL) { // remove the 7.5 kHz half-subcarrier shift: multiply by exp(-j pi i / N) (srsran_enb_ul_fft)
          const float2 rr = __ldg(&c.ul_rot[idx]);
          x               = make_float2(x.x * rr.x - x.y * rr.y, x.x * rr.y + x.y * rr.x);
        }
        v[j] = x;
      }
      fft_bfly(v[0], v[1], w1), fft_bfly(v[2], v[3], w1), fft_bfly(v[4], v[5], w1), fft_bfly(v[6], v[7], w1);
      fft_bfly(v[0], v[2], w20), fft_bfly(v[1], v[3], w21), fft_bfly(v[4], v[6], w20), fft_bfly(v[5], v[7], w21);
      fft_bfly(v[0], v[4], w40), fft_bfly(v[1], v[5], w41), fft_bfly(v[2], v[6], w42), fft_bfly(v[3], v[7], w43);
#pragma unroll
      for (uint32_t j = 0; j < 8; j++) work[fft_swz(8 * g + j)] = v[j];
    }
  }
  __syncthreads();
  uint32_t s = 4;
  while (s + 2 <= L) {
    fft_pass<3>(work, tw_st, M, s, tid, nt);
    __syncthreads();
    s += 3;
  }
  if (s + 1 <= L) {
    fft_pass<2>(work, tw_st, M, s, tid, nt);
    __syncthreads();
    s += 2;
  }
  if (s <= L) {
    fft_pass<1>(work, tw_st, M, s, tid, nt);
    __syncthreads();
  }
  float2*        dst = sym + (((size_t)sf * nant + a) * 14 + l) * c.nsc;
  const uint32_t h   = c.nsc / 2;
  const float2*  all = reinterpret_cast<const float2*>(smem_raw);
  for (uint32_t k = threadIdx.x; k < c.nsc; k += blockDim.x) {
    const uint32_t bin = UL ? (k + n - h) % n : (k < h ? n - h + k : k - h + 1); // no DC gap on the uplink
    if (!R3) {
      dst[k] = all[fft_swz(bin)];
    } else {
      const uint32_t kp = bin % M;
      const float2   f0 = all[fft_swz(kp)], f1 = all[M + fft_swz(kp)], f2 = all[2 * M + fft_swz(kp)];
      const float2   u1 = __ldg(&c.w3[bin]), u2 = __ldg(&c.w3[n + bin]);
      const float    t1r = u1.x * f1.x - u1.y * f1.y, t1i = u1.x * f1.y + u1.y * f1.x;
      const float    t2r = u2.x * f2.x - u2.y * f2.y, t2i = u2.x * f2.y + u2.y * f2.x;
      dst[k]             = make_float2((f0.x + t1r) + t2r, (f0.y + t1i) + t2i);
    }
  }
}

// =================================================================================================
// K2: CRS channel estimate for one (port, antenna, subframe) per CTA.
// Reads 800 pilots (+ CRS table), writes ce[14][nsc].  Restates srsran_chest_dl_estimate_cfg with the
// reference's cfg (src/src/SubframeWorker.cc:376-400).
// =================================================================================================
__global__ void __launch_bounds__(256) chest_kernel(const __grid_constant__ DevCell c, const float2* __restrict__ sym, float2* __restrict__ pilg,
                                                    DevSfInfo* __restrict__ info)
{
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t np = 2 * c.nof_prb, nsc = c.nsc;
  float2*        ls = reinterpret_cast<float2*>(smem_raw); // [4][np]
  float2*        sm = ls + NPILSYM * np;                   // [4][np]
  __shared__ float red[NPILSYM][2];
  __shared__ float cfo_s[2];

  const uint32_t p = blockIdx.x / c.nof_rx, a = blockIdx.x % c.nof_rx, sf = blockIdx.y, tid = threadIdx.x, nt = blockDim.x;
  const uint32_t sf_idx = info[sf].tti % 10;
  const float2*  y      = sym + ((size_t)sf * c.nof_rx + a) * 14 * nsc;
  const float2*  pil    = c.crs + ((size_t)sf_idx * 2 + p) * NPILSYM * np;
  const uint32_t PL[NPILSYM] = {0, 4, 7, 11};

  for (uint32_t i = tid; i < NPILSYM * np; i += nt) {
    const uint32_t li = i / np, m = i % np, l = PL[li], off = c.crs_off[p][li & 1];
    const float2   v = y[l * nsc + 6 * m + off], q = pil[li * np + m];
    ls[i]            = make_float2(v.x * q.x + v.y * q.y, v.y * q.x - v.x * q.y);
  }
  __syncthreads();
  for (uint32_t i = tid; i < NPILSYM * np; i += nt) {
    const uint32_t li = i / np, m = i % np;
    float          ar = 0.0f, ai = 0.0f, ws = 0.0f;
#pragma unroll
    for (int j = 0; j < 5; j++) {
      const int mm = (int)m + j - 2;
      if (mm < 0 || mm >= (int)np) continue;
      ar = ar + c.filt[j] * ls[li * np + mm].x;
      ai = ai + c.filt[j] * ls[li * np + mm].y;
      ws = ws + c.filt[j];
    }
    sm[i] = make_float2(ar / ws, ai / ws);
  }
  __syncthreads();
  const uint32_t warp = tid >> 5, lane = tid & 31;
  if (warp < NPILSYM) {
    float pn = 0.0f, pp = 0.0f;
    for (uint32_t m = lane; m < np; m += 32) {
      const float2 s = sm[warp * np + m], r = ls[warp * np + m];
      const float  dr = r.x - s.x, di = r.y - s.y;
      pn = pn + (dr * dr + di * di);
      pp = pp + (s.x * s.x + s.y * s.y);
    }
    pn = warp_tree_sum(pn);
    pp = warp_tree_sum(pp);
    if (lane == 0) red[warp][0] = pn, red[warp][1] = pp;
  } else if (warp == NPILSYM && p == 0 && a == 0) {
    float cr = 0.0f, ci = 0.0f;
    for (uint32_t m = lane; m < np; m += 32) {
      const float2 u = ls[0 * np + m], v = ls[2 * np + m];
      cr = cr + (u.x * v.x + u.y * v.y);
      ci = ci + (u.x * v.y - u.y * v.x);
    }
    cr = warp_tree_sum(cr);
    ci = warp_tree_sum(ci);
    if (lane == 0) cfo_s[0] = cr, cfo_s[1] = ci;
  }
  __syncthreads();
  if (tid == 0) {
    float nsum = 0.0f, psum = 0.0f;
    for (int li = 0; li < NPILSYM; li++) {
      nsum = nsum + red[li][0];
      psum = psum + red[li][1];
    }
    const float cnt   = (float)(NPILSYM * np);
    info[sf].noise[p][a] = (nsum / cnt) / c.noise_corr;
    info[sf].rsrp[p][a]  = psum / cnt;
    if (p == 0 && a == 0) {
      info[sf].cfo_re = cfo_s[0];
      info[sf].cfo_im = cfo_s[1];
    }
  }
  // the smoothed pilot grid is what the equalisers interpolate from (dev_eq.cuh: ce_at); 6.4 KB per (port, antenna, subframe) instead of 134 KB
  float2* out = pilg + (((size_t)sf * c.nof_ports + p) * c.nof_rx + a) * NPILSYM * np;
  for (uint32_t i = tid; i < NPILSYM * np; i += nt) out[i] = sm[i];
}

// The interpolated grid ce[port][ant][14][nsc] (q->chest_res.ce of the reference), materialised only when somebody asks for it
// (ltephy_tap(LTEPHY_TAP_CE): tests, the srsRAN-compatible shim); grid (ports * rx, subframes)
__global__ void __launch_bounds__(256) chest_interp_kernel(const __grid_constant__ DevCell c, const float2* __restrict__ pilg, float2* __restrict__ ce)
{
  const uint32_t np = 2 * c.nof_prb, nsc = c.nsc, p = blockIdx.x / c.nof_rx, sf = blockIdx.y;
  const float2*  pil = pilg + ((size_t)sf * c.nof_ports * c.nof_rx + blockIdx.x) * NPILSYM * np;
  float2*        out = ce + ((size_t)sf * c.nof_ports * c.nof_rx + blockIdx.x) * 14 * nsc;
  for (uint32_t i = threadIdx.x; i < 14 * nsc; i += blockDim.x) out[i] = ce_at(c, pil, p, i / nsc, i % nsc);
}

// =================================================================================================
// K10: per-PRB mean RE power of antenna 0 (SubframePower::computePower).
// =================================================================================================
__global__ void __launch_bounds__(128) rb_power_kernel(const __grid_constant__ DevCell c, const float2* __restrict__ sym, DevSfInfo* __restrict__ info)
{
  const uint32_t sf = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const float2*  y = sym + (size_t)sf * c.nof_rx * 14 * c.nsc;
  for (uint32_t prb = warp; prb < c.nof_prb; prb += nw) {
    float acc = 0.0f;
    for (uint32_t i = lane; i < 168; i += 32) {
      const float2 v = y[(i / 12) * c.nsc + 12 * prb + (i % 12)];
      acc = acc + (v.x * v.x + v.y * v.y);
    }
    acc = warp_tree_sum(acc);
    if (lane == 0) info[sf].rb_power[prb] = acc / 168.0f;
  }
}

// =================================================================================================
// K3 + K4: PCFICH decode, then PDCCH REG gather + equalise (MRC / SFBC, zero forcing) + QPSK soft
// demodulation + descrambling -> llr[nof_cce * 72], then per-CCE mean |LLR|
// (srsran_pcfich_decode, srsran_pdcch_extract_llr, srsran_pdcch_cce_avg_llr_power falcon_pdcch.c:595-620).
// =================================================================================================

__global__ void __launch_bounds__(256) pdcch_llr_kernel(const __grid_constant__ DevCell c, const float2* __restrict__ sym, const float2* __restrict__ ce,
                                                        float* __restrict__ llr_all, DevSfInfo* __restrict__ info)
{
  __shared__ uint32_t cfi_s;
  const uint32_t sf = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const uint32_t sf_idx = info[sf].tti % 10;
  const SfView   v      = make_view(c, sym, ce, sf);
  const float    ms2    = -1.41421354f;
  if (tid == 0) {
    float    llr[32];
    float2   d[16];
    if (c.nof_ports == 1) {
      for (int i = 0; i < 16; i++) d[i] = eq_port0(c, v, c.pcfich_idx[i]);
    } else {
      for (int i = 0; i < 16; i += 2) eq_sfbc(c, v, c.pcfich_idx[i], c.pcfich_idx[i + 1], d[i], d[i + 1]);
    }
    const uint32_t scr = c.pcfich_scr[sf_idx];
    for (int i = 0; i < 16; i++) {
      const float a = d[i].x * ms2, b = d[i].y * ms2;
      llr[2 * i]     = ((scr >> (2 * i)) & 1u) ? -a : a;
      llr[2 * i + 1] = ((scr >> (2 * i + 1)) & 1u) ? -b : b;
    }
    // codewords 36.212 Table 5.3.4-1: period-3 patterns 011, 101, 110
    uint32_t best = 0;
    float    corr[3];
    for (uint32_t cw = 0; cw < 3; cw++) {
      float acc = 0.0f;
      for (int i = 0; i < 32; i++) {
        const bool bit = ((i + (3 - cw) % 3) % 3) != 0; // cw0: 0,1,1  cw1: 1,0,1  cw2: 1,1,0
        acc            = acc + (bit ? llr[i] : -llr[i]);
      }
      corr[cw] = acc;
      if (acc > corr[best]) best = cw;
    }
    for (int i = 0; i < 3; i++) info[sf].pcfich_corr[i] = corr[i];
    info[sf].cfi           = best + 1;
    info[sf].nof_cce       = c.nof_cce[best];
    info[sf].nof_locations = c.nloc[best];
    cfi_s                  = best + 1;
  }
  __syncthreads();
  const uint32_t  cfi = cfi_s, nof_cce = c.nof_cce[cfi - 1], nq = nof_cce * 9;
  const uint16_t* map = c.pdcch_idx[cfi - 1];
  const uint32_t* scr = c.pdcch_scr + (size_t)sf_idx * c.pdcch_scr_words;
  float*          llr = llr_all + (size_t)sf * LLR_STRIDE;
  for (uint32_t q = tid; q < nq; q += nt) {
    uint32_t idx[4];
    float2   d[4];
#pragma unroll
    for (int j = 0; j < 4; j++) idx[j] = map[4 * q + j];
    if (c.nof_ports == 1) {
#pragma unroll
      for (int j = 0; j < 4; j++) d[j] = eq_port0(c, v, idx[j]);
    } else {
      eq_sfbc(c, v, idx[0], idx[1], d[0], d[1]);
      eq_sfbc(c, v, idx[2], idx[3], d[2], d[3]);
    }
    const uint32_t sb = (scr[(8 * q) >> 5] >> ((8 * q) & 31)) & 0xFFu;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float a = d[j].x * ms2, b = d[j].y * ms2;
      llr[8 * q + 2 * j]     = ((sb >> (2 * j)) & 1u) ? -a : a;
      llr[8 * q + 2 * j + 1] = ((sb >> (2 * j + 1)) & 1u) ? -b : b;
    }
  }
  for (uint32_t i = nq * 8 + tid; i < LLR_STRIDE; i += nt) llr[i] = 0.0f;
  __syncthreads();
  for (uint32_t cce = tid; cce < LTEPHY_MAX_CCE; cce += nt) {
    float pw = 0.0f;
    if (cce < nof_cce) {
      double m = 0.0;
      for (int i = 0; i < 72; i++) m += (double)fabsf(llr[cce * 72 + i]);
      pw = (float)(m / 72.0);
    }
    info[sf].cce_power[cce] = pw;
  }
}

// ---- launchers ----------------------------------------------------------------------------------
extern "C" void launch_chest_interp(const DevCell& c, const float2* pil, float2* ce, uint32_t n, cudaStream_t st, uint64_t* launches)
{
  chest_interp_kernel<<<dim3(c.nof_ports * c.nof_rx, n), 256, 0, st>>>(c, pil, ce);
  *launches += 1;
}

// one launch of the OFDM receive over n subframes of nant antennas (the DL or the UL carrier), in the handle's sample format
template <bool UL>
static void launch_ofdm(const DevCell& c, const void* iq, uint32_t fmt, float2* sym, uint32_t nant, uint32_t n, bool cfo, cudaStream_t st)
{
  const size_t   smem_fft = (size_t)c.fft * sizeof(float2);
  const dim3     grid(14, nant, n);
  const uint32_t nt2 = c.fft / 8 < 32 ? 32 : c.fft / 8, nt3 = 3 * (c.sub / 8);
  with_iq_type(fmt, [&](auto z) {
    using X    = decltype(z);
    const X* x = static_cast<const X*>(iq);
    if (c.sub == c.fft) {
      if (cfo)
        ofdm_rx_kernel<UL, false, true, X><<<grid, nt2, smem_fft, st>>>(c, x, sym);
      else
        ofdm_rx_kernel<UL, false, false, X><<<grid, nt2, smem_fft, st>>>(c, x, sym);
    } else {
      if (cfo)
        ofdm_rx_kernel<UL, true, true, X><<<grid, nt3, smem_fft, st>>>(c, x, sym);
      else
        ofdm_rx_kernel<UL, true, false, X><<<grid, nt3, smem_fft, st>>>(c, x, sym);
    }
    return 0;
  });
}

extern "C" void launch_frontend(const DevCell& c, const void* iq, uint32_t fmt, float2* sym, float2* ce, float* llr, DevSfInfo* info, uint32_t n,
                                cudaStream_t st, uint64_t* launches)
{
  launch_ofdm<false>(c, iq, fmt, sym, c.nof_rx, n, c.cfo_rot != nullptr, st);
  const size_t smem_ch = (size_t)2 * NPILSYM * 2 * c.nof_prb * sizeof(float2);
  chest_kernel<<<dim3(c.nof_ports * c.nof_rx, n), 256, smem_ch, st>>>(c, sym, ce, info);
  rb_power_kernel<<<n, 128, 0, st>>>(c, sym, info);
  pdcch_llr_kernel<<<n, 256, 0, st>>>(c, sym, ce, llr, info);
  *launches += 4;
}

extern "C" void launch_ul_ofdm(const DevCell& c, const void* iq, uint32_t fmt, float2* sym, uint32_t n, cudaStream_t st, uint64_t* launches)
{
  launch_ofdm<true>(c, iq, fmt, sym, c.ul_nof_rx, n, c.ul_cfo_rot != nullptr, st);
  *launches += 1;
}
