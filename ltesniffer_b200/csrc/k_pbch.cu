// k_pbch.cu -- PBCH / MIB decode of subframe 0 (SURVEY 8f-1): what srsran_ue_mib_decode + srsran_pbch_mib_unpack deliver before the hot path
// starts (reference src/src/LTESniffer_Core.cc:382-396: bandwidth, PHICH configuration, SFN; the CRC mask gives the antenna-port count).
// Two kernels serve both ltephy_mib_decode (one frame at a time) and ltephy_mib_decode_combined (soft combining across the 40 ms period,
// DESIGN.md §2 "PBCH combining"):
//   pbch_llr_kernel  one CTA per (subframe 0 of the batch, port count): equalise the 240 resource elements (slot 1, symbols 0..3, central 72 sub-carriers
//                    without the CRS of four ports) for the port counts asked for (1: port 0 zero forcing; 2: SFBC; the combining decoder asks for
//                    every one the handle can equalise, ltephy_mib_decode for the handle's) and store the 480 QPSK soft bits per port count in the
//                    handle's frame store, row 3 + (ordinal of the frame in the batch).
//   pbch_hyp_kernel  one warp per hypothesis (port count, n consecutive frames ending at a given row, their first position dst in the period):
//                    descramble frame j with bits [480 (dst + j), 480 (dst + j) + 480) of c(cell_id), rate-dematch the 1920-value input 480 -> 120
//                    with accumulation in ascending input order (absent frames are zeros, which add exactly and are skipped), quantise like the
//                    PDCCH decoder, tail-biting Viterbi (K = 7, r = 1/3, three concatenated copies, middle kept), CRC16.  Output: the port count
//                    whose mask the remainder is (0x0000 / 0xFFFF / 0x5555 -> 1 / 2 / 4, 0 for none) and the 24 bits.  The host picks the winner.
// A one-frame hypothesis at dst = q is, bit for bit, the decode of position q of lteo_pbch_decode: same arithmetic and tie rules.
#include "dev_common.cuh"
#include "k_launch.cuh"
#include "dev_eq.cuh"

#define PBCH_ROW 960 // floats per frame-store row: [port count - 1][480]

__global__ void __launch_bounds__(128) pbch_llr_kernel(const __grid_constant__ DevCell c, const float2* __restrict__ sym, const float2* __restrict__ pil,
                                                       const uint32_t* __restrict__ frame_sf, uint32_t p_first, float* __restrict__ store)
{
  const uint32_t sf = frame_sf[blockIdx.x], tid = threadIdx.x, p = p_first + blockIdx.y; // p = port count - 1
  float*         row = store + (size_t)(3 + blockIdx.x) * PBCH_ROW + 480 * p;
  const SfView   v   = make_view(c, sym, pil, sf);
  const float    ms2 = -1.41421354f;
  if (p == 0) {
    for (uint32_t i = tid; i < 240; i += blockDim.x) {
      const uint32_t e = c.pbch_re[i];
      const float2   d = eq_port0(c, v, (e >> 16) * c.nsc + (e & 0xFFFFu));
      row[2 * i] = d.x * ms2, row[2 * i + 1] = d.y * ms2;
    }
  } else {
    for (uint32_t i = 2 * tid; i < 240; i += 2 * blockDim.x) {
      const uint32_t e0 = c.pbch_re[i], e1 = c.pbch_re[i + 1];
      float2         d0, d1;
      eq_sfbc(c, v, (e0 >> 16) * c.nsc + (e0 & 0xFFFFu), (e1 >> 16) * c.nsc + (e1 & 0xFFFFu), d0, d1);
      row[2 * i] = d0.x * ms2, row[2 * i + 1] = d0.y * ms2, row[2 * i + 2] = d1.x * ms2, row[2 * i + 3] = d1.y * ms2;
    }
  }
}

// Quantise the 120 dematched values rm (mx = max |rm|, 0: nothing to decode), tail-biting Viterbi, CRC16 -- one warp.  Returns {port count of the
// CRC mask or 0, the 24 MIB bits with the first bit in bit 23}, valid in every lane.
__device__ uint2 pbch_viterbi_crc(const float* rm, float mx, int* rq, int (*pm)[64], unsigned long long* dec, uint32_t lane)
{
  const uint32_t K    = 40;
  const bool     ok   = mx > 0.0f;
  const float    gain = ok ? 32.0f / mx : 0.0f;
  for (uint32_t i = lane; i < 120; i += 32) {
    float x = rm[i] * gain + 127.5f;
    x       = fminf(fmaxf(x, 0.0f), 255.0f);
    rq[i]   = 2 * (int)x - 255;
  }
  pm[0][lane] = 0, pm[0][lane + 32] = 0;
  // output signs of the branches into new states sn = lane and lane + 32: predecessor p, input c = sn & 1; polynomials 133, 171, 165 (octal)
  int sg[2][2][3];
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int w = 0; w < 2; w++) {
      const int sn = (int)lane + 32 * h, cc = sn & 1, s = (sn >> 1) | (w ? 32 : 0);
#define TB(j) ((s >> ((j)-1)) & 1)
      const int o0 = cc ^ TB(2) ^ TB(3) ^ TB(5) ^ TB(6), o1 = cc ^ TB(1) ^ TB(2) ^ TB(3) ^ TB(6), o2 = cc ^ TB(1) ^ TB(2) ^ TB(4) ^ TB(6);
#undef TB
      sg[h][w][0] = o0 ? 1 : -1, sg[h][w][1] = o1 ? 1 : -1, sg[h][w][2] = o2 ? 1 : -1;
    }
  __syncwarp();
  for (uint32_t t = 0; t < 3 * K; t++) {
    const uint32_t k = t % K, cur = t & 1;
    const int      r0 = rq[k], r1 = rq[K + k], r2 = rq[2 * K + k];
    unsigned long long dw = 0;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int sn = (int)lane + 32 * h, p0 = sn >> 1, p1 = p0 | 32;
      const int m0 = pm[cur][p0] + sg[h][0][0] * r0 + sg[h][0][1] * r1 + sg[h][0][2] * r2;
      const int m1 = pm[cur][p1] + sg[h][1][0] * r0 + sg[h][1][1] * r1 + sg[h][1][2] * r2;
      const bool     take1 = m1 > m0; // ties keep the lower predecessor
      pm[cur ^ 1][sn]      = take1 ? m1 : m0;
      const uint32_t bal   = __ballot_sync(0xffffffffu, take1);
      dw |= (unsigned long long)bal << (32 * h);
    }
    if (lane == 0) dec[t] = dw;
    __syncwarp();
  }
  // best end state: the lowest index among the maxima
  const uint32_t fin = (3 * K) & 1;
  int            bv = pm[fin][lane], bs = (int)lane;
  if (pm[fin][lane + 32] > bv) bv = pm[fin][lane + 32], bs = (int)lane + 32;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const int ov = __shfl_xor_sync(0xffffffffu, bv, off), os = __shfl_xor_sync(0xffffffffu, bs, off);
    if (ov > bv || (ov == bv && os < bs)) bv = ov, bs = os;
  }
  uint32_t np = 0, mib = 0;
  if (lane == 0) {
    uint32_t st = (uint32_t)bs;
    unsigned long long data = 0; // bit i of the frame at bit (39 - i)
    for (int t = 3 * (int)K - 1; t >= (int)K; t--) {
      if (t < 2 * (int)K) data |= (unsigned long long)(st & 1u) << (39 - (t - (int)K));
      st = (st >> 1) | ((uint32_t)((dec[t] >> st) & 1ull) << 5);
    }
    mib                = (uint32_t)(data >> 16) & 0xFFFFFFu;
    const uint32_t par = (uint32_t)data & 0xFFFFu;
    uint32_t       crc = 0;
    for (int i = 23; i >= 0; i--) { // CRC16, polynomial 0x11021, zero initial state
      crc ^= ((mib >> i) & 1u) << 15;
      crc = (crc & 0x8000u) ? ((crc << 1) ^ 0x1021u) & 0xFFFFu : (crc << 1) & 0xFFFFu;
    }
    const uint32_t rem = par ^ crc;
    np                 = !ok ? 0u : rem == 0x0000u ? 1u : rem == 0xFFFFu ? 2u : rem == 0x5555u ? 4u : 0u;
  }
  return make_uint2(__shfl_sync(0xffffffffu, np, 0), __shfl_sync(0xffffffffu, mib, 0));
}

// job word: bit 0 port count - 1, bits 1..2 n - 1, bits 3..4 dst, bits 5..31 the frame-store row of the newest of the n frames
__global__ void __launch_bounds__(128) pbch_hyp_kernel(const __grid_constant__ DevCell c, const float* __restrict__ store, const uint32_t* __restrict__ jobs,
                                                       uint32_t njobs, uint2* __restrict__ out)
{
  __shared__ float              rm[4][120];
  __shared__ int                rq[4][120];
  __shared__ int                pm[4][2][64];
  __shared__ unsigned long long dec[4][120];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, j = blockIdx.x * 4 + warp;
  if (j >= njobs) return;
  const uint32_t job = jobs[j], p = job & 1u, n = ((job >> 1) & 3u) + 1, dst = (job >> 3) & 3u, newest = job >> 5;
  const float*   x0  = store + (size_t)(newest + 1 - n) * PBCH_ROW + 480 * p;
  float          mx  = 0.0f;
  for (uint32_t m = lane; m < 120; m += 32) {
    float acc = 0.0f;
    for (uint32_t f = 0; f < n; f++) { // input positions 480 pos + 120 rep + m in ascending order; the other positions hold zeros
      const float* x = x0 + (size_t)f * PBCH_ROW;
#pragma unroll
      for (uint32_t rep = 0; rep < 4; rep++) {
        const uint32_t k = m + 120 * rep, b = 480 * (dst + f) + k, sbit = (c.pbch_scr[b >> 5] >> (b & 31)) & 1u;
        acc = acc + (sbit ? -x[k] : x[k]);
      }
    }
    rm[warp][c.pbch_tab[m]] = acc;
    mx                      = fmaxf(mx, fabsf(acc));
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  __syncwarp();
  const uint2 r = pbch_viterbi_crc(rm[warp], mx, rq[warp], pm[warp], dec[warp], lane);
  if (lane == 0) out[j] = r;
}

extern "C" void launch_pbch(const DevCell& c, const float2* sym, const float2* pil, const uint32_t* frame_sf, uint32_t nframes, uint32_t p_first, uint32_t np,
                            float* store,
                            const uint32_t* jobs, uint32_t njobs, void* out, cudaStream_t st, uint64_t* launches)
{
  if (nframes) {
    pbch_llr_kernel<<<dim3(nframes, np), 128, 0, st>>>(c, sym, pil, frame_sf, p_first, store);
    *launches += 1;
  }
  if (njobs) {
    pbch_hyp_kernel<<<(njobs + 3) / 4, 128, 0, st>>>(c, store, jobs, njobs, static_cast<uint2*>(out));
    *launches += 1;
  }
}
