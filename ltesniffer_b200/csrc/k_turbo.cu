// k_turbo.cu -- K8: max-log-MAP turbo decoder, batched over every code block of the batch.
// One CTA decodes a PAIR of code blocks of equal size K: the two trellises live in the low and high
// halves of packed int16x2 registers (VIADD.16x2 / VIADDMNMX.S16x2 / VIMNMX.S16x2), one thread per
// 32-step window, 8 state metrics per thread in registers, window-boundary metrics carried over from
// the previous iteration (next-iteration initialisation), alpha kept in shared memory for 8 steps at a
// time, the pair's systematic, extrinsic and interleaver arrays in shared memory for the whole pair.
// Restates the srsran_tdec_* behaviour reached through srsran_dlsch_decode2 (reference
// src/src/DL_Sniffer_PDSCH.cc:997): int16 LLRs, CRC24B/CRC24A early stop, at least one iteration.
// The arithmetic is the CPU oracle's (oracle/lte_oracle.c, siso()): outputs are offset-invariant, so
// the int16 normalisation schedule below does not change any decision.
#include "dev_common.cuh"
#include "k_launch.cuh"

#include "turbo_arith.cuh"

struct TurboView {
  const uint32_t *p1T, *p2T, *tails; // global: parity streams [32][NW] of both constituent codes, termination words
  const uint32_t* sys;               // shared: [32][NW] systematic values, window-transposed
  uint32_t*       ext;               // shared: [32][NW] a-priori / extrinsic values, updated in place by both constituent decoders
  const uint16_t* pi;                // shared: [32][NW] natural bit index of step j of window w in the interleaved order
  uint32_t*       bnd;               // global scratch slot: [2 siso][2 (A,B)][NW][8]
  uint32_t        K, NW;
};

#define TD_SUB 8 // alpha is kept in shared memory for TD_SUB steps at a time
#define TD_NSUB (TD_WL / TD_SUB)

// bit index and window-transposed word of step j of window w: the identity in the natural pass, the QPP interleaver in the other
template <bool IL>
__device__ __forceinline__ uint32_t step_bit(const TurboView& tv, uint32_t j, uint32_t w)
{
  return IL ? (uint32_t)tv.pi[j * tv.NW + w] : w * TD_WL + j;
}
__device__ __forceinline__ uint32_t bit_word(uint32_t k, uint32_t NW) { return (k & 31u) * NW + (k >> 5); }

// (2 xa, 2 p) packed for the step at word pos with parity p: xa = systematic + a-priori
__device__ __forceinline__ uint2 branch_in(const TurboView& tv, uint32_t pos, uint32_t p)
{
  const uint32_t xa = vadd(tv.sys[pos], tv.ext[pos]);
  return make_uint2(vadd(xa, xa), vadd(p, p));
}
// parity of the 8 steps j0 .. j0 + 7 of window w (coalesced across the CTA)
template <bool FULL>
__device__ __forceinline__ void load_par(uint32_t (&p)[TD_SUB], const uint32_t* par, uint32_t j0, uint32_t w, uint32_t NW, uint32_t len)
{
#pragma unroll
  for (uint32_t jj = 0; jj < TD_SUB; jj++)
    if (FULL || j0 + jj < len) p[jj] = __ldg(par + (j0 + jj) * NW + w);
}

// one SISO pass for window w.  IL = second constituent decoder (interleaved order); NT = threads per CTA
// (compile time, so every shared-memory access is base + immediate); FULL = every window has 32 steps.
// The systematic and a-priori values come from shared memory when a step needs them, with no staged copy: within a pass window w
// reads and writes ext only at its own 32 words (the identity in the natural pass, the QPP bijection in the interleaved one), and
// reads the a-priori value of step j before it writes the extrinsic value of step j, so no other window's write can reach them.
// The window is walked in 8-step chunks: forward over sub-windows 0 .. 3, then sub-windows 3 .. 0.  The parity words of the next
// chunk are loaded while the current one is computed, so their global-memory latency is hidden behind 8 trellis steps.
// Shared memory per thread: alpha_t[TD_SUB][2] (uint4).
template <bool IL, int NT, bool FULL>
__device__ __forceinline__ void siso_pass(const TdConst& c, const TurboView& tv, uint4* __restrict__ alpha_t, uint32_t* bits_s, uint32_t w,
                                          bool active, const uint32_t* btail)
{
  const uint32_t  K = tv.K, NW = tv.NW;
  const uint32_t  len = FULL ? (uint32_t)TD_WL : (active ? min((uint32_t)TD_WL, K - w * TD_WL) : 0u);
  uint32_t*       A  = tv.bnd + (size_t)(IL ? 2 : 0) * NW * 8;
  uint32_t*       B  = A + (size_t)NW * 8;
  const uint32_t* par = IL ? tv.p2T : tv.p1T;

  St8      a0, b;
  uint32_t pn[TD_SUB]; // parity of the next chunk
  if (active) {
#pragma unroll
    for (int s = 0; s < 8; s++) {
      a0.s[s] = (w == 0) ? (s ? pk2(TD_NINF + (int)TD_BIAS, TD_NINF + (int)TD_BIAS) : TD_BIASW) : A[(size_t)w * 8 + s];
      b.s[s]  = (w == NW - 1) ? btail[s] : B[(size_t)w * 8 + s];
    }
    load_par<FULL>(pn, par, 0, w, NW, len);
  }
  // every window has read its boundary metrics (A, B) before any window overwrites them below: windows w - 1 and w + 1 write
  // the slots window w has just read
  __syncthreads();

  if (active) {
    // ---- forward over the whole window, remembering alpha at the start of every sub-window ----------
    St8 a = a0, ck[TD_NSUB];
#pragma unroll 1
    for (uint32_t sw = 0; sw < TD_NSUB; sw++) {
      ck[sw] = a;
      uint32_t pc[TD_SUB];
#pragma unroll
      for (uint32_t jj = 0; jj < TD_SUB; jj++) pc[jj] = pn[jj];
      load_par<FULL>(pn, par, (sw + 1 < TD_NSUB ? sw + 1 : sw) * TD_SUB, w, NW, len); // after sub-window 3 comes sub-window 3 again
#pragma unroll
      for (uint32_t jj = 0; jj < TD_SUB; jj++) {
        const uint32_t j = sw * TD_SUB + jj;
        if (FULL || j < len) {
          const uint2 g = branch_in(tv, bit_word(step_bit<IL>(tv, j, w), NW), pc[jj]);
          alpha_step(c, a, to32(c, g.x), g.y, vadd(g.x, g.y));
          if ((jj & 1u) == 1u) norm8(c, a);
        }
      }
    }
    norm8(c, a);
    if (w + 1 < NW) {
#pragma unroll
      for (int s = 0; s < 8; s++) A[(size_t)(w + 1) * 8 + s] = a.s[s];
    }
    // ---- sub-windows, last first: forward with storage, then backward with LLR / extrinsic ----------
#pragma unroll 1
    for (int sw = TD_NSUB - 1; sw >= 0; sw--) {
      const uint32_t j0 = (uint32_t)sw * TD_SUB;
      uint32_t       pc[TD_SUB];
#pragma unroll
      for (uint32_t jj = 0; jj < TD_SUB; jj++) pc[jj] = pn[jj];
      if (sw > 0) load_par<FULL>(pn, par, j0 - TD_SUB, w, NW, len);
      if (!FULL && j0 >= len) continue;
      St8 af = ck[sw];
      // inputs of the sub-window's 8 steps, read once for both recursions and before any of its extrinsic values is written
      uint2    g[TD_SUB];
      uint32_t kb[TD_SUB];
#pragma unroll
      for (uint32_t jj = 0; jj < TD_SUB; jj++) {
        const uint32_t j = j0 + jj;
        if (FULL || j < len) {
          kb[jj] = step_bit<IL>(tv, j, w);
          g[jj]  = branch_in(tv, bit_word(kb[jj], NW), pc[jj]);
        }
      }
#pragma unroll
      for (uint32_t jj = 0; jj < TD_SUB; jj++) {
        const uint32_t j = j0 + jj;
        if (FULL || j < len) {
          alpha_t[(jj * 2 + 0) * NT] = make_uint4(af.s[0], af.s[1], af.s[2], af.s[3]);
          alpha_t[(jj * 2 + 1) * NT] = make_uint4(af.s[4], af.s[5], af.s[6], af.s[7]);
          if (jj + 1 < TD_SUB) {
            alpha_step(c, af, to32(c, g[jj].x), g[jj].y, vadd(g[jj].x, g[jj].y));
            if ((jj & 1u) == 1u) norm8(c, af);
          }
        }
      }
#pragma unroll
      for (int jj = TD_SUB - 1; jj >= 0; jj--) {
        const uint32_t j = j0 + (uint32_t)jj;
        if (FULL || j < len) {
          const uint4 u0 = alpha_t[(jj * 2 + 0) * NT], u1 = alpha_t[(jj * 2 + 1) * NT];
          St8         al;
          al.s[0] = u0.x, al.s[1] = u0.y, al.s[2] = u0.z, al.s[3] = u0.w, al.s[4] = u1.x, al.s[5] = u1.y, al.s[6] = u1.z, al.s[7] = u1.w;
          const uint32_t X32 = to32(c, g[jj].x), P32 = to32(c, g[jj].y);
          uint32_t       m1, m0;
          beta_llr_step(c, b, al, X32, P32, add32(c, X32, P32), m1, m0);
          if ((jj & 1) == 0) norm8(c, b);
          const uint32_t L = vsub(m1, m0); // the double bias cancels
          const uint32_t k = kb[jj];
          if (IL) {
            if ((int)(L << 16) > 0) atomicOr(&bits_s[k >> 5], 0x80000000u >> (k & 31u));
            if ((int)L >= 0x10000) atomicOr(&bits_s[(TD_WL * 6) + (k >> 5)], 0x80000000u >> (k & 31u));
          }
          tv.ext[bit_word(k, NW)] = ext_pair(c, L, g[jj].x);
        }
      }
    }
    norm8(c, b);
    if (w > 0) {
#pragma unroll
      for (int s = 0; s < 8; s++) B[(size_t)(w - 1) * 8 + s] = b.s[s];
    }
  }
  __syncthreads();
}

// GF(2) helpers for the parallel CRC24: (a * b) mod poly, degrees < 24
__device__ __forceinline__ uint32_t gf_mulmod24(uint32_t a, uint32_t b, uint32_t poly)
{
  uint32_t r = 0;
#pragma unroll 4
  for (int i = 0; i < 24; i++) {
    if ((b >> i) & 1u) r ^= a;
    a <<= 1;
    if (a & 0x1000000u) a ^= poly;
  }
  return r;
}
__device__ __forceinline__ uint32_t gf_mod24(uint32_t v, uint32_t nbits, uint32_t poly)
{
  uint32_t r = 0;
  for (uint32_t i = 0; i < nbits; i++) {
    r = (r << 1) | ((v >> (31 - i)) & 1u);
    if (r & 0x1000000u) r ^= poly;
  }
  return r;
}

// Persistent CTAs: the grid is sized to the number of CTAs the GPU can hold; each CTA takes code-block pairs from a queue
// (early CRC stop makes the pairs' run times vary by up to 8x).  The pair's systematic values, interleaver table and
// extrinsic values live in shared memory for the whole pair: the systematic stream and the table are read from global memory once
// per pair, and the interleaved pass gathers and scatters in shared memory (a few bank conflicts per warp access) instead of
// touching a different 128-byte line per lane.  The window-boundary metrics stay in the CTA's OWN scratch slot
// (scratch + slot * slot_words), which is rewritten for every pair, so its lines stay dirty in L2 and are never written back
// for a finished pair.  At most 168 registers per thread (384 threads per SM) in every size class: unbounded, the 32-thread
// variants take more and fit fewer CTAs per SM than shared memory allows.
template <int NT, bool FULL>
__global__ void __launch_bounds__(NT, 384 / NT) turbo_kernel(const DevPair* __restrict__ pairs, uint32_t npairs, uint32_t* __restrict__ queue,
                                                    const uint32_t* __restrict__ pool, uint32_t* __restrict__ scratch, uint32_t slot_words,
                                                    const uint16_t* __restrict__ pi_pool,
                                                    const uint32_t* __restrict__ pi_off, const uint32_t* __restrict__ xpowA,
                                                    const uint32_t* __restrict__ xpowB, uint8_t* __restrict__ payload, uint8_t* __restrict__ cb_iters,
                                                    uint8_t* __restrict__ cb_crc, uint32_t max_iter, const TdConst c)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint4*             alpha_t = reinterpret_cast<uint4*>(smem_raw) + threadIdx.x;                          // [TD_SUB][2][NT]
  uint32_t*          sys_s   = reinterpret_cast<uint32_t*>(reinterpret_cast<uint4*>(smem_raw) + TD_SUB * 2 * NT); // [TD_WL][NW], NW <= NT
  uint32_t*          ext_s   = sys_s + TD_WL * NT;                                                         // [TD_WL][NW]
  uint16_t*          pi_s    = reinterpret_cast<uint16_t*>(ext_s + TD_WL * NT);                            // [TD_WL][NW]
  __shared__ uint32_t bits_s[2 * TD_WL * 6];                       // 2 x 6144 bits
  __shared__ uint32_t btail[2][8];
  __shared__ uint32_t red_s[8];
  __shared__ uint32_t done_s[2];
  __shared__ uint32_t next_s;

  const uint32_t tid = threadIdx.x, nthreads = NT;
  uint32_t* const my_scratch = scratch + (size_t)blockIdx.x * slot_words;
  for (;;) {
    __syncthreads(); // the previous pair is completely done (shared memory and scratch slot are free)
    if (tid == 0) next_s = atomicAdd(queue, 1u);
    __syncthreads();
    const uint32_t pidx = next_s;
    if (pidx >= npairs) break;
  const DevPair  P = pairs[pidx];
  const uint32_t K = P.K, NW = P.NW;
  const bool     active = tid < NW;
  const uint32_t* sysT = pool + P.buf_off;
  const uint16_t* piT  = pi_pool + pi_off[pidx];
  TurboView       tv;
  tv.p1T   = sysT + 32 * NW;
  tv.p2T   = tv.p1T + 32 * NW;
  tv.tails = tv.p2T + 32 * NW;
  tv.sys   = sys_s;
  tv.ext   = ext_s;
  tv.pi    = pi_s;
  tv.bnd   = my_scratch;
  tv.K = K, tv.NW = NW;

  // boundary metrics start "unknown" (all equal: the bias); the a-priori input of the very first half iteration is zero
  for (uint32_t i = tid; i < 4 * NW * 8; i += nthreads) tv.bnd[i] = TD_BIASW;
  {
    // the pair's systematic values and interleaver table into shared memory, the a-priori values to zero, in 16-byte chunks (pair
    // buffers are 96 NW + 16 words and tables 32 NW entries, so both start 16-byte aligned; NW <= NT), 4 loads in flight per thread
    const uint4* s4 = reinterpret_cast<const uint4*>(sysT);
    const uint4* p4 = reinterpret_cast<const uint4*>(piT);
#pragma unroll
    for (uint32_t k0 = 0; k0 < 12; k0 += 4) {
      uint4 v[4];
#pragma unroll
      for (uint32_t k = k0; k < k0 + 4; k++) {
        const uint32_t i = (k & 7u) * NT + tid;
        if (i < (k < 8 ? 8 : 4) * NW) v[k - k0] = __ldg((k < 8 ? s4 : p4) + i);
      }
#pragma unroll
      for (uint32_t k = k0; k < k0 + 4; k++) {
        const uint32_t i = (k & 7u) * NT + tid;
        if (k < 8 && i < 8 * NW) {
          reinterpret_cast<uint4*>(sys_s)[i] = v[k - k0];
          reinterpret_cast<uint4*>(ext_s)[i] = make_uint4(0u, 0u, 0u, 0u);
        } else if (k >= 8 && i < 4 * NW)
          reinterpret_cast<uint4*>(pi_s)[i] = v[k - k0];
      }
    }
  }
  if (tid < 2) done_s[tid] = (tid < P.ncb) ? 0u : 1u;
  if (tid == 0) {
    // beta at K from the termination bits, both constituent codes, both code blocks (scalar int32)
    for (int dec = 0; dec < 2; dec++) {
      // d0 = xK, zK+1, x'K, z'K+1 ; d1 = zK, xK+2, z'K, x'K+2 ; d2 = xK+1, zK+2, x'K+1, z'K+2
      const uint32_t* T = tv.tails;
      uint32_t        tx[3], tz[3];
      if (dec == 0) {
        tx[0] = T[0], tx[1] = T[8], tx[2] = T[5];
        tz[0] = T[4], tz[1] = T[1], tz[2] = T[9];
      } else {
        tx[0] = T[2], tx[1] = T[10], tx[2] = T[7];
        tz[0] = T[6], tz[1] = T[3], tz[2] = T[11];
      }
      const uint8_t NEXT[8][2] = {{0, 4}, {4, 0}, {5, 1}, {1, 5}, {2, 6}, {6, 2}, {7, 3}, {3, 7}};
      const uint8_t PAR[8][2]  = {{0, 1}, {0, 1}, {1, 0}, {1, 0}, {1, 0}, {1, 0}, {0, 1}, {0, 1}};
      for (int h = 0; h < 2; h++) {
        int bt[8], bn[8];
        for (int s = 0; s < 8; s++) bt[s] = s ? TD_NINF : 0;
        for (int k = 2; k >= 0; k--) {
          const int x = h ? hi_s(tx[k]) : lo_s(tx[k]), z = h ? hi_s(tz[k]) : lo_s(tz[k]);
          for (int s = 0; s < 8; s++) {
            int best = -(1 << 30);
            for (int u = 0; u < 2; u++) {
              const int g = (u ? x : -x) + (PAR[s][u] ? z : -z), v = bt[NEXT[s][u]] + g;
              best        = v > best ? v : best;
            }
            bn[s] = best;
          }
          for (int s = 0; s < 8; s++) bt[s] = bn[s];
        }
        const int ref = bt[0];
        for (int s = 0; s < 8; s++) {
          const int      v = bt[s] - ref + (int)TD_BIAS;
          const uint32_t o = btail[dec][s];
          btail[dec][s]    = h ? ((o & 0xFFFFu) | ((uint32_t)v << 16)) : ((uint32_t)v & 0xFFFFu);
        }
      }
    }
  }
  __syncthreads();

  uint32_t it = 0;
  while (it < max_iter) {
    for (uint32_t i = tid; i < 2 * TD_WL * 6; i += nthreads) bits_s[i] = 0u;
    siso_pass<false, NT, FULL>(c, tv, alpha_t, bits_s, tid, active, btail[0]);
    siso_pass<true, NT, FULL>(c, tv, alpha_t, bits_s, tid, active, btail[1]);
    it++;
    // ---- CRC over the K decided bits of each code block -------------------------------------------
    bool all_done = true;
    const uint32_t was_done[2] = {done_s[0], done_s[1]}; // read before anybody can set it below (every path to here passed a barrier)
    __syncthreads();
    for (uint32_t h = 0; h < 2; h++) {
      if (was_done[h]) continue;
      const uint32_t ct = P.crc_type[h];
      bool           ok = false;
      if (ct) {
        const uint32_t  poly = ct == 1 ? 0x1864CFBu : 0x1800063u;
        const uint32_t* xp   = ct == 1 ? xpowA : xpowB;
        uint32_t        r    = 0;
        if (active) {
          const uint32_t k0 = tid * TD_WL, nb = min((uint32_t)TD_WL, K - k0), after = K - k0 - nb;
          r                 = gf_mulmod24(gf_mod24(bits_s[h * TD_WL * 6 + tid], nb, poly), xp[after >> 3], poly);
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, off);
        if ((tid & 31u) == 0) red_s[tid >> 5] = r;
        __syncthreads();
        uint32_t tot = 0;
        for (uint32_t i = 0; i < (nthreads + 31) / 32; i++) tot ^= red_s[i];
        ok = (tot == 0);
        __syncthreads();
      }
      if (ok || it == max_iter) {
        // emit the data bits (skip fillers, drop the CB CRC when C > 1): byte aligned by construction
        const uint32_t nbytes = P.out_bits[h] >> 3, skip = P.out_skip[h];
        for (uint32_t i = tid; i < nbytes; i += nthreads) {
          const uint32_t bit0 = skip + 8 * i;
          payload[P.out_byte[h] + i] = (uint8_t)((bits_s[h * TD_WL * 6 + (bit0 >> 5)] >> (24 - (bit0 & 31u))) & 0xFFu);
        }
        if (tid == 0) {
          cb_iters[P.cb_index[h]] = (uint8_t)it;
          cb_crc[P.cb_index[h]]   = ok ? 1 : 0;
          done_s[h]               = 1;
        }
      } else
        all_done = false;
    }
    __syncthreads();
    if (all_done) break;
  }
  } // pair queue
}

// ---- transport-block CRC24A over the assembled payload (tbs/8 data bytes + 3 CRC bytes) -------------
__global__ void __launch_bounds__(256) tb_crc_kernel(const DevTb* __restrict__ tbs, const uint8_t* __restrict__ payload,
                                                     const uint8_t* __restrict__ cb_crc, const uint8_t* __restrict__ cb_iters,
                                                     const uint32_t* __restrict__ xpowA, ltephy_tb_result_t* __restrict__ res)
{
  __shared__ uint32_t red_s[8];
  const DevTb&    tb = tbs[blockIdx.x];
  const uint32_t  tid = threadIdx.x, n = tb.nbytes + 3;
  const uint8_t*  p = payload + tb.byte_off;
  uint32_t        r = 0;
  // each thread folds a contiguous run of bytes, then shifts it to its position
  const uint32_t per = (n + blockDim.x - 1) / blockDim.x, b0 = tid * per, b1 = min(n, b0 + per);
  if (b0 < b1) {
    uint32_t v = 0;
    for (uint32_t i = b0; i < b1; i++) {
      for (int bit = 7; bit >= 0; bit--) {
        v = (v << 1) | ((p[i] >> bit) & 1u);
        if (v & 0x1000000u) v ^= 0x1864CFBu;
      }
    }
    r = gf_mulmod24(v, xpowA[n - b1], 0x1864CFBu);
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, off);
  if ((tid & 31u) == 0) red_s[tid >> 5] = r;
  __syncthreads();
  if (tid == 0) {
    uint32_t tot = 0;
    for (uint32_t i = 0; i < blockDim.x / 32; i++) tot ^= red_s[i];
    uint32_t ok = (tot == 0), its = 0;
    for (uint32_t i = 0; i < tb.ncb; i++) {
      if (tb.ncb > 1 && !cb_crc[tb.cb_first + i]) ok = 0;
      its += cb_iters[tb.cb_first + i];
    }
    res[blockIdx.x].crc       = (uint8_t)ok;
    res[blockIdx.x].avg_iters = (uint8_t)((its + tb.ncb - 1) / tb.ncb);
    res[blockIdx.x].nof_cb    = (uint16_t)tb.ncb;
  }
}

template <int NT, bool FULL>
static void launch_turbo_t(const DevPair* pairs, uint32_t npairs, uint32_t* queue, const uint32_t* pool, uint32_t* scratch, size_t scratch_words,
                           const uint16_t* pi_pool, const uint32_t* pi_off, const uint32_t* xpowA, const uint32_t* xpowB, uint8_t* payload,
                           uint8_t* cb_iters, uint8_t* cb_crc, uint32_t max_iter, cudaStream_t st)
{
  const size_t smem = (size_t)NT * (TD_SUB * 2 * sizeof(uint4) + 2 * TD_WL * sizeof(uint32_t) + TD_WL * sizeof(uint16_t));
  // the attribute belongs to the current device / context (handles may live on different devices): set it on every launch
  cudaFuncSetAttribute(turbo_kernel<NT, FULL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int dev = 0, sms = 132, per_sm = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, turbo_kernel<NT, FULL>, NT, smem);
  const uint32_t slot_words = 32u * NT; // boundary metrics [4][NW][8], NW <= NT
  uint32_t       grid       = (uint32_t)(sms * (per_sm > 0 ? per_sm : 1));
  grid                      = grid < npairs ? grid : npairs;
  if ((size_t)grid * slot_words > scratch_words) grid = (uint32_t)(scratch_words / slot_words);
  const TdConst c{1u, 0xFFFFFFFFu, 0xFFFFFFFEu, 3u};
  turbo_kernel<NT, FULL><<<grid, NT, smem, st>>>(pairs, npairs, queue, pool, scratch, slot_words, pi_pool, pi_off, xpowA, xpowB, payload, cb_iters,
                                                 cb_crc, max_iter, c);
}
// all pairs of one launch share the CTA size class `max_threads` (32..192) and `full` (every K a multiple of 32);
// queue: one zeroed uint32 (the pair counter of this launch); scratch: per-CTA extrinsic / boundary state (see turbo_kernel)
extern "C" void launch_turbo(const DevPair* pairs, uint32_t npairs, uint32_t max_threads, int full, uint32_t* queue, const uint32_t* pool,
                             uint32_t* scratch, size_t scratch_words, const uint16_t* pi_pool, const uint32_t* pi_off, const uint32_t* xpowA,
                             const uint32_t* xpowB, uint8_t* payload, uint8_t* cb_iters, uint8_t* cb_crc, uint32_t max_iter, cudaStream_t st,
                             uint64_t* launches)
{
  if (!npairs) return;
  const uint32_t nt = ((max_threads + 31) / 32) * 32;
#define TURBO_CASE(N)                                                                                                                            \
  case N:                                                                                                                                        \
    if (full)                                                                                                                                    \
      launch_turbo_t<N, true>(pairs, npairs, queue, pool, scratch, scratch_words, pi_pool, pi_off, xpowA, xpowB, payload, cb_iters, cb_crc,      \
                              max_iter, st);                                                                                                     \
    else                                                                                                                                         \
      launch_turbo_t<N, false>(pairs, npairs, queue, pool, scratch, scratch_words, pi_pool, pi_off, xpowA, xpowB, payload, cb_iters, cb_crc,     \
                               max_iter, st);                                                                                                    \
    break;
  switch (nt) {
    TURBO_CASE(32)
    TURBO_CASE(64)
    TURBO_CASE(96)
    TURBO_CASE(128)
    TURBO_CASE(160)
    default: TURBO_CASE(192)
  }
#undef TURBO_CASE
  *launches += 1;
}
extern "C" void launch_tb_crc(const DevTb* tbs, uint32_t ntb, const uint8_t* payload, const uint8_t* cb_crc, const uint8_t* cb_iters,
                              const uint32_t* xpowA, ltephy_tb_result_t* res, cudaStream_t st, uint64_t* launches)
{
  if (!ntb) return;
  tb_crc_kernel<<<ntb, 256, 0, st>>>(tbs, payload, cb_crc, cb_iters, xpowA, res);
  *launches += 1;
}
