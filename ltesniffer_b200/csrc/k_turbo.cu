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

// Per-phase cycle counters for tools/turbo_phases.py, compiled in only with -DLTEPHY_TURBO_PHASES (the default build has none of it):
// thread 0 of a CTA adds the clock64() time since its previous mark to the phase that ends at the mark, in shared memory, and the CTA
// adds its sums to turbo_phase_cycles when it leaves.  Thread 0 waits at every barrier of the CTA, so its clock is the CTA's.
#ifdef LTEPHY_TURBO_PHASES
enum { PH_QUEUE, PH_STAGE, PH_BTAIL, PH_NATURAL, PH_INTERLEAVED, PH_CRC, PH_EMIT, PH_COUNT };
__device__ unsigned long long turbo_phase_cycles[PH_COUNT];
#define PH_BEGIN()                                                                                                                               \
  __shared__ long long          ph_t;                                                                                                            \
  __shared__ unsigned long long ph_s[PH_COUNT];                                                                                                  \
  if (threadIdx.x == 0) {                                                                                                                        \
    for (int i_ = 0; i_ < PH_COUNT; i_++) ph_s[i_] = 0;                                                                                          \
    ph_t = clock64();                                                                                                                            \
  }
#define PH_MARK(p)                                                                                                                               \
  if (threadIdx.x == 0) {                                                                                                                        \
    const long long t_ = clock64();                                                                                                              \
    ph_s[p] += (unsigned long long)(t_ - ph_t);                                                                                                  \
    ph_t = t_;                                                                                                                                   \
  }
#define PH_END()                                                                                                                                 \
  if (threadIdx.x == 0)                                                                                                                          \
    for (int i_ = 0; i_ < PH_COUNT; i_++) atomicAdd(&turbo_phase_cycles[i_], ph_s[i_]);
// reads (and optionally clears) the counters of the current device: PH_COUNT values
extern "C" int ltephy_turbo_phases(unsigned long long* out, int reset)
{
  static const unsigned long long zero[PH_COUNT] = {};
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(out, turbo_phase_cycles, sizeof(zero)) != cudaSuccess) return -1;
  if (reset && cudaMemcpyToSymbol(turbo_phase_cycles, zero, sizeof(zero)) != cudaSuccess) return -1;
  return PH_COUNT;
}
#else
#define PH_BEGIN()
#define PH_MARK(p)
#define PH_END()
#endif

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
// The window is walked in 8-step chunks: forward over sub-windows 0 .. 2, then sub-windows 3 .. 0 forward with storage and backward.
// Sub-window 3 is walked forward once: its stored pass also takes the eighth step, which gives the alpha the next window starts from.
// The parity words of the next chunk are loaded while the current one is computed, so their global-memory latency is hidden behind
// 8 trellis steps.
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
    // ---- forward over all sub-windows but the last, remembering alpha at the start of every sub-window ----------
    St8 a = a0, ck[TD_NSUB];
#pragma unroll 1
    for (uint32_t sw = 0; sw + 1 < TD_NSUB; sw++) {
      ck[sw] = a;
      uint32_t pc[TD_SUB];
#pragma unroll
      for (uint32_t jj = 0; jj < TD_SUB; jj++) pc[jj] = pn[jj];
      load_par<FULL>(pn, par, (sw + 1) * TD_SUB, w, NW, len);
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
    ck[TD_NSUB - 1] = a;
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
          if (jj + 1 < TD_SUB || sw == TD_NSUB - 1) {
            alpha_step(c, af, to32(c, g[jj].x), g[jj].y, vadd(g[jj].x, g[jj].y));
            if ((jj & 1u) == 1u) norm8(c, af);
          }
        }
      }
      if (sw == TD_NSUB - 1 && w + 1 < NW) { // only a full window has a successor
        norm8(c, af);
#pragma unroll
        for (int s = 0; s < 8; s++) A[(size_t)(w + 1) * 8 + s] = af.s[s];
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
// the same product for both code blocks of a pair at once: two independent chains, so the 24 rounds of one hide the latency of the other
__device__ __forceinline__ void gf_mulmod24x2(uint32_t (&a)[2], const uint32_t (&b)[2], const uint32_t (&poly)[2], uint32_t (&r)[2])
{
  r[0] = r[1] = 0;
#pragma unroll
  for (int i = 0; i < 24; i++) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      if ((b[h] >> i) & 1u) r[h] ^= a[h];
      a[h] <<= 1;
      if (a[h] & 0x1000000u) a[h] ^= poly[h];
    }
  }
}
// b(x) x^24 mod CRC24A / CRC24B for every byte b (turbo_arith.cuh); 2 KB of global memory, read through the read-only path
__device__ const Crc24Tab crc24_tab = crc24_make_tab();

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
  __shared__ uint32_t red_s[2][8];
  __shared__ uint32_t done_s[2];
  __shared__ uint32_t next_s;

  const uint32_t tid = threadIdx.x, nthreads = NT;
  uint32_t* const my_scratch = scratch + (size_t)blockIdx.x * slot_words;
  PH_BEGIN()
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

  // the termination words of warp 0's lanes (below), asked for before the staging loads so that they arrive with them
  uint32_t tx[3] = {0u, 0u, 0u}, tz[3] = {0u, 0u, 0u};
  if (tid < 32) {
    // d0 = xK, zK+1, x'K, z'K+1 ; d1 = zK, xK+2, z'K, x'K+2 ; d2 = xK+1, zK+2, x'K+1, z'K+2
    const uint32_t* T = tv.tails + 2 * (tid >> 4); // the second constituent code's words lie two further
    tx[0] = __ldg(T + 0), tx[1] = __ldg(T + 8), tx[2] = __ldg(T + 5);
    tz[0] = __ldg(T + 4), tz[1] = __ldg(T + 1), tz[2] = __ldg(T + 9);
  }
  // boundary metrics start "unknown" (all equal: the bias); the a-priori input of the very first half iteration is zero
  for (uint32_t i = tid; i < 4 * NW * 8; i += nthreads) tv.bnd[i] = TD_BIASW;
  PH_MARK(PH_QUEUE)
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
  PH_MARK(PH_STAGE)
  if (tid < 2) done_s[tid] = (tid < P.ncb) ? 0u : 1u;
  if (tid < 32) {
    // beta at K from the termination bits (int32): one lane per (constituent code, code block, state), lane = 16 dec + 8 h + s.
    // Successor of state s on input u: NEXT[s][u] = {{0,4},{4,0},{5,1},{1,5},{2,6},{6,2},{7,3},{3,7}} (a nibble per state, the other
    // edge is 4 away); parity of that edge: PAR[s][u] = {{0,1},{0,1},{1,0},{1,0},{1,0},{1,0},{0,1},{0,1}} (a bit per state, the other edge
    // has the opposite parity).  The successors' metrics come from the lanes that hold them.
    const uint32_t h = (tid >> 3) & 1u, s = tid & 7u, base = tid & 24u;
    const uint32_t n0 = (0x37621540u >> (4 * s)) & 7u;
    const bool     p0 = (0x3Cu >> s) & 1u;
    int            bt = s ? TD_NINF : 0;
#pragma unroll
    for (int k = 2; k >= 0; k--) {
      const int x = h ? hi_s(tx[k]) : lo_s(tx[k]), z = h ? hi_s(tz[k]) : lo_s(tz[k]), zz = p0 ? z : -z;
      const int v0 = __shfl_sync(0xffffffffu, bt, base + n0) + (zz - x), v1 = __shfl_sync(0xffffffffu, bt, base + (n0 ^ 4u)) + (x - zz);
      bt           = max(v0, v1);
    }
    const int v = bt - __shfl_sync(0xffffffffu, bt, base) + (int)TD_BIAS;
    const int o = __shfl_xor_sync(0xffffffffu, v, 8); // the other code block's value of the same state
    if (!h) btail[tid >> 4][s] = ((uint32_t)v & 0xFFFFu) | ((uint32_t)o << 16);
  }
  __syncthreads();
  PH_MARK(PH_BTAIL)

  uint32_t it = 0;
  while (it < max_iter) {
    for (uint32_t i = tid; i < 2 * TD_WL * 6; i += nthreads) bits_s[i] = 0u;
    siso_pass<false, NT, FULL>(c, tv, alpha_t, bits_s, tid, active, btail[0]);
    PH_MARK(PH_NATURAL)
    siso_pass<true, NT, FULL>(c, tv, alpha_t, bits_s, tid, active, btail[1]);
    PH_MARK(PH_INTERLEAVED)
    it++;
    // ---- CRC over the K decided bits of each code block -------------------------------------------
    bool all_done = true;
    const uint32_t was_done[2] = {done_s[0], done_s[1]}; // read before anybody can set it below (every path to here passed a barrier)
    __syncthreads();
    // syndromes of the unfinished halves that carry a CRC, both in one round: word tid of a half is reduced by the byte table, moved
    // to its place by x^after, and the words are summed over the CTA
    const bool chk[2] = {!was_done[0] && P.crc_type[0], !was_done[1] && P.crc_type[1]};
    uint32_t   tot[2] = {0u, 0u};
    if (chk[0] || chk[1]) {
      uint32_t r[2] = {0u, 0u};
      if (active) {
        const uint32_t k0 = tid * TD_WL, nb = min((uint32_t)TD_WL, K - k0), after = K - k0 - nb;
        uint32_t       a[2], xp[2], poly[2];
#pragma unroll
        for (uint32_t h = 0; h < 2; h++) {
          const bool     tA = P.crc_type[h] == 1; // a half without CRC goes through CRC24B's arithmetic and is ignored
          const uint32_t v  = bits_s[h * TD_WL * 6 + tid] >> (32u - nb);
          a[h]              = crc24_fold_word(__ldg(&crc24_tab.t[tA ? 0 : 1][v >> 24]), v);
          xp[h]             = __ldg((tA ? xpowA : xpowB) + (after >> 3));
          poly[h]           = tA ? TD_CRC24A : TD_CRC24B;
        }
        gf_mulmod24x2(a, xp, poly, r);
      }
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) {
        r[0] ^= __shfl_xor_sync(0xffffffffu, r[0], off);
        r[1] ^= __shfl_xor_sync(0xffffffffu, r[1], off);
      }
      if ((tid & 31u) == 0) red_s[0][tid >> 5] = r[0], red_s[1][tid >> 5] = r[1];
      __syncthreads(); // red_s is next written an iteration (several barriers) later
      for (uint32_t i = 0; i < (nthreads + 31) / 32; i++) tot[0] ^= red_s[0][i], tot[1] ^= red_s[1][i];
    }
    PH_MARK(PH_CRC)
    for (uint32_t h = 0; h < 2; h++) {
      if (was_done[h]) continue;
      const bool ok = chk[h] && tot[h] == 0;
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
    PH_MARK(PH_EMIT)
    if (all_done) break;
  }
  } // pair queue
  PH_END()
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
    for (uint32_t i = b0; i < b1; i++) v = crc24_fold_byte(__ldg(&crc24_tab.t[0][v >> 16]), v, p[i]);
    r = gf_mulmod24(v, xpowA[n - b1], TD_CRC24A);
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
