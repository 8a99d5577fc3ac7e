// k_viterbi.cu -- K5: exhaustive blind-DCI decode.  One warp decodes TWO PDCCH candidates of the same
// payload size at once (their path metrics share registers as packed int16x2); the 64 trellis states are
// spread two per lane.  Restates srsran_pdcch_dci_decode as called from
// srsran_pdcch_decode_msg_limit_avg_llr_power (reference lib/src/phy/falcon_phch/falcon_pdcch.c:110-170):
// conv rate-dematch with accumulation, uint8 quantisation (gain 32 / max|x|), K=7 r=1/3 tail-biting
// Viterbi run over three concatenated copies of which the middle one is kept, CRC16, RNTI = parity ^ crc.
// The table T[location][size] this kernel fills is what DCISearch::inspect_dci_location_recursively
// (src/src/DCISearch.cc:102-447) consults one entry at a time.
//
// Layout (tests/test_viterbi_model.py restates it lane by lane and checks it against the oracle without a GPU):
//  * ROTATING BUTTERFLY.  Before step t (phase f = t mod 5) lane bit i holds state bit ((i + f) mod 5) + 1 and the register index
//    (a0 / a1) holds state bit 0.  One exchange with lane ^ (16 >> f) brings the two predecessors of a butterfly (state bit 5)
//    into one lane; the two new states it produces are already where phase f + 1 wants them.  Round 1 routed every new state back
//    to a fixed owner: 2 SHFL + 4 SEL per step instead of 1 SHFL + 3 LOP3.
//  * DUAL-PIPE ARITHMETIC.  Integer adds issue at 16 lanes / clk on the ALU pipe and on the FMA pipe (IMAD); max / select / logic
//    only on the ALU pipe.  Branch metrics are offset by +765 (the common offset of both competitors of an add-compare-select changes no
//    decision), so every metric field is non-negative and the packed adds can run as 32-bit IMADs (a * 1 + b with the 1 in a
//    kernel parameter): no carry ever crosses from the low into the high field.  Renormalisation every 5 steps subtracts
//    (metric of state 0) - 9180; any two path metrics differ by at most 6 * 1530 = 9180 (every state is reached from every state
//    in 6 steps), so fields stay within [0, 2 * 9180 + 5 * 1530] = [0, 26010].
//  * Survivor decisions are ballot words in the layout of the step; the traceback walks in the same rotated coordinates (one bit
//    of the lane index is replaced per step), so it needs no permutation either.  CRC16 by GF(2) folding across the warp.
#include "dev_common.cuh"
#include "k_launch.cuh"

#define VIT_KMAX 80          // nof_bits <= 64 -> K = nof_bits + 16 <= 80
#define VIT_WARPS 4
#define VIT_OFFS 765         // 3 * 255: makes every branch metric non-negative
#define VIT_SPREAD 9180      // 6 * 2 * 765

struct __align__(16) VitWarpSmem {
  union {
    struct {
      float    rm[2][3 * VIT_KMAX]; // dematched soft bits, stream-major (prologue only)
      uint32_t R[3][VIT_KMAX];      // quantised symbols 2q-255, packed (cand0 lo, cand1 hi) (prologue only)
    } p;
    uint4 dec[2 * VIT_KMAX + 4];    // dec[4 + t - K]: survivor decisions of steps K..3K-1 (the up to 4 steps before K of the first stored group land in dec[0..3]): {c0 u=0, c0 u=1, c1 u=0, c1 u=1}, bit = lane of the step's layout
  };
  uint32_t S[VIT_KMAX + 4][8];      // branch metrics + 765 for the 8 output sign patterns (o0 o1 o2), packed; S[k][p ^ 7] = 1530 - S[k][p];
                                    // rows K..K+3 repeat rows 0..3 so that a group of five steps never wraps inside the table
};

struct VitConst {
  uint32_t one, minus_one; // run-time constants: keep a * 1 + b an IMAD (FMA pipe)
};

__device__ __forceinline__ uint32_t pk(int lo, int hi) { return ((uint32_t)lo & 0xFFFFu) | ((uint32_t)hi << 16); }
__device__ __forceinline__ int      lo16(uint32_t v) { return (int)(short)(v & 0xFFFFu); }
__device__ __forceinline__ int      hi16(uint32_t v) { return (int)(short)(v >> 16); }

// x^(e + 16) mod (x^16 + x^12 + x^5 + 1), e = 0..63: the CRC16 of a message is the XOR of these over its set bits
__device__ const uint16_t vit_xpow[64] = {
    0x1021, 0x2042, 0x4084, 0x8108, 0x1231, 0x2462, 0x48C4, 0x9188, 0x3331, 0x6662, 0xCCC4, 0x89A9, 0x0373, 0x06E6, 0x0DCC, 0x1B98,
    0x3730, 0x6E60, 0xDCC0, 0xA9A1, 0x4363, 0x86C6, 0x1DAD, 0x3B5A, 0x76B4, 0xED68, 0xCAF1, 0x85C3, 0x1BA7, 0x374E, 0x6E9C, 0xDD38,
    0xAA51, 0x4483, 0x8906, 0x022D, 0x045A, 0x08B4, 0x1168, 0x22D0, 0x45A0, 0x8B40, 0x06A1, 0x0D42, 0x1A84, 0x3508, 0x6A10, 0xD420,
    0xB861, 0x60E3, 0xC1C6, 0x93AD, 0x377B, 0x6EF6, 0xDDEC, 0xABF9, 0x47D3, 0x8FA6, 0x0F6D, 0x1EDA, 0x3DB4, 0x7B68, 0xF6D0, 0xFD81};

// Traceback of one candidate in the rotated coordinates of each step: (y, u) = (lane, register) of the state.  Going back one step, the bit of
// y at position pos (the one that held state bit 1) becomes the new u and is replaced by the survivor decision; pos advances by one (mod 5)
// per step, so with the start position as a template parameter every step of a group of five has a compile-time position.
// Steps idx = 2K-1 .. K (third copy) only give traceback depth; idx = K-1 .. 0 (second copy) are the data bits: bit i at position
// 31 - (i & 31) of word i >> 5, collected by a funnel shift and flushed when a word is complete.
template <int P0> __device__ __forceinline__ void vit_traceback(const uint32_t* __restrict__ dw, int K, int idx, uint32_t y, uint32_t u, uint32_t& w0,
                                                                uint32_t& w1, uint32_t& w2)
{
  uint32_t cur = 0;
#define TB_BACK(POS)                                                                                                           \
  {                                                                                                                            \
    const uint32_t d = (dw[idx * 4 + (int)u] >> y) & 1u;                                                                       \
    u                = (y >> (POS)) & 1u;                                                                                      \
    y                = (y & ~(1u << (POS))) | (d << (POS));                                                                    \
    idx--;                                                                                                                     \
  }
#define TB_REC()                                                                                                               \
  {                                                                                                                            \
    cur = __funnelshift_r(cur, u, 1);                                                                                          \
  }
#define TB_SLOW(POS)                                                                                                           \
  {                                                                                                                            \
    if (idx < K) {                                                                                                             \
      TB_REC()                                                                                                                 \
      if ((idx & 31) == 0) {                                                                                                   \
        if (idx == 64)                                                                                                         \
          w2 = cur;                                                                                                            \
        else if (idx == 32)                                                                                                    \
          w1 = cur;                                                                                                            \
        else                                                                                                                   \
          w0 = cur;                                                                                                            \
      }                                                                                                                        \
    }                                                                                                                          \
    TB_BACK(POS)                                                                                                               \
  }
  while (idx >= 4) {
    if (idx - 4 >= K) {
      TB_BACK((P0) % 5) TB_BACK((P0 + 1) % 5) TB_BACK((P0 + 2) % 5) TB_BACK((P0 + 3) % 5) TB_BACK((P0 + 4) % 5)
    } else if (idx < K && ((idx ^ (idx - 4)) & ~31) == 0 && ((idx - 4) & 31) != 0) { // five bits of one word, none of them its last
      TB_REC() TB_BACK((P0) % 5) TB_REC() TB_BACK((P0 + 1) % 5) TB_REC() TB_BACK((P0 + 2) % 5) TB_REC() TB_BACK((P0 + 3) % 5) TB_REC() TB_BACK((P0 + 4) % 5)
    } else {
      TB_SLOW((P0) % 5) TB_SLOW((P0 + 1) % 5) TB_SLOW((P0 + 2) % 5) TB_SLOW((P0 + 3) % 5) TB_SLOW((P0 + 4) % 5)
    }
  }
  if (idx >= 0) TB_SLOW((P0) % 5)
  if (idx >= 0) TB_SLOW((P0 + 1) % 5)
  if (idx >= 0) TB_SLOW((P0 + 2) % 5)
  if (idx >= 0) TB_SLOW((P0 + 3) % 5)
#undef TB_BACK
#undef TB_REC
#undef TB_SLOW
}

// One work item = (subframe, two decodable locations -- or one and VIT_LOC_NONE --, payload size) (vit_worklist_kernel).  Every step below
// is per 16-bit field or per candidate, so a candidate's result does not depend on which location shares its warp.
#define VIT_LOC_NONE 0xFFu
__device__ __forceinline__ void vit_decode_item(const DevCell& c, const float* __restrict__ llr_all, const DevSfInfo* __restrict__ info,
                                                ltephy_cand_t* __restrict__ cands, const VitConst& vc, VitWarpSmem& sm, const uint32_t lane,
                                                const uint32_t loc0, const uint32_t loc1, const uint32_t si, const uint32_t sf)
{
  const uint32_t cfi = info[sf].cfi;
  if (cfi < 1 || cfi > 3) return;
  const uint32_t nloc = c.nloc[cfi - 1];
  if (loc0 >= nloc) return;
  const uint32_t nb = c.sizes[si], K = nb + 16, n3 = 3 * K;
  const float*   llr = llr_all + (size_t)sf * LLR_STRIDE;
  const uint16_t* tab = c.conv_tab[si];

  // ---- which of the two candidates are decoded at all (location exists, every CCE above the power floor) -------------------
  bool     valid[2];
  uint32_t loc_i[2], ncce_c[2], L_c[2];
  for (int cd = 0; cd < 2; cd++) {
    loc_i[cd] = cd ? loc1 : loc0;
    valid[cd] = loc_i[cd] < nloc;
    ncce_c[cd] = 0, L_c[cd] = 0;
    if (valid[cd]) {
      const uint32_t e = c.loc_tab[cfi - 1][loc_i[cd]];
      ncce_c[cd] = e & 0xFFu, L_c[cd] = e >> 8;
      if (c.flags & LTEPHY_FLAG_SKIP_LOW_POWER)
        for (uint32_t i = ncce_c[cd]; i < ncce_c[cd] + (1u << L_c[cd]); i++)
          if (info[sf].cce_power[i] < 0.7f) valid[cd] = false;
    }
  }
  // ---- prologue: rate-dematch (accumulating), quantise -------------------------------------------
  if (valid[0] || valid[1])
    for (int cd = 0; cd < 2; cd++) {
      const uint32_t E  = 72u << L_c[cd];
      const float*   e  = llr + 72 * ncce_c[cd];
      float          mx = 0.0f;
#pragma unroll 1
      for (uint32_t j = lane; j < n3; j += 32) {
        float acc = 0.0f;
        if (valid[cd])
          for (uint32_t k = j; k < E; k += n3) acc = acc + e[k];
        sm.p.rm[cd][tab[j]] = acc;
        mx                  = fmaxf(mx, fabsf(acc));
      }
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      if (!(mx > 0.0f)) valid[cd] = false;
      const float gain = valid[cd] ? 32.0f / mx : 0.0f;
      __syncwarp();
#pragma unroll 1
      for (uint32_t st = 0; st < 3; st++)
#pragma unroll 1
        for (uint32_t k = lane; k < K; k += 32) {
          float v = sm.p.rm[cd][st * K + k] * gain + 127.5f;
          v       = fminf(fmaxf(v, 0.0f), 255.0f);
          const int r = 2 * (int)v - 255;
          reinterpret_cast<uint16_t*>(&sm.p.R[st][k])[cd] = (uint16_t)(short)r;
        }
      __syncwarp();
    }
  if (!valid[0] && !valid[1]) {
    if (lane < 2 && loc_i[lane] < LTEPHY_MAX_LOC) {
      ltephy_cand_t o{};
      cands[((size_t)sf * LTEPHY_MAX_LOC + loc_i[lane]) * LTEPHY_MAX_SIZES + si] = o;
    }
    return;
  }
  // branch-metric table for all 8 output patterns p = o0*4 + o1*2 + o2: 765 + sum_i (o_i ? +r_i : -r_i), both candidates
#pragma unroll 1
  for (uint32_t k = lane; k < K; k += 32) {
    const uint32_t r0 = sm.p.R[0][k], r1 = sm.p.R[1][k], r2 = sm.p.R[2][k];
    const uint32_t n0 = __vneg2(r0), n1 = __vneg2(r1), n2 = __vneg2(r2);
#pragma unroll
    for (uint32_t pat = 0; pat < 8; pat++)
    {
      const uint32_t m = __vadd2(__vadd2(__vadd2((pat & 4u) ? r0 : n0, (pat & 2u) ? r1 : n1), (pat & 1u) ? r2 : n2), pk(VIT_OFFS, VIT_OFFS));
      sm.S[k][pat] = m;
      if (k < 4) sm.S[K + k][pat] = m;
    }
  }
  __syncwarp();

  // ---- per-lane constants of the five phases ---------------------------------------------------------------------------
  // phase f, after the exchange: state bit 0 = lane bit (4 - f) mod 5, state bit k (1..4) = lane bit (k - 1 - f) mod 5; the register
  // index is state bit 5.  pat = output pattern of (old state with bit 5 = 0, input 0): polynomials 133, 171, 165 (octal).
  uint32_t xm[5];      // exchange mask: all ones if this lane's bit (16 >> f) is set
  uint32_t po[5];      // byte offset of this lane's pattern inside a row of S
#pragma unroll
  for (int f = 0; f < 5; f++) {
    uint32_t p = (lane >> ((4 - f + 5) % 5)) & 1u;
#pragma unroll
    for (int k = 1; k < 5; k++) p |= ((lane >> ((k - 1 - f + 10) % 5)) & 1u) << k;
    const uint32_t o0 = __popc(p & 0x36u) & 1u, o1 = __popc(p & 0x27u) & 1u, o2 = __popc(p & 0x2Bu) & 1u;
    po[f] = (o0 * 4 + o1 * 2 + o2) * 4u + 32u * (uint32_t)f; // + the row offset of step f inside its group
    xm[f] = (lane & (16u >> f)) ? 0xFFFFFFFFu : 0u;
  }
  const uint32_t C1530 = pk(2 * VIT_OFFS, 2 * VIT_OFFS), CSPREAD = pk(VIT_SPREAD, VIT_SPREAD);
  const unsigned char* Sb  = reinterpret_cast<const unsigned char*>(&sm.S[0][0]);
  const uint32_t       Kb  = K * 32u; // bytes of S in use
  uint32_t             kb  = 0;       // byte offset of row (t mod K)
  uint32_t a0 = 0, a1 = 0;            // packed path metrics of the lane's two states, non-negative fields
  uint4*   dst = sm.dec;

  // one trellis step in phase F; store: keep the survivor decisions of this step
#define VIT_SEL(D, A, B, C) asm("lop3.b32 %0, %1, %2, %3, 0xE4;" : "=r"(D) : "r"(A), "r"(B), "r"(C)) /* (A & C) | (B & ~C): one LOP3, no compare */
#define VIT_STEP(F, STORE)                                                                                                     \
  {                                                                                                                            \
    uint32_t snd, n0, n1;                                                                                                      \
    VIT_SEL(snd, a0, a1, xm[F]);                                                                                               \
    const uint32_t rcv = __shfl_xor_sync(0xffffffffu, snd, 16u >> F);                                                          \
    VIT_SEL(n0, rcv, a0, xm[F]);                                                                                               \
    VIT_SEL(n1, a1, rcv, xm[F]);                                                                                               \
    a0 = n0, a1 = n1;                                                                                                          \
    const uint32_t m   = *reinterpret_cast<const uint32_t*>(Sb + kb + po[F]);                                                  \
    const uint32_t mn  = m * vc.minus_one + C1530;                                                                             \
    bool           p0h, p0l, p1h, p1l;                                                                                         \
    const uint32_t N0 = __vibmax_s16x2(a0 * vc.one + m, a1 * vc.one + mn, &p0h, &p0l);                                         \
    const uint32_t N1 = __vibmax_s16x2(a0 * vc.one + mn, a1 * vc.one + m, &p1h, &p1l);                                         \
    if (STORE) {                                                                                                               \
      uint4 d;                                                                                                                 \
      d.x = __ballot_sync(0xffffffffu, !p0l);                                                                                  \
      d.y = __ballot_sync(0xffffffffu, !p1l);                                                                                  \
      d.z = __ballot_sync(0xffffffffu, !p0h);                                                                                  \
      d.w = __ballot_sync(0xffffffffu, !p1h);                                                                                  \
      if (lane == 0) *dst = d;                                                                                                 \
      dst++;                                                                                                                   \
    }                                                                                                                          \
    a0 = N0, a1 = N1;                                                                                                          \
  }
#define VIT_GROUP_END()  /* five rows further; the table has K rows (+ 4 repeated ones) */                                      \
  {                                                                                                                            \
    kb += 160u;                                                                                                                \
    if (kb >= Kb) kb -= Kb;                                                                                                    \
  }
#define VIT_RENORM()                                                                                                           \
  {                                                                                                                            \
    const uint32_t ref = __shfl_sync(0xffffffffu, a0, 0) * vc.one + (0u - CSPREAD); /* state 0 sits in a0 of lane 0 in every phase */ \
    a0                 = ref * vc.minus_one + a0;                                                                              \
    a1                 = ref * vc.minus_one + a1;                                                                              \
  }
  // three concatenated copies of the K-step frame = 3K steps in groups of five phases; decisions are kept from the group that contains step K on
  // (its steps before K are stored too, into dec[0..3], and never read)
  const uint32_t T3 = 3 * K, t0 = (K / 5u) * 5u;
  uint32_t       t  = 0;
  dst               = sm.dec + 4 - (K - t0);
#pragma unroll 1
  for (; t < t0; t += 5) {
    VIT_STEP(0, false) VIT_STEP(1, false) VIT_STEP(2, false) VIT_STEP(3, false) VIT_STEP(4, false)
    VIT_GROUP_END()
    VIT_RENORM()
  }
#pragma unroll 1
  for (; t + 5 <= T3; t += 5) {
    VIT_STEP(0, true) VIT_STEP(1, true) VIT_STEP(2, true) VIT_STEP(3, true) VIT_STEP(4, true)
    VIT_GROUP_END()
    VIT_RENORM()
  }
  const uint32_t tail = T3 - t; // 0..4 steps left, phases 0..
  if (tail > 0) VIT_STEP(0, true)
  if (tail > 1) VIT_STEP(1, true)
  if (tail > 2) VIT_STEP(2, true)
  if (tail > 3) VIT_STEP(3, true)
#undef VIT_STEP
#undef VIT_RENORM
#undef VIT_GROUP_END
#undef VIT_SEL
  __syncwarp();
  // ---- best final state (lowest index on ties), per candidate ------------------------------------
  // layout after the last step: phase psi = T3 mod 5 before an exchange: lane bit i = state bit ((i + psi) mod 5) + 1, register = bit 0
  const uint32_t psi = T3 % 5u;
  uint32_t       sidx = 0;
#pragma unroll
  for (uint32_t i = 0; i < 5; i++) sidx |= ((lane >> i) & 1u) << (((i + psi) % 5u) + 1u);
  uint32_t best_y[2], best_u[2];
  for (int cd = 0; cd < 2; cd++) {
    const int v0 = cd ? hi16(a0) : lo16(a0), v1 = cd ? hi16(a1) : lo16(a1);
    int       bv = v0, bs = (int)sidx;
    if (v1 > bv) bv = v1, bs = (int)sidx + 1; // same lane: the state with bit 0 set is the larger index
    uint32_t by = lane;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      const int      ov = __shfl_xor_sync(0xffffffffu, bv, off), os = __shfl_xor_sync(0xffffffffu, bs, off);
      const uint32_t oy = __shfl_xor_sync(0xffffffffu, by, off);
      if (ov > bv || (ov == bv && os < bs)) bv = ov, bs = os, by = oy;
    }
    best_y[cd] = by, best_u[cd] = (uint32_t)bs & 1u;
  }
  // ---- traceback (lanes 0,1: one candidate each) in the rotated coordinates of each step: (y, u) = (lane, register) of the state;
  // going back one step, the bit of y that held state bit 1 becomes the new u and is replaced by the decision
  uint32_t w0 = 0, w1 = 0, w2 = 0;
  if (lane < 2) {
    const int       cd = (int)lane;
    const uint32_t* dw = reinterpret_cast<const uint32_t*>(sm.dec + 4) + cd * 2; // word (t-K)*4 + cd*2 + u
    uint32_t        y = best_y[cd], u = best_u[cd], pos = (5u - psi) % 5u;
    int             idx = 2 * (int)K - 1;
    while (pos != 0) { // up to four steps (third copy, nothing recorded) bring the rotation to position 0; the rest runs with compile-time positions
      const uint32_t d = (dw[idx * 4 + (int)u] >> y) & 1u;
      u                = (y >> pos) & 1u;
      y                = (y & ~(1u << pos)) | (d << pos);
      pos              = pos == 4 ? 0 : pos + 1;
      idx--;
    }
    vit_traceback<0>(dw, (int)K, idx, y, u, w0, w1, w2);
  }
  // ---- CRC16 (poly 0x11021, zero init) over the first nb bits of both candidates at once: XOR over the set bits of
  // x^(nb - 1 - i + 16) mod P, folded across the warp; candidate 0 in the low half, candidate 1 in the high half
  uint32_t cw0[2], cw1[2], cw2[2];
#pragma unroll
  for (int cd = 0; cd < 2; cd++) {
    cw0[cd] = __shfl_sync(0xffffffffu, w0, cd), cw1[cd] = __shfl_sync(0xffffffffu, w1, cd), cw2[cd] = __shfl_sync(0xffffffffu, w2, cd);
  }
  uint32_t acc = 0;
#pragma unroll
  for (int cd = 0; cd < 2; cd++) {
    uint32_t r = 0;
    if (lane < nb && ((cw0[cd] >> (31 - lane)) & 1u)) r ^= vit_xpow[nb - 1 - lane];
    if (lane + 32 < nb && ((cw1[cd] >> (31 - lane)) & 1u)) r ^= vit_xpow[nb - 1 - (lane + 32)];
    acc |= r << (16 * cd);
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) acc ^= __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane < 2) {
    const int      cd  = (int)lane;
    const uint32_t reg = (acc >> (16 * cd)) & 0xFFFFu;
    const unsigned long long lo64 = ((unsigned long long)w0 << 32) | (unsigned long long)w1; // bits 0..63, bit i at 63 - i
    // the 16 parity bits nb .. nb+15 of the frame (bit i at position 31 - (i & 31) of word i >> 5): top 16 bits of the 96-bit string shifted left by nb
    const unsigned long long nx64 = (unsigned long long)w2 << 32;
    const unsigned long long win  = nb >= 64 ? (nx64 << (nb - 64)) : (nb == 0 ? lo64 : ((lo64 << nb) | (nx64 >> (64 - nb))));
    const uint32_t           par  = (uint32_t)(win >> 48);
    ltephy_cand_t o{};
    unsigned long long bits = lo64;
    if (nb < 64) bits &= ~((~0ull) >> nb);
    o.bits  = bits;
    o.rnti  = (uint16_t)((par ^ reg) & 0xFFFFu);
    o.valid = valid[cd] ? 1 : 0;
    if (!valid[cd]) o.bits = 0, o.rnti = 0;
    if (loc_i[cd] < LTEPHY_MAX_LOC) cands[((size_t)sf * LTEPHY_MAX_LOC + loc_i[cd]) * LTEPHY_MAX_SIZES + si] = o;
  }
}

// Work list of the decoder.  A location is decodable when it exists and, with LTEPHY_FLAG_SKIP_LOW_POWER, all its CCEs are above the power
// floor (the rule the decoder applies itself).  The decodable locations of a subframe are paired in index order, an odd count leaving one
// single-candidate item, so a warp never decodes an idle half beside a valid one.  Table entries of every other location are zeroed here,
// so nothing stale survives a change of CFI.  One CTA per subframe, one thread per location; work[0] = item count, item i =
// (work[16 + 2 i], work[17 + 2 i]) = (subframe, loc0 | loc1 << 8 | size << 16), loc1 = VIT_LOC_NONE for a single candidate.
#define VIT_WORK_HDR 16u
__global__ void __launch_bounds__(LTEPHY_MAX_LOC) vit_worklist_kernel(const __grid_constant__ DevCell c, const DevSfInfo* __restrict__ info,
                                                                      uint32_t* __restrict__ work, ltephy_cand_t* __restrict__ cands)
{
  static_assert(LTEPHY_MAX_LOC % 32 == 0 && LTEPHY_MAX_LOC <= VIT_LOC_NONE, "layout");
  __shared__ uint32_t wcnt[LTEPHY_MAX_LOC / 32];
  __shared__ uint8_t  order[LTEPHY_MAX_LOC]; // decodable locations, ascending
  __shared__ uint32_t base_s;
  const uint32_t sf = blockIdx.x, li = threadIdx.x, lane = li & 31u, warp = li >> 5, cfi = info[sf].cfi;
  const uint32_t nloc = (cfi >= 1 && cfi <= 3) ? c.nloc[cfi - 1] : 0;
  bool           v    = li < nloc;
  if (v && (c.flags & LTEPHY_FLAG_SKIP_LOW_POWER)) {
    const uint32_t e = c.loc_tab[cfi - 1][li], ncce = e & 0xFFu, L = e >> 8;
    for (uint32_t i = ncce; i < ncce + (1u << L); i++)
      if (info[sf].cce_power[i] < 0.7f) v = false;
  }
  if (!v) {
    const ltephy_cand_t z{};
    for (uint32_t si = 0; si < c.nsizes; si++) cands[((size_t)sf * LTEPHY_MAX_LOC + li) * LTEPHY_MAX_SIZES + si] = z;
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, v);
  if (lane == 0) wcnt[warp] = __popc(bal);
  __syncthreads();
  uint32_t rank = __popc(bal & ((1u << lane) - 1u)), total = 0;
#pragma unroll
  for (uint32_t w = 0; w < LTEPHY_MAX_LOC / 32; w++) {
    if (w < warp) rank += wcnt[w];
    total += wcnt[w];
  }
  if (v) order[rank] = (uint8_t)li;
  const uint32_t nitems = (total + 1) / 2;
  if (li == 0) base_s = atomicAdd(&work[0], nitems * c.nsizes);
  __syncthreads();
  if (li < nitems) {
    const uint32_t l0 = order[2 * li], l1 = 2 * li + 1 < total ? order[2 * li + 1] : VIT_LOC_NONE;
    uint2*         dst = reinterpret_cast<uint2*>(work + VIT_WORK_HDR) + base_s + li * c.nsizes;
    for (uint32_t si = 0; si < c.nsizes; si++) dst[si] = make_uint2(sf, l0 | (l1 << 8) | (si << 16));
  }
}

__global__ void __launch_bounds__(VIT_WARPS * 32) dci_viterbi_kernel(const __grid_constant__ DevCell c, const float* __restrict__ llr_all,
                                                                      const DevSfInfo* __restrict__ info, ltephy_cand_t* __restrict__ cands,
                                                                      const uint32_t* __restrict__ work, const VitConst vc)
{
  __shared__ VitWarpSmem sm_all[VIT_WARPS];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, count = work[0];
  const uint2*   items = reinterpret_cast<const uint2*>(work + VIT_WORK_HDR);
  for (uint32_t it = blockIdx.x * VIT_WARPS + warp; it < count; it += gridDim.x * VIT_WARPS) { // every warp of the grid decodes real work
    const uint2 item = items[it];
    vit_decode_item(c, llr_all, info, cands, vc, sm_all[warp], lane, item.y & 0xFFu, (item.y >> 8) & 0xFFu, item.y >> 16, item.x);
    __syncwarp(); // the next item's prologue reuses the decision store
  }
}

extern "C" void launch_viterbi(const DevCell& c, const float* llr, const DevSfInfo* info, ltephy_cand_t* cands, uint32_t* work, uint32_t n,
                               cudaStream_t st, uint64_t* launches)
{
  if (!n) return;
  const VitConst vc{1u, 0xFFFFFFFFu};
  int            dev = 0, sms = 132, per_sm = 8;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dci_viterbi_kernel, VIT_WARPS * 32, 0);
  cudaMemsetAsync(work, 0, VIT_WORK_HDR * sizeof(uint32_t), st);
  vit_worklist_kernel<<<n, LTEPHY_MAX_LOC, 0, st>>>(c, info, work, cands);
  const uint32_t max_items = n * (LTEPHY_MAX_LOC / 2) * c.nsizes, want = (max_items + VIT_WARPS - 1) / VIT_WARPS;
  const uint32_t grid = (uint32_t)sms * (uint32_t)(per_sm > 0 ? per_sm : 1);
  dci_viterbi_kernel<<<grid < want ? grid : want, VIT_WARPS * 32, 0, st>>>(c, llr, info, cands, work, vc);
  *launches += 2;
}

// ---------------------------------------------------------------------------------------------------
// Survivor selection (ltephy_compact_t, include/ltephy_b200.h): the RNTI-history-independent part of
// DCISearch::inspect_dci_location_recursively (src/src/DCISearch.cc:133-190) done for every entry of the table at once:
// sufficient-power rule (:473-489), srsran_pdcch_validate_location (falcon_pdcch.c:223-250), zero-RNTI and
// first-child-equals-parent (shortcut, :163-178) tests.  One CTA per subframe, one thread per location; the block-wide
// exclusive scan makes the list order (location, then size column) deterministic.
__device__ __forceinline__ bool dev_in_ue_space(uint32_t nof_cce, uint32_t ncce, uint32_t l, uint32_t Yk)
{
  const uint32_t L = 1u << l, M = l < 2 ? 6u : 2u;
  if (nof_cce < L || (ncce & (L - 1))) return false;
  const uint32_t n = nof_cce >> l, q = ncce >> l;
  if (q >= n) return false;
  return (q + n - Yk % n) % n < M;
}
__device__ __forceinline__ bool dev_in_common_space(uint32_t nof_cce, uint32_t ncce, uint32_t l)
{
  if (l < 2) return false;
  const uint32_t L = 1u << l;
  if (nof_cce < L || (ncce & (L - 1))) return false;
  const uint32_t lim = min(nof_cce, 16u) >> l, q = ncce >> l;
  return q < lim && q < (nof_cce >> l);
}
__device__ __forceinline__ uint32_t dev_validate_location(uint32_t nof_cce, uint32_t ncce, uint32_t l, uint32_t sf_idx, uint32_t rnti)
{
  bool ue = false, common = false;
  if (rnti >= 0x0001u && rnti <= 0x000Au)
    common = true;
  else if (rnti >= 0x000Bu && rnti <= 0xFFF3u)
    ue = common = true;
  else if (rnti >= 0xFFFDu)
    common = true;
  else
    return 0;
  uint32_t Yk = rnti;
  if (ue)
    for (uint32_t m = 0; m < sf_idx + 1; m++) Yk = (39827u * Yk) % 65537u;
  const bool valid = (ue && dev_in_ue_space(nof_cce, ncce, l, Yk)) || (common && dev_in_common_space(nof_cce, ncce, l));
  if (!valid) return 0;
  const bool amb = l > 0 && ((ue && dev_in_ue_space(nof_cce, ncce, l - 1, Yk)) || (common && dev_in_common_space(nof_cce, ncce, l - 1)));
  return amb ? 1u : 2u;
}

__global__ void __launch_bounds__(LTEPHY_MAX_LOC) cand_compact_kernel(const __grid_constant__ DevCell c, const DevSfInfo* __restrict__ info,
                                                                       const ltephy_cand_t* __restrict__ cands, ltephy_compact_t* __restrict__ out)
{
  static_assert(LTEPHY_MAX_LOC % 32 == 0 && LTEPHY_MAX_SIZES == 8, "layout");
  __shared__ uint32_t wtot[LTEPHY_MAX_LOC / 32];
  __shared__ uint8_t  smask[LTEPHY_MAX_LOC];
  const uint32_t sf = blockIdx.x, li = threadIdx.x, lane = li & 31u, warp = li >> 5;
  const uint32_t cfi = info[sf].cfi;
  const bool     ok  = cfi >= 1 && cfi <= 3;
  const uint32_t nloc = ok ? c.nloc[cfi - 1] : 0;
  uint4          e[LTEPHY_MAX_SIZES];
  uint32_t       mask = 0, my_L = 0, my_q = 0, lim = 0;
  if (li < nloc) {
    const uint32_t ent = c.loc_tab[cfi - 1][li], ncce = ent & 0xFFu, L = ent >> 8;
    const uint32_t ncce_sf = c.nof_cce[cfi - 1], sf_idx = info[sf].tti % 10;
    lim = min(ncce_sf, (uint32_t)LTEPHY_SEARCH_MAX_CCE), my_L = L, my_q = ncce >> L;
    bool           suff = true;
    for (uint32_t i = ncce; i < ncce + (1u << L); i++)
      if (i < lim && info[sf].cce_power[i] < 0.7f) suff = false;
    if (suff) {
      int par = -1; // location index of (L + 1, ncce): levels are laid out 3,2,1,0 with lim >> l entries each
      if (L < 3 && (ncce & ((2u << L) - 1u)) == 0) {
        const uint32_t lp = L + 1, q = ncce >> lp;
        uint32_t       base = 0;
        for (uint32_t l2 = 3; l2 > lp; l2--) base += lim >> l2;
        if (q < (lim >> lp) && base + q < nloc) par = (int)(base + q);
      }
      const uint4* row  = reinterpret_cast<const uint4*>(cands + ((size_t)sf * LTEPHY_MAX_LOC + li) * LTEPHY_MAX_SIZES);
      const uint4* prow = reinterpret_cast<const uint4*>(cands + ((size_t)sf * LTEPHY_MAX_LOC + (par >= 0 ? par : 0)) * LTEPHY_MAX_SIZES);
#pragma unroll
      for (uint32_t si = 0; si < LTEPHY_MAX_SIZES; si++) {
        if (si >= c.nsizes) continue;
        uint4          v  = row[si];
        const uint32_t vl = (v.z >> 16) & 0xFFu, r = vl ? (v.z & 0xFFFFu) : 0u;
        const uint32_t sm = dev_validate_location(ncce_sf, ncce, L, sf_idx, r);
        bool           eq = false;
        if (par >= 0) {
          const uint4 pv = prow[si];
          eq             = (((pv.z >> 16) & 0xFFu) ? (pv.z & 0xFFFFu) : 0u) == r;
        }
        if (sm == 0 && r != 0 && !eq) continue;
        mask |= 1u << si;
        if (!vl) v.x = 0, v.y = 0;
        v.z   = r | (vl << 16) | ((sm | ((r == 0) << 2) | ((uint32_t)eq << 3)) << 24);
        v.w   = li | (si << 8);
        e[si] = v;
      }
    }
  }
  const uint32_t cnt = __popc(mask);
  uint32_t       inc = cnt;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, off);
    if ((int)lane >= off) inc += t;
  }
  if (lane == 31) wtot[warp] = inc;
  smask[li] = (uint8_t)mask;
  __syncthreads();
  uint32_t sub = mask; // union of the masks over the location's subtree: levels are laid out 3,2,1,0 with lim >> l entries each
  if (li < nloc)
    for (uint32_t l2 = 0; l2 < my_L; l2++) {
      uint32_t b = 0;
      for (uint32_t l3 = 3; l3 > l2; l3--) b += lim >> l3;
      const uint32_t span = 1u << (my_L - l2);
      for (uint32_t j = 0; j < span; j++) {
        const uint32_t q2 = my_q * span + j;
        if (q2 < (lim >> l2) && b + q2 < nloc) sub |= smask[b + q2];
      }
    }
  uint32_t base = 0, total = 0;
#pragma unroll
  for (uint32_t w = 0; w < LTEPHY_MAX_LOC / 32; w++) {
    if (w < warp) base += wtot[w];
    total += wtot[w];
  }
  ltephy_compact_t& o   = out[sf];
  uint32_t          pos = base + inc - cnt;
  ltephy_cloc_t     cl;
  cl.off = li < nloc ? (uint16_t)min(pos, 0xFFFFu) : (uint16_t)0, cl.mask = (uint8_t)mask, cl.pad = (uint8_t)sub;
  o.loc[li] = cl;
  if (li == 0) o.count = total, o.reserved = 0;
  uint4* lst = reinterpret_cast<uint4*>(o.list);
#pragma unroll
  for (uint32_t si = 0; si < LTEPHY_MAX_SIZES; si++)
    if ((mask >> si) & 1u) {
      if (pos < LTEPHY_COMPACT_CAP) lst[pos] = e[si];
      pos++;
    }
}

extern "C" void launch_compact(const DevCell& c, const DevSfInfo* info, const ltephy_cand_t* cands, ltephy_compact_t* out, uint32_t n, cudaStream_t st,
                               uint64_t* launches)
{
  cand_compact_kernel<<<n, LTEPHY_MAX_LOC, 0, st>>>(c, info, cands, out);
  *launches += 1;
}
