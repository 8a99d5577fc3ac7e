// turbo_arith.cuh -- arithmetic core of the max-log-MAP decoder (K8), shared by the kernel (k_turbo.cu) and by the host model that
// checks it against the CPU oracle without a GPU (tools/turbo_model.cpp, tests/test_turbo_model.py): the packed int16x2 intrinsics
// get bit-identical host definitions below when this header is compiled for the host.
#pragma once
#include <cstdint>
#ifdef __CUDACC__
#define TD_HD __host__ __device__ __forceinline__
#else
#define TD_HD inline
#endif
#if !defined(__CUDA_ARCH__)
// host definitions of the SIMD-in-a-word intrinsics (per 16-bit field, two's complement, wrap-around like the hardware)
namespace td_host {
inline uint32_t f2(int lo, int hi) { return ((uint32_t)lo & 0xFFFFu) | ((uint32_t)hi << 16); }
inline int      slo(uint32_t v) { return (int)(short)(v & 0xFFFFu); }
inline int      shi(uint32_t v) { return (int)(short)(v >> 16); }
inline int      ulo(uint32_t v) { return (int)(v & 0xFFFFu); }
inline int      uhi(uint32_t v) { return (int)(v >> 16); }
inline uint32_t vadd2(uint32_t a, uint32_t b) { return f2(slo(a) + slo(b), shi(a) + shi(b)); }
inline uint32_t vsub2(uint32_t a, uint32_t b) { return f2(slo(a) - slo(b), shi(a) - shi(b)); }
inline uint32_t vmaxs2(uint32_t a, uint32_t b) { return f2(slo(a) > slo(b) ? slo(a) : slo(b), shi(a) > shi(b) ? shi(a) : shi(b)); }
inline uint32_t vmins2(uint32_t a, uint32_t b) { return f2(slo(a) < slo(b) ? slo(a) : slo(b), shi(a) < shi(b) ? shi(a) : shi(b)); }
inline uint32_t viaddmax_s(uint32_t a, uint32_t b, uint32_t c) { return vmaxs2(vadd2(a, b), c); }
inline uint32_t viaddmax_u(uint32_t a, uint32_t b, uint32_t c)
{
  const uint32_t s = vadd2(a, b);
  return f2(ulo(s) > ulo(c) ? ulo(s) : ulo(c), uhi(s) > uhi(c) ? uhi(s) : uhi(c));
}
} // namespace td_host
#define TD_VADD2(a, b) td_host::vadd2(a, b)
#define TD_VSUB2(a, b) td_host::vsub2(a, b)
#define TD_VMAXS2(a, b) td_host::vmaxs2(a, b)
#define TD_VMINS2(a, b) td_host::vmins2(a, b)
#define TD_VIADDMAX_S(a, b, c) td_host::viaddmax_s(a, b, c)
#define TD_VIADDMAX_U(a, b, c) td_host::viaddmax_u(a, b, c)
#else
#define TD_VADD2(a, b) __vadd2(a, b)
#define TD_VSUB2(a, b) __vsub2(a, b)
#define TD_VMAXS2(a, b) __vmaxs2(a, b)
#define TD_VMINS2(a, b) __vmins2(a, b)
#define TD_VIADDMAX_S(a, b, c) __viaddmax_s16x2(a, b, c)
#define TD_VIADDMAX_U(a, b, c) __viaddmax_u16x2(a, b, c)
#endif

#define TD_WL 32
#define TD_NINF (-8192)
#define TD_BIAS 0x4C00u                 // every state metric is kept as (true value + TD_BIAS) in both 16-bit fields
#define TD_BIASW 0x4C004C00u

// ---- arithmetic model ------------------------------------------------------------------------------------------------
// Integer adds issue on two pipes of an SM sub-partition at 16 lanes / clk each: the ALU pipe (IADD3, LOP3, VIADD.16x2,
// VIMNMX.S16x2, VIADDMNMX.S16x2) and the FMA pipe (IMAD).  A decoder written only with packed 16x2 adds and maxes is bound by the
// ALU pipe at half the issue rate (round-1 ncu: math-pipe-throttle stalls, 51-62 % issue slots).  Here every plain add runs as a
// 32-bit IMAD (a * 1 + b, with the 1 in a kernel parameter so that it stays an IMAD), which is exact field-wise as long as the low
// field of the left operand and of the result is non-negative: state metrics therefore carry a bias of 0x4C00 per field (bounds
// below), and the signed addends (branch metrics, normalisation reference) are used in "32-form" hi * 65536 + lo.  Maxes and add-max stay packed on the ALU pipe.  The decisions are offset-
// invariant, so bias, branch-metric offset and normalisation schedule do not change any output (oracle/lte_oracle.c, siso()).
//
// Branch metrics: the oracle's edge metric for (u, parity) is +-xa +- p.  Adding xa + p to all 16 edges of a step gives
//   (0,0) -> 0,  (1,1) -> G0 = 2 (xa + p),  (1,0) -> X = 2 xa,  (0,1) -> P = 2 p,
// so 4 of the 8 add-compare-selects of a step need one add instead of two.  |X| <= 1532, |P| <= 510, |G0| <= 2042.
// Ranges, inputs |sys|, |par| <= 255 and |a-priori| <= 511 (true values relative to the last normalisation, which sets state 0 to 0
// and happens every 2 steps): the metrics of any two states differ by at most 3 * 2042 = 6126 (every state is reached from every
// state in 3 steps), state 0 drifts by at most 2 * 2042 between normalisations, an add-compare-select candidate adds one more
// edge: stored values lie in [-10210, +10210], candidates in [-12252, +12252].  The first window starts from (0, -8192 x 7): its
// -8192-derived values survive two steps (after three steps every state has a path from state 0): stored >= -16360, candidates
// >= -18402.  The termination metrics are real after the three tail steps (>= -3060).  With the bias 0x4C00 = 19456 every field
// stays in [1054, 31708] (signed and unsigned compares agree), and alpha + (beta + edge), which carries the bias twice and is
// compared unsigned, stays below 61374 < 65536.
struct TdConst {
  uint32_t one, minus_one, minus_two, three; // run-time constants: keep the multiplies in IMAD form (FMA pipe)
};
TD_HD uint32_t vadd(uint32_t a, uint32_t b) { return TD_VADD2(a, b); }
TD_HD uint32_t vsub(uint32_t a, uint32_t b) { return TD_VSUB2(a, b); }
TD_HD uint32_t vamax(uint32_t a, uint32_t b, uint32_t c) { return TD_VIADDMAX_S(a, b, c); }  // max(a+b, c), signed fields
TD_HD uint32_t vamaxu(uint32_t a, uint32_t b, uint32_t c) { return TD_VIADDMAX_U(a, b, c); } // unsigned fields
TD_HD uint32_t vmax(uint32_t a, uint32_t b) { return TD_VMAXS2(a, b); }
TD_HD uint32_t vmin(uint32_t a, uint32_t b) { return TD_VMINS2(a, b); }
TD_HD uint32_t pk2(int lo, int hi) { return ((uint32_t)lo & 0xFFFFu) | ((uint32_t)hi << 16); }
TD_HD int      lo_s(uint32_t v) { return (int)(short)(v & 0xFFFFu); }
TD_HD int      hi_s(uint32_t v) { return (int)(short)(v >> 16); }
TD_HD uint32_t add32(const TdConst& c, uint32_t a, uint32_t b) { return a * c.one + b; }       // a + b on the FMA pipe
TD_HD uint32_t sub32(const TdConst& c, uint32_t a, uint32_t b) { return b * c.minus_one + a; } // a - b on the FMA pipe
// packed signed pair -> 32-form (hi * 65536 + lo): subtract 0x10000 when the low field is negative
TD_HD uint32_t to32(const TdConst& c, uint32_t p) { return (p & 0x8000u) * c.minus_two + p; }

struct St8 {
  uint32_t s[8];
};

// X32: 2 xa in 32-form; Pp: 2 p packed; G0p: 2 (xa + p) packed
TD_HD void alpha_step(const TdConst& c, St8& a, uint32_t X32, uint32_t Pp, uint32_t G0p)
{
  St8 n;
  n.s[0] = vamax(a.s[1], G0p, a.s[0]);
  n.s[4] = vamax(a.s[0], G0p, a.s[1]);
  n.s[1] = vamax(a.s[3], Pp, add32(c, a.s[2], X32));
  n.s[5] = vamax(a.s[2], Pp, add32(c, a.s[3], X32));
  n.s[2] = vamax(a.s[4], Pp, add32(c, a.s[5], X32));
  n.s[6] = vamax(a.s[5], Pp, add32(c, a.s[4], X32));
  n.s[3] = vamax(a.s[6], G0p, a.s[7]);
  n.s[7] = vamax(a.s[7], G0p, a.s[6]);
  a      = n;
}
TD_HD void norm8(const TdConst& c, St8& a)
{
  const uint32_t r = sub32(c, a.s[0], TD_BIASW); // 32-form of (state 0 - bias)
#pragma unroll
  for (int i = 0; i < 8; i++) a.s[i] = sub32(c, a.s[i], r);
}
// beta update + LLR numerators. b = beta_{k+1} in, beta_k out; al = alpha_k.  m1, m0 carry a double bias (compare unsigned).
TD_HD void beta_llr_step(const TdConst& c, St8& b, const St8& al, uint32_t X32, uint32_t P32, uint32_t G032, uint32_t& m1,
                                              uint32_t& m0)
{
  uint32_t c0[8], c1[8];
  c0[0] = b.s[0], c1[0] = add32(c, b.s[4], G032);
  c0[1] = b.s[4], c1[1] = add32(c, b.s[0], G032);
  c0[2] = add32(c, b.s[5], P32), c1[2] = add32(c, b.s[1], X32);
  c0[3] = add32(c, b.s[1], P32), c1[3] = add32(c, b.s[5], X32);
  c0[4] = add32(c, b.s[2], P32), c1[4] = add32(c, b.s[6], X32);
  c0[5] = add32(c, b.s[6], P32), c1[5] = add32(c, b.s[2], X32);
  c0[6] = b.s[7], c1[6] = add32(c, b.s[3], G032);
  c0[7] = b.s[3], c1[7] = add32(c, b.s[7], G032);
  m1    = add32(c, al.s[0], c1[0]);
  m0    = add32(c, al.s[0], c0[0]);
#pragma unroll
  for (int s = 1; s < 8; s++) {
    m1 = vamaxu(al.s[s], c1[s], m1);
    m0 = vamaxu(al.s[s], c0[s], m0);
  }
#pragma unroll
  for (int s = 0; s < 8; s++) b.s[s] = vmax(c0[s], c1[s]);
}
// extrinsic of both code blocks: clamp((3 (L - 2 xa)) >> 3, +-511) per field, L = m1 - m0, Xp = 2 xa packed.
// |3 v >> 3| reaches 512 at |v| >= 1366, so v is clamped to +-1365 first; then t = v + 1400 >= 0 per field, 3 t is a plain
// multiply, (3 t) >> 3 - 525 = floor(3 v / 8) (4200 = 8 * 525), and only the negative side can still land on -512.
TD_HD uint32_t ext_pair(const TdConst& c, uint32_t L, uint32_t Xp)
{
  uint32_t v = vsub(L, Xp);
  v          = vmax(vmin(v, 0x05550555u), 0xFAABFAABu);          // +-1365
  const uint32_t t = vadd(v, 0x05780578u) * c.three;             // 3 (v + 1400), fields < 8400: no carry between fields
  const uint32_t e = vsub((t >> 3) & 0x07FF07FFu, 0x020D020Du);  // - 525
  return vmax(e, 0xFE01FE01u);                                   // -511
}

// ---- CRC24 of the hard decisions ---------------------------------------------------------------------------------------
// Remainder of a 32-bit word v(x) modulo a CRC24 generator g: the low 24 bits are their own remainder, and the top byte b
// contributes b(x) x^24 mod g, one entry of a 256-entry table per generator.  A word that holds only nb < 32 bits (in its top
// bits) is shifted down first: leading zeros do not change a remainder.
#define TD_CRC24A 0x1864CFBu
#define TD_CRC24B 0x1800063u
struct Crc24Tab {
  uint32_t t[2][256]; // [0] CRC24A, [1] CRC24B: t[.][b] = b(x) x^24 mod g
};
constexpr Crc24Tab crc24_make_tab()
{
  Crc24Tab r{};
  for (int p = 0; p < 2; p++)
    for (uint32_t b = 0; b < 256; b++) {
      uint32_t v = b << 16; // b(x) x^16, then 8 more shifts with reduction
      for (int i = 0; i < 8; i++) {
        v <<= 1;
        if (v & 0x1000000u) v ^= (p ? TD_CRC24B : TD_CRC24A);
      }
      r.t[p][b] = v;
    }
  return r;
}
// top: the table entry of v's top byte (the caller reads it: __ldg on the device)
TD_HD uint32_t crc24_fold_word(uint32_t top, uint32_t v) { return top ^ (v & 0xFFFFFFu); }
// (r x^8 + byte) mod g for a remainder r < 2^24, top = table entry of r >> 16
TD_HD uint32_t crc24_fold_byte(uint32_t top, uint32_t r, uint32_t byte) { return top ^ ((r << 8) & 0xFFFFFFu) ^ byte; }
