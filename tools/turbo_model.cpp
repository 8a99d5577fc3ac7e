// turbo_model.cpp -- HOST model of the K8 turbo kernel (test infrastructure): the same packed-int16x2 / biased / dual-form arithmetic
// (ltesniffer_b200/csrc/turbo_arith.cuh, compiled for the host with bit-identical definitions of the SIMD intrinsics), the same
// window / sub-window / normalisation schedule and boundary hand-over as turbo_kernel, executed one "thread" after the other.
// tests/test_turbo_model.py compares its hard decisions after every iteration with the CPU oracle (oracle/lte_oracle.c, siso()),
// so the arithmetic design of the kernel is checked bit for bit without a GPU.  Not part of the product.
#include "../ltesniffer_b200/csrc/turbo_arith.cuh"
#include <cstring>
#include <vector>

#define TD_SUB 8
#define TD_NSUB (TD_WL / TD_SUB)

namespace {
struct Pair {
  uint32_t              K, NW;
  std::vector<uint32_t> sys, p1, p2, ext, bnd; // natural order (not window-transposed: layout is not what is modelled)
  std::vector<uint16_t> pi;
  uint32_t              tails[12];
  uint32_t              btail[2][8];
  std::vector<uint8_t>  bits[2];
};
void siso_pass(const TdConst& c, Pair& P, bool IL, bool first_iter)
{
  const uint32_t K = P.K, NW = P.NW;
  uint32_t*      A = P.bnd.data() + (size_t)(IL ? 2 : 0) * NW * 8;
  uint32_t*      B = A + (size_t)NW * 8;
  const std::vector<uint32_t>& par = IL ? P.p2 : P.p1;
  // stage every window first (the kernel's barrier): g, pos
  std::vector<uint32_t> gx((size_t)NW * TD_WL), gy((size_t)NW * TD_WL), pos((size_t)NW * TD_WL);
  std::vector<St8>      a0(NW), b0(NW);
  for (uint32_t w = 0; w < NW; w++) {
    const uint32_t len = K - w * TD_WL < TD_WL ? K - w * TD_WL : TD_WL;
    for (int s = 0; s < 8; s++) {
      a0[w].s[s] = (w == 0) ? (s ? pk2(TD_NINF + (int)TD_BIAS, TD_NINF + (int)TD_BIAS) : TD_BIASW) : A[(size_t)w * 8 + s];
      b0[w].s[s] = (w == NW - 1) ? P.btail[IL ? 1 : 0][s] : B[(size_t)w * 8 + s];
    }
    for (uint32_t j = 0; j < len; j++) {
      const uint32_t k = w * TD_WL + j, ps = IL ? P.pi[k] : k;
      const uint32_t sy = P.sys[ps], ap = (!IL && first_iter) ? 0u : P.ext[ps], p = par[k];
      const uint32_t xa = vadd(sy, ap);
      gx[(size_t)w * TD_WL + j] = vadd(xa, xa), gy[(size_t)w * TD_WL + j] = vadd(p, p), pos[(size_t)w * TD_WL + j] = ps;
    }
  }
  std::vector<uint32_t> newA((size_t)NW * 8), newB((size_t)NW * 8);
  memcpy(newA.data(), A, sizeof(uint32_t) * NW * 8), memcpy(newB.data(), B, sizeof(uint32_t) * NW * 8);
  for (uint32_t w = 0; w < NW; w++) {
    const uint32_t  len = K - w * TD_WL < TD_WL ? K - w * TD_WL : TD_WL;
    const uint32_t *X = &gx[(size_t)w * TD_WL], *Y = &gy[(size_t)w * TD_WL], *PS = &pos[(size_t)w * TD_WL];
    St8             a = a0[w], b = b0[w], ck[TD_NSUB];
    for (uint32_t sw = 0; sw < TD_NSUB; sw++) {
      ck[sw] = a;
      for (uint32_t jj = 0; jj < TD_SUB; jj++) {
        const uint32_t j = sw * TD_SUB + jj;
        if (j < len) {
          alpha_step(c, a, to32(c, X[j]), Y[j], vadd(X[j], Y[j]));
          if ((jj & 1u) == 1u) norm8(c, a);
        }
      }
    }
    norm8(c, a);
    if (w + 1 < NW)
      for (int s = 0; s < 8; s++) newA[(size_t)(w + 1) * 8 + s] = a.s[s];
    for (int sw = TD_NSUB - 1; sw >= 0; sw--) {
      const uint32_t j0 = (uint32_t)sw * TD_SUB;
      if (j0 >= len) continue;
      St8 af = ck[sw], al[TD_SUB];
      for (uint32_t jj = 0; jj < TD_SUB; jj++) {
        const uint32_t j = j0 + jj;
        if (j < len) {
          al[jj] = af;
          if (jj + 1 < TD_SUB) {
            alpha_step(c, af, to32(c, X[j]), Y[j], vadd(X[j], Y[j]));
            if ((jj & 1u) == 1u) norm8(c, af);
          }
        }
      }
      for (int jj = TD_SUB - 1; jj >= 0; jj--) {
        const uint32_t j = j0 + (uint32_t)jj;
        if (j < len) {
          const uint32_t X32 = to32(c, X[j]), P32 = to32(c, Y[j]);
          uint32_t       m1, m0;
          beta_llr_step(c, b, al[jj], X32, P32, add32(c, X32, P32), m1, m0);
          if ((jj & 1) == 0) norm8(c, b);
          const uint32_t L = vsub(m1, m0);
          if (IL) {
            P.bits[0][PS[j]] = (int)(L << 16) > 0;
            P.bits[1][PS[j]] = (int)L >= 0x10000;
          }
          P.ext[PS[j]] = ext_pair(c, L, X[j]);
        }
      }
    }
    norm8(c, b);
    if (w > 0)
      for (int s = 0; s < 8; s++) newB[(size_t)(w - 1) * 8 + s] = b.s[s];
  }
  memcpy(A, newA.data(), sizeof(uint32_t) * NW * 8), memcpy(B, newB.data(), sizeof(uint32_t) * NW * 8);
}
} // namespace

extern "C" int turbo_model_decode(const int16_t* d0, const int16_t* d1, uint32_t K, uint32_t f1, uint32_t f2, uint32_t iters, uint8_t* bits0, uint8_t* bits1)
{
  const TdConst c{1u, 0xFFFFFFFFu, 0xFFFFFFFEu, 3u};
  const uint32_t D = K + 4;
  Pair           P;
  P.K = K, P.NW = (K + TD_WL - 1) / TD_WL;
  P.sys.resize(K), P.p1.resize(K), P.p2.resize(K), P.ext.assign(K, 0), P.bnd.assign((size_t)4 * P.NW * 8, TD_BIASW), P.pi.resize(K);
  P.bits[0].assign(K, 0), P.bits[1].assign(K, 0);
  for (uint64_t i = 0; i < K; i++) {
    P.sys[i] = pk2(d0[i], d1[i]), P.p1[i] = pk2(d0[D + i], d1[D + i]), P.p2[i] = pk2(d0[2 * D + i], d1[2 * D + i]);
    P.pi[i]  = (uint16_t)((f1 * i + f2 * i * i) % K);
  }
  // termination metrics exactly as the kernel's thread 0 computes them (int32, both constituent codes, both code blocks)
  for (uint32_t s = 0; s < 3; s++)
    for (uint32_t i = 0; i < 4; i++) P.tails[s * 4 + i] = pk2(d0[s * D + K + i], d1[s * D + K + i]);
  static const uint8_t NEXT[8][2] = {{0, 4}, {4, 0}, {5, 1}, {1, 5}, {2, 6}, {6, 2}, {7, 3}, {3, 7}};
  static const uint8_t PAR[8][2]  = {{0, 1}, {0, 1}, {1, 0}, {1, 0}, {1, 0}, {1, 0}, {0, 1}, {0, 1}};
  for (int dec = 0; dec < 2; dec++) {
    const uint32_t* T = P.tails;
    uint32_t        tx[3], tz[3];
    if (dec == 0)
      tx[0] = T[0], tx[1] = T[8], tx[2] = T[5], tz[0] = T[4], tz[1] = T[1], tz[2] = T[9];
    else
      tx[0] = T[2], tx[1] = T[10], tx[2] = T[7], tz[0] = T[6], tz[1] = T[3], tz[2] = T[11];
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
        memcpy(bt, bn, sizeof(bt));
      }
      const int ref = bt[0];
      for (int s = 0; s < 8; s++) {
        const int      v = bt[s] - ref + (int)TD_BIAS;
        const uint32_t o = P.btail[dec][s];
        P.btail[dec][s]  = h ? ((o & 0xFFFFu) | ((uint32_t)v << 16)) : ((uint32_t)v & 0xFFFFu);
      }
    }
  }
  for (uint32_t it = 0; it < iters; it++) {
    siso_pass(c, P, false, it == 0);
    siso_pass(c, P, true, false);
  }
  memcpy(bits0, P.bits[0].data(), K), memcpy(bits1, P.bits[1].data(), K);
  return 0;
}

// The CRC24 byte tables of turbo_arith.cuh and the kernel's use of them: remainder of the top nb bits of a decision word
// (which: 0 CRC24A, 1 CRC24B), and one byte folded into a remainder as tb_crc_kernel does it.
static constexpr Crc24Tab crc24_tab_h = crc24_make_tab();
extern "C" void turbo_model_crc24_table(uint32_t which, uint32_t* out) { memcpy(out, crc24_tab_h.t[which & 1u], sizeof(crc24_tab_h.t[0])); }
extern "C" uint32_t turbo_model_crc24_word(uint32_t which, uint32_t word, uint32_t nb)
{
  const uint32_t v = word >> (32u - nb);
  return crc24_fold_word(crc24_tab_h.t[which & 1u][v >> 24], v);
}
extern "C" uint32_t turbo_model_crc24_byte(uint32_t which, uint32_t r, uint32_t byte)
{
  return crc24_fold_byte(crc24_tab_h.t[which & 1u][r >> 16], r, byte);
}
