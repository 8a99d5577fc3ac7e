// lte_host.cpp -- see lte_host.hpp.  Product code (host side, C++17).
#include "lte_host.hpp"
#include "../../include/ltephy_b200.h"
#include "../../include/lte_tables.h"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace ltehost {

uint32_t fft_size(uint32_t n)
{
  return n <= 6 ? 128 : n <= 15 ? 256 : n <= 25 ? 512 : n <= 50 ? 1024 : 2048;
}
uint32_t cp_len(uint32_t fft, uint32_t s) { return (s == 0 ? 160u : 144u) * fft / 2048u; }

// ------------------------------------------------------------------------------------------------
// Gold sequences.  x1/x2 are length-31 LFSRs; state kept as a 31-bit word, bit i = x(n+i).
namespace {
inline uint32_t step_x1(uint32_t s) { return (s >> 1) | ((((s >> 3) ^ s) & 1u) << 30); }
inline uint32_t step_x2(uint32_t s) { return (s >> 1) | ((((s >> 3) ^ (s >> 2) ^ (s >> 1) ^ s) & 1u) << 30); }
std::vector<uint32_t> lfsr_words(uint32_t init, bool is_x2, uint32_t nbits)
{
  uint32_t s = init & 0x7FFFFFFFu;
  for (int i = 0; i < 1600; i++) s = is_x2 ? step_x2(s) : step_x1(s);
  std::vector<uint32_t> w((nbits + 31) / 32, 0u);
  for (uint32_t i = 0; i < nbits; i++) {
    w[i >> 5] |= (s & 1u) << (i & 31);
    s = is_x2 ? step_x2(s) : step_x1(s);
  }
  return w;
}
} // namespace

std::vector<uint32_t> gold_words(uint32_t c_init, uint32_t nbits)
{
  auto a = lfsr_words(1u, false, nbits), b = lfsr_words(c_init, true, nbits);
  for (size_t i = 0; i < a.size(); i++) a[i] ^= b[i];
  return a;
}
GoldBasis gold_basis(uint32_t nbits)
{
  GoldBasis g;
  g.nwords = (nbits + 31) / 32;
  g.x1     = lfsr_words(1u, false, g.nwords * 32);
  g.basis.resize(31u * g.nwords);
  for (uint32_t b = 0; b < 31; b++) {
    auto w = lfsr_words(1u << b, true, g.nwords * 32);
    std::copy(w.begin(), w.end(), g.basis.begin() + (size_t)b * g.nwords);
  }
  return g;
}

// ------------------------------------------------------------------------------------------------
uint32_t crc_bits(uint32_t poly, uint32_t order, const uint8_t* bits, uint32_t n)
{
  uint32_t r = 0, top = 1u << order;
  for (uint32_t i = 0; i < n + order; i++) {
    r = (r << 1) | (i < n ? (bits[i] & 1u) : 0u);
    if (r & top) r ^= poly;
  }
  return r & (top - 1);
}
std::vector<uint32_t> crc24_xpow8(uint32_t poly, uint32_t n)
{
  std::vector<uint32_t> t(n);
  uint32_t              v = 1;
  for (uint32_t i = 0; i < n; i++) {
    t[i] = v;
    for (int b = 0; b < 8; b++) {
      v <<= 1;
      if (v & 0x1000000u) v ^= poly;
    }
  }
  return t;
}

// ------------------------------------------------------------------------------------------------
uint32_t crs_offset(const Cell& c, uint32_t port, uint32_t s)
{
  uint32_t v = port == 0 ? (s == 0 ? 0u : 3u) : (s == 0 ? 3u : 0u);
  return (v + c.cell_id % 6) % 6;
}
std::vector<float> crs_table(const Cell& c)
{
  const uint32_t     np = 2 * c.nof_prb;
  static const int   PL[4] = {0, 4, 7, 11};
  std::vector<float> t((size_t)10 * 2 * 4 * np * 2);
  const float        a = (float)M_SQRT1_2;
  for (uint32_t sf = 0; sf < 10; sf++)
    for (uint32_t p = 0; p < 2; p++)
      for (uint32_t li = 0; li < 4; li++) {
        uint32_t ns = 2 * sf + PL[li] / 7, l = PL[li] % 7;
        uint32_t ci = 1024u * (7u * (ns + 1) + l + 1) * (2u * c.cell_id + 1) + 2u * c.cell_id + 1u;
        auto     w  = gold_words(ci, 4 * 110);
        float*   o  = &t[(((size_t)sf * 2 + p) * 4 + li) * np * 2];
        for (uint32_t m = 0; m < np; m++) {
          uint32_t mp  = m + 110 - c.nof_prb;
          uint32_t b0  = (w[(2 * mp) >> 5] >> ((2 * mp) & 31)) & 1u, b1 = (w[(2 * mp + 1) >> 5] >> ((2 * mp + 1) & 31)) & 1u;
          o[2 * m]     = b0 ? -a : a;
          o[2 * m + 1] = b1 ? -a : a;
        }
      }
  return t;
}

// ------------------------------------------------------------------------------------------------
// Control region: REGs, PCFICH/PHICH reservation, PDCCH interleaver (36.211 6.2.4, 6.7.4, 6.9.3, 6.8.5)
namespace {
const uint8_t kConvPerm[32] = {1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31,
                               0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30};
struct Reg {
  uint16_t k0;
  uint8_t  l, kind;
  uint16_t k[4];
};
} // namespace

bool build_ctrl_map(const Cell& c, CtrlMap& out)
{
  if (c.nof_prb <= 10 || c.nof_prb > 110 || c.nof_ports < 1 || c.nof_ports > 2 || c.phich_ng > 3 || c.phich_ext > 1) return false;
  const uint32_t   nsc = 12 * c.nof_prb, v3 = c.cell_id % 3;
  std::vector<Reg> regs;
  uint32_t         sym_base[4] = {0, 0, 0, 0};
  for (uint32_t l = 0; l < 3; l++) {
    sym_base[l]      = (uint32_t)regs.size();
    const uint32_t w = l == 0 ? 6 : 4;
    for (uint32_t k0 = 0; k0 < nsc; k0 += w) {
      Reg r{};
      r.k0 = (uint16_t)k0, r.l = (uint8_t)l;
      uint32_t q = 0;
      for (uint32_t k = k0; k < k0 + w; k++)
        if (l != 0 || k % 3 != v3) r.k[q++] = (uint16_t)k;
      regs.push_back(r);
    }
  }
  sym_base[3] = (uint32_t)regs.size();
  auto reg_at = [&](uint32_t l, uint32_t k0) -> int {
    const uint32_t w = l == 0 ? 6 : 4;
    return k0 % w ? -1 : (int)(sym_base[l] + k0 / w);
  };
  // PCFICH
  const uint32_t kbar = 6 * (c.cell_id % (2 * c.nof_prb));
  for (uint32_t i = 0; i < 4; i++) {
    int j = reg_at(0, (kbar + (i * c.nof_prb / 2) * 6) % nsc);
    if (j < 0) return false;
    regs[j].kind = 1;
    for (int q = 0; q < 4; q++) out.pcfich_idx[4 * i + q] = regs[j].k[q];
  }
  // PHICH, normal duration (36.211 6.9): N_group = ceil(Ng N_RB / 8), Ng = 1/6, 1/2, 1, 2 from the MIB (srsran_cell_t.phich_resources; the
  // reference's file mode presets 1/6, src/src/LTESniffer_Core.cc:242-247, its live mode takes the MIB's value, :196, :389)
  {
    std::vector<uint32_t> free0;
    for (uint32_t j = sym_base[0]; j < sym_base[1]; j++)
      if (regs[j].kind == 0) free0.push_back(j);
    static const uint32_t ng_x6[4] = {1, 3, 6, 12};
    const uint32_t        n0 = (uint32_t)free0.size(), ngroups = (ng_x6[c.phich_ng] * c.nof_prb + 47) / 48;
    if (3 * ngroups > n0) return false;
    if (!c.phich_ext) {
      for (uint32_t m = 0; m < ngroups; m++)
        for (uint32_t i = 0; i < 3; i++) regs[free0[(c.cell_id + m + i * n0 / 3) % n0]].kind = 2;
    } else { // extended duration, ordinary FDD subframes (36.211 6.9.3): quadruplet i of a group goes to symbol l' = i, to the REG numbered
             // (floor(N_id n_l' / n_0) + m' + floor(i n_l' / 3)) mod n_l' among the n_l' REGs of that symbol that do not carry the PCFICH
      for (uint32_t m = 0; m < ngroups; m++)
        for (uint32_t i = 0; i < 3; i++) {
          const uint32_t nl = i == 0 ? n0 : sym_base[i + 1] - sym_base[i];
          const uint32_t ni = (uint32_t)(((uint64_t)c.cell_id * nl / n0 + m + i * nl / 3) % nl);
          regs[i == 0 ? free0[ni] : sym_base[i] + ni].kind = 2;
        }
    }
  }
  for (uint32_t cfi = 1; cfi <= 3; cfi++) {
    std::vector<uint32_t> F;
    for (uint32_t k = 0; k < nsc; k++)
      for (uint32_t l = 0; l < cfi; l++) {
        int j = reg_at(l, k);
        if (j >= 0 && regs[j].kind == 0) F.push_back((uint32_t)j);
      }
    const uint32_t M     = (uint32_t)F.size();
    out.nof_cce[cfi - 1] = M / 9;
    std::vector<uint32_t> carrier(M);
    const uint32_t        nrows = (M - 1) / 32 + 1, ndummy = 32 * nrows - M;
    uint32_t              kk = 0;
    for (uint32_t col = 0; col < 32; col++)
      for (uint32_t row = 0; row < nrows; row++) {
        uint32_t idx = row * 32 + kConvPerm[col];
        if (idx < ndummy) continue;
        carrier[idx - ndummy] = F[(kk + M - c.cell_id % M) % M];
        kk++;
      }
    auto& v = out.pdcch_idx[cfi - 1];
    v.resize((size_t)out.nof_cce[cfi - 1] * 9 * 4);
    for (uint32_t q = 0; q < out.nof_cce[cfi - 1] * 9; q++)
      for (int i = 0; i < 4; i++) v[4 * q + i] = (uint16_t)(regs[carrier[q]].l * nsc + regs[carrier[q]].k[i]);
  }
  return true;
}

// ------------------------------------------------------------------------------------------------
namespace {
uint32_t clog2(uint32_t v)
{
  uint32_t n = 0;
  while ((1u << n) < v) n++;
  return n;
}
uint32_t rbg(uint32_t n) { return n <= 10 ? 1 : n <= 26 ? 2 : n <= 63 ? 3 : 4; }
bool     ambiguous(uint32_t n)
{
  for (uint32_t a : {12u, 14u, 16u, 20u, 24u, 26u, 32u, 40u, 44u, 56u})
    if (a == n) return true;
  return false;
}
uint32_t gap1(uint32_t n) { return n <= 10 ? (n + 1) / 2 : n == 11 ? 4 : n <= 19 ? 8 : n <= 26 ? 12 : n <= 44 ? 18 : n <= 63 ? 27 : n <= 79 ? 32 : 48; }
} // namespace

uint32_t dci_sizeof(const Cell& c, Format f)
{
  const uint32_t N = c.nof_prb, P = rbg(N), hdr = N > 10, bm = (N + P - 1) / P, riv = clog2(N * (N + 1) / 2);
  uint32_t       base = std::max(1 + 1 + riv + 5 + 1 + 2 + 3 + 1, 1 + 1 + riv + 5 + 3 + 1 + 2 + 2);
  while (ambiguous(base)) base++;
  const uint32_t tpmi = c.nof_ports == 2 ? 2 : c.nof_ports == 4 ? 4 : 0;
  uint32_t       n    = 0;
  switch (f) {
    case F0:
    case F1A: return base;
    case F1:
      n = hdr + bm + 13;
      if (n == base) n++;
      while (ambiguous(n) || n == base) n++;
      return n;
    case F1B:
    case F1D: n = 1 + riv + 13 + tpmi + 1; break;
    case F1C: {
      uint32_t g = gap1(N), nv = 2 * std::min(g, N - g) / (N < 50 ? 2 : 4);
      return (N >= 50 ? 1 : 0) + clog2(nv * (nv + 1) / 2) + 5;
    }
    case F2: n = hdr + bm + 22 + (c.nof_ports == 2 ? 3 : c.nof_ports == 4 ? 6 : 0); break;
    case F2A: n = hdr + bm + 22 + (c.nof_ports == 4 ? 2 : 0); break;
    case F2B: n = hdr + bm + 22; break;
    default: return 0;
  }
  while (ambiguous(n)) n++;
  return n;
}
SizeTable dci_size_table(const Cell& c)
{
  SizeTable t;
  for (int f = 0; f < NOF_FORMATS; f++) {
    uint32_t s  = dci_sizeof(c, (Format)f);
    auto     it = std::find(t.sizes.begin(), t.sizes.end(), s);
    if (it == t.sizes.end()) {
      t.index_of[f] = (uint32_t)t.sizes.size();
      t.sizes.push_back(s);
    } else
      t.index_of[f] = (uint32_t)(it - t.sizes.begin());
  }
  return t;
}
std::vector<uint16_t> conv_rm_table(uint32_t K)
{
  std::vector<uint16_t> t;
  const uint32_t        R = (K + 31) / 32, ND = 32 * R - K;
  for (uint32_t s = 0; s < 3; s++)
    for (uint32_t k = 0; k < 32 * R; k++) {
      uint32_t y = (k % R) * 32 + kConvPerm[k / R];
      if (y >= ND) t.push_back((uint16_t)(s * K + y - ND));
    }
  return t;
}
std::vector<Location> all_locations(uint32_t nof_cce)
{
  std::vector<Location> v;
  if (!nof_cce) return v;
  const uint32_t lim = std::min<uint32_t>(nof_cce, 84);
  for (int l = 3; l >= 0; l--) {
    const uint32_t L = 1u << l;
    for (uint32_t i = 0; i < lim / L; i++)
      if (v.size() < 160 && nof_cce / L) v.push_back({(uint16_t)(L * (i % (nof_cce / L))), (uint8_t)l});
  }
  return v;
}

// ------------------------------------------------------------------------------------------------
bool cb_segmentation(uint32_t tbs, Segm& s)
{
  s     = Segm{};
  s.tbs = tbs;
  uint32_t B = tbs + 24, Bp = B;
  s.C = 1;
  if (B > 6144) {
    s.C = (B + 6119) / 6120;
    Bp  = B + 24 * s.C;
  }
  int ip = lte_qpp_index_ge((Bp + s.C - 1) / s.C);
  if (ip < 0) return false;
  s.Kp = lte_qpp_K((uint32_t)ip);
  s.Cp = 1;
  if (s.C > 1) {
    s.Km = ip > 0 ? lte_qpp_K((uint32_t)ip - 1) : 0;
    s.Cm = (s.C * s.Kp - Bp) / (s.Kp - s.Km);
    s.Cp = s.C - s.Cm;
  }
  s.F = s.Cp * s.Kp + s.Cm * s.Km - Bp;
  return true;
}
bool uci_layout(uint32_t L_prb, uint32_t qm, uint32_t tbs, uint32_t nof_ack, uint32_t ri_len, uint32_t cqi_len, uint32_t I_ack, uint32_t I_ri, uint32_t I_cqi,
                UciLayout& out)
{
  // betaOffset tables, 36.213 8.6.3 (-1: reserved index)
  static const float B_ACK[16] = {2.000f, 2.500f, 3.125f, 4.000f, 5.000f, 6.250f, 8.000f, 10.000f, 12.625f, 15.875f, 20.000f, 31.000f, 50.000f, 80.000f, 126.000f, -1.0f};
  static const float B_RI[16]  = {1.250f, 1.625f, 2.000f, 2.500f, 3.125f, 4.000f, 5.000f, 6.250f, 8.000f, 10.000f, 12.625f, 15.875f, 20.000f, -1.0f, -1.0f, -1.0f};
  static const float B_CQI[16] = {-1.0f, -1.0f, 1.125f, 1.250f, 1.375f, 1.625f, 1.750f, 2.000f, 2.250f, 2.500f, 2.875f, 3.125f, 3.500f, 4.000f, 5.000f, 6.250f};
  out = UciLayout{};
  const uint32_t M = 12 * L_prb, nsymb = 12; // no SRS: 12 data SC-FDMA symbols (ul_sf.shortened = false, src/src/DL_Sniffer_PDSCH.cc:655)
  Segm           sg;
  if (!cb_segmentation(tbs, sg)) return false;
  const uint32_t Ksum = sg.Cm * sg.Km + sg.Cp * sg.Kp;
  if (!Ksum) return false;
  // Q' = min(ceil(O M_sc N_symb beta / sum K_r), 4 M_sc), in float like srsRAN's Q_prime_ri_ack / Q_prime_cqi
  auto qprime = [&](uint32_t O, float beta) { return (uint32_t)ceilf((float)O * (float)M * (float)nsymb * beta / (float)Ksum); };
  if (ri_len) {
    const float b = B_RI[I_ri & 15];
    if (b < 0) return false;
    out.Qp_ri = std::min(qprime(ri_len, b), 4 * M);
  }
  if (nof_ack) {
    const float b = B_ACK[I_ack & 15];
    if (b < 0) return false;
    out.Qp_ack = std::min(qprime(nof_ack, b), 4 * M);
  }
  if (cqi_len) {
    const float b = B_CQI[I_cqi & 15];
    if (b < 0) return false;
    out.Qp_cqi = std::min(qprime(cqi_len + (cqi_len <= 11 ? 0u : 8u), b), M * nsymb - out.Qp_ri); // CRC-8 from 12 bits on (36.212 5.2.2.6.4)
  }
  out.G = (M * nsymb - out.Qp_cqi - out.Qp_ri) * qm;
  return true;
}
bool qpp_params(uint32_t K, uint32_t& f1, uint32_t& f2)
{
  int i = lte_qpp_index_ge(K);
  if (i < 0 || lte_qpp_K((uint32_t)i) != K) return false;
  f1 = lte_qpp_f1[i], f2 = lte_qpp_f2[i];
  return true;
}
uint32_t rm_turbo_E(uint32_t G, uint32_t C, uint32_t r, uint32_t Qm, uint32_t NL)
{
  const uint32_t Gp = G / (NL * Qm), gamma = Gp % C;
  return r + gamma + 1 <= C ? NL * Qm * (Gp / C) : NL * Qm * ((Gp + C - 1) / C);
}
RmTurboTable rm_turbo_table(uint32_t K, uint32_t F, uint32_t rv)
{
  static const uint8_t P[32] = {0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30,
                                1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31};
  const uint32_t D = K + 4, R = (D + 31) / 32, Kpi = 32 * R, ND = Kpi - D, Kw = 3 * Kpi;
  std::vector<uint32_t> w(Kw, 0xFFFFFFFFu); // circular buffer position -> stream position
  for (uint32_t k = 0; k < Kpi; k++) {
    uint32_t y = P[k / R] + 32 * (k % R), y2 = (y + 1) % Kpi;
    if (y >= ND) {
      w[k]           = y - ND;
      w[Kpi + 2 * k] = D + y - ND;
    }
    if (y2 >= ND) w[Kpi + 2 * k + 1] = 2 * D + y2 - ND;
  }
  RmTurboTable t;
  t.order.reserve(Kw);
  const uint32_t k0 = R * (2 * ((Kw + 8 * R - 1) / (8 * R)) * rv + 2);
  for (uint32_t j = 0; j < Kw; j++) {
    uint32_t s = w[(k0 + j) % Kw];
    if (s == 0xFFFFFFFFu) continue;
    if (s / D < 2 && s % D < F) continue; // filler bits are <NULL> in d0/d1
    t.order.push_back(s);
  }
  t.nn = (uint32_t)t.order.size();
  return t;
}
uint32_t rm_turbo_word(uint32_t K, uint32_t s)
{
  const uint32_t D = K + 4, NW = (K + 31) / 32, st = s / D, i = s % D;
  return i < K ? st * 32 * NW + (i & 31u) * NW + (i >> 5) : 3 * 32 * NW + st * 4 + (i - K);
}
RmTurboInverse rm_turbo_inverse(uint32_t K, uint32_t F)
{
  const uint32_t D = K + 4, NW = (K + 31) / 32;
  RmTurboInverse r;
  r.inv.assign((size_t)96 * NW + 16, (uint16_t)LTEPHY_RM_NONE);
  for (uint32_t st = 0; st < 2; st++)
    for (uint32_t i = 0; i < F; i++) r.inv[rm_turbo_word(K, st * D + i)] = (uint16_t)LTEPHY_RM_FILLER;
  for (uint32_t rv = 0; rv < 4; rv++) {
    const RmTurboTable t = rm_turbo_table(K, F, rv);
    if (rv == 0) {
      r.nn = t.nn;
      for (uint32_t j = 0; j < t.nn; j++) r.inv[rm_turbo_word(K, t.order[j])] = (uint16_t)j;
    }
    r.rot[rv] = t.nn ? r.inv[rm_turbo_word(K, t.order[0])] : 0;
  }
  return r;
}

// ------------------------------------------------------------------------------------------------
uint32_t pdsch_re_in_prb(const Cell& c, uint32_t sf_idx, uint32_t cfi, uint32_t l, uint32_t prb, uint16_t* kk)
{
  if (l < (c.nof_prb <= 10 ? cfi + 1 : cfi)) return 0;
  const uint32_t lo = 6 * c.nof_prb - 36, hi = lo + 72;
  const bool     crs = (l % 7 == 0) || (l % 7 == 4);
  uint32_t       n = 0;
  for (uint32_t k = 12 * prb; k < 12 * prb + 12; k++) {
    if (crs && (c.nof_ports == 1 ? k % 6 == crs_offset(c, 0, l % 7) : k % 3 == c.cell_id % 3)) continue;
    if (k >= lo && k < hi) {
      if ((sf_idx == 0 || sf_idx == 5) && (l == 5 || l == 6)) continue;
      if (sf_idx == 0 && l >= 7 && l <= 10) continue;
    }
    kk[n++] = (uint16_t)k;
  }
  return n;
}

} // namespace ltehost
