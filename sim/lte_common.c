/*
 * lte_common.c -- see lte_common.h.  Plain C99 restatement of the 3GPP procedures that the
 * reference reaches through srsRAN.  TEST INFRASTRUCTURE (synthetic eNB + oracle only).
 */
#include "lte_common.h"
#include "../include/lte_tables.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ numerology */
uint32_t lte_fft_size(uint32_t nof_prb)
{
  if (nof_prb <= 6) return 128;
  if (nof_prb <= 15) return 256;
  if (nof_prb <= 25) return 512;
  if (nof_prb <= 50) return 1024;
  return 2048;
}
uint32_t lte_cp_len(uint32_t fft, uint32_t symbol_in_slot) { return (symbol_in_slot == 0 ? 160u : 144u) * fft / 2048u; }
uint32_t lte_sf_len(uint32_t nof_prb) { return 15u * lte_fft_size(nof_prb); }
uint32_t lte_cell_fft(const lte_cell_t* c) { return c->symbol_sz ? c->symbol_sz : lte_fft_size(c->nof_prb); }

/* ------------------------------------------------------------------ Gold sequence, 36.211 7.2 */
void lte_gold_bits(uint32_t c_init, uint8_t* c, uint32_t len)
{
  const uint32_t Nc = 1600;
  uint32_t       n  = len + Nc + 31;
  uint8_t*       x1 = (uint8_t*)calloc(n, 1);
  uint8_t*       x2 = (uint8_t*)calloc(n, 1);
  x1[0]             = 1;
  for (uint32_t i = 0; i < 31; i++) x2[i] = (c_init >> i) & 1;
  for (uint32_t i = 0; i + 31 < n; i++) {
    x1[i + 31] = x1[i + 3] ^ x1[i];
    x2[i + 31] = x2[i + 3] ^ x2[i + 2] ^ x2[i + 1] ^ x2[i];
  }
  for (uint32_t i = 0; i < len; i++) c[i] = x1[i + Nc] ^ x2[i + Nc];
  free(x1);
  free(x2);
}

/* ------------------------------------------------------------------ CRC (restates srsran_crc_checksum, falcon_pdcch.c:401) */
uint32_t lte_crc(uint32_t poly, uint32_t order, const uint8_t* bits, uint32_t n)
{
  uint32_t reg = 0, top = 1u << order;
  for (uint32_t i = 0; i < n + order; i++) {
    reg = (reg << 1) | (i < n ? (bits[i] & 1u) : 0u);
    if (reg & top) reg ^= poly;
  }
  return reg & (top - 1);
}
void lte_bits_pack(const uint8_t* bits, uint32_t nbits, uint8_t* bytes)
{
  for (uint32_t i = 0; i < (nbits + 7) / 8; i++) bytes[i] = 0;
  for (uint32_t i = 0; i < nbits; i++) bytes[i / 8] |= (uint8_t)((bits[i] & 1) << (7 - (i % 8)));
}
void lte_bits_unpack(const uint8_t* bytes, uint32_t nbits, uint8_t* bits)
{
  for (uint32_t i = 0; i < nbits; i++) bits[i] = (bytes[i / 8] >> (7 - (i % 8))) & 1;
}

/* ------------------------------------------------------------------ CRS, 36.211 6.10.1 */
uint32_t lte_crs_offset(const lte_cell_t* c, uint32_t port, uint32_t l_in_slot)
{
  uint32_t v = (port == 0) ? (l_in_slot == 0 ? 0 : 3) : (l_in_slot == 0 ? 3 : 0);
  return (v + c->cell_id % 6) % 6;
}
uint32_t lte_crs(const lte_cell_t* c, uint32_t port, uint32_t ns, uint32_t l, cf_t* pilots)
{
  uint8_t  seq[2 * 2 * LTE_MAX_PRB];
  uint32_t c_init = 1024u * (7u * (ns + 1) + l + 1) * (2u * c->cell_id + 1) + 2u * c->cell_id + 1u;
  lte_gold_bits(c_init, seq, 2 * 2 * LTE_MAX_PRB);
  const float a = (float)M_SQRT1_2;
  for (uint32_t m = 0; m < 2 * c->nof_prb; m++) {
    uint32_t mp  = m + LTE_MAX_PRB - c->nof_prb;
    pilots[m].re = seq[2 * mp] ? -a : a;
    pilots[m].im = seq[2 * mp + 1] ? -a : a;
  }
  return lte_crs_offset(c, port, l);
}

/* ------------------------------------------------------------------ control-region REGs */
static const uint8_t CONV_PERM[32] = {1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31,
                                      0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30};

int lte_regs_init(lte_regs_t* r, const lte_cell_t* cell)
{
  memset(r, 0, sizeof(*r));
  r->cell = *cell;
  if (cell->nof_prb <= 10 || cell->nof_prb > LTE_MAX_PRB || cell->nof_ports < 1 || cell->nof_ports > 2 || cell->phich_ng > 3 || cell->phich_ext > 1) return -1;
  uint32_t n = 0, vs3 = cell->cell_id % 3;
  for (uint32_t l = 0; l < 3; l++) {
    uint32_t cnt = 0;
    for (uint32_t prb = 0; prb < cell->nof_prb; prb++) {
      uint32_t nreg = (l == 0) ? 2 : 3, w = 12 / nreg;
      for (uint32_t i = 0; i < nreg; i++) {
        lte_reg_t* g = &r->regs[n++];
        g->k0        = (uint16_t)(12 * prb + i * w);
        g->l         = (uint8_t)l;
        uint32_t q   = 0;
        for (uint32_t k = g->k0; k < g->k0 + w; k++)
          if (l != 0 || (k % 3) != vs3) g->k[q++] = (uint16_t)k;
        cnt++;
      }
    }
    r->nof_regs_sym[l] = cnt;
  }
  r->nof_regs_total = n;
  /* PCFICH, 36.211 6.7.4 */
  uint32_t nsc  = 12 * cell->nof_prb;
  uint32_t kbar = 6 * (cell->cell_id % (2 * cell->nof_prb));
  for (uint32_t i = 0; i < 4; i++) {
    uint32_t k = (kbar + (i * cell->nof_prb / 2) * 6) % nsc;
    uint32_t found = 0;
    for (uint32_t j = 0; j < r->nof_regs_sym[0]; j++)
      if (r->regs[j].k0 == k) {
        r->regs[j].kind  = 1;
        r->pcfich_reg[i] = j;
        found            = 1;
      }
    if (!found) return -2;
  }
  /* PHICH, normal duration, 36.211 6.9: N_group = ceil(Ng N_RB / 8), Ng = 1/6 (the reference's file mode, LTESniffer_Core.cc:242-247), 1/2, 1 or 2 */
  static const uint32_t ng_x6[4] = {1, 3, 6, 12};
  r->nof_phich_groups = (ng_x6[cell->phich_ng] * cell->nof_prb + 47) / 48;
  uint32_t n0 = 0, idx0[2 * LTE_MAX_PRB];
  for (uint32_t j = 0; j < r->nof_regs_sym[0]; j++)
    if (r->regs[j].kind != 1) idx0[n0++] = j;
  if (3 * r->nof_phich_groups > n0 || r->nof_phich_groups > 28) return -2;
  for (uint32_t m = 0; m < r->nof_phich_groups; m++)
    for (uint32_t i = 0; i < 3; i++) {
      uint32_t reg;
      if (!cell->phich_ext || i == 0) { /* symbol 0: the REGs that do not carry the PCFICH, numbered upwards in frequency */
        reg = idx0[(cell->cell_id + m + (i * n0) / 3) % n0];
      } else { /* extended duration (36.211 6.9.3, FDD, no MBSFN): quadruplet i in symbol i, every REG of that symbol counts */
        uint32_t first = r->nof_regs_sym[0] + (i == 2 ? r->nof_regs_sym[1] : 0), nl = r->nof_regs_sym[i];
        reg            = first + (uint32_t)(((uint64_t)cell->cell_id * nl / n0 + m + (i * nl) / 3) % nl);
      }
      r->regs[reg].kind       = 2;
      r->phich_reg[3 * m + i] = reg;
    }
  /* PDCCH REG order and interleaver, 36.211 6.8.5 */
  for (uint32_t cfi = 1; cfi <= 3; cfi++) {
    static uint16_t F[3 * 3 * LTE_MAX_PRB];
    uint32_t        M = 0;
    /* k-first-then-l ordering: walk subcarriers, for each k' take symbols in order */
    for (uint32_t k = 0; k < nsc; k++)
      for (uint32_t l = 0; l < cfi; l++) {
        /* find REG in symbol l starting at k */
        uint32_t base = 0;
        for (uint32_t ll = 0; ll < l; ll++) base += r->nof_regs_sym[ll];
        uint32_t nreg = (l == 0) ? 2 : 3, w = 12 / nreg;
        if (k % w) continue;
        uint32_t j = base + (k / 12) * nreg + (k % 12) / w;
        if (r->regs[j].kind == 0) F[M++] = (uint16_t)j;
      }
    r->nof_cce[cfi - 1]        = M / 9;
    r->nof_pdcch_regs[cfi - 1] = (M / 9) * 9;
    uint32_t nrows = (M - 1) / 32 + 1, ndummy = 32 * nrows - M, kk = 0;
    for (uint32_t j = 0; j < 32; j++)
      for (uint32_t i = 0; i < nrows; i++) {
        uint32_t idx = i * 32 + CONV_PERM[j];
        if (idx >= ndummy) {
          uint32_t m  = idx - ndummy;
          uint32_t kp = (kk + M - (cell->cell_id % M)) % M;
          r->pdcch_map[cfi - 1][m] = F[kp];
          kk++;
        }
      }
  }
  return 0;
}

/* ------------------------------------------------------------------ convolutional code */
void lte_conv_encode(const uint8_t* in, uint32_t K, uint8_t* out)
{
  uint32_t sr = 0; /* bit j = c_{k-1-j} */
  for (uint32_t j = 0; j < 6; j++) sr |= (uint32_t)(in[K - 1 - j] & 1) << j;
  for (uint32_t k = 0; k < K; k++) {
    uint32_t c = in[k] & 1;
#define T(j) ((sr >> ((j)-1)) & 1u)
    out[0 * K + k] = (uint8_t)(c ^ T(2) ^ T(3) ^ T(5) ^ T(6)); /* 133 */
    out[1 * K + k] = (uint8_t)(c ^ T(1) ^ T(2) ^ T(3) ^ T(6)); /* 171 */
    out[2 * K + k] = (uint8_t)(c ^ T(1) ^ T(2) ^ T(4) ^ T(6)); /* 165 */
#undef T
    sr = ((sr << 1) | c) & 63u;
  }
}
void lte_rm_conv_table(uint32_t K, uint16_t* tab)
{
  uint32_t R = (K + 31) / 32, ND = 32 * R - K, n = 0;
  for (uint32_t s = 0; s < 3; s++)
    for (uint32_t k = 0; k < 32 * R; k++) {
      uint32_t y = (k % R) * 32 + CONV_PERM[k / R];
      if (y >= ND) tab[n++] = (uint16_t)(s * K + (y - ND));
    }
}
void lte_rm_conv_tx(const uint8_t* d, uint32_t K, uint8_t* e, uint32_t E)
{
  uint16_t tab[3 * (LTE_DCI_MAX_BITS + 16)];
  lte_rm_conv_table(K, tab);
  for (uint32_t k = 0; k < E; k++) e[k] = d[tab[k % (3 * K)]];
}

/* ------------------------------------------------------------------ turbo code */
int lte_cbsegm(lte_cbsegm_t* s, uint32_t tbs)
{
  memset(s, 0, sizeof(*s));
  s->tbs      = tbs;
  uint32_t B  = tbs + 24, Bp;
  if (B <= 6144) {
    s->C = 1;
    Bp   = B;
  } else {
    s->C = (B + 6119) / 6120;
    Bp   = B + 24 * s->C;
  }
  int ip = lte_qpp_index_ge((Bp + s->C - 1) / s->C);
  if (ip < 0) return -1;
  s->Kp = lte_qpp_K((uint32_t)ip);
  if (s->C == 1) {
    s->Cp = 1;
    s->Km = 0;
    s->Cm = 0;
  } else {
    s->Km        = ip > 0 ? lte_qpp_K((uint32_t)ip - 1) : 0;
    uint32_t dK  = s->Kp - s->Km;
    s->Cm        = (s->C * s->Kp - Bp) / dK;
    s->Cp        = s->C - s->Cm;
  }
  s->F = s->Cp * s->Kp + s->Cm * s->Km - Bp;
  return 0;
}
uint32_t lte_cb_K(const lte_cbsegm_t* s, uint32_t r) { return r < s->Cm ? s->Km : s->Kp; }

void lte_qpp(uint32_t K, uint16_t* pi)
{
  int      idx = lte_qpp_index_ge(K);
  uint64_t f1 = lte_qpp_f1[idx], f2 = lte_qpp_f2[idx];
  for (uint64_t i = 0; i < K; i++) pi[i] = (uint16_t)((f1 * i + f2 * i * i) % K);
}

static void rsc_encode(const uint8_t* in, uint32_t K, uint8_t* z, uint8_t* xt, uint8_t* zt)
{
  uint32_t r1 = 0, r2 = 0, r3 = 0;
  for (uint32_t k = 0; k < K; k++) {
    uint32_t a = (in[k] & 1) ^ r2 ^ r3;
    z[k]       = (uint8_t)(a ^ r1 ^ r3);
    r3 = r2, r2 = r1, r1 = a;
  }
  for (uint32_t k = 0; k < 3; k++) {
    xt[k] = (uint8_t)(r2 ^ r3);
    zt[k] = (uint8_t)(r1 ^ r3);
    r3 = r2, r2 = r1, r1 = 0;
  }
}
void lte_turbo_encode(const uint8_t* in, uint32_t K, uint8_t* d0, uint8_t* d1, uint8_t* d2)
{
  static __thread uint16_t pi[6144];
  static __thread uint8_t  il[6144];
  uint8_t                  xt[3], zt[3], xpt[3], zpt[3];
  lte_qpp(K, pi);
  for (uint32_t i = 0; i < K; i++) {
    d0[i] = in[i] & 1;
    il[i] = in[pi[i]] & 1;
  }
  rsc_encode(in, K, d1, xt, zt);
  rsc_encode(il, K, d2, xpt, zpt);
  d0[K] = xt[0], d0[K + 1] = zt[1], d0[K + 2] = xpt[0], d0[K + 3] = zpt[1];
  d1[K] = zt[0], d1[K + 1] = xt[2], d1[K + 2] = zpt[0], d1[K + 3] = xpt[2];
  d2[K] = xt[1], d2[K + 1] = zt[2], d2[K + 2] = xpt[1], d2[K + 3] = zpt[2];
}

static const uint8_t TURBO_PERM[32] = {0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30,
                                       1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31};
uint32_t lte_rm_turbo_table(uint32_t K, uint32_t* tab)
{
  uint32_t D = K + 4, R = (D + 31) / 32, Kpi = 32 * R, ND = Kpi - D;
  for (uint32_t k = 0; k < Kpi; k++) {
    uint32_t y01 = TURBO_PERM[k / R] + 32 * (k % R);
    uint32_t y2  = (TURBO_PERM[k / R] + 32 * (k % R) + 1) % Kpi;
    tab[k]               = y01 >= ND ? 0 * D + (y01 - ND) : 0xFFFFFFFFu;
    tab[Kpi + 2 * k]     = y01 >= ND ? 1 * D + (y01 - ND) : 0xFFFFFFFFu;
    tab[Kpi + 2 * k + 1] = y2 >= ND ? 2 * D + (y2 - ND) : 0xFFFFFFFFu;
  }
  return Kpi;
}
uint32_t lte_rm_turbo_k0(uint32_t K, uint32_t rv)
{
  uint32_t R = (K + 4 + 31) / 32, Ncb = 3 * 32 * R;
  return R * (2 * ((Ncb + 8 * R - 1) / (8 * R)) * rv + 2);
}
void lte_rm_turbo_tx(const uint8_t* d, uint32_t K, uint32_t F, uint32_t rv, uint8_t* e, uint32_t E)
{
  static __thread uint32_t tab[3 * 6176];
  uint32_t Kpi = lte_rm_turbo_table(K, tab), Kw = 3 * Kpi, D = K + 4;
  uint32_t j = lte_rm_turbo_k0(K, rv), k = 0;
  while (k < E) {
    uint32_t t = tab[j % Kw];
    j++;
    if (t == 0xFFFFFFFFu) continue;
    uint32_t s = t / D, i = t % D;
    if (s < 2 && i < F) continue; /* filler bits are <NULL> in d0, d1 */
    e[k++] = d[t];
  }
}
uint32_t lte_rm_turbo_E(uint32_t G, uint32_t C, uint32_t r, uint32_t Qm, uint32_t NL)
{
  uint32_t Gp = G / (NL * Qm), gamma = Gp % C;
  if (r + gamma + 1 <= C) return NL * Qm * (Gp / C);
  return NL * Qm * ((Gp + C - 1) / C);
}

/* ------------------------------------------------------------------ modulation, 36.211 7.1 */
void lte_modulate(const uint8_t* b, uint32_t nsym, uint32_t Qm, cf_t* out)
{
  for (uint32_t i = 0; i < nsym; i++) {
    const uint8_t* p = &b[i * Qm];
    float          I, Q;
    switch (Qm) {
      case 2:
        I = (1 - 2 * p[0]) * (float)M_SQRT1_2;
        Q = (1 - 2 * p[1]) * (float)M_SQRT1_2;
        break;
      case 4:
        I = (1 - 2 * p[0]) * (p[2] ? 3.0f : 1.0f) / sqrtf(10.0f);
        Q = (1 - 2 * p[1]) * (p[3] ? 3.0f : 1.0f) / sqrtf(10.0f);
        break;
      case 6: {
        static const float lv[4] = {3, 1, 5, 7}; /* (b2 b4): 00->3 01->1 10->5 11->7 */
        I = (1 - 2 * p[0]) * lv[2 * p[2] + p[4]] / sqrtf(42.0f);
        Q = (1 - 2 * p[1]) * lv[2 * p[3] + p[5]] / sqrtf(42.0f);
      } break;
      default: {
        static const float lv[8] = {5, 7, 3, 1, 11, 9, 13, 15};
        I = (1 - 2 * p[0]) * lv[4 * p[2] + 2 * p[4] + p[6]] / sqrtf(170.0f);
        Q = (1 - 2 * p[1]) * lv[4 * p[3] + 2 * p[5] + p[7]] / sqrtf(170.0f);
      } break;
    }
    out[i].re = I;
    out[i].im = Q;
  }
}

/* ------------------------------------------------------------------ DCI sizes (FDD, no CIF) */
static uint32_t ceil_log2(uint32_t v)
{
  uint32_t n = 0;
  while ((1u << n) < v) n++;
  return n;
}
static uint32_t rbg_size(uint32_t nprb) { return nprb <= 10 ? 1 : nprb <= 26 ? 2 : nprb <= 63 ? 3 : 4; }
static uint32_t riv_nbits(uint32_t nprb) { return ceil_log2(nprb * (nprb + 1) / 2); }
static int      is_ambiguous(uint32_t n)
{
  static const uint32_t a[10] = {12, 14, 16, 20, 24, 26, 32, 40, 44, 56};
  for (int i = 0; i < 10; i++)
    if (a[i] == n) return 1;
  return 0;
}
static uint32_t ngap1(uint32_t n)
{
  if (n <= 10) return (n + 1) / 2;
  if (n == 11) return 4;
  if (n <= 19) return 8;
  if (n <= 26) return 12;
  if (n <= 44) return 18;
  if (n <= 63) return 27;
  if (n <= 79) return 32;
  return 48;
}
static uint32_t ngap2(uint32_t n) { return n < 50 ? 0 : n <= 63 ? 9 : n <= 79 ? 16 : 16; }
static uint32_t nvrb_gap(uint32_t n, int gap2)
{
  if (!gap2) {
    uint32_t g = ngap1(n);
    return 2 * (g < n - g ? g : n - g);
  }
  uint32_t g = ngap2(n);
  return (n / (2 * g)) * 2 * g;
}
static uint32_t f1c_riv_bits(uint32_t nprb)
{
  uint32_t step = nprb < 50 ? 2 : 4, nv = nvrb_gap(nprb, 0) / step;
  return ceil_log2(nv * (nv + 1) / 2);
}
static uint32_t size_01a(const lte_cell_t* c)
{
  uint32_t f0 = 1 + 1 + riv_nbits(c->nof_prb) + 5 + 1 + 2 + 3 + 1;
  uint32_t f1a = 1 + 1 + riv_nbits(c->nof_prb) + 5 + 3 + 1 + 2 + 2;
  uint32_t n  = f0 > f1a ? f0 : f1a;
  while (is_ambiguous(n)) n++;
  return n;
}
uint32_t lte_dci_sizeof(const lte_cell_t* c, lte_dci_format_t f)
{
  uint32_t N = c->nof_prb, P = rbg_size(N), hdr = N > 10 ? 1 : 0, bm = (N + P - 1) / P;
  uint32_t s01a = size_01a(c), n = 0;
  uint32_t tpmi = c->nof_ports == 2 ? 2 : c->nof_ports == 4 ? 4 : 0;
  switch (f) {
    case LTE_DCI_FORMAT0:
    case LTE_DCI_FORMAT1A: return s01a;
    case LTE_DCI_FORMAT1:
      n = hdr + bm + 5 + 3 + 1 + 2 + 2;
      if (n == s01a) n++;
      while (is_ambiguous(n) || n == s01a) n++;
      return n;
    case LTE_DCI_FORMAT1B: n = 1 + riv_nbits(N) + 5 + 3 + 1 + 2 + 2 + tpmi + 1; break;
    case LTE_DCI_FORMAT1D: n = 1 + riv_nbits(N) + 5 + 3 + 1 + 2 + 2 + tpmi + 1; break;
    case LTE_DCI_FORMAT1C: return (N >= 50 ? 1 : 0) + f1c_riv_bits(N) + 5;
    case LTE_DCI_FORMAT2: n = hdr + bm + 2 + 3 + 1 + 8 + 8 + (c->nof_ports == 2 ? 3 : c->nof_ports == 4 ? 6 : 0); break;
    case LTE_DCI_FORMAT2A: n = hdr + bm + 2 + 3 + 1 + 8 + 8 + (c->nof_ports == 4 ? 2 : 0); break;
    case LTE_DCI_FORMAT2B: n = hdr + bm + 2 + 3 + 1 + 8 + 8; break;
    default: return 0;
  }
  while (is_ambiguous(n)) n++;
  return n;
}

/* ------------------------------------------------------------------ DCI pack / unpack */
static void put(uint8_t** p, uint32_t v, uint32_t n)
{
  for (uint32_t i = 0; i < n; i++) *(*p)++ = (uint8_t)((v >> (n - 1 - i)) & 1);
}
static uint32_t get(const uint8_t** p, uint32_t n)
{
  uint32_t v = 0;
  for (uint32_t i = 0; i < n; i++) v = (v << 1) | (*(*p)++ & 1);
  return v;
}
int lte_dci_pack(const lte_cell_t* c, const lte_dci_t* d, uint8_t* bits, uint32_t* nbits)
{
  uint32_t N = c->nof_prb, P = rbg_size(N), bm = (N + P - 1) / P, hdr = N > 10 ? 1 : 0;
  uint32_t size = lte_dci_sizeof(c, (lte_dci_format_t)d->format);
  uint8_t* p    = bits;
  memset(bits, 0, LTE_DCI_MAX_BITS);
  switch (d->format) {
    case LTE_DCI_FORMAT0:
      put(&p, 0, 1);
      put(&p, d->hop, 1);
      put(&p, d->riv, riv_nbits(N));
      put(&p, d->mcs[0], 5);
      put(&p, d->ndi[0], 1);
      put(&p, d->tpc, 2);
      put(&p, d->n_dmrs, 3);
      put(&p, d->cqi_req, 1);
      break;
    case LTE_DCI_FORMAT1A:
      put(&p, 1, 1);
      put(&p, d->t2_dist, 1);
      if (d->t2_dist && N >= 50) {
        put(&p, d->t2_ngap2, 1);
        put(&p, d->riv, riv_nbits(N) - 1);
      } else {
        put(&p, d->riv, riv_nbits(N));
      }
      put(&p, d->mcs[0], 5);
      put(&p, d->pid, 3);
      put(&p, d->ndi[0], 1);
      put(&p, d->rv[0], 2);
      if (LTE_RNTI_ISUSER(d->rnti))
        put(&p, d->tpc, 2);
      else
        put(&p, d->n_prb1a == 3 ? 1 : 0, 2); /* MSB reserved, LSB selects N_PRB^1A */
      break;
    case LTE_DCI_FORMAT1:
    case LTE_DCI_FORMAT2:
    case LTE_DCI_FORMAT2A:
      if (hdr) put(&p, d->alloc_type == 1, 1);
      if (d->alloc_type == 0) {
        put(&p, d->rbg_bitmask, bm);
      } else if (d->alloc_type == 1) {
        uint32_t sb = ceil_log2(P);
        put(&p, d->t1_subset, sb);
        put(&p, d->t1_shift, 1);
        put(&p, d->t1_vrb_bitmask, bm - sb - 1);
      } else
        return -1;
      if (d->format == LTE_DCI_FORMAT1) {
        put(&p, d->mcs[0], 5);
        put(&p, d->pid, 3);
        put(&p, d->ndi[0], 1);
        put(&p, d->rv[0], 2);
        put(&p, d->tpc, 2);
      } else {
        put(&p, d->tpc, 2);
        put(&p, d->pid, 3);
        put(&p, d->tb_cw_swap, 1);
        for (int i = 0; i < 2; i++) {
          if (d->tb_en[i]) {
            put(&p, d->mcs[i], 5);
            put(&p, d->ndi[i], 1);
            put(&p, d->rv[i], 2);
          } else { /* disabled TB: mcs 0, rv 1 (36.213 7.1.7.2) */
            put(&p, 0, 5);
            put(&p, d->ndi[i], 1);
            put(&p, 1, 2);
          }
        }
        if (d->format == LTE_DCI_FORMAT2) put(&p, d->pinfo, c->nof_ports == 2 ? 3 : c->nof_ports == 4 ? 6 : 0);
        if (d->format == LTE_DCI_FORMAT2A && c->nof_ports == 4) put(&p, d->pinfo, 2);
      }
      break;
    case LTE_DCI_FORMAT1C:
      if (N >= 50) put(&p, d->t2_ngap2, 1);
      put(&p, d->riv, f1c_riv_bits(N));
      put(&p, d->mcs[0], 5);
      break;
    default: return -1;
  }
  if ((uint32_t)(p - bits) > size) return -2;
  *nbits = size;
  return 0;
}

/* restates srsran_dci_msg_unpack_pdsch / _pusch as called from srsran_dci_msg_to_trace_timestamp
 * (lib/src/phy/falcon_phch/falcon_dci.c:208,271) */
int lte_dci_unpack(const lte_cell_t* c, lte_dci_format_t f, uint16_t rnti, const uint8_t* bits, uint32_t nbits, lte_dci_t* d)
{
  uint32_t N = c->nof_prb, P = rbg_size(N), bm = (N + P - 1) / P, hdr = N > 10 ? 1 : 0;
  const uint8_t* p = bits;
  memset(d, 0, sizeof(*d));
  if (nbits != lte_dci_sizeof(c, f)) return -1;
  d->rnti   = rnti;
  d->format = (uint8_t)f;
  switch (f) {
    case LTE_DCI_FORMAT0:
      if (get(&p, 1) != 0) return -2;
      d->hop        = (uint8_t)get(&p, 1);
      d->alloc_type = 2;
      d->riv        = get(&p, riv_nbits(N));
      d->mcs[0]     = (uint8_t)get(&p, 5);
      d->ndi[0]     = (uint8_t)get(&p, 1);
      d->tpc        = (uint8_t)get(&p, 2);
      d->n_dmrs     = (uint8_t)get(&p, 3);
      d->cqi_req    = (uint8_t)get(&p, 1);
      d->tb_en[0]   = 1;
      break;
    case LTE_DCI_FORMAT1A:
      if (get(&p, 1) != 1) return -2;
      d->alloc_type = 2;
      d->t2_dist    = (uint8_t)get(&p, 1);
      if (d->t2_dist && N >= 50) {
        d->t2_ngap2 = (uint8_t)get(&p, 1);
        d->riv      = get(&p, riv_nbits(N) - 1);
      } else
        d->riv = get(&p, riv_nbits(N));
      d->mcs[0] = (uint8_t)get(&p, 5);
      d->pid    = (uint8_t)get(&p, 3);
      d->ndi[0] = (uint8_t)get(&p, 1);
      d->rv[0]  = (uint8_t)get(&p, 2);
      {
        uint32_t t = get(&p, 2);
        if (LTE_RNTI_ISUSER(rnti))
          d->tpc = (uint8_t)t;
        else
          d->n_prb1a = (t & 1) ? 3 : 2;
      }
      d->tb_en[0] = 1;
      break;
    case LTE_DCI_FORMAT1:
    case LTE_DCI_FORMAT2:
    case LTE_DCI_FORMAT2A:
      d->alloc_type = hdr ? (uint8_t)get(&p, 1) : 0;
      if (d->alloc_type == 0)
        d->rbg_bitmask = get(&p, bm);
      else {
        uint32_t sb       = ceil_log2(P);
        d->t1_subset      = get(&p, sb);
        d->t1_shift       = get(&p, 1);
        d->t1_vrb_bitmask = get(&p, bm - sb - 1);
      }
      if (f == LTE_DCI_FORMAT1) {
        d->mcs[0]   = (uint8_t)get(&p, 5);
        d->pid      = (uint8_t)get(&p, 3);
        d->ndi[0]   = (uint8_t)get(&p, 1);
        d->rv[0]    = (uint8_t)get(&p, 2);
        d->tpc      = (uint8_t)get(&p, 2);
        d->tb_en[0] = 1;
      } else {
        d->tpc        = (uint8_t)get(&p, 2);
        d->pid        = (uint8_t)get(&p, 3);
        d->tb_cw_swap = (uint8_t)get(&p, 1);
        for (int i = 0; i < 2; i++) {
          d->mcs[i]   = (uint8_t)get(&p, 5);
          d->ndi[i]   = (uint8_t)get(&p, 1);
          d->rv[i]    = (uint8_t)get(&p, 2);
          d->tb_en[i] = !(d->mcs[i] == 0 && d->rv[i] == 1);
        }
        if (f == LTE_DCI_FORMAT2) d->pinfo = (uint8_t)get(&p, c->nof_ports == 2 ? 3 : c->nof_ports == 4 ? 6 : 0);
        if (f == LTE_DCI_FORMAT2A && c->nof_ports == 4) d->pinfo = (uint8_t)get(&p, 2);
      }
      break;
    case LTE_DCI_FORMAT1C:
      d->alloc_type = 2;
      d->t2_dist    = 1;
      if (N >= 50) d->t2_ngap2 = (uint8_t)get(&p, 1);
      d->riv      = get(&p, f1c_riv_bits(N));
      d->mcs[0]   = (uint8_t)get(&p, 5);
      d->tb_en[0] = 1;
      break;
    default: return -3; /* 1B/1D/2B: rejected downstream by dl_sniffer_config_mimo_type (dl_sniffer_pdsch.c:168-175) */
  }
  return 0;
}

/* ------------------------------------------------------------------ resource allocation -> PRB mask */
static void riv_decode(uint32_t riv, uint32_t N, uint32_t* L, uint32_t* S)
{
  *L = riv / N + 1;
  *S = riv % N;
  if (*L + *S > N) {
    *L = N - *L + 2;
    *S = N - 1 - *S;
  }
}
/* 36.211 6.2.3.2 distributed VRB -> PRB for slot 0/1 */
static void dvrb_to_prb(uint32_t N, int gap2, uint32_t nvrb, uint32_t* prb0, uint32_t* prb1)
{
  uint32_t P = rbg_size(N), Ngap = gap2 ? ngap2(N) : ngap1(N);
  uint32_t Nt = gap2 ? 2 * Ngap : nvrb_gap(N, 0);
  uint32_t Nrow = ((Nt + 4 * P - 1) / (4 * P)) * P, Nnull = 4 * Nrow - Nt;
  uint32_t nt = nvrb % Nt, blk = nvrb / Nt;
  int32_t  np1 = (int32_t)(2 * Nrow * (nt % 2) + nt / 2 + Nt * blk);
  int32_t  np2 = (int32_t)(Nrow * (nt % 4) + nt / 4 + Nt * blk);
  int32_t  e;
  if (Nnull && nt >= Nt - Nnull && (nt % 2) == 1)
    e = np1 - (int32_t)Nrow;
  else if (Nnull && nt >= Nt - Nnull && (nt % 2) == 0)
    e = np1 - (int32_t)Nrow + (int32_t)Nnull / 2;
  else if (Nnull && nt < Nt - Nnull && (nt % 4) >= 2)
    e = np2 - (int32_t)Nnull / 2;
  else
    e = np2;
  int32_t o  = (int32_t)(((uint32_t)e + Nt / 2) % Nt + Nt * blk);
  uint32_t a = (uint32_t)e, b = (uint32_t)o;
  *prb0      = (a % Nt) < Nt / 2 ? a : a + Ngap - Nt / 2;
  *prb1      = (b % Nt) < Nt / 2 ? b : b + Ngap - Nt / 2;
}
static int ra_to_prb_mask(const lte_cell_t* c, const lte_dci_t* d, lte_dl_grant_t* g)
{
  uint32_t N = c->nof_prb, P = rbg_size(N), nrbg = (N + P - 1) / P;
  memset(g->prb_mask, 0, sizeof(g->prb_mask));
  g->nof_prb = 0;
  if (d->alloc_type == 0) {
    for (uint32_t i = 0; i < nrbg; i++)
      if (d->rbg_bitmask & (1u << (nrbg - 1 - i)))
        for (uint32_t j = i * P; j < (i + 1) * P && j < N; j++) {
          g->prb_mask[0][j] = g->prb_mask[1][j] = 1;
          g->nof_prb++;
        }
  } else if (d->alloc_type == 1) {
    uint32_t sb = ceil_log2(P), nb = nrbg - sb - 1, p = d->t1_subset;
    uint32_t q = (N - 1) / (P * P), pm = ((N - 1) / P) % P, nsub;
    if (p < pm)
      nsub = q * P + P;
    else if (p == pm)
      nsub = q * P + (N - 1) % P + 1;
    else
      nsub = q * P;
    uint32_t shift = d->t1_shift ? nsub - nb : 0;
    for (uint32_t i = 0; i < nb; i++)
      if (d->t1_vrb_bitmask & (1u << (nb - 1 - i))) {
        uint32_t v = ((i + shift) / P) * P * P + p * P + (i + shift) % P;
        if (v >= N) return -1;
        g->prb_mask[0][v] = g->prb_mask[1][v] = 1;
        g->nof_prb++;
      }
  } else {
    uint32_t L, S;
    if (d->format == LTE_DCI_FORMAT1C) {
      uint32_t step = N < 50 ? 2 : 4, nv = nvrb_gap(N, d->t2_ngap2) / step;
      riv_decode(d->riv, nv, &L, &S);
      L *= step, S *= step;
    } else if (d->t2_dist) {
      riv_decode(d->riv, nvrb_gap(N, d->t2_ngap2), &L, &S);
    } else
      riv_decode(d->riv, N, &L, &S);
    {
      uint32_t lim = d->t2_dist ? nvrb_gap(N, d->t2_ngap2) : N; /* an out-of-range RIV decodes to nonsense: reject it */
      if (L < 1 || L > lim || S >= lim || S + L > lim) return -1;
    }
    if (!d->t2_dist) {
      for (uint32_t j = S; j < S + L; j++) g->prb_mask[0][j] = g->prb_mask[1][j] = 1;
    } else {
      for (uint32_t v = S; v < S + L; v++) {
        uint32_t p0, p1;
        dvrb_to_prb(N, d->t2_ngap2, v, &p0, &p1);
        if (p0 >= N || p1 >= N) return -1;
        g->prb_mask[0][p0] = 1;
        g->prb_mask[1][p1] = 1;
      }
    }
    g->nof_prb = L;
  }
  return g->nof_prb ? 0 : -1;
}

int lte_tbs_from_idx(int itbs, uint32_t nprb)
{
  if (itbs < 0 || itbs >= LTE_TBS_NOF_ITBS || nprb < 1 || nprb > LTE_TBS_NOF_PRB) return -1;
  return lte_tbs_table[itbs][nprb - 1];
}

uint32_t lte_pdsch_re_in_prb(const lte_cell_t* c, uint32_t sf_idx, uint32_t cfi, uint32_t l, uint32_t prb, uint16_t* kk)
{
  uint32_t n = 0, nctrl = c->nof_prb <= 10 ? cfi + 1 : cfi;
  if (l < nctrl) return 0;
  uint32_t lo = 6 * c->nof_prb - 36, hi = 6 * c->nof_prb + 36; /* centre 72 subcarriers */
  int      crs_sym = (l % 7 == 0) || (l % 7 == 4);
  for (uint32_t k = 12 * prb; k < 12 * prb + 12; k++) {
    if (crs_sym) {
      if (c->nof_ports == 1) {
        if (k % 6 == lte_crs_offset(c, 0, l % 7)) continue;
      } else if (k % 3 == c->cell_id % 3)
        continue;
    }
    if (k >= lo && k < hi) {
      if ((sf_idx == 0 || sf_idx == 5) && (l == 5 || l == 6)) continue; /* SSS, PSS (FDD) */
      if (sf_idx == 0 && l >= 7 && l <= 10) continue;                    /* PBCH */
    }
    kk[n++] = (uint16_t)k;
  }
  return n;
}

int lte_dl_dci_to_grant(const lte_cell_t* c, uint32_t sf_idx, uint32_t cfi, int alt, const lte_dci_t* d, lte_dl_grant_t* g)
{
  memset(g, 0, sizeof(*g));
  if (ra_to_prb_mask(c, d, g)) return -1;
  /* dl_sniffer_compute_tb, dl_sniffer_pdsch.c:14-92 */
  for (int i = 0; i < 2; i++) {
    g->tb[i].mcs = d->mcs[i];
    g->tb[i].rv  = d->rv[i];
    if ((d->tb_en[i] && d->format >= LTE_DCI_FORMAT2) || (d->format < LTE_DCI_FORMAT2 && i == 0)) {
      g->tb[i].enabled = 1;
      g->nof_tb++;
    }
  }
  g->cw_swap = (uint8_t)(d->format >= LTE_DCI_FORMAT2 && g->nof_tb == 2 && d->tb_cw_swap); /* one TB: always codeword 0 (Table 5.3.3.1.5-2) */
  if (d->format == LTE_DCI_FORMAT1A || !LTE_RNTI_ISUSER(d->rnti)) alt = 0;
  if (!LTE_RNTI_ISUSER(d->rnti)) {
    int tbs;
    if (d->format == LTE_DCI_FORMAT1A)
      tbs = lte_tbs_from_idx(d->mcs[0], d->n_prb1a == 2 ? 2 : 3);
    else if (d->format == LTE_DCI_FORMAT1C)
      tbs = d->mcs[0] < 32 ? lte_tbs_format1c[d->mcs[0]] : -1;
    else
      return -2;
    if (tbs < 0) return -2;
    g->tb[0].qm  = 2;
    g->tb[0].tbs = tbs;
  } else {
    for (int i = 0; i < 2; i++) {
      if (!g->tb[i].enabled) continue;
      uint32_t m = d->mcs[i];
      int      itbs = alt ? lte_dl_mcs_itbs_alt[m] : lte_dl_mcs_itbs[m];
      g->tb[i].qm   = (uint8_t)(alt ? lte_dl_mcs_qm_alt[m] : lte_dl_mcs_qm[m]);
      g->tb[i].tbs  = itbs >= 0 ? lte_tbs_from_idx(itbs, g->nof_prb) : 0; /* retx MCS: last_tbs = 0 after bzero */
      if (g->tb[i].tbs < 0) return -2;
    }
  }
  /* srsran_ra_dl_compute_nof_re (dl_sniffer_pdsch.c:110) */
  uint16_t kk[12];
  for (uint32_t l = 0; l < LTE_NSYMB_SF; l++)
    for (uint32_t prb = 0; prb < c->nof_prb; prb++)
      if (g->prb_mask[l / 7][prb]) g->nof_re += lte_pdsch_re_in_prb(c, sf_idx, cfi, l, prb, kk);
  for (int i = 0; i < 2; i++)
    if (g->tb[i].enabled) g->tb[i].nof_bits = g->nof_re * g->tb[i].qm;
  if (d->format == LTE_DCI_FORMAT1C && (d->rnti <= LTE_RARNTI_END || d->rnti == LTE_PRNTI))
    for (int i = 0; i < 2; i++) g->tb[i].rv = 0;
  /* dl_sniffer_config_mimo (dl_sniffer_pdsch.c:134-276) */
  switch (d->format) {
    case LTE_DCI_FORMAT1:
    case LTE_DCI_FORMAT1A:
    case LTE_DCI_FORMAT1C: g->tx_scheme = c->nof_ports == 1 ? LTE_TX_PORT0 : LTE_TX_DIVERSITY; break;
    case LTE_DCI_FORMAT2: g->tx_scheme = (g->nof_tb == 1 && d->pinfo == 0) ? LTE_TX_DIVERSITY : LTE_TX_SPATIALMUX; break;
    case LTE_DCI_FORMAT2A: g->tx_scheme = (g->nof_tb == 1 && d->pinfo == 0) ? LTE_TX_DIVERSITY : LTE_TX_CDD; break;
    default: return -3;
  }
  if (g->tx_scheme == LTE_TX_SPATIALMUX) {
    if (g->nof_tb == 1) {
      if (d->pinfo > 0 && d->pinfo < 5)
        g->pmi = d->pinfo - 1;
      else
        return -4;
    } else {
      if (d->pinfo >= 2) return -4;
      g->pmi = d->pinfo % 2;
    }
  }
  switch (g->tx_scheme) {
    case LTE_TX_PORT0:
      if (g->nof_tb != 1) return -5;
      g->nof_layers = 1;
      break;
    case LTE_TX_DIVERSITY:
      if (g->nof_tb != 1) return -5;
      g->nof_layers = (uint8_t)c->nof_ports;
      break;
    case LTE_TX_SPATIALMUX:
      if (g->nof_tb < 1 || g->nof_tb > 2) return -5;
      g->nof_layers = (uint8_t)g->nof_tb;
      break;
    default:
      if (g->nof_tb != 2) return -5;
      g->nof_layers = 2;
      break;
  }
  return 0;
}

/* ------------------------------------------------------------------ search spaces, 36.213 9.1.1 */
uint32_t lte_pdcch_ue_locations(uint32_t nof_cce, uint32_t sf_idx, uint16_t rnti, uint16_t* ncce, uint8_t* Lv, uint32_t max)
{
  static const uint32_t M[4] = {6, 6, 2, 2};
  uint32_t              Yk = rnti, k = 0;
  for (uint32_t m = 0; m < sf_idx + 1; m++) Yk = (39827u * Yk) % 65537u;
  for (int l = 3; l >= 0; l--) {
    uint32_t L = 1u << l;
    for (uint32_t i = 0; i < M[l]; i++) {
      if (nof_cce >= L) {
        uint32_t n = L * ((Yk + i) % (nof_cce / L));
        if (k < max && n + L <= nof_cce) {
          ncce[k] = (uint16_t)n;
          Lv[k]   = (uint8_t)l;
          k++;
        }
      }
    }
  }
  return k;
}
uint32_t lte_pdcch_common_locations(uint32_t nof_cce, uint16_t* ncce, uint8_t* Lv, uint32_t max)
{
  uint32_t k = 0;
  for (int l = 3; l > 1; l--) {
    uint32_t L = 1u << l, lim = (nof_cce < 16 ? nof_cce : 16) / L;
    for (uint32_t i = 0; i < lim; i++) {
      uint32_t n = L * (i % (nof_cce / L));
      if (k < max && n + L <= nof_cce) {
        ncce[k] = (uint16_t)n;
        Lv[k]   = (uint8_t)l;
        k++;
      }
    }
  }
  return k;
}
uint32_t lte_pdcch_validate_location(uint32_t nof_cce, uint32_t ncce, uint32_t l, uint32_t sf_idx, uint16_t rnti)
{
  uint16_t nc[22];
  uint8_t  Lv[22];
  uint32_t n = 0;
  if (rnti >= LTE_RARNTI_START && rnti <= LTE_RARNTI_END)
    n = lte_pdcch_common_locations(nof_cce, nc, Lv, 22);
  else if (rnti >= LTE_CRNTI_START && rnti <= LTE_CRNTI_END) {
    n = lte_pdcch_ue_locations(nof_cce, sf_idx, rnti, nc, Lv, 22);
    n += lte_pdcch_common_locations(nof_cce, &nc[n], &Lv[n], 22 - n);
  } else if (rnti >= 0xFFFD)
    n = lte_pdcch_common_locations(nof_cce, nc, Lv, 22);
  uint32_t amb = 0, valid = 0;
  for (uint32_t i = 0; i < n; i++)
    if (nc[i] == ncce) {
      if (l > 0 && l - 1 == Lv[i]) amb = 1;
      if (Lv[i] == l) valid = 1;
    }
  if (valid && !amb) valid = 2;
  return valid;
}

/* ------------------------------------------------------------------ PCFICH codewords, 36.212 Table 5.3.4-1 */
const uint8_t lte_cfi_codeword[3][32] = {
    {0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1},
    {1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0},
    {1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 0, 1, 1}};

/* ------------------------------------------------------------------ RNG (xoshiro256**) */
static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
void            lte_rng_seed(lte_rng_t* r, uint64_t seed)
{
  for (int i = 0; i < 4; i++) {
    uint64_t z = (seed += 0x9E3779B97F4A7C15ull);
    z          = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z          = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    r->s[i]    = z ^ (z >> 31);
  }
}
uint64_t lte_rng_u64(lte_rng_t* r)
{
  uint64_t res = rotl(r->s[1] * 5, 7) * 9, t = r->s[1] << 17;
  r->s[2] ^= r->s[0];
  r->s[3] ^= r->s[1];
  r->s[1] ^= r->s[2];
  r->s[0] ^= r->s[3];
  r->s[2] ^= t;
  r->s[3] = rotl(r->s[3], 45);
  return res;
}
double lte_rng_uniform(lte_rng_t* r) { return (double)(lte_rng_u64(r) >> 11) * (1.0 / 9007199254740992.0); }
double lte_rng_gauss(lte_rng_t* r)
{
  double u1 = lte_rng_uniform(r), u2 = lte_rng_uniform(r);
  if (u1 < 1e-300) u1 = 1e-300;
  return sqrt(-2.0 * log(u1)) * cos(2.0 * M_PI * u2);
}

/* ================================================================== uplink */
int lte_ul_valid_prb(uint32_t L)
{
  if (L == 0) return 0;
  while (L % 2 == 0) L /= 2;
  while (L % 3 == 0) L /= 3;
  while (L % 5 == 0) L /= 5;
  return L == 1;
}
uint32_t lte_largest_prime_below(uint32_t n)
{
  for (uint32_t p = n - 1; p >= 2; p--) {
    int ok = 1;
    for (uint32_t d = 2; d * d <= p; d++)
      if (p % d == 0) {
        ok = 0;
        break;
      }
    if (ok) return p;
  }
  return 2;
}
int lte_ul_dci_to_grant(const lte_cell_t* c, const lte_dci_t* d, int table, lte_ul_grant_t* g) { return lte_ul_dci_to_grant_hop(c, NULL, d, table, g); }
int lte_ul_dci_to_grant_hop(const lte_cell_t* c, const lte_ul_cfg_t* ucfg, const lte_dci_t* d, int table, lte_ul_grant_t* g)
{
  static const uint8_t dmrs2_map[8] = {0, 6, 3, 4, 2, 8, 10, 9}; /* 36.211 Table 5.5.2.1.1-1 */
  memset(g, 0, sizeof(*g));
  if (d->format != LTE_DCI_FORMAT0) return -1;
  uint32_t L, S, riv = d->riv, hop_kind = 0xFF;
  const uint32_t N = c->nof_prb;
  if (d->hop) { /* the N_UL_hop most significant bits of the allocation field select the hop (36.213 Tables 8.4-1 / 8.4-2) */
    uint32_t rivb = 0, nh = N < 50 ? 1 : 2;
    while ((1u << rivb) < N * (N + 1) / 2) rivb++;
    uint32_t hb = riv >> (rivb - nh);
    riv &= (1u << (rivb - nh)) - 1;
    hop_kind = nh == 1 ? (hb == 0 ? 2 : 3) : hb; /* 0 +1/4, 1 -1/4, 2 +1/2, 3 type 2 */
  }
  riv_decode(riv, N, &L, &S);
  if (L < 1 || L > N || S + L > N) return -1;
  g->n_prb_slot1 = S;
  if (hop_kind < 3) { /* type 1: ul_sniffer_ra_ul_grant_to_grant_prb_allocation, lib/src/phy/falcon_phch/ul_sniffer_pusch.c:48-80 */
    uint32_t ho = ucfg ? ucfg->n_rb_ho : 0;
    if (ho % 2) ho++;
    const uint32_t nrb = N - ho - (N % 2);
    if (S < ho / 2) return -1;
    uint32_t s1 = S;
    if (hop_kind == 0)
      s1 = (nrb / 4 + S) % nrb;
    else if (hop_kind == 1)
      s1 = S < nrb / 4 ? nrb + S - nrb / 4 : S - nrb / 4;
    else
      s1 = (nrb / 2 + S) % nrb;
    if (s1 + L > N) return -1;
    g->hop = 1, g->n_prb_slot1 = s1;
  }
  g->rnti = d->rnti, g->L_prb = L, g->n_prb = S, g->mcs = d->mcs[0], g->n_dmrs2 = dmrs2_map[d->n_dmrs & 7];
  uint32_t m = d->mcs[0];
  int      itbs;
  if (m > 28) return -2; /* retransmission MCS: needs the HARQ state the sniffer does not have */
  if (table == 2) {      /* 36.213 Table 8.6.1-3 (256QAM), ul_fill_ra_mcs_256, lib/src/phy/falcon_phch/ul_sniffer_pusch.c:91-135 */
    if (m < 6)
      g->qm = 2, itbs = 2 * (int)m;
    else if (m < 10)
      g->qm = 4, itbs = (int)m + 5;
    else if (m < 14)
      g->qm = 4, itbs = (int)m + 6;
    else if (m < 19)
      g->qm = 6, itbs = (int)m + 6;
    else if (m < 23)
      g->qm = 6, itbs = (int)m + 7;
    else if (m < 26)
      g->qm = 8, itbs = (int)m + 7;
    else if (m == 26)
      g->qm = 8, itbs = -32; /* row 32A */
    else
      g->qm = 8, itbs = (int)m + 6;
  } else if (m <= 10)
    g->qm = 2, itbs = (int)m;
  else if (m <= 20)
    g->qm = 4, itbs = (int)m - 1;
  else
    g->qm = table ? 6 : 4, itbs = (int)m - 2;
  g->rv  = 0;
  g->tbs = itbs == -32 ? lte_tbs_32a(L) : lte_tbs_from_idx(itbs, L);
  if (g->tbs <= 0) return -2;
  g->nof_re   = 12 * L * 12; /* 12 data SC-FDMA symbols, no SRS */
  g->nof_bits = g->nof_re * g->qm;
  return 0;
}
void lte_pusch_uv(const lte_cell_t* c, const lte_ul_cfg_t* u, uint32_t ns, uint32_t M, uint32_t* u_out, uint32_t* v_out)
{
  const uint32_t fss = ((c->cell_id % 30) + u->delta_ss) % 30; /* f_ss^PUSCH */
  uint32_t       fgh = 0, v = 0;
  uint8_t        cb[8 * 20 + 8];
  if (u->group_hopping) { /* f_gh(ns) = sum c(8 ns + i) 2^i mod 30, c_init = floor(cell_id / 30) */
    lte_gold_bits(c->cell_id / 30, cb, 8 * 20);
    for (uint32_t i = 0; i < 8; i++) fgh += (uint32_t)cb[8 * ns + i] << i;
    fgh %= 30;
  } else if (u->seq_hopping && M >= 72) { /* v = c(ns), c_init = floor(cell_id / 30) 2^5 + f_ss^PUSCH */
    lte_gold_bits((c->cell_id / 30) * 32 + fss, cb, 20);
    v = cb[ns];
  }
  *u_out = (fgh + fss) % 30, *v_out = v;
}
int lte_pusch_dmrs(const lte_cell_t* c, const lte_ul_cfg_t* u, uint32_t ns, uint32_t n_dmrs2, uint32_t M, cf_t* r)
{
  if (M < 36) return -1;
  uint32_t fss = ((c->cell_id % 30) + u->delta_ss) % 30, useq, v;
  lte_pusch_uv(c, u, ns, M, &useq, &v);
  /* n_PRS(ns), 36.211 5.5.2.1.1 */
  uint8_t  cbits[8 * 7 * 20 + 8];
  lte_gold_bits((c->cell_id / 30) * 32 + fss, cbits, 8 * 7 * 20 + 8);
  uint32_t nprs = 0;
  for (uint32_t i = 0; i < 8; i++) nprs += (uint32_t)cbits[8 * 7 * ns + i] << i;
  static const uint8_t n_dmrs1_of[8] = {0, 2, 3, 4, 6, 8, 9, 10}; /* cyclicShift -> n_DMRS^(1), 36.211 Table 5.5.2.1.1-2 */
  uint32_t ncs = (n_dmrs1_of[u->n_dmrs1 & 7u] + n_dmrs2 + nprs) % 12;
  uint32_t Nzc = lte_largest_prime_below(M);
  double   qb  = (double)Nzc * (useq + 1) / 31.0;
  uint32_t q   = (uint32_t)floor(qb + 0.5);
  if (v) q = ((uint32_t)floor(2.0 * qb) & 1u) ? q - 1 : q + 1; /* q = floor(qb + 1/2) + v (-1)^floor(2 qb) */
  for (uint32_t n = 0; n < M; n++) {
    uint64_t m  = n % Nzc;
    uint64_t t  = ((uint64_t)q * m * (m + 1)) % (2ull * Nzc);   /* phase = -pi t / Nzc */
    uint32_t a  = (ncs * n) % 12;                               /* + 2 pi a / 12 */
    double   ph = -M_PI * (double)t / (double)Nzc + 2.0 * M_PI * (double)a / 12.0;
    r[n].re     = (float)cos(ph);
    r[n].im     = (float)sin(ph);
  }
  return 0;
}

/* ---- control information on PUSCH (36.212 5.2.2.6 - 5.2.2.8) ---- */
static const float BETA_ACK[16] = {2.000f, 2.500f, 3.125f, 4.000f, 5.000f, 6.250f, 8.000f, 10.000f, 12.625f, 15.875f, 20.000f, 31.000f, 50.000f, 80.000f, 126.000f, -1.0f};
static const float BETA_RI[16]  = {1.250f, 1.625f, 2.000f, 2.500f, 3.125f, 4.000f, 5.000f, 6.250f, 8.000f, 10.000f, 12.625f, 15.875f, 20.000f, -1.0f, -1.0f, -1.0f};
static const float BETA_CQI[16] = {-1.0f, -1.0f, 1.125f, 1.250f, 1.375f, 1.625f, 1.750f, 2.000f, 2.250f, 2.500f, 2.875f, 3.125f, 3.500f, 4.000f, 5.000f, 6.250f};
void lte_uci_layout(const lte_ul_grant_t* g, lte_uci_layout_t* L)
{
  const uint32_t M = 12 * g->L_prb, nsymb = 12;
  lte_cbsegm_t   sg;
  uint32_t       K = 0;
  memset(L, 0, sizeof(*L));
  if (g->tbs > 0 && lte_cbsegm(&sg, (uint32_t)g->tbs) == 0)
    for (uint32_t r = 0; r < sg.C; r++) K += lte_cb_K(&sg, r);
  if (K) {
    /* Q' = min(ceil(O M_sc N_symb beta / sum K_r), 4 M_sc), evaluated in float like srsRAN's Q_prime_ri_ack */
    if (g->ri_len) {
      float    b = BETA_RI[g->I_offset_ri & 15];
      uint32_t x = (uint32_t)ceilf((float)g->ri_len * (float)M * (float)nsymb * b / (float)K);
      L->Qp_ri   = x < 4 * M ? x : 4 * M;
    }
    if (g->nof_ack) {
      float    b = BETA_ACK[g->I_offset_ack & 15];
      uint32_t x = (uint32_t)ceilf((float)g->nof_ack * (float)M * (float)nsymb * b / (float)K);
      L->Qp_ack  = x < 4 * M ? x : 4 * M;
    }
    if (g->cqi_len) { /* CRC-8 is attached from 12 bits on */
      float    b   = BETA_CQI[g->I_offset_cqi & 15];
      uint32_t Lc  = g->cqi_len <= 11 ? 0 : 8;
      uint32_t x   = (uint32_t)ceilf((float)(g->cqi_len + Lc) * (float)M * (float)nsymb * b / (float)K);
      uint32_t lim = M * nsymb - L->Qp_ri;
      L->Qp_cqi    = x < lim ? x : lim;
    }
  }
  L->G = (M * nsymb - L->Qp_cqi - L->Qp_ri) * g->qm;
}
void lte_uci_map(uint32_t M, const lte_uci_layout_t* L, uint8_t* kind, uint32_t* dpos)
{
  static const uint32_t RI_COL[4] = {1, 4, 7, 10}, ACK_COL[4] = {2, 3, 8, 9}; /* normal CP, 36.212 Tables 5.2.2.8-1 / -2 */
  memset(kind, 0, 12 * M);
  for (uint32_t i = 0, j = 0; i < L->Qp_ri; i++, j = (j + 3) % 4) kind[(M - 1 - i / 4) * 12 + RI_COL[j]] = 2;
  uint32_t k = 0;
  for (uint32_t p = 0; p < 12 * M; p++) {
    if (kind[p] == 2) {
      dpos[p] = 0;
      continue;
    }
    if (k < L->Qp_cqi)
      kind[p] = 1, dpos[p] = k;
    else
      dpos[p] = k - L->Qp_cqi;
    k++;
  }
  for (uint32_t i = 0, j = 0; i < L->Qp_ack; i++, j = (j + 3) % 4) {
    uint32_t p = (M - 1 - i / 4) * 12 + ACK_COL[j];
    if (kind[p] == 0) kind[p] = 3; /* the data symbol is overwritten (an ACK over a CQI symbol cannot happen: Q'_cqi rows come first) */
    else if (kind[p] == 1) kind[p] = 4;
  }
}

/* ---- PBCH / MIB ---- */
uint32_t lte_pbch_re(const lte_cell_t* c, uint16_t* k, uint8_t* l)
{
  const uint32_t nsc = 12 * c->nof_prb, k0 = nsc / 2 - 36;
  uint32_t       n = 0;
  for (uint32_t sym = 7; sym < 11; sym++)
    for (uint32_t kk = k0; kk < k0 + 72; kk++) {
      if (sym < 9 && kk % 3 == c->cell_id % 3) continue; /* CRS of ports 0/1 (symbol 0) and 2/3 (symbol 1), reserved whatever the port count */
      k[n] = (uint16_t)kk, l[n] = (uint8_t)sym;
      n++;
    }
  return n;
}
void lte_mib_pack(uint32_t nof_prb, uint32_t phich_ext, uint32_t phich_res, uint32_t sfn, uint8_t* bits)
{
  static const uint32_t BW[6] = {6, 15, 25, 50, 75, 100};
  uint32_t bw = 0;
  for (uint32_t i = 0; i < 6; i++)
    if (BW[i] == nof_prb) bw = i;
  memset(bits, 0, 24);
  for (int i = 0; i < 3; i++) bits[i] = (bw >> (2 - i)) & 1;
  bits[3] = phich_ext & 1;
  bits[4] = (phich_res >> 1) & 1, bits[5] = phich_res & 1;
  for (int i = 0; i < 8; i++) bits[6 + i] = ((sfn >> 2) >> (7 - i)) & 1;
}
int lte_mib_unpack(const uint8_t* bits, uint32_t* nof_prb, uint32_t* phich_ext, uint32_t* phich_res, uint32_t* sfn)
{
  static const uint32_t BW[8] = {6, 15, 25, 50, 75, 100, 0, 0};
  uint32_t bw = (bits[0] << 2) | (bits[1] << 1) | bits[2], f = 0;
  for (int i = 0; i < 8; i++) f = (f << 1) | bits[6 + i];
  *nof_prb = BW[bw], *phich_ext = bits[3], *phich_res = (bits[4] << 1) | bits[5], *sfn = f << 2;
  return BW[bw] ? 0 : -1;
}
uint32_t lte_pbch_crc_mask(uint32_t nof_ports) { return nof_ports == 1 ? 0x0000u : nof_ports == 2 ? 0xFFFFu : nof_ports == 4 ? 0x5555u : 0u; }

/* ------------------------------------------------------------------ PSS / SSS, 36.211 6.11.1.1 / 6.11.2.1 */
void lte_pss(uint32_t n_id_2, cf_t* d)
{
  static const uint32_t ROOT[3] = {25, 29, 34};
  const uint32_t        u       = ROOT[n_id_2 % 3];
  for (uint32_t n = 0; n < 62; n++) {
    const uint32_t m  = n < 31 ? n * (n + 1) : (n + 1) * (n + 2);
    const double   ph = -M_PI * (double)((u * m) % 126u) / 63.0; /* exp(-j pi u m / 63) */
    d[n]              = (cf_t){(float)cos(ph), (float)sin(ph)};
  }
}

void lte_sss(uint32_t n_id_1, uint32_t n_id_2, uint32_t sf5, float* d)
{
  uint8_t xs[31] = {0, 0, 0, 0, 1}, xc[31] = {0, 0, 0, 0, 1}, xz[31] = {0, 0, 0, 0, 1};
  for (uint32_t i = 0; i + 5 < 31; i++) {
    xs[i + 5] = (xs[i + 2] + xs[i]) & 1;
    xc[i + 5] = (xc[i + 3] + xc[i]) & 1;
    xz[i + 5] = (xz[i + 4] + xz[i + 2] + xz[i + 1] + xz[i]) & 1;
  }
  const uint32_t qp = n_id_1 / 30, q = (n_id_1 + qp * (qp + 1) / 2) / 30, mp = n_id_1 + q * (q + 1) / 2;
  const uint32_t m0 = mp % 31, m1 = (m0 + mp / 31 + 1) % 31;
  for (uint32_t n = 0; n < 31; n++) {
    const int s0 = 1 - 2 * xs[(n + m0) % 31], s1 = 1 - 2 * xs[(n + m1) % 31];
    const int c0 = 1 - 2 * xc[(n + n_id_2) % 31], c1 = 1 - 2 * xc[(n + n_id_2 + 3) % 31];
    const int z0 = 1 - 2 * xz[(n + m0 % 8) % 31], z1 = 1 - 2 * xz[(n + m1 % 8) % 31];
    d[2 * n]     = (float)(sf5 ? s1 * c0 : s0 * c0);
    d[2 * n + 1] = (float)(sf5 ? s0 * c1 * z1 : s1 * c1 * z0);
  }
}
