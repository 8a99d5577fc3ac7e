/* lte_pusch_rx_oracle.c -- PUSCH receive with one or two antennas (lte_pusch_rx_oracle.h, DESIGN.md §2 "uplink receive diversity") */
#include "lte_pusch_rx_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

static float eq_div(float n, float d) { return d == 0.0f ? 0.0f : n / d; } /* no channel on any antenna: 0, not 0/0 = NaN */
static int16_t f2s(float v)
{
  if (isnan(v)) return 0;
  if (v > 32767.0f) v = 32767.0f;
  if (v < -32767.0f) v = -32767.0f;
  return (int16_t)v;
}
/* srsran_demod_soft_demodulate_s, QPSK .. 256QAM */
static void demod_s(cf_t x, uint32_t Qm, int16_t* z)
{
  static const float   scale[4] = {141.421356f, 400.0f, 700.0f, 1000.0f};
  static const int16_t off[4][3] = {{0, 0, 0}, {252, 0, 0}, {432, 216, 0}, {613, 306, 153}};
  const uint32_t       m = Qm / 2 - 1;
  const int16_t        yr = f2s(x.re * scale[m]), yi = f2s(x.im * scale[m]);
  z[0] = (int16_t)-yr, z[1] = (int16_t)-yi;
  for (uint32_t j = 1; j < Qm / 2; j++) {
    z[2 * j]     = (int16_t)(abs(j == 1 ? yr : z[2 * j - 2]) - off[m][j - 1]);
    z[2 * j + 1] = (int16_t)(abs(j == 1 ? yi : z[2 * j - 1]) - off[m][j - 1]);
  }
}

int lteo_pusch_decode_rx(const lte_cell_t* cell, const lte_ul_cfg_t* ucfg, uint32_t sf_idx, const lte_ul_grant_t* g, const cf_t* const* sym,
                         uint32_t nof_rx, uint32_t max_iter, uint8_t* payload, int* crc_ok, lteo_ul_chest_t* chest, int16_t* llr_out, cf_t* eq_out)
{
  static const uint32_t DATA_SYM[12] = {0, 1, 2, 4, 5, 6, 7, 8, 9, 11, 12, 13};
  const uint32_t        M = 12 * g->L_prb, nsc = 12 * cell->nof_prb, Qm = g->qm, A = nof_rx;
  const uint32_t        k0s[2] = {12 * g->n_prb, 12 * (g->hop ? g->n_prb_slot1 : g->n_prb)};
  const int             hop = k0s[0] != k0s[1];
  if (A < 1 || A > 2 || M < 36 || k0s[0] + M > nsc || k0s[1] + M > nsc || !lte_ul_valid_prb(g->L_prb)) return -1;
  lte_uci_layout_t L;
  lte_uci_layout(g, &L);
  const uint32_t G = L.G;
  cf_t*          r   = (cf_t*)malloc(sizeof(cf_t) * M);
  cf_t*          ls  = (cf_t*)malloc(sizeof(cf_t) * 2 * M);
  cf_t*          sm  = (cf_t*)malloc(sizeof(cf_t) * A * 2 * M); /* [a][slot][M] */
  float*         tmp = (float*)malloc(sizeof(float) * M);
  const float    f[3] = {0.3333f, 1.0f - 2.0f * 0.3333f, 0.3333f};
  const float    ncorr = (1.0f - 2.0f * f[1]) + (f[0] * f[0] + f[1] * f[1] + f[2] * f[2]);
  float          pn[2][2], pp[2][2], cr[2][2], ci[2][2]; /* [a][slot] */
  for (uint32_t a = 0; a < A; a++)
    for (uint32_t sl = 0; sl < 2; sl++) {
      if (lte_pusch_dmrs(cell, ucfg, 2 * sf_idx + sl, g->n_dmrs2, M, r)) {
        free(r), free(ls), free(sm), free(tmp);
        return -2;
      }
      cf_t* e = ls + sl * M;
      cf_t* s = sm + (a * 2 + sl) * M;
      for (uint32_t n = 0; n < M; n++) {
        cf_t y  = sym[a][(7 * sl + 3) * nsc + k0s[sl] + n];
        e[n].re = y.re * r[n].re + y.im * r[n].im;
        e[n].im = y.im * r[n].re - y.re * r[n].im;
      }
      for (uint32_t n = 0; n < M; n++) {
        float ar = 0.0f, ai = 0.0f, ws = 0.0f;
        for (int j = 0; j < 3; j++) {
          int nn = (int)n + j - 1;
          if (nn < 0 || nn >= (int)M) continue;
          ar = ar + f[j] * e[nn].re;
          ai = ai + f[j] * e[nn].im;
          ws = ws + f[j];
        }
        s[n].re = ar / ws;
        s[n].im = ai / ws;
      }
      for (uint32_t n = 0; n < M; n++) {
        float dr = e[n].re - s[n].re, di = e[n].im - s[n].im;
        tmp[n]   = dr * dr + di * di;
      }
      pn[a][sl] = lteo_det_sum(tmp, M);
      for (uint32_t n = 0; n < M; n++) tmp[n] = s[n].re * s[n].re + s[n].im * s[n].im;
      pp[a][sl] = lteo_det_sum(tmp, M);
      for (uint32_t n = 0; n + 1 < M; n++) tmp[n] = e[n + 1].re * e[n].re + e[n + 1].im * e[n].im;
      tmp[M - 1] = 0.0f;
      cr[a][sl]  = lteo_det_sum(tmp, M);
      for (uint32_t n = 0; n + 1 < M; n++) tmp[n] = e[n + 1].im * e[n].re - e[n + 1].re * e[n].im;
      ci[a][sl] = lteo_det_sum(tmp, M);
    }
  if (chest) { /* sums antenna-major, then slot; the timing offset from the per-slot correlations summed over the antennas */
    float nsum = 0.0f, psum = 0.0f, ta = 0.0f;
    for (uint32_t a = 0; a < A; a++) nsum = nsum + pn[a][0], nsum = nsum + pn[a][1];
    for (uint32_t a = 0; a < A; a++) psum = psum + pp[a][0], psum = psum + pp[a][1];
    for (uint32_t sl = 0; sl < 2; sl++) {
      float c_r = cr[0][sl], c_i = ci[0][sl];
      for (uint32_t a = 1; a < A; a++) c_r = c_r + cr[a][sl], c_i = c_i + ci[a][sl];
      ta = ta + (-atan2f(c_i, c_r) / 6.28318530717958647692f) / 2.0f;
    }
    chest->noise  = (nsum / (float)(2 * M * A)) / ncorr;
    chest->rsrp   = psum / (float)(2 * M * A);
    chest->snr_db = 10.0f * log10f(chest->rsrp / chest->noise);
    chest->ta_us  = isnormal(ta) ? ta / 15e-3f : 0.0f;
  }
  const float scl  = 1.0f / sqrtf((float)M);
  cf_t*       x    = (cf_t*)malloc(sizeof(cf_t) * M);
  cf_t*       z    = (cf_t*)malloc(sizeof(cf_t) * M);
  int16_t*    e    = (int16_t*)calloc(G + 16, sizeof(int16_t));
  uint8_t*    scr  = (uint8_t*)malloc(12 * M * Qm);
  uint8_t*    kind = (uint8_t*)malloc(12 * M);
  uint32_t*   dpos = (uint32_t*)malloc(sizeof(uint32_t) * 12 * M);
  lte_uci_map(M, &L, kind, dpos);
  lte_gold_bits(((uint32_t)g->rnti << 14) + (sf_idx << 9) + cell->cell_id, scr, 12 * M * Qm);
  for (uint32_t c = 0; c < 12; c++) {
    const uint32_t l = DATA_SYM[c], sl = c / 6, k0 = k0s[sl];
    const float    t = (float)((int)l - 3) / 7.0f;
    for (uint32_t n = 0; n < M; n++) {
      float nr = 0.0f, ni = 0.0f, den = 0.0f;
      for (uint32_t a = 0; a < A; a++) { /* antenna 0's terms start the sums */
        const cf_t* s  = sm + a * 2 * M;
        cf_t        hA = s[n], hB = s[M + n];
        cf_t        h  = hop ? s[sl * M + n] : (cf_t){hA.re + (hB.re - hA.re) * t, hA.im + (hB.im - hA.im) * t};
        cf_t        y  = sym[a][l * nsc + k0 + n];
        float       tr = y.re * h.re + y.im * h.im, ti = y.im * h.re - y.re * h.im, td = h.re * h.re + h.im * h.im;
        nr  = a ? nr + tr : tr;
        ni  = a ? ni + ti : ti;
        den = a ? den + td : td;
      }
      x[n].re = eq_div(nr, den);
      x[n].im = eq_div(ni, den);
    }
    if (eq_out) memcpy(eq_out + c * M, x, sizeof(cf_t) * M);
    lteo_idft(M, x, z);
    for (uint32_t k = 0; k < M; k++) {
      cf_t    zs   = {z[k].re * scl, z[k].im * scl};
      int16_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (z[k].re != 0.0f || z[k].im != 0.0f) demod_s(zs, Qm, v); /* an exactly zero de-precoded sample is an erasure: LLR 0 */
      const uint32_t p = k * 12 + c, kd = kind[p];
      if (kd != 0 && kd != 3) continue; /* CQI / RI symbol */
      for (uint32_t b = 0; b < Qm; b++) {
        uint32_t hb         = (c * M + k) * Qm + b;
        int16_t  d          = scr[hb] ? (int16_t)-v[b] : v[b];
        e[dpos[p] * Qm + b] = kd == 3 ? 0 : d; /* ACK over data: erasure */
      }
    }
  }
  if (llr_out) memcpy(llr_out, e, sizeof(int16_t) * G);
  *crc_ok = lteo_dlsch_decode(e, G, (uint32_t)g->tbs, g->rv, Qm, 1, max_iter, 1, payload, NULL);
  free(r), free(ls), free(sm), free(tmp), free(x), free(z), free(e), free(scr), free(kind), free(dpos);
  return 0;
}
