/* lte_mib_oracle.c -- PBCH soft bits per port count and the srsRAN-style combiner across the 40 ms period (lte_mib_oracle.h, DESIGN.md §2). */
#include "lte_mib_oracle.h"
#include <stdlib.h>
#include <string.h>

/* the zero-forcing equalisers of lte_oracle.c (static there), same operation order: an exactly zero denominator equalises to 0 */
static float eq_div(float n, float d) { return d == 0.0f ? 0.0f : n / d; }
static cf_t eq_port0(uint32_t A, const cf_t* const* sym, const cf_t* const* ce, uint32_t idx)
{
  float nr = 0.0f, ni = 0.0f, den = 0.0f;
  for (uint32_t a = 0; a < A; a++) {
    cf_t y = sym[a][idx], h = ce[a][idx];
    nr  = nr + (y.re * h.re + y.im * h.im);
    ni  = ni + (y.im * h.re - y.re * h.im);
    den = den + (h.re * h.re + h.im * h.im);
  }
  return (cf_t){eq_div(nr, den), eq_div(ni, den)};
}
static void eq_sfbc(uint32_t A, const cf_t* const* sym, const cf_t* const* ce, uint32_t i0, uint32_t i1, cf_t* x0, cf_t* x1)
{
  float n0r = 0.0f, n0i = 0.0f, n1r = 0.0f, n1i = 0.0f, d0 = 0.0f, d1 = 0.0f;
  for (uint32_t a = 0; a < A; a++) {
    cf_t r0 = sym[a][i0], r1 = sym[a][i1];
    cf_t h00 = ce[0 * A + a][i0], h01 = ce[0 * A + a][i1];
    cf_t h10 = ce[1 * A + a][i0], h11 = ce[1 * A + a][i1];
    n0r = n0r + ((h00.re * r0.re + h00.im * r0.im) + (h11.re * r1.re + h11.im * r1.im));
    n0i = n0i + ((h00.re * r0.im - h00.im * r0.re) + (h11.im * r1.re - h11.re * r1.im));
    n1r = n1r + ((h01.re * r1.re + h01.im * r1.im) - (h10.re * r0.re + h10.im * r0.im));
    n1i = n1i + ((h01.re * r1.im - h01.im * r1.re) - (h10.im * r0.re - h10.re * r0.im));
    d0  = d0 + ((h00.re * h00.re + h00.im * h00.im) + (h11.re * h11.re + h11.im * h11.im));
    d1  = d1 + ((h01.re * h01.re + h01.im * h01.im) + (h10.re * h10.re + h10.im * h10.im));
  }
  const float s2 = 1.41421354f;
  x0->re = eq_div(n0r, d0) * s2;
  x0->im = eq_div(n0i, d0) * s2;
  x1->re = eq_div(n1r, d1) * s2;
  x1->im = eq_div(n1i, d1) * s2;
}

int lteo_pbch_llr(const lte_cell_t* c, const cf_t* const* sym, const cf_t* const* ce, uint32_t nant, float* llr)
{
  if (nant < 1 || nant > 2 || nant > c->nof_ports) return -1;
  uint16_t       ks[240];
  uint8_t        ls[240];
  const uint32_t nre = lte_pbch_re(c, ks, ls), nsc = 12 * c->nof_prb;
  cf_t           d[240];
  if (nant == 1) {
    for (uint32_t i = 0; i < nre; i++) d[i] = eq_port0(c->nof_rx, sym, ce, ls[i] * nsc + ks[i]);
  } else {
    for (uint32_t i = 0; i + 1 < nre; i += 2) eq_sfbc(c->nof_rx, sym, ce, ls[i] * nsc + ks[i], ls[i + 1] * nsc + ks[i + 1], &d[i], &d[i + 1]);
  }
  const float ms2 = -1.41421354f;
  for (uint32_t i = 0; i < nre; i++) llr[2 * i] = d[i].re * ms2, llr[2 * i + 1] = d[i].im * ms2;
  return 0;
}

struct lteo_mib {
  lte_cell_t cell;
  uint8_t    scr[1920];        /* c(cell_id) over the four frames of the period */
  float      buf[2][4][480];   /* [nant - 1][frame] soft bits, oldest frame first */
  uint32_t   frame_idx;        /* frames held */
  int32_t    last_sfn;         /* SFN of the last frame consumed, -1 after a reset */
};

lteo_mib_t* lteo_mib_create(const lte_cell_t* cell)
{
  if (cell->nof_ports < 1 || cell->nof_ports > 2) return NULL;
  lteo_mib_t* q = (lteo_mib_t*)calloc(1, sizeof(lteo_mib_t));
  if (!q) return NULL;
  q->cell = *cell;
  lte_gold_bits(cell->cell_id, q->scr, 1920);
  lteo_mib_reset(q);
  return q;
}
void lteo_mib_destroy(lteo_mib_t* q) { free(q); }
void lteo_mib_reset(lteo_mib_t* q)
{
  q->frame_idx = 0;
  q->last_sfn  = -1;
}

int lteo_mib_decode(lteo_mib_t* q, uint32_t tti, const cf_t* const* sym, const cf_t* const* ce, int search_ports, lteo_mib_res_t* res)
{
  memset(res, 0, sizeof(*res));
  const int32_t sfn = (int32_t)((tti / 10) % 1024);
  if (q->frame_idx && sfn != (q->last_sfn + 1) % 1024) lteo_mib_reset(q); /* a gap: the held frames are not the ones before this one */
  q->last_sfn = sfn;
  for (uint32_t p = 0; p < q->cell.nof_ports; p++) lteo_pbch_llr(&q->cell, sym, ce, p + 1, q->buf[p][q->frame_idx]);
  q->frame_idx++;
  uint32_t tries[2], ntries = 0;
  if (search_ports)
    for (uint32_t p = 1; p <= q->cell.nof_ports; p++) tries[ntries++] = p;
  else
    tries[ntries++] = q->cell.nof_ports;
  float e[1920];
  for (uint32_t t = 0; t < ntries; t++) {
    const uint32_t nant = tries[t];
    const uint16_t mask = nant == 1 ? 0x0000 : 0xFFFF;
    for (uint32_t nb = 0; nb < q->frame_idx; nb++)
      for (uint32_t dst = 0; dst < 4 - nb; dst++)
        for (uint32_t src = 0; src < q->frame_idx - nb; src++) {
          memset(e, 0, sizeof(e)); /* the positions of absent frames stay 0 (srsRAN's RX_NULL) */
          for (uint32_t j = 0; j <= nb; j++) {
            const float*   x   = q->buf[nant - 1][src + j];
            const uint8_t* scr = q->scr + 480 * (dst + j);
            for (uint32_t i = 0; i < 480; i++) e[480 * (dst + j) + i] = scr[i] ? -x[i] : x[i];
          }
          uint8_t  bits[64];
          uint16_t rem = 0;
          if (lteo_dci_decode(e, 1920, 24, bits, &rem)) continue;
          if (rem != mask) continue;
          res->found = 1, res->nof_ports = (uint8_t)nant, res->nof_frames = (uint8_t)(nb + 1), res->src = (uint8_t)src, res->dst = (uint8_t)dst;
          res->window     = (uint8_t)q->frame_idx;
          res->sfn_offset = (uint8_t)(dst - src + q->frame_idx - 1);
          memcpy(res->mib, bits, 24);
          uint32_t msb = 0;
          for (uint32_t i = 6; i < 14; i++) msb = (msb << 1) | bits[i];
          res->sfn = ((msb << 2) + res->sfn_offset) % 1024;
          q->frame_idx = 0; /* a success resets the buffers; the SFN stays, so the next frame is still checked against it */
          return 1;
        }
  }
  if (q->frame_idx == 4) { /* nothing passed with a full buffer: drop the oldest frame */
    for (uint32_t p = 0; p < q->cell.nof_ports; p++) memmove(q->buf[p][0], q->buf[p][1], 3 * 480 * sizeof(float));
    q->frame_idx = 3;
  }
  return 0;
}
