/*
 * lte_oracle.c -- CPU ORACLE (test infrastructure, parity unpinned; see lte_oracle.h header).
 * Build with -ffp-contract=off: every float expression is evaluated exactly as written.
 */
#include "lte_oracle.h"
#include "../include/lte_tables.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define NPILSYM 4
static const uint32_t PIL_L[NPILSYM] = {0, 4, 7, 11};

struct lteo {
  lte_cell_t cell;
  lte_regs_t regs;
  uint32_t   fft, nsc, sf_len, log2n, sub; /* sub: length of the power-of-two transforms (fft or fft / 3) */
  cf_t*      w3;                        /* radix-3 twiddles of a 3 * 2^k symbol size, NULL otherwise */
  float *    tw_re, *tw_im; /* tw[k] = exp(-2 pi i k / N), k < N/2, rounded from double */
  uint16_t*  bitrev;
  uint32_t   sym_off[14];
  /* CRS pilots [sf_idx 10][port 2][pilsym 4][2*nof_prb] */
  cf_t*   crs;
  float   filt[5];
  float   noise_corr;                   /* 1 - 2 f_c + sum f^2 */
  float   interp_c[17];                 /* (float)j / 6.0f for j = -5..11 */
  uint8_t* pdcch_scr[10];               /* PDCCH scrambling bits per subframe */
  uint8_t  pcfich_scr[10][32];
};

/* ---------------------------------------------------------------- deterministic reduction */
float lteo_det_sum(const float* x, uint32_t n)
{
  float p[32];
  for (uint32_t j = 0; j < 32; j++) {
    float a = 0.0f;
    for (uint32_t i = j; i < n; i += 32) a = a + x[i];
    p[j] = a;
  }
  for (uint32_t off = 16; off >= 1; off >>= 1)
    for (uint32_t j = 0; j < off; j++) p[j] = p[j] + p[j + off];
  return p[0];
}

/* ---------------------------------------------------------------- create */
lteo_t* lteo_create(const lte_cell_t* cell)
{
  lteo_t* q = (lteo_t*)calloc(1, sizeof(*q));
  q->cell   = *cell;
  if (lte_regs_init(&q->regs, cell)) {
    free(q);
    return NULL;
  }
  q->fft    = lte_cell_fft(cell);
  q->nsc    = 12 * cell->nof_prb;
  q->sf_len = 15u * q->fft;
  /* 3 * 2^k symbol sizes (srsRAN's default rates): three power-of-two transforms of length sub = fft / 3 and one radix-3 step */
  q->sub    = q->fft % 3 ? q->fft : q->fft / 3;
  for (q->log2n = 0; (1u << q->log2n) < q->sub; q->log2n++) {
  }
  q->tw_re  = (float*)malloc(sizeof(float) * q->sub / 2);
  q->tw_im  = (float*)malloc(sizeof(float) * q->sub / 2);
  q->bitrev = (uint16_t*)malloc(sizeof(uint16_t) * q->sub);
  for (uint32_t k = 0; k < q->sub / 2; k++) {
    double a    = -2.0 * M_PI * (double)k / (double)q->sub;
    q->tw_re[k] = (float)cos(a);
    q->tw_im[k] = (float)sin(a);
  }
  q->w3 = NULL;
  if (q->sub != q->fft) {
    q->w3 = (cf_t*)malloc(sizeof(cf_t) * 2 * q->fft); /* w3[k] = W_N^k, w3[N + k] = W_N^(2k) */
    for (uint32_t k = 0; k < q->fft; k++)
      for (uint32_t r = 1; r < 3; r++) {
        double a = -2.0 * M_PI * (double)((uint64_t)r * k % q->fft) / (double)q->fft;
        q->w3[(r - 1) * q->fft + k] = (cf_t){(float)cos(a), (float)sin(a)};
      }
  }
  for (uint32_t i = 0; i < q->sub; i++) {
    uint32_t r = 0;
    for (uint32_t b = 0; b < q->log2n; b++)
      if (i & (1u << b)) r |= 1u << (q->log2n - 1 - b);
    q->bitrev[i] = (uint16_t)r;
  }
  uint32_t pos = 0;
  for (uint32_t l = 0; l < 14; l++) {
    pos += lte_cp_len(q->fft, l % 7);
    q->sym_off[l] = pos;
    pos += q->fft;
  }
  q->crs = (cf_t*)malloc(sizeof(cf_t) * 10 * 2 * NPILSYM * 2 * cell->nof_prb);
  for (uint32_t sf = 0; sf < 10; sf++)
    for (uint32_t p = 0; p < 2; p++)
      for (uint32_t li = 0; li < NPILSYM; li++)
        lte_crs(cell, p, 2 * sf + PIL_L[li] / 7, PIL_L[li] % 7, &q->crs[((sf * 2 + p) * NPILSYM + li) * 2 * cell->nof_prb]);
  /* gaussian smoothing filter, order 4 / sigma 1: chest cfg filter_coef {4,1}, src/src/SubframeWorker.cc:379-389 */
  {
    float s = 0.0f;
    for (int i = 0; i < 5; i++) {
      q->filt[i] = (float)exp(-(double)((i - 2) * (i - 2)) / 2.0);
      s          = s + q->filt[i];
    }
    float s2 = 0.0f;
    for (int i = 0; i < 5; i++) {
      q->filt[i] = q->filt[i] / s;
      s2         = s2 + q->filt[i] * q->filt[i];
    }
    q->noise_corr = (1.0f - 2.0f * q->filt[2]) + s2;
  }
  for (int j = -5; j <= 11; j++) q->interp_c[j + 5] = (float)j / 6.0f;
  for (uint32_t sf = 0; sf < 10; sf++) {
    q->pdcch_scr[sf] = (uint8_t*)malloc(LTE_MAX_CCE * 72);
    lte_gold_bits((sf << 9) + cell->cell_id, q->pdcch_scr[sf], LTE_MAX_CCE * 72);
    lte_gold_bits((sf + 1) * (2 * cell->cell_id + 1) * 512u + cell->cell_id, q->pcfich_scr[sf], 32);
  }
  return q;
}
void lteo_destroy(lteo_t* q)
{
  if (!q) return;
  free(q->tw_re), free(q->tw_im), free(q->bitrev), free(q->crs), free(q->w3);
  for (int i = 0; i < 10; i++) free(q->pdcch_scr[i]);
  free(q);
}
uint32_t lteo_nof_cce(lteo_t* q, uint32_t cfi) { return (cfi >= 1 && cfi <= 3) ? q->regs.nof_cce[cfi - 1] : 0; }

/* ---------------------------------------------------------------- K1: OFDM receive
 * restates srsran_ofdm_rx_sf as reached from srsran_ue_dl_decode_fft_estimate (DCISearch.cc:562):
 * CP removed, forward DFT without scaling, guard bands and DC dropped.
 * FFT = iterative radix-2 decimation-in-time, twiddles from the rounded table. */
static void fft_pow2(const lteo_t* q, const cf_t* in, uint32_t stride, float* re, float* im)
{
  uint32_t n = q->sub;
  for (uint32_t i = 0; i < n; i++) {
    re[q->bitrev[i]] = in[i * stride].re;
    im[q->bitrev[i]] = in[i * stride].im;
  }
  for (uint32_t s = 1; s <= q->log2n; s++) {
    uint32_t m = 1u << s, h = m >> 1, step = n / m;
    for (uint32_t j = 0; j < n; j += m)
      for (uint32_t k = 0; k < h; k++) {
        float wr = q->tw_re[k * step], wi = q->tw_im[k * step];
        float br = re[j + k + h], bi = im[j + k + h];
        float tr = wr * br - wi * bi;
        float ti = wr * bi + wi * br;
        float ar = re[j + k], ai = im[j + k];
        re[j + k]     = ar + tr;
        im[j + k]     = ai + ti;
        re[j + k + h] = ar - tr;
        im[j + k + h] = ai - ti;
      }
  }
}
/* X[k] = (F0[k mod M] + W_N^k F1[k mod M]) + W_N^(2k) F2[k mod M], F_r = FFT_M of x[3 m + r] (M = N / 3); plain FFT_N when N is a power of two */
static void fft_fwd(const lteo_t* q, const cf_t* in, float* re, float* im)
{
  if (q->sub == q->fft) {
    fft_pow2(q, in, 1, re, im);
    return;
  }
  const uint32_t N = q->fft, M = q->sub;
  float*         f = (float*)malloc(sizeof(float) * 6 * M);
  for (uint32_t r = 0; r < 3; r++) fft_pow2(q, in + r, 3, f + 2 * r * M, f + (2 * r + 1) * M);
  for (uint32_t k = 0; k < N; k++) {
    const uint32_t kp = k % M;
    const cf_t     w1 = q->w3[k], w2 = q->w3[N + k];
    const float    t1r = w1.re * f[2 * M + kp] - w1.im * f[3 * M + kp], t1i = w1.re * f[3 * M + kp] + w1.im * f[2 * M + kp];
    const float    t2r = w2.re * f[4 * M + kp] - w2.im * f[5 * M + kp], t2i = w2.re * f[5 * M + kp] + w2.im * f[4 * M + kp];
    re[k] = (f[kp] + t1r) + t2r;
    im[k] = (f[M + kp] + t1i) + t2i;
  }
  free(f);
}
void lteo_ofdm_rx(lteo_t* q, const cf_t* iq, cf_t* sym)
{
  float*   re = (float*)malloc(sizeof(float) * q->fft);
  float*   im = (float*)malloc(sizeof(float) * q->fft);
  uint32_t h  = q->nsc / 2;
  for (uint32_t l = 0; l < 14; l++) {
    fft_fwd(q, iq + q->sym_off[l], re, im);
    for (uint32_t k = 0; k < q->nsc; k++) {
      uint32_t bin        = (k < h) ? q->fft - h + k : k - h + 1;
      sym[l * q->nsc + k] = (cf_t){re[bin], im[bin]};
    }
  }
  free(re);
  free(im);
}

/* ---------------------------------------------------------------- K2: channel estimation
 * restates srsran_chest_dl_estimate_cfg with the reference's configuration
 * (src/src/SubframeWorker.cc:376-400): LS at the CRS, gaussian frequency smoothing (edge taps
 * renormalised), noise from LS - smoothed (NOISE_ALG_REFS), linear interpolation in frequency then
 * time (ESTIMATOR_ALG_INTERPOLATE). */
void lteo_chest(lteo_t* q, uint32_t sf_idx, const cf_t* const* sym, cf_t* const* ce, lteo_chest_res_t* res)
{
  const uint32_t N = q->cell.nof_prb, np = 2 * N, nsc = q->nsc;
  cf_t*          ls  = (cf_t*)malloc(sizeof(cf_t) * NPILSYM * np);
  cf_t*          sm  = (cf_t*)malloc(sizeof(cf_t) * NPILSYM * np);
  cf_t*          fi  = (cf_t*)malloc(sizeof(cf_t) * NPILSYM * nsc);
  float*         tmp = (float*)malloc(sizeof(float) * np);
  memset(res, 0, sizeof(*res));
  for (uint32_t p = 0; p < q->cell.nof_ports; p++)
    for (uint32_t a = 0; a < q->cell.nof_rx; a++) {
      float nsum = 0.0f, psum = 0.0f;
      for (uint32_t li = 0; li < NPILSYM; li++) {
        uint32_t    l = PIL_L[li], off = lte_crs_offset(&q->cell, p, l % 7);
        const cf_t* pil = &q->crs[((sf_idx * 2 + p) * NPILSYM + li) * np];
        for (uint32_t m = 0; m < np; m++) {
          cf_t y  = sym[a][l * nsc + 6 * m + off];
          cf_t pl = pil[m];
          ls[li * np + m].re = y.re * pl.re + y.im * pl.im;
          ls[li * np + m].im = y.im * pl.re - y.re * pl.im;
        }
        for (uint32_t m = 0; m < np; m++) {
          float ar = 0.0f, ai = 0.0f, ws = 0.0f;
          for (int j = 0; j < 5; j++) {
            int mm = (int)m + j - 2;
            if (mm < 0 || mm >= (int)np) continue;
            ar = ar + q->filt[j] * ls[li * np + mm].re;
            ai = ai + q->filt[j] * ls[li * np + mm].im;
            ws = ws + q->filt[j];
          }
          sm[li * np + m].re = ar / ws;
          sm[li * np + m].im = ai / ws;
        }
        for (uint32_t m = 0; m < np; m++) {
          float dr = ls[li * np + m].re - sm[li * np + m].re, di = ls[li * np + m].im - sm[li * np + m].im;
          tmp[m]   = dr * dr + di * di;
        }
        nsum = nsum + lteo_det_sum(tmp, np);
        for (uint32_t m = 0; m < np; m++) tmp[m] = sm[li * np + m].re * sm[li * np + m].re + sm[li * np + m].im * sm[li * np + m].im;
        psum = psum + lteo_det_sum(tmp, np);
        /* frequency interpolation */
        for (uint32_t k = 0; k < nsc; k++) {
          int m = ((int)k - (int)off) / 6;
          if ((int)k < (int)off) m = 0;
          if (m > (int)np - 2) m = (int)np - 2;
          int   j = (int)k - (6 * m + (int)off);
          float c = q->interp_c[j + 5];
          cf_t  A = sm[li * np + m], B = sm[li * np + m + 1];
          fi[li * nsc + k].re = A.re + (B.re - A.re) * c;
          fi[li * nsc + k].im = A.im + (B.im - A.im) * c;
        }
      }
      float cnt                = (float)(NPILSYM * np);
      res->noise[p][a]         = (nsum / cnt) / q->noise_corr;
      res->rsrp[p][a]          = psum / cnt;
      if (p == 0 && a == 0) {
        for (uint32_t m = 0; m < np; m++) tmp[m] = ls[0 * np + m].re * ls[2 * np + m].re + ls[0 * np + m].im * ls[2 * np + m].im;
        res->cfo_re = lteo_det_sum(tmp, np);
        for (uint32_t m = 0; m < np; m++) tmp[m] = ls[0 * np + m].re * ls[2 * np + m].im - ls[0 * np + m].im * ls[2 * np + m].re;
        res->cfo_im = lteo_det_sum(tmp, np);
      }
      /* time interpolation */
      cf_t* out = ce[p * q->cell.nof_rx + a];
      for (uint32_t l = 0; l < 14; l++) {
        uint32_t ia, ib;
        float    t;
        if (l < 4)
          ia = 0, ib = 1, t = (float)l / 4.0f;
        else if (l < 7)
          ia = 1, ib = 2, t = (float)(l - 4) / 3.0f;
        else if (l < 11)
          ia = 2, ib = 3, t = (float)(l - 7) / 4.0f;
        else
          ia = 2, ib = 3, t = (float)(l - 11) / 4.0f;
        for (uint32_t k = 0; k < nsc; k++) {
          cf_t A = fi[ia * nsc + k], B = fi[ib * nsc + k];
          if (l < 11) {
            out[l * nsc + k].re = A.re + (B.re - A.re) * t;
            out[l * nsc + k].im = A.im + (B.im - A.im) * t;
          } else {
            out[l * nsc + k].re = B.re + (B.re - A.re) * t;
            out[l * nsc + k].im = B.im + (B.im - A.im) * t;
          }
        }
      }
    }
  float ns = 0.0f, ps = 0.0f;
  for (uint32_t p = 0; p < q->cell.nof_ports; p++)
    for (uint32_t a = 0; a < q->cell.nof_rx; a++) {
      ns = ns + res->noise[p][a];
      ps = ps + res->rsrp[p][a];
    }
  float npa      = (float)(q->cell.nof_ports * q->cell.nof_rx);
  res->noise_avg = ns / npa;
  res->rsrp_avg  = ps / npa;
  res->snr_db    = 10.0f * log10f(res->rsrp_avg / res->noise_avg);
  res->cfo       = atan2f(res->cfo_im, res->cfo_re) / (2.0f * (float)M_PI * 7.5f);
  free(ls), free(sm), free(fi), free(tmp);
}

void lteo_rb_power(lteo_t* q, const cf_t* sym0, float* pwr)
{
  float t[14 * 12];
  for (uint32_t prb = 0; prb < q->cell.nof_prb; prb++) {
    for (uint32_t l = 0; l < 14; l++)
      for (uint32_t k = 0; k < 12; k++) {
        cf_t v        = sym0[l * q->nsc + 12 * prb + k];
        t[l * 12 + k] = v.re * v.re + v.im * v.im;
      }
    pwr[prb] = lteo_det_sum(t, 168) / 168.0f;
  }
}

/* ---------------------------------------------------------------- equalisers (ZF; decoder_type 0, SURVEY App. B.7)
 * an exactly zero denominator (no channel: zero-filled samples, a dead antenna, a singular 2x2) equalises to 0, an erasure, instead of 0/0 = NaN */
static float eq_div(float n, float d) { return d == 0.0f ? 0.0f : n / d; }
static cf_t eq_port0(const lteo_t* q, const cf_t* const* sym, const cf_t* const* ce, uint32_t idx)
{
  float nr = 0.0f, ni = 0.0f, den = 0.0f;
  for (uint32_t a = 0; a < q->cell.nof_rx; a++) {
    cf_t y = sym[a][idx], h = ce[a][idx];
    nr  = nr + (y.re * h.re + y.im * h.im);
    ni  = ni + (y.im * h.re - y.re * h.im);
    den = den + (h.re * h.re + h.im * h.im);
  }
  return (cf_t){eq_div(nr, den), eq_div(ni, den)};
}
/* SFBC pair at grid indices i0, i1 -> x0, x1 (36.211 6.3.4.3 inverted) */
static void eq_sfbc(const lteo_t* q, const cf_t* const* sym, const cf_t* const* ce, uint32_t i0, uint32_t i1, cf_t* x0, cf_t* x1)
{
  const uint32_t A  = q->cell.nof_rx;
  float          n0r = 0.0f, n0i = 0.0f, n1r = 0.0f, n1i = 0.0f, d0 = 0.0f, d1 = 0.0f;
  for (uint32_t a = 0; a < A; a++) {
    cf_t r0 = sym[a][i0], r1 = sym[a][i1];
    cf_t h00 = ce[0 * A + a][i0], h01 = ce[0 * A + a][i1]; /* port 0 at RE0 / RE1 */
    cf_t h10 = ce[1 * A + a][i0], h11 = ce[1 * A + a][i1]; /* port 1 */
    /* x0 += conj(h00) r0 + h11 conj(r1) */
    n0r = n0r + ((h00.re * r0.re + h00.im * r0.im) + (h11.re * r1.re + h11.im * r1.im));
    n0i = n0i + ((h00.re * r0.im - h00.im * r0.re) + (h11.im * r1.re - h11.re * r1.im));
    /* x1 += conj(h01) r1 - h10 conj(r0) */
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
/* 2x2 large-delay CDD zero forcing: r = H (1/2)[[1,1],[s,-s]] x */
static void eq_cdd(const lteo_t* q, const cf_t* const* sym, const cf_t* const* ce, uint32_t idx, int odd, cf_t* x0, cf_t* x1)
{
  (void)q;
  cf_t  r0 = sym[0][idx], r1 = sym[1][idx];
  cf_t  h00 = ce[0][idx], h10 = ce[1][idx]; /* port0: ant0, ant1 */
  cf_t  h01 = ce[2][idx], h11 = ce[3][idx]; /* port1: ant0, ant1 */
  float s = odd ? -1.0f : 1.0f;
  /* E = 2 Heff = [[h00 + s h01, h00 - s h01],[h10 + s h11, h10 - s h11]] */
  cf_t e00 = {h00.re + s * h01.re, h00.im + s * h01.im}, e01 = {h00.re - s * h01.re, h00.im - s * h01.im};
  cf_t e10 = {h10.re + s * h11.re, h10.im + s * h11.im}, e11 = {h10.re - s * h11.re, h10.im - s * h11.im};
  cf_t det = {(e00.re * e11.re - e00.im * e11.im) - (e01.re * e10.re - e01.im * e10.im),
              (e00.re * e11.im + e00.im * e11.re) - (e01.re * e10.im + e01.im * e10.re)};
  cf_t a0  = {(e11.re * r0.re - e11.im * r0.im) - (e01.re * r1.re - e01.im * r1.im),
              (e11.re * r0.im + e11.im * r0.re) - (e01.re * r1.im + e01.im * r1.re)};
  cf_t a1  = {(e00.re * r1.re - e00.im * r1.im) - (e10.re * r0.re - e10.im * r0.im),
              (e00.re * r1.im + e00.im * r1.re) - (e10.re * r0.im + e10.im * r0.re)};
  float dd = det.re * det.re + det.im * det.im;
  /* x = 2 a conj(det) / |det|^2 */
  x0->re = eq_div(a0.re * det.re + a0.im * det.im, dd) * 2.0f;
  x0->im = eq_div(a0.im * det.re - a0.re * det.im, dd) * 2.0f;
  x1->re = eq_div(a1.re * det.re + a1.im * det.im, dd) * 2.0f;
  x1->im = eq_div(a1.im * det.re - a1.re * det.im, dd) * 2.0f;
}

/* closed-loop spatial multiplexing, 2 CRS ports (36.211 Table 6.3.4.2.3-1).  w = second precoder entry:
 * 1 layer: W = (1/sqrt2)[1, w]^T, w in {1,-1,j,-j} (pmi 0..3); 2 layers: W = (1/2)[[1,1],[w,-w]], w in {1, j} (pmi 0,1) */
static void spmux_w(uint32_t nof_layers, uint32_t pmi, float* wr, float* wi)
{
  static const float W1[4][2] = {{1, 0}, {-1, 0}, {0, 1}, {0, -1}};
  static const float W2[2][2] = {{1, 0}, {0, 1}};
  if (nof_layers == 1)
    *wr = W1[pmi & 3][0], *wi = W1[pmi & 3][1];
  else
    *wr = W2[pmi & 1][0], *wi = W2[pmi & 1][1];
}
static cf_t eq_spmux1(const lteo_t* q, const cf_t* const* sym, const cf_t* const* ce, uint32_t idx, float wr, float wi)
{
  const uint32_t A = q->cell.nof_rx;
  float          nr = 0.0f, ni = 0.0f, den = 0.0f;
  for (uint32_t a = 0; a < A; a++) {
    cf_t y = sym[a][idx], h0 = ce[0 * A + a][idx], h1 = ce[1 * A + a][idx];
    cf_t e = {h0.re + (wr * h1.re - wi * h1.im), h0.im + (wr * h1.im + wi * h1.re)};
    nr  = nr + (e.re * y.re + e.im * y.im);
    ni  = ni + (e.re * y.im - e.im * y.re);
    den = den + (e.re * e.re + e.im * e.im);
  }
  const float s2 = 1.41421354f;
  return (cf_t){eq_div(nr, den) * s2, eq_div(ni, den) * s2};
}
/* x = 2 E^-1 r for E = [[e00, e01], [e10, e11]] (rows: rx antennas, columns: layers) */
static void zf2x2(cf_t e00, cf_t e01, cf_t e10, cf_t e11, cf_t r0, cf_t r1, cf_t* x0, cf_t* x1)
{
  cf_t det = {(e00.re * e11.re - e00.im * e11.im) - (e01.re * e10.re - e01.im * e10.im),
              (e00.re * e11.im + e00.im * e11.re) - (e01.re * e10.im + e01.im * e10.re)};
  cf_t a0  = {(e11.re * r0.re - e11.im * r0.im) - (e01.re * r1.re - e01.im * r1.im),
              (e11.re * r0.im + e11.im * r0.re) - (e01.re * r1.im + e01.im * r1.re)};
  cf_t a1  = {(e00.re * r1.re - e00.im * r1.im) - (e10.re * r0.re - e10.im * r0.im),
              (e00.re * r1.im + e00.im * r1.re) - (e10.re * r0.im + e10.im * r0.re)};
  float dd = det.re * det.re + det.im * det.im;
  x0->re = eq_div(a0.re * det.re + a0.im * det.im, dd) * 2.0f;
  x0->im = eq_div(a0.im * det.re - a0.re * det.im, dd) * 2.0f;
  x1->re = eq_div(a1.re * det.re + a1.im * det.im, dd) * 2.0f;
  x1->im = eq_div(a1.im * det.re - a1.re * det.im, dd) * 2.0f;
}
static void eq_spmux2(const cf_t* const* sym, const cf_t* const* ce, uint32_t idx, float wr, float wi, cf_t* x0, cf_t* x1)
{
  cf_t h00 = ce[0][idx], h10 = ce[1][idx], h01 = ce[2][idx], h11 = ce[3][idx]; /* [port*2 + ant] */
  cf_t w0 = {wr * h01.re - wi * h01.im, wr * h01.im + wi * h01.re}; /* w * h(ant0, port1) */
  cf_t w1 = {wr * h11.re - wi * h11.im, wr * h11.im + wi * h11.re};
  cf_t e00 = {h00.re + w0.re, h00.im + w0.im}, e01 = {h00.re - w0.re, h00.im - w0.im};
  cf_t e10 = {h10.re + w1.re, h10.im + w1.im}, e11 = {h10.re - w1.re, h10.im - w1.im};
  zf2x2(e00, e01, e10, e11, sym[0][idx], sym[1][idx], x0, x1);
}

/* equalise n control-channel REs given by grid indices (n multiple of 2 for 2 ports) */
static void eq_ctrl(const lteo_t* q, const cf_t* const* sym, const cf_t* const* ce, const uint32_t* idx, uint32_t n, cf_t* d)
{
  if (q->cell.nof_ports == 1) {
    for (uint32_t i = 0; i < n; i++) d[i] = eq_port0(q, sym, ce, idx[i]);
  } else {
    for (uint32_t i = 0; i + 1 < n; i += 2) eq_sfbc(q, sym, ce, idx[i], idx[i + 1], &d[i], &d[i + 1]);
  }
}

/* ---------------------------------------------------------------- K3: PCFICH (srsran_pcfich_decode) */
uint32_t lteo_pcfich_decode(lteo_t* q, uint32_t sf_idx, const cf_t* const* sym, const cf_t* const* ce, float* corr)
{
  uint32_t idx[16];
  cf_t     d[16];
  float    llr[32];
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) idx[4 * i + j] = q->regs.regs[q->regs.pcfich_reg[i]].k[j]; /* symbol 0 */
  eq_ctrl(q, sym, ce, idx, 16, d);
  const float ms2 = -1.41421354f;
  for (int i = 0; i < 16; i++) {
    llr[2 * i]     = d[i].re * ms2;
    llr[2 * i + 1] = d[i].im * ms2;
  }
  for (int i = 0; i < 32; i++)
    if (q->pcfich_scr[sf_idx][i]) llr[i] = -llr[i];
  uint32_t best = 0;
  for (uint32_t c = 0; c < 3; c++) {
    float acc = 0.0f;
    for (int i = 0; i < 32; i++) acc = acc + (lte_cfi_codeword[c][i] ? llr[i] : -llr[i]);
    corr[c] = acc;
    if (acc > corr[best]) best = c;
  }
  return best + 1;
}

/* ---------------------------------------------------------------- K4: PDCCH LLRs (srsran_pdcch_extract_llr) */
uint32_t lteo_pdcch_extract_llr(lteo_t* q, uint32_t sf_idx, uint32_t cfi, const cf_t* const* sym, const cf_t* const* ce, float* llr)
{
  uint32_t    nof_cce = q->regs.nof_cce[cfi - 1], nq = nof_cce * 9;
  const float ms2     = -1.41421354f;
  for (uint32_t qq = 0; qq < nq; qq++) {
    const lte_reg_t* rg = &q->regs.regs[q->regs.pdcch_map[cfi - 1][qq]];
    uint32_t         idx[4];
    cf_t             d[4];
    for (int j = 0; j < 4; j++) idx[j] = rg->l * q->nsc + rg->k[j];
    eq_ctrl(q, sym, ce, idx, 4, d);
    for (int j = 0; j < 4; j++) {
      float a = d[j].re * ms2, b = d[j].im * ms2;
      llr[8 * qq + 2 * j]     = q->pdcch_scr[sf_idx][8 * qq + 2 * j] ? -a : a;
      llr[8 * qq + 2 * j + 1] = q->pdcch_scr[sf_idx][8 * qq + 2 * j + 1] ? -b : b;
    }
  }
  return nof_cce;
}
/* geometry only: grid index l * nsc + k of every RE lteo_pdcch_extract_llr reads, in its order (test accessor) */
uint32_t lteo_pdcch_re_index(lteo_t* q, uint32_t cfi, uint16_t* idx, uint16_t* pcfich_idx)
{
  uint32_t nq = q->regs.nof_cce[cfi - 1] * 9;
  for (uint32_t qq = 0; qq < nq; qq++) {
    const lte_reg_t* rg = &q->regs.regs[q->regs.pdcch_map[cfi - 1][qq]];
    for (int j = 0; j < 4; j++) idx[4 * qq + j] = (uint16_t)(rg->l * q->nsc + rg->k[j]);
  }
  if (pcfich_idx)
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) pcfich_idx[4 * i + j] = q->regs.regs[q->regs.pcfich_reg[i]].k[j];
  return q->regs.nof_cce[cfi - 1];
}
void lteo_cce_power(const float* llr, uint32_t nof_cce, float* pwr)
{
  for (uint32_t c = 0; c < nof_cce; c++) {
    double m = 0;
    for (int i = 0; i < 72; i++) m += fabsf(llr[c * 72 + i]);
    pwr[c] = (float)(m / 72);
  }
}

/* ---------------------------------------------------------------- K5: DCI decode
 * restates srsran_pdcch_dci_decode (falcon_pdcch.c:142 -> rm_conv_rx + viterbi_decode_f + crc):
 * accumulate-dematch, quantise to uint8 with gain 32/max (falcon_pdcch.c:432 mirrors the constants),
 * K=7 r=1/3 tail-biting Viterbi run over 3 copies keeping the middle one, CRC16 remainder XOR. */
int lteo_dci_decode(const float* e, uint32_t E, uint32_t nof_bits, uint8_t* bits, uint16_t* crc_rem)
{
  const uint32_t K = nof_bits + 16, n3 = 3 * K;
  uint16_t       tab[3 * (LTE_DCI_MAX_BITS + 16)];
  float          rm[3 * (LTE_DCI_MAX_BITS + 16)];
  int            r[3 * (LTE_DCI_MAX_BITS + 16)];
  lte_rm_conv_table(K, tab);
  for (uint32_t i = 0; i < n3; i++) rm[i] = 0.0f;
  for (uint32_t k = 0; k < E; k++) rm[tab[k % n3]] = rm[tab[k % n3]] + e[k];
  float mx = 0.0f;
  for (uint32_t i = 0; i < n3; i++)
    if (fabsf(rm[i]) > mx) mx = fabsf(rm[i]);
  if (!(mx > 0.0f)) return -1;
  float gain = 32.0f / mx;
  for (uint32_t i = 0; i < n3; i++) {
    float v = rm[i] * gain + 127.5f;
    if (!(v >= 0.0f)) v = 0.0f; /* NaN (a NaN soft bit, 0 * an infinite gain, an infinite sum * 0) quantises as fmaxf does: to 0 */
    if (v > 255.0f) v = 255.0f;
    int qv = (int)v;
    r[i]   = 2 * qv - 255;
  }
  /* outputs for (state, input): state bit j = c_{k-1-j} */
  static int8_t sgn[64][2][3];
  static int    init = 0;
  if (!init) {
    for (int s = 0; s < 64; s++)
      for (int c = 0; c < 2; c++) {
#define T(j) ((s >> ((j)-1)) & 1)
        int o0 = c ^ T(2) ^ T(3) ^ T(5) ^ T(6), o1 = c ^ T(1) ^ T(2) ^ T(3) ^ T(6), o2 = c ^ T(1) ^ T(2) ^ T(4) ^ T(6);
#undef T
        sgn[s][c][0] = o0 ? 1 : -1, sgn[s][c][1] = o1 ? 1 : -1, sgn[s][c][2] = o2 ? 1 : -1;
      }
    init = 1;
  }
  const uint32_t T3 = 3 * K;
  int            pm[64], nm[64];
  uint64_t*      dec = (uint64_t*)malloc(sizeof(uint64_t) * T3);
  memset(pm, 0, sizeof(pm));
  for (uint32_t t = 0; t < T3; t++) {
    uint32_t k  = t % K;
    int      r0 = r[k], r1 = r[K + k], r2 = r[2 * K + k];
    uint64_t dw = 0;
    for (int sn = 0; sn < 64; sn++) {
      int c = sn & 1, p0 = sn >> 1, p1 = (sn >> 1) | 32;
      int m0 = pm[p0] + sgn[p0][c][0] * r0 + sgn[p0][c][1] * r1 + sgn[p0][c][2] * r2;
      int m1 = pm[p1] + sgn[p1][c][0] * r0 + sgn[p1][c][1] * r1 + sgn[p1][c][2] * r2;
      if (m1 > m0) {
        nm[sn] = m1;
        dw |= 1ull << sn;
      } else
        nm[sn] = m0;
    }
    memcpy(pm, nm, sizeof(pm));
    dec[t] = dw;
  }
  int best = 0;
  for (int s = 1; s < 64; s++)
    if (pm[s] > pm[best]) best = s;
  uint8_t data[LTE_DCI_MAX_BITS + 16];
  int     st = best;
  for (int t = (int)T3 - 1; t >= (int)K; t--) {
    if (t < (int)(2 * K)) data[t - K] = (uint8_t)(st & 1);
    st = (st >> 1) | ((int)((dec[t] >> st) & 1) << 5);
  }
  free(dec);
  memcpy(bits, data, nof_bits);
  uint32_t p = 0;
  for (uint32_t i = 0; i < 16; i++) p = (p << 1) | data[nof_bits + i];
  *crc_rem = (uint16_t)(p ^ lte_crc(LTE_CRC16, 16, data, nof_bits));
  return 0;
}

/* ---------------------------------------------------------------- K6: PDSCH symbols -> int16 LLRs
 * restates the front half of srsran_pdsch_decode (DL_Sniffer_PDSCH.cc:997): srsran_predecoding_type,
 * layer demapping, srsran_demod_soft_demodulate_s, descrambling. */
static int16_t f2s(float v)
{
  if (isnan(v)) return 0; /* converting NaN to an integer is undefined */
  if (v > 32767.0f) v = 32767.0f;
  if (v < -32767.0f) v = -32767.0f;
  return (int16_t)v; /* truncation toward zero, as the C cast in the int16 demodulator */
}
static void demod_s(cf_t x, uint32_t Qm, int16_t* z)
{
  switch (Qm) {
    case 2:
      z[0] = (int16_t)-f2s(x.re * 141.421356f);
      z[1] = (int16_t)-f2s(x.im * 141.421356f);
      break;
    case 4: {
      int16_t yr = f2s(x.re * 400.0f), yi = f2s(x.im * 400.0f);
      z[0] = (int16_t)-yr, z[1] = (int16_t)-yi;
      z[2] = (int16_t)(abs(yr) - 252), z[3] = (int16_t)(abs(yi) - 252);
    } break;
    case 6: {
      int16_t yr = f2s(x.re * 700.0f), yi = f2s(x.im * 700.0f);
      z[0] = (int16_t)-yr, z[1] = (int16_t)-yi;
      z[2] = (int16_t)(abs(yr) - 432), z[3] = (int16_t)(abs(yi) - 432);
      z[4] = (int16_t)(abs(z[2]) - 216), z[5] = (int16_t)(abs(z[3]) - 216);
    } break;
    default: {
      int16_t yr = f2s(x.re * 1000.0f), yi = f2s(x.im * 1000.0f);
      z[0] = (int16_t)-yr, z[1] = (int16_t)-yi;
      z[2] = (int16_t)(abs(yr) - 613), z[3] = (int16_t)(abs(yi) - 613);
      z[4] = (int16_t)(abs(z[2]) - 306), z[5] = (int16_t)(abs(z[3]) - 306);
      z[6] = (int16_t)(abs(z[4]) - 153), z[7] = (int16_t)(abs(z[5]) - 153);
    } break;
  }
}
int lteo_pdsch_llr(lteo_t* q, uint32_t sf_idx, uint32_t cfi, uint16_t rnti, const lte_dl_grant_t* g, const cf_t* const* sym,
                   const cf_t* const* ce, int16_t* const* llr, cf_t* const* eq_out)
{
  const uint32_t N = q->cell.nof_prb, nsc = q->nsc;
  uint32_t*      idx = (uint32_t*)malloc(sizeof(uint32_t) * (g->nof_re + 16));
  uint16_t       kk[12];
  uint32_t       n = 0;
  for (uint32_t l = 0; l < 14; l++)
    for (uint32_t prb = 0; prb < N; prb++)
      if (g->prb_mask[l / 7][prb]) {
        uint32_t c = lte_pdsch_re_in_prb(&q->cell, sf_idx, cfi, l, prb, kk);
        for (uint32_t i = 0; i < c; i++) idx[n++] = l * nsc + kk[i];
      }
  if (n != g->nof_re) {
    free(idx);
    return -1;
  }
  cf_t* x[2] = {(cf_t*)malloc(sizeof(cf_t) * (n + 2)), (cf_t*)malloc(sizeof(cf_t) * (n + 2))};
  uint32_t ncw = 0, qm[2] = {0, 0};
  for (int t = 0; t < 2; t++)
    if (g->tb[t].enabled) qm[g->cw_swap ? 1 - ncw : ncw] = g->tb[t].qm, ncw++; /* srsran_ra_tb_t.cw_idx (dl_sniffer_pdsch.c:24) */
  if (g->tx_scheme == LTE_TX_PORT0) {
    for (uint32_t i = 0; i < n; i++) x[0][i] = eq_port0(q, sym, ce, idx[i]);
  } else if (g->tx_scheme == LTE_TX_DIVERSITY) {
    for (uint32_t i = 0; i + 1 < n; i += 2) eq_sfbc(q, sym, ce, idx[i], idx[i + 1], &x[0][i], &x[0][i + 1]);
  } else if (g->tx_scheme == LTE_TX_CDD && q->cell.nof_rx == 2 && q->cell.nof_ports == 2) {
    for (uint32_t i = 0; i < n; i++) eq_cdd(q, sym, ce, idx[i], (int)(i & 1), &x[0][i], &x[1][i]);
  } else if (g->tx_scheme == LTE_TX_SPATIALMUX && q->cell.nof_ports == 2 && (g->nof_layers == 1 || q->cell.nof_rx == 2)) {
    float wr, wi;
    spmux_w(g->nof_layers, g->pmi, &wr, &wi);
    if (g->nof_layers == 1)
      for (uint32_t i = 0; i < n; i++) x[0][i] = eq_spmux1(q, sym, ce, idx[i], wr, wi);
    else
      for (uint32_t i = 0; i < n; i++) eq_spmux2(sym, ce, idx[i], wr, wi, &x[0][i], &x[1][i]);
  } else {
    free(idx), free(x[0]), free(x[1]);
    return -2;
  }
  static __thread uint8_t scr[110 * 12 * 14 * 8];
  for (uint32_t cw = 0; cw < ncw; cw++) {
    uint32_t G = n * qm[cw];
    lte_gold_bits(((uint32_t)rnti << 14) + (cw << 13) + (sf_idx << 9) + q->cell.cell_id, scr, G);
    for (uint32_t i = 0; i < n; i++) {
      if (x[cw][i].re == 0.0f && x[cw][i].im == 0.0f) /* an erasure: zero denominator or zero samples -- LLR 0, not the -threshold of the folds */
        memset(&llr[cw][i * qm[cw]], 0, sizeof(int16_t) * qm[cw]);
      else
        demod_s(x[cw][i], qm[cw], &llr[cw][i * qm[cw]]);
    }
    for (uint32_t i = 0; i < G; i++)
      if (scr[i]) llr[cw][i] = (int16_t)-llr[cw][i];
    if (eq_out && eq_out[cw]) memcpy(eq_out[cw], x[cw], sizeof(cf_t) * n);
  }
  free(idx), free(x[0]), free(x[1]);
  return 0;
}

/* ---------------------------------------------------------------- K7: turbo rate de-matching
 * restates srsran_rm_turbo_rx_lut: saturating int16 accumulation into the circular buffer
 * (N_cb = K_w), then de-interleave to the three streams; turbo input conditioning
 * v = clamp(w >> sh(Qm), +-255), sh = {QPSK 0, 16QAM 1, 64QAM 2, 256QAM 2}. */
static int sat16(int v) { return v > 32767 ? 32767 : v < -32768 ? -32768 : v; }
void lteo_rm_turbo_rx_harq(const int16_t* e, uint32_t E, uint32_t K, uint32_t F, uint32_t rv, uint32_t Qm, int16_t* d, int16_t* soft, int combine);
void lteo_rm_turbo_rx(const int16_t* e, uint32_t E, uint32_t K, uint32_t F, uint32_t rv, uint32_t Qm, int16_t* d) { lteo_rm_turbo_rx_harq(e, E, K, F, rv, Qm, d, NULL, 0); }
/* soft != NULL: the circular-buffer accumulators (stream-major, 3 (K + 4) values) live in the caller's HARQ buffer -- cleared first unless
 * combine is set (srsran_softbuffer_rx_reset_tbs for a new transmission, plain accumulation for a retransmission; HARQ.cc:71-135) */
void lteo_rm_turbo_rx_harq(const int16_t* e, uint32_t E, uint32_t K, uint32_t F, uint32_t rv, uint32_t Qm, int16_t* d, int16_t* soft, int combine)
{
  static __thread uint32_t tab[3 * 6176];
  static __thread int16_t  wloc[3 * 6176];
  static __thread uint32_t order[3 * 6176];
  int16_t*                 w = soft ? soft : wloc;
  uint32_t                 Kpi = lte_rm_turbo_table(K, tab), Kw = 3 * Kpi, D = K + 4;
  /* list of transmittable circular-buffer positions in order starting from k0 */
  uint32_t nn = 0, k0 = lte_rm_turbo_k0(K, rv);
  for (uint32_t j = 0; j < Kw; j++) {
    uint32_t pos = (k0 + j) % Kw, t = tab[pos];
    if (t == 0xFFFFFFFFu) continue;
    if (t / D < 2 && t % D < F) continue;
    order[nn++] = t;
  }
  if (!soft || !combine) memset(w, 0, sizeof(int16_t) * 3 * D);
  for (uint32_t k = 0; k < E; k++) {
    uint32_t t = order[k % nn];
    w[t]       = (int16_t)sat16((int)w[t] + (int)e[k]);
  }
  int sh = Qm == 2 ? 0 : Qm == 4 ? 1 : 2;
  for (uint32_t i = 0; i < 3 * D; i++) {
    int v = w[i] >> sh;
    d[i]  = (int16_t)(v > 255 ? 255 : v < -255 ? -255 : v);
  }
  for (uint32_t i = 0; i < F; i++) d[i] = -255, d[D + i] = -255; /* filler bits are known zeros */
}

/* ---------------------------------------------------------------- K8: turbo decoder
 * restates srsran_tdec_* behaviour (max-log-MAP, int16 LLRs, CRC early stop, do-while so at least
 * one iteration) as a windowed decoder: windows of 32 trellis steps, boundary state metrics carried
 * over from the previous iteration (next-iteration initialisation), extrinsic scaled by 3/8 of the
 * doubled-metric difference (= 0.75 of the true extrinsic) and clamped to +-511. */
#define TD_WL 32
#define TD_NINF (-8192)
static const uint8_t TD_NEXT[8][2] = {{0, 4}, {4, 0}, {5, 1}, {1, 5}, {2, 6}, {6, 2}, {7, 3}, {3, 7}};
static const uint8_t TD_PAR[8][2]  = {{0, 1}, {0, 1}, {1, 0}, {1, 0}, {1, 0}, {1, 0}, {0, 1}, {0, 1}};
/* state s = 4 r1 + 2 r2 + r3;  a = u^r2^r3;  z = a^r1^r3;  next = 4a + 2 r1 + r2 */

typedef struct {
  int A[(6144 / TD_WL) + 1][8], B[(6144 / TD_WL) + 1][8];
} td_bound_t;

static void siso(const int* sys, const int* par, const int* apr, uint32_t K, const int tx[3], const int tz[3], td_bound_t* bd,
                 int* ext, int* llr2x)
{
  uint32_t NW = (K + TD_WL - 1) / TD_WL;
  static __thread td_bound_t nb;
  /* beta at K from the tail: beta_{K+3} = state 0 */
  int bt[8], bn[8];
  for (int s = 0; s < 8; s++) bt[s] = s ? TD_NINF : 0;
  for (int k = 2; k >= 0; k--) {
    for (int s = 0; s < 8; s++) {
      int best = -(1 << 30);
      for (int u = 0; u < 2; u++) {
        int g = (u ? tx[k] : -tx[k]) + (TD_PAR[s][u] ? tz[k] : -tz[k]);
        int v = bt[TD_NEXT[s][u]] + g;
        if (v > best) best = v;
      }
      bn[s] = best;
    }
    memcpy(bt, bn, sizeof(bt));
  }
  for (int s = 7; s >= 0; s--) bt[s] -= bt[0];
  for (uint32_t w = 0; w < NW; w++) {
    uint32_t k0 = w * TD_WL, k1 = k0 + TD_WL < K ? k0 + TD_WL : K;
    int      al[TD_WL + 1][8], be[8], t[8];
    if (w == 0)
      for (int s = 0; s < 8; s++) al[0][s] = s ? TD_NINF : 0;
    else
      memcpy(al[0], bd->A[w], sizeof(int) * 8);
    for (uint32_t k = k0; k < k1; k++) {
      int xa = sys[k] + apr[k], p = par[k];
      int* a = al[k - k0];
      for (int s = 0; s < 8; s++) t[s] = -(1 << 30);
      for (int s = 0; s < 8; s++)
        for (int u = 0; u < 2; u++) {
          int g = (u ? xa : -xa) + (TD_PAR[s][u] ? p : -p);
          int v = a[s] + g, n = TD_NEXT[s][u];
          if (v > t[n]) t[n] = v;
        }
      memcpy(al[k - k0 + 1], t, sizeof(t));
    }
    for (int s = 7; s >= 0; s--) nb.A[w + 1][s] = al[k1 - k0][s] - al[k1 - k0][0];
    if (w == NW - 1)
      memcpy(be, bt, sizeof(be));
    else
      memcpy(be, bd->B[w], sizeof(be));
    for (int k = (int)k1 - 1; k >= (int)k0; k--) {
      int  xa = sys[k] + apr[k], p = par[k];
      int* a  = al[k - (int)k0];
      int  m1 = -(1 << 30), m0 = -(1 << 30);
      for (int s = 0; s < 8; s++) {
        int best = -(1 << 30);
        for (int u = 0; u < 2; u++) {
          int g = (u ? xa : -xa) + (TD_PAR[s][u] ? p : -p);
          int v = be[TD_NEXT[s][u]] + g;
          if (v > best) best = v;
          int tot = a[s] + v;
          if (u) {
            if (tot > m1) m1 = tot;
          } else if (tot > m0)
            m0 = tot;
        }
        t[s] = best;
      }
      memcpy(be, t, sizeof(be));
      int L     = m1 - m0;
      llr2x[k]  = L;
      int e     = (3 * (L - 2 * xa)) >> 3;
      ext[k]    = e > 511 ? 511 : e < -511 ? -511 : e;
    }
    if (w > 0)
      for (int s = 7; s >= 0; s--) nb.B[w - 1][s] = be[s] - be[0];
  }
  for (uint32_t w = 1; w < NW; w++) memcpy(bd->A[w], nb.A[w], sizeof(int) * 8);
  for (uint32_t w = 0; w + 1 < NW; w++) memcpy(bd->B[w], nb.B[w], sizeof(int) * 8);
}

uint32_t lteo_turbo_decode(const int16_t* d, uint32_t K, uint32_t max_iter, int crc_type, uint8_t* bits, int* crc_ok)
{
  static __thread int        sys[6144], p1[6144], p2[6144], sysi[6144], apr1[6144], apr2[6144], ext[6144], l2[6144];
  static __thread uint16_t   pi[6144];
  static __thread td_bound_t b1, b2;
  uint32_t                   D = K + 4;
  lte_qpp(K, pi);
  for (uint32_t k = 0; k < K; k++) {
    sys[k] = d[k], p1[k] = d[D + k], p2[k] = d[2 * D + k];
    apr1[k] = 0;
  }
  for (uint32_t i = 0; i < K; i++) sysi[i] = sys[pi[i]];
  /* tails: d0 = xK, zK+1, x'K, z'K+1 ; d1 = zK, xK+2, z'K, x'K+2 ; d2 = xK+1, zK+2, x'K+1, z'K+2 */
  int tx1[3] = {d[K], d[2 * D + K], d[D + K + 1]}, tz1[3] = {d[D + K], d[K + 1], d[2 * D + K + 1]};
  int tx2[3] = {d[K + 2], d[2 * D + K + 2], d[D + K + 3]}, tz2[3] = {d[D + K + 2], d[K + 3], d[2 * D + K + 3]};
  memset(&b1, 0, sizeof(b1));
  memset(&b2, 0, sizeof(b2));
  if (max_iter < 1) max_iter = 1;
  uint32_t it = 0;
  *crc_ok     = 0;
  while (it < max_iter) {
    siso(sys, p1, apr1, K, tx1, tz1, &b1, ext, l2);
    for (uint32_t i = 0; i < K; i++) apr2[i] = ext[pi[i]];
    siso(sysi, p2, apr2, K, tx2, tz2, &b2, ext, l2);
    for (uint32_t i = 0; i < K; i++) {
      apr1[pi[i]] = ext[i];
      bits[pi[i]] = l2[i] > 0;
    }
    it++;
    if (crc_type) {
      uint32_t poly = crc_type == 1 ? LTE_CRC24A : LTE_CRC24B, c = lte_crc(poly, 24, bits, K - 24), r = 0;
      for (uint32_t i = 0; i < 24; i++) r = (r << 1) | bits[K - 24 + i];
      if (c == r) {
        *crc_ok = 1;
        break;
      }
    }
  }
  return it;
}

int lteo_dlsch_decode(const int16_t* e, uint32_t G, uint32_t tbs, uint32_t rv, uint32_t Qm, uint32_t NL, uint32_t max_iter,
                      int early_stop, uint8_t* payload, uint32_t* iters_out)
{
  return lteo_dlsch_decode_harq(e, G, tbs, rv, Qm, NL, max_iter, early_stop, payload, iters_out, NULL, 0);
}
int lteo_dlsch_decode_harq(const int16_t* e, uint32_t G, uint32_t tbs, uint32_t rv, uint32_t Qm, uint32_t NL, uint32_t max_iter, int early_stop,
                           uint8_t* payload, uint32_t* iters_out, int16_t* soft /* C x LTEO_HARQ_CB_STRIDE or NULL */, int combine)
{
  lte_cbsegm_t s;
  if (lte_cbsegm(&s, tbs)) return -1;
  static __thread int16_t d[3 * 6148];
  static __thread uint8_t cb[6144];
  uint8_t*                tb = (uint8_t*)malloc(tbs + 24 + 64);
  uint32_t                rp = 0, wp = 0;
  int                     all_cb_ok = 1;
  for (uint32_t r = 0; r < s.C; r++) {
    uint32_t K = lte_cb_K(&s, r), F = (r == 0) ? s.F : 0, E = lte_rm_turbo_E(G, s.C, r, Qm, NL);
    lteo_rm_turbo_rx_harq(e + rp, E, K, F, rv, Qm, d, soft ? soft + (size_t)r * LTEO_HARQ_CB_STRIDE : NULL, combine);
    rp += E;
    int      ok = 0;
    uint32_t it = lteo_turbo_decode(d, K, max_iter, early_stop ? (s.C > 1 ? 2 : 1) : 0, cb, &ok);
    if (!early_stop && s.C > 1) {
      uint32_t c = lte_crc(LTE_CRC24B, 24, cb, K - 24), rr = 0;
      for (uint32_t i = 0; i < 24; i++) rr = (rr << 1) | cb[K - 24 + i];
      ok = (c == rr);
    }
    if (s.C > 1 && !ok) all_cb_ok = 0;
    if (iters_out) iters_out[r] = it;
    uint32_t nd = K - F - (s.C > 1 ? 24 : 0);
    memcpy(tb + wp, cb + F, nd);
    wp += nd;
  }
  uint32_t c = lte_crc(LTE_CRC24A, 24, tb, tbs), rr = 0;
  for (uint32_t i = 0; i < 24; i++) rr = (rr << 1) | tb[tbs + i];
  lte_bits_pack(tb, tbs, payload);
  free(tb);
  return (c == rr && all_cb_ok) ? 1 : 0;
}

int lteo_pdsch_decode(lteo_t* q, uint32_t sf_idx, uint32_t cfi, uint16_t rnti, const lte_dl_grant_t* g, const cf_t* const* sym,
                      const cf_t* const* ce, uint32_t max_iter, uint8_t* const* payload, int* crc_ok)
{
  int16_t* none[2] = {NULL, NULL};
  int      comb[2] = {0, 0};
  return lteo_pdsch_decode_harq(q, sf_idx, cfi, rnti, g, sym, ce, max_iter, payload, crc_ok, none, comb);
}
int lteo_pdsch_decode_harq(lteo_t* q, uint32_t sf_idx, uint32_t cfi, uint16_t rnti, const lte_dl_grant_t* g, const cf_t* const* sym,
                           const cf_t* const* ce, uint32_t max_iter, uint8_t* const* payload, int* crc_ok, int16_t* const* soft, const int* combine)
{
  int16_t* llr[2] = {(int16_t*)malloc(sizeof(int16_t) * (g->nof_re * 8 + 16)), (int16_t*)malloc(sizeof(int16_t) * (g->nof_re * 8 + 16))};
  int      ret    = lteo_pdsch_llr(q, sf_idx, cfi, rnti, g, sym, ce, llr, NULL);
  if (ret == 0) {
    uint32_t cw = 0;
    for (int t = 0; t < 2; t++) {
      crc_ok[t] = 0;
      if (!g->tb[t].enabled) continue;
      uint32_t NL = g->tx_scheme == LTE_TX_DIVERSITY ? 2 : 1;
      if (g->tb[t].tbs > 0)
        crc_ok[t] = lteo_dlsch_decode_harq(llr[g->cw_swap ? 1 - cw : cw], g->tb[t].nof_bits, (uint32_t)g->tb[t].tbs, g->tb[t].rv, g->tb[t].qm, NL, max_iter,
                                           1, payload[t], NULL, soft[t], combine[t]);
      cw++;
    }
  }
  free(llr[0]), free(llr[1]);
  return ret;
}

/* ---------------------------------------------------------------- whole phase A for one subframe (convenience for the
 * CPU baseline and the end-to-end tests): OFDM rx, channel estimate, PCFICH, PDCCH LLRs. sym/ce are caller buffers. */
int lteo_phase_a(lteo_t* q, const cf_t* iq, uint32_t sf_idx, cf_t* sym /* [nof_rx][14*nsc] */, cf_t* ce /* [ports*rx][14*nsc] */,
                 float* llr /* [88*72] */, lteo_chest_res_t* res, uint32_t* cfi_out)
{
  const uint32_t g = 14 * q->nsc;
  const cf_t*    symp[LTE_MAX_ANT];
  cf_t*          cep[LTE_MAX_PORTS * LTE_MAX_ANT];
  for (uint32_t a = 0; a < q->cell.nof_rx; a++) {
    lteo_ofdm_rx(q, iq + (size_t)a * q->sf_len, sym + (size_t)a * g);
    symp[a] = sym + (size_t)a * g;
  }
  for (uint32_t i = 0; i < q->cell.nof_ports * q->cell.nof_rx; i++) cep[i] = ce + (size_t)i * g;
  lteo_chest(q, sf_idx, symp, cep, res);
  float corr[3];
  *cfi_out = lteo_pcfich_decode(q, sf_idx, symp, (const cf_t* const*)cep, corr);
  return (int)lteo_pdcch_extract_llr(q, sf_idx, *cfi_out, symp, (const cf_t* const*)cep, llr);
}

/* ================================================================== PBCH / MIB, CFO correction (SURVEY 8f-1) */
int lteo_pbch_decode(lteo_t* q, const cf_t* const* sym, const cf_t* const* ce, uint8_t* mib, uint32_t* nof_ports, uint32_t* frame_q)
{
  const lte_cell_t* c = &q->cell;
  uint16_t          ks[240];
  uint8_t           ls[240];
  const uint32_t    nre = lte_pbch_re(c, ks, ls), nsc = q->nsc;
  cf_t              d[240];
  if (c->nof_ports == 1) {
    for (uint32_t i = 0; i < nre; i++) d[i] = eq_port0(q, sym, ce, ls[i] * nsc + ks[i]);
  } else {
    for (uint32_t i = 0; i + 1 < nre; i += 2) eq_sfbc(q, sym, ce, ls[i] * nsc + ks[i], ls[i + 1] * nsc + ks[i + 1], &d[i], &d[i + 1]);
  }
  float   llr[480], e[480];
  uint8_t sc[1920];
  const float ms2 = -1.41421354f;
  for (uint32_t i = 0; i < nre; i++) llr[2 * i] = d[i].re * ms2, llr[2 * i + 1] = d[i].im * ms2;
  lte_gold_bits(c->cell_id, sc, 1920);
  for (uint32_t fq = 0; fq < 4; fq++) {
    for (uint32_t i = 0; i < 480; i++) e[i] = sc[480 * fq + i] ? -llr[i] : llr[i];
    uint8_t  bits[64];
    uint16_t rem = 0;
    if (lteo_dci_decode(e, 480, 24, bits, &rem)) continue;
    const uint32_t np = rem == 0x0000 ? 1 : rem == 0xFFFF ? 2 : rem == 0x5555 ? 4 : 0;
    if (!np) continue;
    memcpy(mib, bits, 24);
    *nof_ports = np, *frame_q = fq;
    return 1;
  }
  return 0;
}
void lteo_cfo_correct(lteo_t* q, float cfo_hz, const cf_t* in, cf_t* out)
{
  for (uint32_t n = 0; n < q->sf_len; n++) {
    double ph = -2.0 * M_PI * (double)cfo_hz * (double)n / (15000.0 * (double)q->fft);
    float  cr = (float)cos(ph), ci = (float)sin(ph);
    out[n]    = (cf_t){in[n].re * cr - in[n].im * ci, in[n].re * ci + in[n].im * cr};
  }
}

/* ================================================================== uplink (PUSCH) */
void lteo_ul_ofdm(lteo_t* q, const cf_t* iq, cf_t* sym)
{
  const uint32_t N = q->fft, h = q->nsc / 2;
  float*         re = (float*)malloc(sizeof(float) * N);
  float*         im = (float*)malloc(sizeof(float) * N);
  cf_t*          x  = (cf_t*)malloc(sizeof(cf_t) * N);
  for (uint32_t l = 0; l < 14; l++) {
    const cf_t* in = iq + q->sym_off[l];
    for (uint32_t n = 0; n < N; n++) { /* multiply by exp(-j pi n / N) */
      double ph = M_PI * (double)n / (double)N;
      float  cr = (float)cos(ph), ci = (float)-sin(ph);
      x[n].re   = in[n].re * cr - in[n].im * ci;
      x[n].im   = in[n].re * ci + in[n].im * cr;
    }
    fft_fwd(q, x, re, im);
    for (uint32_t kk = 0; kk < q->nsc; kk++) {
      uint32_t bin          = (kk + N - h) % N;
      sym[l * q->nsc + kk] = (cf_t){re[bin], im[bin]};
    }
  }
  free(re), free(im), free(x);
}

/* M-point inverse DFT, M = 2^a 3^b 5^c: Stockham autosort, decimation in time, radices in the order 5.., 3.., 4.., 2; every butterfly is the
 * plain sum over its inputs in index order (twiddle first), W[m] = exp(+j 2 pi m / M).  The CUDA kernel evaluates the same expression tree. */
static uint32_t idft_radices(uint32_t M, uint32_t* rad)
{
  uint32_t n = 0;
  while (M % 5 == 0) rad[n++] = 5, M /= 5;
  while (M % 3 == 0) rad[n++] = 3, M /= 3;
  while (M % 4 == 0) rad[n++] = 4, M /= 4;
  if (M % 2 == 0) rad[n++] = 2, M /= 2;
  return M == 1 ? n : 0;
}
static cf_t* idft_mixed(const cf_t* W, uint32_t M, cf_t* a, cf_t* b)
{
  uint32_t rad[16], ns = idft_radices(M, rad), Ns = 1;
  cf_t *   src = a, *dst = b;
  for (uint32_t st = 0; st < ns; st++) {
    const uint32_t R = rad[st], Q = M / R;
    for (uint32_t j = 0; j < Q; j++) {
      const uint32_t k = j % Ns, tstep = k * (M / (Ns * R));
      cf_t           v[5];
      for (uint32_t r = 0; r < R; r++) {
        cf_t x = src[j + r * Q];
        if (r * tstep != 0) {
          cf_t w = W[r * tstep];
          v[r]   = (cf_t){x.re * w.re - x.im * w.im, x.re * w.im + x.im * w.re};
        } else
          v[r] = x;
      }
      const uint32_t o0 = (j / Ns) * Ns * R + k;
      for (uint32_t qq = 0; qq < R; qq++) {
        float ar = v[0].re, ai = v[0].im;
        for (uint32_t r = 1; r < R; r++) {
          cf_t w = W[((r * qq) % R) * Q];
          ar     = ar + (v[r].re * w.re - v[r].im * w.im);
          ai     = ai + (v[r].re * w.im + v[r].im * w.re);
        }
        dst[o0 + qq * Ns] = (cf_t){ar, ai};
      }
    }
    cf_t* t = src;
    src = dst, dst = t, Ns *= R;
  }
  return src;
}
/* test accessor: the M-point inverse DFT of the transform de-precoder exactly as lteo_pusch_decode runs it (unscaled); M = 2^a 3^b 5^c */
int lteo_idft(uint32_t M, const cf_t* in, cf_t* out)
{
  if (!lte_ul_valid_prb(M / 12) || M % 12) return -1;
  cf_t* W = (cf_t*)malloc(sizeof(cf_t) * M);
  cf_t* a = (cf_t*)malloc(sizeof(cf_t) * M);
  cf_t* b = (cf_t*)malloc(sizeof(cf_t) * M);
  for (uint32_t m = 0; m < M; m++) {
    double ph = 2.0 * M_PI * (double)m / (double)M;
    W[m]      = (cf_t){(float)cos(ph), (float)sin(ph)};
  }
  memcpy(a, in, sizeof(cf_t) * M);
  const cf_t* z = idft_mixed(W, M, a, b);
  memcpy(out, z, sizeof(cf_t) * M);
  free(W), free(a), free(b);
  return 0;
}

int lteo_pusch_decode(lteo_t* q, const lte_ul_cfg_t* ucfg, uint32_t sf_idx, const lte_ul_grant_t* g, const cf_t* sym, uint32_t max_iter,
                      uint8_t* payload, int* crc_ok, lteo_ul_chest_t* chest, int16_t* llr_out)
{
  static const uint32_t DATA_SYM[12] = {0, 1, 2, 4, 5, 6, 7, 8, 9, 11, 12, 13};
  const uint32_t        M = 12 * g->L_prb, nsc = q->nsc, Qm = g->qm;
  const uint32_t        k0s[2] = {12 * g->n_prb, 12 * (g->hop ? g->n_prb_slot1 : g->n_prb)};
  const int             hop = k0s[0] != k0s[1];
  lte_uci_layout_t      L;
  lte_uci_layout(g, &L);
  const uint32_t G = L.G;
  if (M < 36 || k0s[0] + M > nsc || k0s[1] + M > nsc || !lte_ul_valid_prb(g->L_prb)) return -1;
  cf_t*  r   = (cf_t*)malloc(sizeof(cf_t) * M);
  cf_t*  ls  = (cf_t*)malloc(sizeof(cf_t) * 2 * M);
  cf_t*  sm  = (cf_t*)malloc(sizeof(cf_t) * 2 * M);
  float* tmp = (float*)malloc(sizeof(float) * M);
  /* smoothing taps (w, 1-2w, w), w = 0.3333 (srsRAN chest_ul default 3-tap filter), edges renormalised */
  const float f[3] = {0.3333f, 1.0f - 2.0f * 0.3333f, 0.3333f};
  const float ncorr = (1.0f - 2.0f * f[1]) + (f[0] * f[0] + f[1] * f[1] + f[2] * f[2]);
  float       nsum = 0.0f, psum = 0.0f, ta = 0.0f;
  for (uint32_t sl = 0; sl < 2; sl++) {
    if (lte_pusch_dmrs(&q->cell, ucfg, 2 * sf_idx + sl, g->n_dmrs2, M, r)) {
      free(r), free(ls), free(sm), free(tmp);
      return -2;
    }
    for (uint32_t n = 0; n < M; n++) {
      cf_t y = sym[(7 * sl + 3) * nsc + k0s[sl] + n];
      ls[sl * M + n].re = y.re * r[n].re + y.im * r[n].im;
      ls[sl * M + n].im = y.im * r[n].re - y.re * r[n].im;
    }
    for (uint32_t n = 0; n < M; n++) {
      float ar = 0.0f, ai = 0.0f, ws = 0.0f;
      for (int j = 0; j < 3; j++) {
        int nn = (int)n + j - 1;
        if (nn < 0 || nn >= (int)M) continue;
        ar = ar + f[j] * ls[sl * M + nn].re;
        ai = ai + f[j] * ls[sl * M + nn].im;
        ws = ws + f[j];
      }
      sm[sl * M + n].re = ar / ws;
      sm[sl * M + n].im = ai / ws;
    }
    for (uint32_t n = 0; n < M; n++) {
      float dr = ls[sl * M + n].re - sm[sl * M + n].re, di = ls[sl * M + n].im - sm[sl * M + n].im;
      tmp[n]   = dr * dr + di * di;
    }
    nsum = nsum + lteo_det_sum(tmp, M);
    for (uint32_t n = 0; n < M; n++) tmp[n] = sm[sl * M + n].re * sm[sl * M + n].re + sm[sl * M + n].im * sm[sl * M + n].im;
    psum = psum + lteo_det_sum(tmp, M);
    /* timing offset from the phase slope of the least-squares estimates (srsran_vec_estimate_frequency over the pilots of one slot, meas_ta_en,
     * UL_Sniffer_PUSCH.cc:424): -arg(sum ls[n+1] conj(ls[n])) / 2 pi, averaged over the slots, / 15e-3 -> microseconds */
    const cf_t* e = ls + sl * M;
    for (uint32_t n = 0; n + 1 < M; n++) tmp[n] = e[n + 1].re * e[n].re + e[n + 1].im * e[n].im;
    tmp[M - 1] = 0.0f;
    float cr = lteo_det_sum(tmp, M);
    for (uint32_t n = 0; n + 1 < M; n++) tmp[n] = e[n + 1].im * e[n].re - e[n + 1].re * e[n].im;
    float ci = lteo_det_sum(tmp, M);
    ta       = ta + (-atan2f(ci, cr) / 6.28318530717958647692f) / 2.0f;
  }
  if (chest) {
    chest->noise  = (nsum / (float)(2 * M)) / ncorr;
    chest->rsrp   = psum / (float)(2 * M);
    chest->snr_db = 10.0f * log10f(chest->rsrp / chest->noise);
    chest->ta_us  = isnormal(ta) ? ta / 15e-3f : 0.0f;
  }
  /* IDFT twiddles W[m] = exp(+j 2 pi m / M) */
  cf_t* W = (cf_t*)malloc(sizeof(cf_t) * M);
  for (uint32_t m = 0; m < M; m++) {
    double ph = 2.0 * M_PI * (double)m / (double)M;
    W[m]      = (cf_t){(float)cos(ph), (float)sin(ph)};
  }
  const float scl = 1.0f / sqrtf((float)M);
  cf_t*       x   = (cf_t*)malloc(sizeof(cf_t) * M);
  cf_t*       x2  = (cf_t*)malloc(sizeof(cf_t) * M);
  int16_t*    e   = (int16_t*)calloc(G + 16, sizeof(int16_t));
  uint8_t*    scr = (uint8_t*)malloc(12 * M * Qm);
  uint8_t*    kind = (uint8_t*)malloc(12 * M);
  uint32_t*   dpos = (uint32_t*)malloc(sizeof(uint32_t) * 12 * M);
  lte_uci_map(M, &L, kind, dpos);
  lte_gold_bits(((uint32_t)g->rnti << 14) + (sf_idx << 9) + q->cell.cell_id, scr, 12 * M * Qm);
  for (uint32_t c = 0; c < 12; c++) {
    const uint32_t l = DATA_SYM[c], sl = c / 6, k0 = k0s[sl];
    const float    t = (float)((int)l - 3) / 7.0f;
    for (uint32_t n = 0; n < M; n++) {
      cf_t A = sm[n], B = sm[M + n];
      cf_t h = hop ? sm[sl * M + n] : (cf_t){A.re + (B.re - A.re) * t, A.im + (B.im - A.im) * t}; /* hopping: each slot stands alone */
      cf_t y = sym[l * nsc + k0 + n];
      float den = h.re * h.re + h.im * h.im;
      x[n].re   = eq_div(y.re * h.re + y.im * h.im, den); /* no channel (zero-filled samples): 0, not 0/0 = NaN */
      x[n].im   = eq_div(y.im * h.re - y.re * h.im, den);
    }
    const cf_t* zt = idft_mixed(W, M, x, x2);
    for (uint32_t k = 0; k < M; k++) {
      cf_t    z    = {zt[k].re * scl, zt[k].im * scl};
      int16_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (zt[k].re != 0.0f || zt[k].im != 0.0f) demod_s(z, Qm, v); /* an exactly zero de-precoded sample is an erasure: LLR 0 */
      const uint32_t p = k * 12 + c, kd = kind[p]; /* row k, column c of the channel interleaver (36.212 5.2.2.8) */
      if (kd != 0 && kd != 3) continue;            /* CQI / RI symbol: not part of the UL-SCH codeword */
      for (uint32_t b = 0; b < Qm; b++) {
        uint32_t hb = (c * M + k) * Qm + b; /* position in the interleaved (transmitted) order */
        int16_t  d  = scr[hb] ? (int16_t)-v[b] : v[b];
        e[dpos[p] * Qm + b] = kd == 3 ? 0 : d; /* an ACK symbol overwrote these coded bits: erasure */
      }
    }
  }
  free(x2), free(kind), free(dpos);
  if (llr_out) memcpy(llr_out, e, sizeof(int16_t) * G);
  *crc_ok = lteo_dlsch_decode(e, G, (uint32_t)g->tbs, g->rv, Qm, 1, max_iter, 1, payload, NULL);
  free(r), free(ls), free(sm), free(tmp), free(W), free(x), free(e), free(scr);
  return 0;
}
