/*
 * lte_sync_oracle.c -- see lte_sync_oracle.h.
 */
#include "lte_sync_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ================================================================== cell search (DESIGN.md §2, "cell search")
 * Every sum over samples or sub-carriers is a float sum in ascending index order that starts from 0.0f, except the SSS inner sum over the
 * 62 sub-carriers, which is lteo_det_sum.  The tables (replicas, PSS values, DFT twiddles) are computed in double and rounded to float. */
static int sync_symbol_ok(uint32_t N)
{
  const uint32_t M = N % 3 ? N : N / 3;
  return N >= 128 && N <= 2048 && N % 128 == 0 && !(M & (M - 1));
}

/* p_u[k] = (1/sqrt N) sum_n d_u(n) exp(+j 2 pi f_n k / N) over the 62 PSS sub-carriers f_n; E_p = sum_k |p_u[k]|^2 */
static void sync_replicas(uint32_t N, cf_t* rep, float* ep, cf_t* dpss)
{
  const double sc = 1.0 / sqrt((double)N);
  for (uint32_t u = 0; u < 3; u++) {
    cf_t* d = dpss + 62 * u;
    lte_pss(u, d);
    double e = 0.0;
    for (uint32_t k = 0; k < N; k++) {
      double re = 0.0, im = 0.0;
      for (uint32_t n = 0; n < 62; n++) {
        const int64_t  f   = n < 31 ? (int64_t)n - 31 : (int64_t)n - 30;
        const uint32_t idx = (uint32_t)(((f * (int64_t)k) % (int64_t)N + (int64_t)N) % (int64_t)N);
        const double   ph = 2.0 * M_PI * (double)idx / (double)N, c = cos(ph), s = sin(ph);
        re += (double)d[n].re * c - (double)d[n].im * s;
        im += (double)d[n].re * s + (double)d[n].im * c;
      }
      rep[u * N + k] = (cf_t){(float)(re * sc), (float)(im * sc)};
      e += (double)rep[u * N + k].re * rep[u * N + k].re + (double)rep[u * N + k].im * rep[u * N + k].im;
    }
    ep[u] = (float)e;
  }
}

/* m_u(t) = sum_a |c_a|^2 / (E_p sum_a E_a), 0 when the denominator is 0 */
static float sync_metric(const cf_t* x, uint64_t lda, uint32_t A, uint64_t t, const cf_t* p, uint32_t N, float ep)
{
  float P = 0.0f, E = 0.0f;
  for (uint32_t a = 0; a < A; a++) {
    const cf_t* xa = x + a * lda + t;
    float       cr = 0.0f, ci = 0.0f, e = 0.0f;
    for (uint32_t k = 0; k < N; k++) {
      cr = cr + (xa[k].re * p[k].re + xa[k].im * p[k].im);
      ci = ci + (xa[k].im * p[k].re - xa[k].re * p[k].im);
      e  = e + (xa[k].re * xa[k].re + xa[k].im * xa[k].im);
    }
    P = P + (cr * cr + ci * ci);
    E = E + e;
  }
  const float den = ep * E;
  return den == 0.0f ? 0.0f : P / den;
}

/* Y[n] = sum_m x[m] exp(-j 2 pi f_n m / N) over the 62 PSS / SSS sub-carriers, twiddles W[i] = exp(-j 2 pi i / N) */
static void sync_dft62(const cf_t* x, uint32_t N, const cf_t* W, cf_t* Y)
{
  for (uint32_t n = 0; n < 62; n++) {
    const uint32_t f = n < 31 ? N + n - 31 : n - 30;
    float          yr = 0.0f, yi = 0.0f;
    for (uint32_t m = 0; m < N; m++) {
      const cf_t w = W[(uint32_t)(((uint64_t)f * m) % N)];
      yr           = yr + (x[m].re * w.re - x[m].im * w.im);
      yi           = yi + (x[m].re * w.im + x[m].im * w.re);
    }
    Y[n] = (cf_t){yr, yi};
  }
}

int lteo_cell_search(uint32_t N, uint32_t A, const cf_t* x, uint64_t L, lteo_cell_t* out, const lteo_sync_taps_t* taps)
{
  if (!sync_symbol_ok(N) || A < 1 || A > 2 || !x || !out) return -2;
  const uint32_t D = N / 128, NB = LTEO_SYNC_BINS, NR = 2 * D - 1, CP6 = 9 * D; /* CP of symbols 1..6: 144 N / 2048 */
  const uint64_t HF = 75ull * N, FR = 150ull * N;
  if (L < HF + N) return -2;
  const uint64_t J = (L - N) / D + 1; /* coarse offsets whose window fits */
  cf_t*          rep  = (cf_t*)malloc(sizeof(cf_t) * 3 * N);
  cf_t*          W    = (cf_t*)malloc(sizeof(cf_t) * N);
  float*         fold = (float*)malloc(sizeof(float) * 3 * NB);
  float*         sss  = (float*)malloc(sizeof(float) * 3 * 168 * 2);
  float          ep[3], ref[3 * 32], S[3][2];
  cf_t           dpss[3 * 62];
  lteo_cell_t    res[3];
  sync_replicas(N, rep, ep, dpss);
  for (uint32_t i = 0; i < N; i++) {
    const double ph = -2.0 * M_PI * (double)i / (double)N;
    W[i]            = (cf_t){(float)cos(ph), (float)sin(ph)};
  }
  for (uint32_t u = 0; u < 3; u++) {
    const cf_t*  p = rep + u * N;
    lteo_cell_t* o = &res[u];
    memset(o, 0, sizeof(*o));
    o->n_id_2 = (uint8_t)u;
    /* coarse: tau = j D, folded over half-frames (bin j mod 9600), averaged over the windows that fit */
    for (uint32_t b = 0; b < NB; b++) {
      float    sum = 0.0f;
      uint32_t cnt = 0;
      for (uint64_t j = b; j < J; j += NB, cnt++) sum = sum + sync_metric(x, L, A, j * D, p, N, ep[u]);
      fold[u * NB + b] = sum / (float)cnt;
    }
    uint32_t bp = 0;
    for (uint32_t b = 1; b < NB; b++)
      if (fold[u * NB + b] > fold[u * NB + bp]) bp = b; /* ties: lowest bin */
    float side = 0.0f;
    for (uint32_t b = 0; b < NB; b++) {
      const uint32_t d = b > bp ? b - bp : bp - b, dc = d < NB - d ? d : NB - d;
      if (dc > 2 && fold[u * NB + b] > side) side = fold[u * NB + b];
    }
    const float peak = fold[u * NB + bp];
    o->psr           = side > 0.0f ? peak / side : (peak > 0.0f ? INFINITY : 0.0f);
    /* refinement at stride 1 around the coarse peak, circular in the half-frame */
    uint32_t ib = 0;
    uint64_t tau = 0;
    for (uint32_t i = 0; i < NR; i++) {
      const uint64_t t0  = ((uint64_t)bp * D + HF + i - (D - 1)) % HF;
      float          sum = 0.0f;
      uint32_t       cnt = 0;
      for (uint64_t t = t0; t + N <= L; t += HF, cnt++) sum = sum + sync_metric(x, L, A, t, p, N, ep[u]);
      ref[u * 32 + i] = sum / (float)cnt;
      if (i == 0 || ref[u * 32 + i] > ref[u * 32 + ib]) ib = i, tau = t0; /* ties: lowest delta */
    }
    o->pss_peak = ref[u * 32 + ib];
    /* CFO: S = sum_h sum_a c2 conj(c1), the correlation at tau split at N / 2 */
    float sr = 0.0f, si = 0.0f;
    for (uint64_t t = tau; t + N <= L; t += HF)
      for (uint32_t a = 0; a < A; a++) {
        const cf_t* xa = x + a * L + t;
        float       c1r = 0.0f, c1i = 0.0f, c2r = 0.0f, c2i = 0.0f;
        for (uint32_t k = 0; k < N / 2; k++) {
          c1r = c1r + (xa[k].re * p[k].re + xa[k].im * p[k].im);
          c1i = c1i + (xa[k].im * p[k].re - xa[k].re * p[k].im);
        }
        for (uint32_t k = N / 2; k < N; k++) {
          c2r = c2r + (xa[k].re * p[k].re + xa[k].im * p[k].im);
          c2i = c2i + (xa[k].im * p[k].re - xa[k].re * p[k].im);
        }
        sr = sr + (c2r * c1r + c2i * c1i);
        si = si + (c2i * c1r - c2r * c1i);
      }
    S[u][0] = sr, S[u][1] = si;
    o->cfo_re = sr, o->cfo_im = si;
    o->cfo_hz = atan2f(si, sr) * (float)(15000.0 / M_PI);
    /* SSS: every half-frame h whose PSS (tau + h HF) and SSS (N + CP6 earlier) windows lie inside the capture */
    const double phi = 2.0 * M_PI * (double)o->cfo_hz * (double)(N + CP6) / (15000.0 * (double)N);
    const float  rc = (float)cos(phi), rs = (float)-sin(phi); /* exp(-j phi): the channel of the PSS symbol carried back to the SSS symbol */
    float*       Au = sss + u * 336;
    for (uint32_t i = 0; i < 336; i++) Au[i] = 0.0f;
    uint32_t nh = 0;
    for (uint64_t h = 0, tp = tau; tp + N <= L; h++, tp += HF) {
      if (tp < N + CP6) continue;
      cf_t  Yp[62], Ys[62];
      float zr[62], tmp[62], s0[62], s1[62];
      for (uint32_t n = 0; n < 62; n++) zr[n] = 0.0f;
      for (uint32_t a = 0; a < A; a++) {
        sync_dft62(x + a * L + tp, N, W, Yp);
        sync_dft62(x + a * L + tp - N - CP6, N, W, Ys);
        for (uint32_t n = 0; n < 62; n++) {
          const cf_t  d  = dpss[62 * u + n];
          const float hr = Yp[n].re * d.re + Yp[n].im * d.im, hi = Yp[n].im * d.re - Yp[n].re * d.im;
          const float gr = hr * rc - hi * rs, gi = hr * rs + hi * rc;
          zr[n]          = zr[n] + (Ys[n].re * gr + Ys[n].im * gi);
        }
      }
      for (uint32_t n1 = 0; n1 < 168; n1++) {
        lte_sss(n1, u, 0, s0);
        lte_sss(n1, u, 1, s1);
        for (uint32_t n = 0; n < 62; n++) tmp[n] = zr[n] * s0[n];
        const float a0 = lteo_det_sum(tmp, 62);
        for (uint32_t n = 0; n < 62; n++) tmp[n] = zr[n] * s1[n];
        const float a1 = lteo_det_sum(tmp, 62);
        /* hypothesis q: half-frame 0 of the fold is subframe 5 q; half-frame h then carries the SSS of subframe 5 (q xor h mod 2) */
        Au[2 * n1 + 0] = Au[2 * n1 + 0] + ((h & 1) ? a1 : a0);
        Au[2 * n1 + 1] = Au[2 * n1 + 1] + ((h & 1) ? a0 : a1);
      }
      nh++;
    }
    o->nof_half_frames = nh;
    const int64_t s = (int64_t)tau - (int64_t)(13 * N / 2); /* first sample of the subframe whose symbol 6 starts at tau */
    if (nh == 0) {
      o->n_id_1 = 0xFFFF, o->pci = 0xFFFF;
      o->frame_offset = (uint64_t)(((s % (int64_t)FR) + (int64_t)FR) % (int64_t)FR);
      continue;
    }
    uint32_t best = 0;
    for (uint32_t i = 1; i < 336; i++)
      if (Au[i] > Au[best]) best = i; /* ties: lowest N_ID_1, then q = 0 */
    float second = -INFINITY;
    for (uint32_t i = 0; i < 336; i++)
      if (i != best && Au[i] > second) second = Au[i];
    o->n_id_1    = (uint16_t)(best / 2);
    o->pci       = (uint16_t)(3 * (best / 2) + u);
    o->sss_peak  = Au[best];
    o->sss_ratio = second > 0.0f ? Au[best] / second : (Au[best] > 0.0f ? INFINITY : 0.0f);
    const int64_t fs = (best & 1) ? s - (int64_t)HF : s;
    o->frame_offset  = (uint64_t)(((fs % (int64_t)FR) + (int64_t)FR) % (int64_t)FR);
    o->detected      = o->psr >= LTEO_SYNC_PSR_MIN && o->sss_ratio >= LTEO_SYNC_SSS_MIN;
  }
  /* one result per N_ID_2, by pss_peak descending, ties to the lower N_ID_2 */
  uint32_t ord[3] = {0, 1, 2};
  for (uint32_t i = 0; i < 3; i++)
    for (uint32_t j = i + 1; j < 3; j++)
      if (res[ord[j]].pss_peak > res[ord[i]].pss_peak || (res[ord[j]].pss_peak == res[ord[i]].pss_peak && ord[j] < ord[i])) {
        uint32_t t = ord[i];
        ord[i] = ord[j], ord[j] = t;
      }
  for (uint32_t i = 0; i < 3; i++) out[i] = res[ord[i]];
  if (taps) {
    if (taps->coarse) memcpy(taps->coarse, fold, sizeof(float) * 3 * NB);
    if (taps->refined)
      for (uint32_t u = 0; u < 3; u++) memcpy(taps->refined + u * NR, ref + u * 32, sizeof(float) * NR);
    if (taps->cfo) memcpy(taps->cfo, S, sizeof(S));
    if (taps->sss) memcpy(taps->sss, sss, sizeof(float) * 3 * 336);
  }
  free(rep), free(W), free(fold), free(sss);
  return 0;
}
