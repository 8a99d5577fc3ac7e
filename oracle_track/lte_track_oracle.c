/*
 * lte_track_oracle.c -- see lte_track_oracle.h.
 */
#include "lte_track_oracle.h"
#include "../oracle/lte_sync_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

struct lteo_track {
  uint32_t    N, A, W, flags, first_tti, pci;
  float       ep, thr;
  lteo_tcf_t* rep;   /* [N] replica of the PSS of N_ID_2 */
  lteo_tcf_t* tabA;  /* [15 N / 128] exp(-j theta 128 i) of the current subframe */
  lteo_tcf_t* tabB;  /* [128]         exp(-j theta j) */
  /* state */
  int64_t  s;        /* start of the next subframe */
  uint32_t k;        /* its number since frame_offset */
  float    f, d, acc; /* carrier offset (Hz), drift (samples per half-frame), fractional step accumulator */
  uint32_t miss, nhf, ncor;
  uint32_t nl;       /* locked half-frames since the last correction */
  int64_t  sd, sh, shh, shd; /* their sums of delta, h, h^2, h delta (h: half-frame number) */
  int64_t  base;     /* start of subframe 0 of the drift estimate's grid: frame_offset, after a find s' - k' 15 N */
  /* find state (LTEO_TRACK_REACQUIRE) */
  int      find;     /* searching: no subframe is cut */
  int64_t  f0;       /* first sample of the next find window */
  uint32_t kn;       /* subframe number predicted at f0 */
  int      reacq;    /* the next subframe cut is the first after a successful find */
  uint32_t finds;    /* find windows searched */
  lteo_tcf_t* win;   /* [A][150 N + N] copy of a find window */
  /* uplink carrier (lteo_track_set_ul) */
  int      pushed;   /* a push was accepted: the uplink can no longer be set */
  int      ul;       /* set: pushes go through lteo_track_push_ul */
  double   ul_ratio; /* f_UL / f_DL */
  int32_t  ul_off;   /* UL subframe start - DL subframe start */
  uint32_t ul_A;     /* UL antennas */
};

static int track_symbol_ok(uint32_t N)
{
  const uint32_t M = N % 3 ? N : N / 3;
  return N >= 128 && N <= 2048 && N % 128 == 0 && !(M & (M - 1));
}

lteo_track_t* lteo_track_create(uint32_t N, uint32_t A, uint32_t pci, uint32_t first_tti, uint64_t frame_offset, float cfo_hz, uint32_t flags)
{
  if (!track_symbol_ok(N) || A < 1 || A > 2 || pci > 503 || first_tti > 10239 || !(fabsf(cfo_hz) <= 7500.0f)) return NULL;
  if (flags & ~(LTEO_TRACK_NO_CFO | LTEO_TRACK_REACQUIRE)) return NULL;
  lteo_track_t* t = (lteo_track_t*)calloc(1, sizeof(*t));
  t->N = N, t->A = A, t->W = 9 * N / 128, t->flags = flags, t->first_tti = first_tti, t->pci = pci, t->base = (int64_t)frame_offset;
  t->rep  = (lteo_tcf_t*)malloc(sizeof(lteo_tcf_t) * N);
  t->tabA = (lteo_tcf_t*)malloc(sizeof(lteo_tcf_t) * (15 * N / 128));
  t->tabB = (lteo_tcf_t*)malloc(sizeof(lteo_tcf_t) * 128);
  if (flags & LTEO_TRACK_REACQUIRE) t->win = (lteo_tcf_t*)malloc(sizeof(lteo_tcf_t) * A * (151 * N));
  /* d_u(n) = exp(-j pi u m / 63) (36.211 6.11.1.1); p[k] = (1/sqrt N) sum_n d_u(n) exp(+j 2 pi f_n k / N); E_p = sum_k |p[k]|^2; all in double */
  static const uint32_t ROOT[3] = {25, 29, 34};
  double                dr[62], di[62];
  for (uint32_t n = 0; n < 62; n++) {
    const uint32_t m  = n < 31 ? n * (n + 1) : (n + 1) * (n + 2);
    const double   ph = -M_PI * (double)((ROOT[pci % 3] * m) % 126u) / 63.0;
    dr[n] = (double)(float)cos(ph), di[n] = (double)(float)sin(ph);
  }
  const double sc = 1.0 / sqrt((double)N);
  double       e  = 0.0;
  for (uint32_t k = 0; k < N; k++) {
    double re = 0.0, im = 0.0;
    for (uint32_t n = 0; n < 62; n++) {
      const int64_t  f   = n < 31 ? (int64_t)n - 31 : (int64_t)n - 30;
      const uint32_t idx = (uint32_t)(((f * (int64_t)k) % (int64_t)N + (int64_t)N) % (int64_t)N);
      const double   ph = 2.0 * M_PI * (double)idx / (double)N, c = cos(ph), s = sin(ph);
      re += dr[n] * c - di[n] * s;
      im += dr[n] * s + di[n] * c;
    }
    t->rep[k] = (lteo_tcf_t){(float)(re * sc), (float)(im * sc)};
    e += (double)t->rep[k].re * t->rep[k].re + (double)t->rep[k].im * t->rep[k].im;
  }
  t->ep  = (float)e;
  t->thr = LTEO_TRACK_LOCK_K / (float)N;
  t->s   = (int64_t)frame_offset;
  t->f   = cfo_hz;
  return t;
}

void lteo_track_destroy(lteo_track_t* t)
{
  if (!t) return;
  free(t->rep), free(t->tabA), free(t->tabB), free(t->win), free(t);
}

/* the cell search's stride-1 metric: sum_a |c_a|^2 / (E_p sum_a E_a), every sum ascending from 0.0f; 0 when the denominator is 0 */
static float track_metric(const lteo_tcf_t* x, uint64_t lda, uint32_t A, uint64_t t, const lteo_tcf_t* p, uint32_t N, float ep)
{
  float P = 0.0f, E = 0.0f;
  for (uint32_t a = 0; a < A; a++) {
    const lteo_tcf_t* xa = x + a * lda + t;
    float             cr = 0.0f, ci = 0.0f, e = 0.0f;
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

/* one half-frame at the expected PSS position tau (relative to x): argmax over delta = 0, -1, +1, -2, +2, ... (ties: smallest |delta|, then the
 * negative side), then S = sum_a c2 conj(c1) at the argmax, with the correlation split at N / 2 */
static void track_measure(const lteo_track_t* t, const lteo_tcf_t* x, uint64_t lda, uint64_t tau, lteo_track_hf_t* o)
{
  const uint32_t N = t->N;
  int32_t        best = 0;
  float          peak = track_metric(x, lda, t->A, tau, t->rep, N, t->ep);
  for (int32_t m = 1; m <= (int32_t)t->W; m++)
    for (int32_t sg = -1; sg <= 1; sg += 2) {
      const float v = track_metric(x, lda, t->A, tau + (int64_t)(sg * m), t->rep, N, t->ep);
      if (v > peak) peak = v, best = sg * m;
    }
  float sr = 0.0f, si = 0.0f;
  for (uint32_t a = 0; a < t->A; a++) {
    const lteo_tcf_t* xa = x + a * lda + (int64_t)tau + best;
    float             c1r = 0.0f, c1i = 0.0f, c2r = 0.0f, c2i = 0.0f;
    for (uint32_t k = 0; k < N / 2; k++) {
      c1r = c1r + (xa[k].re * t->rep[k].re + xa[k].im * t->rep[k].im);
      c1i = c1i + (xa[k].im * t->rep[k].re - xa[k].re * t->rep[k].im);
    }
    for (uint32_t k = N / 2; k < N; k++) {
      c2r = c2r + (xa[k].re * t->rep[k].re + xa[k].im * t->rep[k].im);
      c2i = c2i + (xa[k].im * t->rep[k].re - xa[k].re * t->rep[k].im);
    }
    sr = sr + (c2r * c1r + c2i * c1i);
    si = si + (c2i * c1r - c2r * c1i);
  }
  o->delta  = best;
  o->peak   = peak;
  o->s_re   = sr, o->s_im = si;
  o->f_meas = atan2f(si, sr) * (float)(15000.0 / M_PI);
}

/* y[n] = x[n] exp(-j theta n), theta = 2 pi f / (15000 N), n = 128 i + j: the factors exp(-j theta 128 i) and exp(-j theta j) in double, rounded
 * to float, multiplied in float (a b), then x (a b) */
static void track_cut(lteo_track_t* t, const lteo_tcf_t* x, uint64_t lda, uint32_t A, float f, uint64_t s, lteo_tcf_t* out)
{
  const uint32_t N = t->N, SF = 15 * N;
  const double   th = 2.0 * M_PI * (double)f / (15000.0 * (double)N);
  for (uint32_t i = 0; i < SF / 128; i++) t->tabA[i] = (lteo_tcf_t){(float)cos(-th * 128.0 * (double)i), (float)sin(-th * 128.0 * (double)i)};
  for (uint32_t j = 0; j < 128; j++) t->tabB[j] = (lteo_tcf_t){(float)cos(-th * (double)j), (float)sin(-th * (double)j)};
  for (uint32_t a = 0; a < A; a++) {
    const lteo_tcf_t* xa = x + a * lda + s;
    lteo_tcf_t*       ya = out + (uint64_t)a * SF;
    for (uint32_t n = 0; n < SF; n++) {
      const lteo_tcf_t A = t->tabA[n >> 7], B = t->tabB[n & 127];
      const float      rr = A.re * B.re - A.im * B.im, ri = A.re * B.im + A.im * B.re;
      ya[n] = (lteo_tcf_t){xa[n].re * rr - xa[n].im * ri, xa[n].re * ri + xa[n].im * rr};
    }
  }
}

int lteo_track_set_ul_rx(lteo_track_t* t, double cfo_ratio, int32_t ul_offset, uint32_t nof_rx)
{
  if (!t || t->pushed || t->ul || !(cfo_ratio > 0.0 && cfo_ratio <= 2.0) || nof_rx > 2) return -2;
  if ((int64_t)(ul_offset < 0 ? -(int64_t)ul_offset : ul_offset) >= 15 * (int64_t)t->N || t->base + ul_offset < 0) return -2;
  t->ul = 1, t->ul_ratio = cfo_ratio, t->ul_off = ul_offset, t->ul_A = nof_rx ? nof_rx : 1;
  return 0;
}
int lteo_track_set_ul(lteo_track_t* t, double cfo_ratio, int32_t ul_offset) { return lteo_track_set_ul_rx(t, cfo_ratio, ul_offset, 1); }

/* the lowest absolute sample the pending DL window, and with the uplink set its UL window, still needs; in the find state the window's start */
static int64_t track_needed(const lteo_track_t* t)
{
  const int64_t s = t->find ? t->f0 : t->s;
  return t->ul && t->ul_off < 0 ? s + t->ul_off : s;
}

uint32_t lteo_track_finds(const lteo_track_t* t) { return t ? t->finds : 0; }

/* one find window [f0, f0 + FR + N) (DESIGN.md §2, "tracking"): the cell search on exactly these samples, the result of N_ID_2 = pci mod 3.  Found:
 * resume at the first subframe boundary of the window with the subframe number its SSS gives; otherwise step to the next frame. */
static void track_find(lteo_track_t* t, const lteo_tcf_t* x, uint64_t first, uint64_t n)
{
  const uint32_t N = t->N, SF = 15 * N;
  const uint64_t FR = 150ull * N, L = FR + N;
  for (uint32_t a = 0; a < t->A; a++) memcpy(t->win + a * L, x + a * n + (uint64_t)(t->f0 - (int64_t)first), sizeof(lteo_tcf_t) * L);
  lteo_cell_t res[3];
  lteo_cell_search(N, t->A, (const cf_t*)t->win, L, res, NULL);
  t->finds++;
  const lteo_cell_t* c = NULL;
  for (uint32_t i = 0; i < 3; i++)
    if (res[i].n_id_2 == t->pci % 3) c = &res[i];
  if (!c->detected || c->pci != t->pci) {
    t->f0 += (int64_t)FR, t->kn += 10;
    return;
  }
  const uint64_t fo   = c->frame_offset;
  const uint32_t sfno = (uint32_t)((10 - fo / SF) % 10);
  const uint32_t k    = t->kn + (sfno + 10 - (t->first_tti + t->kn) % 10) % 10;
  t->s = t->f0 + (int64_t)(fo % SF), t->k = k;
  if (!(t->flags & LTEO_TRACK_NO_CFO)) t->f = c->cfo_hz;
  t->miss = 0, t->acc = 0.0f;
  t->nl = 0, t->sd = t->sh = t->shh = t->shd = 0, t->ncor = 0;
  t->base = t->s - (int64_t)k * SF, t->nhf = 0; /* the drift d is kept: a clock does not change with a gap */
  t->find = 0, t->reacq = 1;
}

/* a subframe is processed only when its DL window (and its UL window) lie inside first .. first + n - 1 */
static int track_fits(const lteo_track_t* t, uint64_t first, uint64_t n)
{
  const uint32_t SF = 15 * t->N;
  if (!(t->s >= (int64_t)first && (uint64_t)t->s + SF <= first + n)) return 0;
  if (!t->ul) return 1;
  const int64_t su = t->s + t->ul_off;
  return su >= (int64_t)first && (uint64_t)su + SF <= first + n;
}

static int track_push(lteo_track_t* t, const lteo_tcf_t* x, const lteo_tcf_t* xu, uint64_t first, uint64_t n, uint32_t max_sf, lteo_track_sf_t* sf,
                      uint32_t* nsf, lteo_track_hf_t* hf, uint32_t* nhf, lteo_tcf_t* cut, lteo_tcf_t* cut_ul, uint64_t* next)
{
  if (!t || !x || !sf || !nsf || !hf || !nhf || !next || (int64_t)first > track_needed(t)) return -2;
  const uint32_t N = t->N, SF = 15 * N, P = LTEO_TRACK_P;
  uint32_t       ns = 0, nh = 0;
  t->pushed = 1;
  while (ns < max_sf) {
    if (t->find) { /* a window is searched once all of its samples have been fed */
      if ((uint64_t)t->f0 + 151ull * N > first + n) break;
      track_find(t, x, first, n);
      continue;
    }
    if (!track_fits(t, first, n)) break;
    const uint64_t   s   = (uint64_t)t->s - first;
    const uint32_t   tti = (t->first_tti + t->k) % 10240;
    lteo_track_sf_t* o   = &sf[ns];
    memset(o, 0, sizeof(*o));
    o->start  = t->s, o->tti = tti, o->cfo_hz = t->f, o->index = t->k;
    o->flags  = (t->miss == 0 ? LTEO_TRACK_LOCKED : 0) | (t->miss >= LTEO_TRACK_MISS ? LTEO_TRACK_LOST : 0) | (t->reacq ? LTEO_TRACK_REACQUIRED : 0);
    t->reacq  = 0;
    if (cut) track_cut(t, x, n, t->A, t->f, s, cut + (uint64_t)ns * t->A * SF);
    /* UL: every UL antenna at start + ul_offset, rotated by f_ul = (float)(f cfo_ratio) with the DL rule */
    if (xu && cut_ul)
      track_cut(t, xu, n, t->ul_A, (float)((double)t->f * t->ul_ratio), (uint64_t)(t->s + t->ul_off) - first, cut_ul + (uint64_t)ns * t->ul_A * SF);
    ns++;
    int lost_now = 0;
    if (tti % 5 == 0) {
      lteo_track_hf_t* h = &hf[nh++];
      memset(h, 0, sizeof(*h));
      h->tau   = t->s + 13 * N / 2;
      h->index = t->k;
      track_measure(t, x, n, s + 13 * N / 2, h);
      const int64_t hn = t->nhf++;
      if (h->peak >= t->thr) {
        h->flags |= LTEO_TRACK_LOCKED;
        t->miss = 0;
        if (!(t->flags & LTEO_TRACK_NO_CFO)) t->f = t->f + LTEO_TRACK_ALPHA * (h->f_meas - t->f);
        t->nl++, t->sd += h->delta, t->sh += hn, t->shh += hn * hn, t->shd += hn * h->delta;
        if (t->nl == P) {
          const int64_t c = t->sd >= 0 ? (t->sd + P / 2) / P : -((-t->sd + P / 2) / P);
          t->s += c;
          t->ncor++;
          if (t->ncor == 1) { /* first correction: the least-squares slope of delta over the half-frame numbers */
            const int64_t num = (int64_t)P * t->shd - t->sh * t->sd, den = (int64_t)P * t->shh - t->sh * t->sh;
            t->d = t->d + (float)num / (float)den;
          } else { /* then: the whole movement of the start beyond the nominal grid over the half-frames seen, less half a correction period */
            const int64_t moved = t->s - t->base - (int64_t)t->k * SF;
            t->d = (float)moved / ((float)t->nhf - 0.5f * (float)(P - 1));
          }
          t->nl = 0, t->sd = t->sh = t->shh = t->shd = 0;
        }
      } else
        lost_now = ++t->miss == LTEO_TRACK_MISS;
      if (t->miss >= LTEO_TRACK_MISS) h->flags |= LTEO_TRACK_LOST;
    }
    t->acc         = t->acc + t->d / 5.0f;
    const float r  = roundf(t->acc);
    t->acc         = t->acc - r;
    t->s           = t->s + SF + (int64_t)r;
    t->k++;
    if (lost_now && (t->flags & LTEO_TRACK_REACQUIRE)) t->find = 1, t->f0 = t->s, t->kn = t->k;
  }
  *nsf = ns, *nhf = nh, *next = (uint64_t)track_needed(t);
  return 0;
}

int lteo_track_push(lteo_track_t* t, const lteo_tcf_t* x, uint64_t first, uint64_t n, uint32_t max_sf, lteo_track_sf_t* sf, uint32_t* nsf,
                    lteo_track_hf_t* hf, uint32_t* nhf, lteo_tcf_t* cut, uint64_t* next)
{
  if (t && t->ul) return -2;
  return track_push(t, x, NULL, first, n, max_sf, sf, nsf, hf, nhf, cut, NULL, next);
}

int lteo_track_push_ul(lteo_track_t* t, const lteo_tcf_t* x, const lteo_tcf_t* x_ul, uint64_t first, uint64_t n, uint32_t max_sf, lteo_track_sf_t* sf,
                       uint32_t* nsf, lteo_track_hf_t* hf, uint32_t* nhf, lteo_tcf_t* cut, lteo_tcf_t* cut_ul, uint64_t* next)
{
  if (!t || !t->ul || !x_ul) return -2;
  return track_push(t, x, x_ul, first, n, max_sf, sf, nsf, hf, nhf, cut, cut_ul, next);
}
