/* lte_chan_poly_oracle.c -- CPU oracle of the channeliser's rational carriers and integer sample formats (DESIGN.md §2 "channeliser").  Tables
 * in double precision rounded to float, then each output as a serial k-ascending sum of separate fp32 products and adds, rotated once:
 * y[m] = r[m mod P] * sum_{k=-Kb..Ka} g_phi[k] x[n - k], n = floor(m M / L), phi = m M mod L.  Integer carriers are lteo_chan_design's. */
#include "lte_chan_poly_oracle.h"
#include "lte_chan_oracle.h"
#include <math.h>
#include <stdlib.h>

#define CHAN_MAX_FS 245760000u
#define CHAN_ATTEN 70.0
#define CHAN_MAX_L 1024u
#define CHAN_MAX_TABLE 32768u

/* largest PRB count a symbol size carries: the pass band is 90 kHz per PRB */
static uint32_t max_prb(uint32_t N)
{
  switch (N) {
    case 128: return 6;
    case 256: return 15;
    case 384: case 512: return 25;
    case 768: case 1024: return 50;
    case 1536: case 2048: return 100;
    default: return 0;
  }
}

/* modified Bessel function I0, power series summed until the term no longer changes the sum */
static double bessel_i0(double x)
{
  double s = 1.0, t = 1.0, q = 0.25 * x * x;
  for (int k = 1; k < 500; k++) {
    t = t * q / ((double)k * (double)k);
    s = s + t;
    if (t < 1e-17 * s) break;
  }
  return s;
}

static int64_t mod_fs(int64_t a, int64_t fs) { return ((a % fs) + fs) % fs; }

static int64_t gcd64(int64_t a, int64_t b)
{
  while (b) {
    const int64_t t = a % b;
    a = b, b = t;
  }
  return a;
}

/* geometry of a rational carrier: L, M, Tp, Ka, Kb, Kp and P; 0 or -2 */
static int poly_geometry(uint32_t fs_in, int32_t offset_hz, uint32_t N, lteo_chan_poly_t* q)
{
  const uint32_t prb = max_prb(N);
  if (!prb || fs_in == 0 || fs_in > CHAN_MAX_FS || offset_hz % 1000) return -2;
  const int64_t fs_out = 15000ll * N, gg = gcd64(fs_out, fs_in), L = fs_out / gg, M = fs_in / gg;
  if (L > CHAN_MAX_L || M > 128 * L || L > 2 * M) return -2;
  const int64_t f_pass = 90000ll * prb, aoff = llabs((long long)offset_hz), mn = fs_out < (int64_t)fs_in ? fs_out : (int64_t)fs_in;
  if (2 * (aoff + f_pass) > (int64_t)fs_in) return -2;
  if (mn <= 2 * f_pass) return -2; /* no transition band [f_pass, min(fs_in, fs_out) - f_pass] */
  /* Kaiser's length for 70 dB over [f_pass, min(fs_in, fs_out) - f_pass] at the prototype's rate L fs_in, made odd */
  const double width = (double)(mn - 2 * f_pass) / (0.5 * (double)(L * (int64_t)fs_in));
  const double nt    = (CHAN_ATTEN - 7.95) / 2.285 / (M_PI * width) + 1.0;
  const int64_t tp = (int64_t)ceil(nt) | 1, hp = (tp - 1) / 2;
  const int64_t ka = hp / L, kb = (hp + L - 1) / L;
  if (L * (ka + kb + 1) > CHAN_MAX_TABLE) return -2;
  q->L = (uint32_t)L, q->M = (uint32_t)M, q->Tp = (uint32_t)tp, q->Ka = (uint32_t)ka, q->Kb = (uint32_t)kb, q->Kp = (uint32_t)(ka + kb + 1);
  q->P = (uint32_t)(fs_out / gcd64(mod_fs(offset_hz, fs_out), fs_out));
  return 0;
}

int lteo_chan_design_poly(uint32_t fs_in, int32_t offset_hz, uint32_t N, uint32_t flags, lteo_chan_poly_t* out, float* hp, float* g, float* rot)
{
  if (flags & ~(uint32_t)LTEO_CHAN_RATIONAL) return -2;
  lteo_chan_poly_t q;
  uint32_t         T, D, P;
  if (lteo_chan_design(fs_in, offset_hz, N, NULL, NULL, NULL, &T, &D, &P) == 0) { /* an integer carrier: lteo_chan_design's rule and tables */
    q.L = 1, q.M = D, q.Tp = T, q.Kp = T, q.Ka = (T - 1) / 2, q.Kb = (T - 1) / 2, q.P = P;
    if (out) *out = q;
    return (hp || g || rot) ? lteo_chan_design(fs_in, offset_hz, N, hp, g, rot, &T, &D, &P) : 0;
  }
  if (!(flags & LTEO_CHAN_RATIONAL) || poly_geometry(fs_in, offset_hz, N, &q)) return -2;
  if (out) *out = q;
  const int64_t L = q.L, Hp = (q.Tp - 1) / 2, Lfs = L * (int64_t)fs_in, fs_out = 15000ll * N;
  if (hp || g) {
    /* windowed sinc with cutoff min(fs_in, fs_out) / 2 at rate L fs_in, scaled to DC gain L */
    double* hd = (double*)malloc(sizeof(double) * q.Tp);
    if (!hd) return -1;
    const double beta = 0.1102 * (CHAN_ATTEN - 8.7), a = 0.5 * (double)(q.Tp - 1), i0b = bessel_i0(beta);
    const double c = 1.0 / (double)(q.L > q.M ? q.L : q.M);
    double       s = 0.0;
    for (int64_t j = 0; j < (int64_t)q.Tp; j++) {
      const double m  = (double)(j - Hp) * c;
      const double sn = m == 0.0 ? 1.0 : sin(M_PI * m) / (M_PI * m);
      const double r  = ((double)j - a) / a;
      const double w  = bessel_i0(beta * sqrt(1.0 - r * r)) / i0b;
      hd[j]           = c * sn * w;
      s               = s + hd[j];
    }
    const double sl = s / (double)L;
    for (int64_t j = 0; j < (int64_t)q.Tp; j++) hd[j] = hd[j] / sl;
    if (hp)
      for (int64_t j = 0; j < (int64_t)q.Tp; j++) hp[j] = (float)hd[j];
    if (g) /* g_phi[k] at [phi][k + Kb]: hp[Hp + phi + L k] e^{+j 2 pi offset (phi + L k) / (L fs_in)}, zero outside the prototype */
      for (int64_t ph = 0; ph < L; ph++)
        for (int64_t k = -(int64_t)q.Kb; k <= (int64_t)q.Ka; k++) {
          const int64_t idx = Hp + ph + L * k;
          const double  tap = idx >= 0 && idx < (int64_t)q.Tp ? hd[idx] : 0.0;
          const double  a2  = 2.0 * M_PI * (double)mod_fs((int64_t)offset_hz * (ph + L * k), Lfs) / (double)Lfs;
          float*        o   = g + 2 * ((size_t)ph * q.Kp + (size_t)(k + q.Kb));
          o[0]              = (float)(tap * cos(a2));
          o[1]              = (float)(tap * sin(a2));
        }
    free(hd);
  }
  if (rot) {
    /* r[i] = e^{-j 2 pi offset i / fs_out} */
    const int64_t step = mod_fs(offset_hz, fs_out);
    for (int64_t i = 0; i < (int64_t)q.P; i++) {
      const double ph = -2.0 * M_PI * (double)((step * i) % fs_out) / (double)fs_out;
      rot[2 * i]      = (float)cos(ph);
      rot[2 * i + 1]  = (float)sin(ph);
    }
  }
  return 0;
}

/* sample s (0-based in the call) of antenna a, converted to cf32 */
static void load_iq(uint32_t fmt, const void* x, uint64_t n, uint32_t a, int64_t s, float* re, float* im)
{
  const size_t i = 2 * ((size_t)a * n + (size_t)s);
  if (fmt == LTEO_IQ_SC16) {
    *re = (float)((const int16_t*)x)[i] * (1.0f / 32768.0f);
    *im = (float)((const int16_t*)x)[i + 1] * (1.0f / 32768.0f);
  } else if (fmt == LTEO_IQ_SC8) {
    *re = (float)((const int8_t*)x)[i] * (1.0f / 128.0f);
    *im = (float)((const int8_t*)x)[i + 1] * (1.0f / 128.0f);
  } else {
    *re = ((const float*)x)[i];
    *im = ((const float*)x)[i + 1];
  }
}

int lteo_chan_run_poly(uint32_t fs_in, uint32_t flags, uint32_t iq_format, uint32_t nof_rx, uint32_t nof_carriers, const int32_t* offset_hz,
                       const uint32_t* N, const void* x, uint64_t first, uint64_t n, float* const* out, uint64_t cap, uint64_t* m_first, uint64_t* count,
                       uint64_t* next)
{
  if (nof_rx < 1 || nof_rx > 2 || nof_carriers < 1 || nof_carriers > 8 || n < 1 || iq_format > LTEO_IQ_SC8) return -2;
  uint64_t nx = UINT64_MAX;
  for (uint32_t c = 0; c < nof_carriers; c++) {
    lteo_chan_poly_t q;
    if (lteo_chan_design_poly(fs_in, offset_hz[c], N[c], flags, &q, NULL, NULL, NULL)) return -2;
    float* g   = (float*)malloc(sizeof(float) * 2 * (size_t)q.L * q.Kp);
    float* rot = (float*)malloc(sizeof(float) * 2 * q.P);
    if (!g || !rot) {
      free(g), free(rot);
      return -1;
    }
    lteo_chan_design_poly(fs_in, offset_hz[c], N[c], flags, &q, NULL, g, rot);
    /* outputs m >= 0 whose window [n - Ka, n + Kb], n = floor(m M / L), has every non-negative sample inside [first, first + n) */
    const unsigned __int128 L = q.L, M = q.M, last = first + n - 1;
    const uint64_t lo   = first == 0 ? 0 : (uint64_t)(((first + q.Ka) * L + M - 1) / M);
    const uint64_t hi_n = last >= q.Kb ? (uint64_t)(((last - q.Kb + 1) * L - 1) / M + 1) : 0; /* one past the last output */
    const uint64_t cnt  = hi_n > lo ? hi_n - lo : 0;
    if (cnt > cap) {
      free(g), free(rot);
      return -1;
    }
    m_first[c] = lo, count[c] = cnt;
    const uint64_t mn = cnt ? hi_n : lo, nn = (uint64_t)(mn * M / L);
    const uint64_t need = nn >= q.Ka ? nn - q.Ka : 0;
    if (need < nx) nx = need;
    for (uint32_t a = 0; a < nof_rx; a++) {
      float* ya = out[c] + 2 * (size_t)a * cnt;
      for (uint64_t i = 0; i < cnt; i++) {
        const unsigned __int128 mm = lo + i;
        const int64_t  s0 = (int64_t)(mm * M / L);
        const uint32_t ph = (uint32_t)(mm * M % L);
        const float*   gp = g + 2 * (size_t)ph * q.Kp;
        float          ar = 0.0f, ai = 0.0f;
        for (int64_t k = -(int64_t)q.Kb; k <= (int64_t)q.Ka; k++) { /* k ascending: sample n - k */
          const int64_t s = s0 - k;
          float         xr = 0.0f, xi = 0.0f;
          if (s >= 0) load_iq(iq_format, x, n, a, s - (int64_t)first, &xr, &xi);
          const float gr = gp[2 * (k + q.Kb)], gi = gp[2 * (k + q.Kb) + 1];
          ar = ar + (gr * xr - gi * xi);
          ai = ai + (gr * xi + gi * xr);
        }
        const uint64_t r  = (uint64_t)(mm % q.P);
        const float    rr = rot[2 * r], ri = rot[2 * r + 1];
        ya[2 * i]     = rr * ar - ri * ai;
        ya[2 * i + 1] = rr * ai + ri * ar;
      }
    }
    free(g), free(rot);
  }
  *next = nx;
  return 0;
}
