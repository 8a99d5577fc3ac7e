/* lte_chan_oracle.c -- CPU oracle of the channeliser (DESIGN.md §2 "channeliser").  Tables in double precision rounded to float, then each output
 * as a serial k-ascending sum of separate fp32 products and adds, rotated once: y[m] = r[m mod P] * sum_{k=-H..H} g[k] x[m D - k]. */
#include "lte_chan_oracle.h"
#include <math.h>
#include <stdlib.h>

#define CHAN_MAX_FS 245760000u
#define CHAN_ATTEN 70.0

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

/* the carrier's decimation, filter length and rotation period; 0 or -2 */
static int chan_geometry(uint32_t fs_in, int32_t offset_hz, uint32_t N, uint32_t* T, uint32_t* D, uint32_t* P)
{
  const uint32_t prb = max_prb(N);
  if (!prb || fs_in == 0 || fs_in > CHAN_MAX_FS || offset_hz % 1000) return -2;
  const uint64_t fs_out = 15000ull * N;
  if (fs_in % fs_out) return -2;
  const uint64_t d = fs_in / fs_out;
  if (d < 2 || d > 128) return -2;
  const uint64_t f_pass = 90000ull * prb, aoff = (uint64_t)llabs((long long)offset_hz);
  if (2 * (aoff + f_pass) > fs_in) return -2;
  /* Kaiser's length for 70 dB over the transition band [f_pass, fs_out - f_pass], width relative to fs_in / 2 (scipy.signal.kaiserord), made odd */
  const double width = (double)(fs_out - 2 * f_pass) / (0.5 * (double)fs_in);
  const double nt    = (CHAN_ATTEN - 7.95) / 2.285 / (M_PI * width) + 1.0;
  *T = (uint32_t)ceil(nt) | 1u;
  *D = (uint32_t)d;
  const int64_t step = mod_fs((int64_t)d * offset_hz, fs_in);
  *P = (uint32_t)(fs_in / gcd64(step, fs_in));
  return 0;
}

int lteo_chan_design(uint32_t fs_in, int32_t offset_hz, uint32_t N, float* h, float* g, float* rot, uint32_t* T, uint32_t* D, uint32_t* P)
{
  uint32_t t, d, p;
  if (chan_geometry(fs_in, offset_hz, N, &t, &d, &p)) return -2;
  if (T) *T = t;
  if (D) *D = d;
  if (P) *P = p;
  const int64_t H = (t - 1) / 2, fs = fs_in;
  if (h || g) {
    /* windowed sinc with cutoff fs_out / 2 = fs_in / (2 D), scaled to DC gain 1 (scipy.signal.firwin) */
    double* hd = (double*)malloc(sizeof(double) * t);
    if (!hd) return -1;
    const double beta = 0.1102 * (CHAN_ATTEN - 8.7), a = 0.5 * (double)(t - 1), i0b = bessel_i0(beta), c = 1.0 / (double)d;
    double       s = 0.0;
    for (int64_t j = 0; j < (int64_t)t; j++) {
      const double m  = (double)(j - H) * c;
      const double sn = m == 0.0 ? 1.0 : sin(M_PI * m) / (M_PI * m);
      const double r  = ((double)j - a) / a;
      const double w  = bessel_i0(beta * sqrt(1.0 - r * r)) / i0b;
      hd[j]           = c * sn * w;
      s               = s + hd[j];
    }
    for (int64_t j = 0; j < (int64_t)t; j++) {
      const double hn = hd[j] / s;
      if (h) h[j] = (float)hn;
      if (g) {
        /* g[k] = h[k] e^{+j omega k}, omega = 2 pi offset / fs_in: the phase reduced in integers first */
        const double ph = 2.0 * M_PI * (double)mod_fs((int64_t)offset_hz * (j - H), fs) / (double)fs;
        g[2 * j]        = (float)(hn * cos(ph));
        g[2 * j + 1]    = (float)(hn * sin(ph));
      }
    }
    free(hd);
  }
  if (rot) {
    /* r[i] = e^{-j omega i D} */
    const int64_t step = mod_fs((int64_t)d * offset_hz, fs);
    for (int64_t i = 0; i < (int64_t)p; i++) {
      const double ph = -2.0 * M_PI * (double)((step * i) % fs) / (double)fs;
      rot[2 * i]      = (float)cos(ph);
      rot[2 * i + 1]  = (float)sin(ph);
    }
  }
  return 0;
}

int lteo_chan_run(uint32_t fs_in, uint32_t nof_rx, uint32_t nof_carriers, const int32_t* offset_hz, const uint32_t* N, const float* x, uint64_t first,
                  uint64_t n, float* const* out, uint64_t cap, uint64_t* m_first, uint64_t* count, uint64_t* next)
{
  if (nof_rx < 1 || nof_rx > 2 || nof_carriers < 1 || nof_carriers > 8 || n < 1) return -2;
  uint64_t nx = UINT64_MAX;
  for (uint32_t c = 0; c < nof_carriers; c++) {
    uint32_t T, D, P;
    if (lteo_chan_design(fs_in, offset_hz[c], N[c], NULL, NULL, NULL, &T, &D, &P)) return -2;
    float* g   = (float*)malloc(sizeof(float) * 2 * T);
    float* rot = (float*)malloc(sizeof(float) * 2 * P);
    if (!g || !rot) {
      free(g), free(rot);
      return -1;
    }
    lteo_chan_design(fs_in, offset_hz[c], N[c], NULL, g, rot, &T, &D, &P);
    /* outputs m >= 0 whose window [m D - H, m D + H] has every non-negative sample inside [first, first + n) */
    const uint64_t H = (T - 1) / 2, last = first + n - 1;
    const uint64_t lo = first == 0 ? 0 : (first + H + D - 1) / D;
    const uint64_t hi_n = last >= H ? (last - H) / D + 1 : 0; /* one past the last output */
    const uint64_t cnt = hi_n > lo ? hi_n - lo : 0;
    if (cnt > cap) {
      free(g), free(rot);
      return -1;
    }
    m_first[c] = lo, count[c] = cnt;
    const uint64_t mn = cnt ? hi_n : lo;
    const uint64_t need = mn * D >= H ? mn * D - H : 0;
    if (need < nx) nx = need;
    for (uint32_t a = 0; a < nof_rx; a++) {
      const float* xa = x + 2 * (size_t)a * n;
      float*       ya = out[c] + 2 * (size_t)a * cnt;
      for (uint64_t i = 0; i < cnt; i++) {
        const uint64_t m  = lo + i;
        float          ar = 0.0f, ai = 0.0f;
        for (int64_t j = 0; j < (int64_t)T; j++) { /* k = j - H ascending: sample m D - k */
          const int64_t s = (int64_t)(m * D) + (int64_t)H - j;
          float         xr = 0.0f, xi = 0.0f;
          if (s >= 0) {
            xr = xa[2 * (s - (int64_t)first)];
            xi = xa[2 * (s - (int64_t)first) + 1];
          }
          const float gr = g[2 * j], gi = g[2 * j + 1];
          ar = ar + (gr * xr - gi * xi);
          ai = ai + (gr * xi + gi * xr);
        }
        const float rr = rot[2 * (m % P)], ri = rot[2 * (m % P) + 1];
        ya[2 * i]     = rr * ar - ri * ai;
        ya[2 * i + 1] = rr * ai + ri * ar;
      }
    }
    free(g), free(rot);
  }
  *next = nx;
  return 0;
}
