// chan.cu -- host side of the channeliser (include/ltephy_b200.h, DESIGN.md §2 "channeliser"): the per-carrier filter design in double precision,
// the output range of a call, and one launch of k_chan.cu over every (carrier, antenna, tile).  An integer carrier is computed as the rational
// one at L = 1, M = D; the tables equal lteo_chan_design's and lteo_chan_design_poly's bit for bit.
#include "../../include/ltephy_b200.h"
#include "k_chan.cuh"
#include "ltephy_internal.cuh"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

#define CHAN_ATTEN 70.0  // stop-band target (dB) of Kaiser's formulas
#define CHAN_SPAN 4096   // input samples an integer tile aims to stage: R = min(1024, max(64, (CHAN_SPAN - T) / D + 1)) outputs
#define CHAN_PSPAN 12288 // input samples a rational tile may stage: R = (CHAN_PSPAN - Kp) / M rows per phase class, at least 1
#define CHAN_MAX_L 1024u
#define CHAN_MAX_TABLE 32768u

struct ltephy_chan {
  ltephy_chan_cfg_t cfg{};
  Stream            stream;
  struct Carrier {
    ltephy_chan_poly_t q{};
    uint32_t           R = 0, Q = 0, rows = 0; // tiles of L R outputs, their span staged in Q phases of rows samples (ChanSeg)
    uint64_t           cap = 0;                // outputs per antenna the buffer holds
    DevBuf<float2>     g, rot, out;
  } car[LTEPHY_CHAN_MAX_CARRIERS];
  DevBuf<float2> d_x;
  size_t         smem = 0;
};

static size_t chan_sample_bytes(uint32_t fmt) { return fmt == LTEPHY_IQ_SC16 ? 4 : fmt == LTEPHY_IQ_SC8 ? 2 : 8; }

static uint32_t chan_max_prb(uint32_t N)
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

static double chan_i0(double x) // modified Bessel function I0, power series until the term no longer changes the sum
{
  double s = 1.0, t = 1.0, q = 0.25 * x * x;
  for (int k = 1; k < 500; k++) {
    t = t * q / ((double)k * (double)k);
    s = s + t;
    if (t < 1e-17 * s) break;
  }
  return s;
}

static int64_t chan_mod(int64_t a, int64_t fs) { return ((a % fs) + fs) % fs; }

static int64_t chan_gcd(int64_t a, int64_t b)
{
  while (b) {
    const int64_t t = a % b;
    a = b, b = t;
  }
  return a;
}

// geometry of a carrier under the plan's flags (DESIGN.md §2): fs_out / fs_in = L / M in lowest terms; an integer decimation D = 2..128 is L = 1,
// M = D, Tp = Kp = T, Ka = Kb = H, flag or not, and with LTEPHY_CHAN_RATIONAL any other ratio within the limits is accepted.  0, or
// INVALID_INPUTS with the reason in the last error
static int chan_geometry(uint32_t fs_in, int32_t offset_hz, uint32_t N, uint32_t flags, ltephy_chan_poly_t* q)
{
  const uint32_t prb = chan_max_prb(N);
  if (!prb) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: symbol size %u not supported", N);
  if (fs_in == 0 || fs_in > LTEPHY_CHAN_MAX_FS) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: fs_in %u outside 1..245760000", fs_in);
  if (offset_hz % 1000) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: offset %d Hz is not a multiple of 1 kHz", offset_hz);
  const int64_t fs_out = 15000ll * N, gg = chan_gcd(fs_out, fs_in), L = fs_out / gg, M = fs_in / gg;
  if (!(L == 1 && M >= 2 && M <= 128)) {
    if (!(flags & LTEPHY_CHAN_RATIONAL))
      return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: fs_in %u / %lld is not an integer decimation 2..128", fs_in, (long long)fs_out);
    if (L > CHAN_MAX_L) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: fs_out / fs_in = %lld / %lld, L above 1024", (long long)L, (long long)M);
    if (M > 128 * L) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: fs_out / fs_in = %lld / %lld is below 1 / 128", (long long)L, (long long)M);
    if (L > 2 * M) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: fs_out / fs_in = %lld / %lld upsamples more than 2x", (long long)L, (long long)M);
  }
  const int64_t f_pass = 90000ll * prb, aoff = std::llabs((long long)offset_hz), mn = std::min<int64_t>(fs_out, fs_in);
  if (2 * (aoff + f_pass) > (int64_t)fs_in)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: band of the carrier at %d Hz (N %u) reaches outside the capture", offset_hz, N);
  if (mn <= 2 * f_pass) // the transition band [f_pass, min(fs_in, fs_out) - f_pass] would be empty, and Kaiser's length infinite
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: carrier at %d Hz (N %u) leaves no transition band: min(fs_in, fs_out) %lld <= 2 f_pass %lld", offset_hz,
                N, (long long)mn, (long long)(2 * f_pass));
  // Kaiser's length for 70 dB over [f_pass, min(fs_in, fs_out) - f_pass] at the prototype's rate L fs_in (scipy.signal.kaiserord), made odd
  const double  width = (double)(mn - 2 * f_pass) / (0.5 * (double)(L * (int64_t)fs_in));
  const double  nt    = (CHAN_ATTEN - 7.95) / 2.285 / (M_PI * width) + 1.0;
  const int64_t tp = (int64_t)std::ceil(nt) | 1, hp = (tp - 1) / 2, ka = hp / L, kb = (hp + L - 1) / L;
  if (L * (ka + kb + 1) > CHAN_MAX_TABLE)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: phase table of %lld taps (L %lld x Kp %lld) above 2^15", (long long)(L * (ka + kb + 1)), (long long)L,
                (long long)(ka + kb + 1));
  q->L = (uint32_t)L, q->M = (uint32_t)M, q->Tp = (uint32_t)tp, q->Ka = (uint32_t)ka, q->Kb = (uint32_t)kb, q->Kp = (uint32_t)(ka + kb + 1);
  q->P = (uint32_t)(fs_out / chan_gcd(chan_mod(offset_hz, fs_out), fs_out));
  return LTEPHY_SUCCESS;
}

// the tables of a carrier under the plan's flags, in the arithmetic of lteo_chan_design_poly, and at L = 1 of lteo_chan_design
static int chan_design(uint32_t fs_in, int32_t offset_hz, uint32_t N, uint32_t flags, ltephy_chan_poly_t* out, float* hp, float* g, float* rot)
{
  ltephy_chan_poly_t q;
  if (int r = chan_geometry(fs_in, offset_hz, N, flags, &q)) return r;
  if (out) *out = q;
  const int64_t L = q.L, Hp = (q.Tp - 1) / 2, Lfs = L * (int64_t)fs_in, fs_out = 15000ll * N;
  if (hp || g) {
    // windowed sinc with cutoff min(fs_in, fs_out) / 2 at rate L fs_in, scaled to DC gain L (scipy.signal.firwin, times L)
    std::vector<double> hd(q.Tp);
    const double        beta = 0.1102 * (CHAN_ATTEN - 8.7), a = 0.5 * (double)(q.Tp - 1), i0b = chan_i0(beta), c = 1.0 / (double)std::max(q.L, q.M);
    double              s = 0.0;
    for (int64_t j = 0; j < (int64_t)q.Tp; j++) {
      const double m  = (double)(j - Hp) * c;
      const double sn = m == 0.0 ? 1.0 : std::sin(M_PI * m) / (M_PI * m);
      const double r  = ((double)j - a) / a;
      const double w  = chan_i0(beta * std::sqrt(1.0 - r * r)) / i0b;
      hd[j]           = c * sn * w;
      s               = s + hd[j];
    }
    const double sl = s / (double)L;
    for (int64_t j = 0; j < (int64_t)q.Tp; j++) hd[j] = hd[j] / sl;
    if (hp)
      for (int64_t j = 0; j < (int64_t)q.Tp; j++) hp[j] = (float)hd[j];
    if (g) // g_phi[k] at [phi][k + Kb]: hp[Hp + phi + L k] e^{+j 2 pi offset (phi + L k) / (L fs_in)}, zero outside the prototype
      for (int64_t ph = 0; ph < L; ph++)
        for (int64_t k = -(int64_t)q.Kb; k <= (int64_t)q.Ka; k++) {
          const int64_t idx = Hp + ph + L * k;
          const double  tap = idx >= 0 && idx < (int64_t)q.Tp ? hd[idx] : 0.0;
          const double  a2  = 2.0 * M_PI * (double)chan_mod((int64_t)offset_hz * (ph + L * k), Lfs) / (double)Lfs;
          float*        o   = g + 2 * ((size_t)ph * q.Kp + (size_t)(k + q.Kb));
          o[0]              = (float)(tap * std::cos(a2));
          o[1]              = (float)(tap * std::sin(a2));
        }
  }
  if (rot) {
    // r[i] = e^{-j 2 pi offset i / fs_out}, the angle reduced in int64 over F before it is divided: at L = 1 over fs_in, as (D offset i) mod fs_in
    // (DESIGN.md §2 "channeliser"; the same angle as over fs_out, but not the same last bit when D is not a power of 2), else over fs_out
    const int64_t F = L == 1 ? (int64_t)fs_in : fs_out, step = chan_mod((int64_t)offset_hz * (F / fs_out), F);
    for (int64_t i = 0; i < (int64_t)q.P; i++) {
      const double ph = -2.0 * M_PI * (double)((step * i) % F) / (double)F;
      rot[2 * i]      = (float)std::cos(ph);
      rot[2 * i + 1]  = (float)std::sin(ph);
    }
  }
  return LTEPHY_SUCCESS;
}

static int chan_check_cfg(const ltephy_chan_cfg_t* cfg)
{
  if (!cfg) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: null configuration");
  if (cfg->nof_rx < 1 || cfg->nof_rx > 2) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: %u antennas not supported", cfg->nof_rx);
  if (cfg->nof_carriers < 1 || cfg->nof_carriers > LTEPHY_CHAN_MAX_CARRIERS)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: %u carriers, not 1..8", cfg->nof_carriers);
  if (cfg->max_samples < 1 || cfg->max_samples > (1ull << 31)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: max_samples outside 1..2^31");
  if (cfg->flags & ~LTEPHY_CHAN_RATIONAL) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: unknown flags 0x%x", cfg->flags);
  if (cfg->iq_format > LTEPHY_IQ_SC8) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan: unknown iq_format %u", cfg->iq_format);
  for (uint32_t c = 0; c < cfg->nof_carriers; c++) {
    ltephy_chan_poly_t q;
    if (int r = chan_geometry(cfg->fs_in, cfg->carrier[c].offset_hz, cfg->carrier[c].symbol_sz, cfg->flags, &q)) return r;
  }
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_chan_taps(const ltephy_chan_cfg_t* cfg, uint32_t c, float* h, float* g, float* rot, uint32_t* T, uint32_t* D, uint32_t* P)
{
  if (!cfg || !T || !D || !P) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_taps: null argument");
  if (c >= cfg->nof_carriers || c >= LTEPHY_CHAN_MAX_CARRIERS)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_taps: carrier %u of %u", c, cfg->nof_carriers);
  const ltephy_chan_carrier_t& k = cfg->carrier[c];
  ltephy_chan_poly_t           q;
  if ((cfg->flags & LTEPHY_CHAN_RATIONAL) && chan_geometry(cfg->fs_in, k.offset_hz, k.symbol_sz, cfg->flags, &q) == LTEPHY_SUCCESS &&
      !(q.L == 1 && q.M > 1))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_taps: carrier %u is rational (L %u / M %u): its tables come from ltephy_chan_design", c, q.L, q.M);
  if (int r = chan_design(cfg->fs_in, k.offset_hz, k.symbol_sz, 0, &q, h, g, rot)) return r; // without the flag: L = 1, M = D = 2..128
  *T = q.Tp, *D = q.M, *P = q.P;
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_chan_design(const ltephy_chan_cfg_t* cfg, uint32_t c, ltephy_chan_poly_t* out, float* hp, float* g, float* rot)
{
  if (!cfg || !out) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_design: null argument");
  if (c >= cfg->nof_carriers || c >= LTEPHY_CHAN_MAX_CARRIERS)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_design: carrier %u of %u", c, cfg->nof_carriers);
  if (cfg->flags & ~LTEPHY_CHAN_RATIONAL) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_design: unknown flags 0x%x", cfg->flags);
  return chan_design(cfg->fs_in, cfg->carrier[c].offset_hz, cfg->carrier[c].symbol_sz, cfg->flags, out, hp, g, rot);
}

extern "C" int ltephy_chan_create(const ltephy_chan_cfg_t* cfg, ltephy_chan_t** out)
{
  if (!out) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_create: null argument");
  if (int r = chan_check_cfg(cfg)) return r;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(LTEPHY_ERROR, "no CUDA device: this library has no CPU path");
  CU(cudaSetDevice(cfg->device));
  std::unique_ptr<ltephy_chan, decltype(&ltephy_chan_destroy)> owner(new ltephy_chan(), ltephy_chan_destroy);
  ltephy_chan* const                                           h = owner.get();
  h->cfg                                                         = *cfg;
  CU(cudaStreamCreateWithFlags(&h->stream.raw, cudaStreamNonBlocking));
  const size_t xbytes = (size_t)cfg->nof_rx * cfg->max_samples * chan_sample_bytes(cfg->iq_format);
  if (h->d_x.reserve((xbytes + sizeof(float2) - 1) / sizeof(float2))) return fail(LTEPHY_ERROR, "chan_create: device allocation failed");
  for (uint32_t c = 0; c < cfg->nof_carriers; c++) {
    ltephy_chan::Carrier& k = h->car[c];
    ltephy_chan_poly_t&   q = k.q;
    chan_geometry(cfg->fs_in, cfg->carrier[c].offset_hz, cfg->carrier[c].symbol_sz, cfg->flags, &q);
    std::vector<float> g(2 * (size_t)q.L * q.Kp), rot(2 * (size_t)q.P);
    chan_design(cfg->fs_in, cfg->carrier[c].offset_hz, cfg->carrier[c].symbol_sz, cfg->flags, nullptr, nullptr, g.data(), rot.data());
    k.Q = q.L == 1 ? q.M : 1;
    if (k.Q > 1) { // an integer carrier: R = min(1024, max(64, (CHAN_SPAN - T) / D + 1)) outputs, the span split into its D phases
      k.R = (uint32_t)std::min<int64_t>(1024, std::max<int64_t>(64, ((int64_t)CHAN_SPAN - (int64_t)q.Kp) / (int64_t)q.M + 1));
    } else { // rows per phase class: the span R M + Kp within CHAN_PSPAN; from 32 rows up, whole warps per class and about 4096 outputs a tile
      k.R = (uint32_t)std::max<int64_t>(1, ((int64_t)CHAN_PSPAN - (int64_t)q.Kp) / (int64_t)q.M);
      if (k.R >= 32) k.R = std::max<uint32_t>(32, std::min<uint32_t>(k.R, 4096 / q.L) / 32 * 32);
    }
    const uint64_t span = ((uint64_t)(q.L - 1) + ((uint64_t)q.L * k.R - 1) * q.M) / q.L + q.Kp; // the longest span of a tile
    k.rows              = (uint32_t)((span + k.Q - 1) / k.Q);
    k.cap               = (uint64_t)(((unsigned __int128)cfg->max_samples * q.L) / q.M) + 2;
    h->smem             = std::max(h->smem, ((q.L == 1 ? q.Kp : 0) + (size_t)k.Q * k.rows) * sizeof(float2)); // taps at L = 1, and the span
    if (k.g.reserve(g.size() / 2) || k.rot.reserve(q.P) || k.out.reserve((size_t)cfg->nof_rx * k.cap))
      return fail(LTEPHY_ERROR, "chan_create: device allocation failed");
    CU(cudaMemcpy(k.g.p, g.data(), g.size() * sizeof(float), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(k.rot.p, rot.data(), rot.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  *out = owner.release();
  return LTEPHY_SUCCESS;
}

extern "C" void ltephy_chan_destroy(ltephy_chan_t* h)
{
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

static int chan_check(ltephy_chan_t* h, const void* iq, uint64_t first, uint64_t n, ltephy_chan_out_t* out, uint64_t* next)
{
  if (!h || !iq || !out || !next) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_run: null argument");
  if (n < 1 || n > h->cfg.max_samples) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_run: %llu samples, not 1..max_samples", (unsigned long long)n);
  if (first > UINT64_MAX / 2) return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_run: first_sample too large");
  return LTEPHY_SUCCESS;
}

static int chan_run(ltephy_chan_t* h, const void* x, uint64_t first, uint64_t n, ltephy_chan_out_t* out, uint64_t* next)
{
  const uint32_t A = h->cfg.nof_rx;
  ChanArgs       g{};
  g.x = x, g.lda = n, g.first = first;
  uint32_t ntiles = 0;
  uint64_t nx     = UINT64_MAX;
  for (uint32_t c = 0; c < h->cfg.nof_carriers; c++) {
    const ltephy_chan::Carrier& k = h->car[c];
    const ltephy_chan_poly_t&   q = k.q;
    // outputs m >= 0 whose window [n - Ka, n + Kb], n = floor(m M / L), has every non-negative sample inside [first, first + n)
    const unsigned __int128 L = q.L, M = q.M, last = first + n - 1;
    const uint64_t          lo   = first == 0 ? 0 : (uint64_t)(((first + q.Ka) * L + M - 1) / M);
    const uint64_t          hi_n = last >= q.Kb ? (uint64_t)(((last - q.Kb + 1) * L - 1) / M + 1) : 0;
    const uint64_t          cnt  = hi_n > lo ? hi_n - lo : 0;
    const uint64_t          mn = cnt ? hi_n : lo, nn = (uint64_t)(mn * M / L);
    nx                         = std::min<uint64_t>(nx, nn >= q.Ka ? nn - q.Ka : 0);
    out[c].first = lo, out[c].count = cnt, out[c].iq_dev = k.out.p;
    if (!cnt) continue;
    const uint64_t per   = (uint64_t)q.L * k.R;
    const uint32_t tiles = (uint32_t)((cnt + per - 1) / per);
    for (uint32_t a = 0; a < A; a++) {
      ChanSeg& s = g.seg[g.nseg++];
      s.g = k.g.p, s.rot = k.rot.p, s.out = k.out.p + (size_t)a * cnt, s.n0 = (uint64_t)(lo * M / L), s.count = cnt;
      s.phi0 = (uint32_t)(lo * M % L), s.r0 = (uint32_t)(lo % q.P), s.L = q.L, s.M = q.M, s.Kp = q.Kp, s.Ka = q.Ka, s.P = q.P, s.R = k.R;
      s.Q = k.Q, s.rows = k.rows, s.tile0 = ntiles, s.a = a;
      ntiles += tiles;
    }
  }
  *next = nx;
  if (launch_chan(g, ntiles, h->smem, h->cfg.iq_format, h->stream))
    return fail(LTEPHY_ERROR, "chan_run: kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
  CU(cudaStreamSynchronize(h->stream));
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_chan_run(ltephy_chan_t* h, const void* iq, uint64_t first_sample, uint64_t nof_samples, ltephy_chan_out_t* out, uint64_t* next_sample)
{
  if (int r = chan_check(h, iq, first_sample, nof_samples, out, next_sample)) return r;
  CU(cudaSetDevice(h->cfg.device));
  CU(cudaMemcpyAsync(h->d_x.p, iq, (size_t)h->cfg.nof_rx * nof_samples * chan_sample_bytes(h->cfg.iq_format), cudaMemcpyHostToDevice, h->stream));
  return chan_run(h, h->d_x.p, first_sample, nof_samples, out, next_sample);
}

extern "C" int ltephy_chan_run_device(ltephy_chan_t* h, const void* iq_dev, uint64_t first_sample, uint64_t nof_samples, ltephy_chan_out_t* out,
                                      uint64_t* next_sample)
{
  if (int r = chan_check(h, iq_dev, first_sample, nof_samples, out, next_sample)) return r;
  if (h->cfg.iq_format != LTEPHY_IQ_CF32 && (uintptr_t)iq_dev % chan_sample_bytes(h->cfg.iq_format))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "chan_run_device: iq_dev not aligned to its %zu-byte samples", chan_sample_bytes(h->cfg.iq_format));
  CU(cudaSetDevice(h->cfg.device));
  return chan_run(h, iq_dev, first_sample, nof_samples, out, next_sample);
}
