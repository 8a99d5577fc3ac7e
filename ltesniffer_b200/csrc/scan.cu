// scan.cu -- the raster scan (include/ltephy_b200.h, DESIGN.md §2 "raster scan"): the N = 128 stream and the cell search of every 100 kHz raster
// point of a capture, a chunk of points per pass.  A pass is one launch of the channeliser kernel over a device table of (point, antenna)
// segments (k_chan.cu, g.tab) and one batched cell search over the chunk's streams (sync_run_batch): two host round trips per chunk.  Every
// point's taps are chan_design's, built once when the handle is created.
#include "../../include/ltephy_b200.h"
#include "k_chan.cuh"
#include "k_sync.cuh"
#include "ltephy_internal.cuh"
#include <algorithm>
#include <vector>

#define SCAN_N 128
#define SCAN_RASTER 100000ll
#define SCAN_BUDGET (2ull << 30) // device bytes the streams and search intermediates of one pass may take when max_points_per_pass = 0

struct ltephy_scan {
  ltephy_scan_cfg_t          cfg{};
  ltephy_chan_poly_t         q{};      // geometry shared by every point (only P differs)
  uint32_t                   R = 0, Q = 0, rows = 0, Pmax = 0, chunk = 0;
  size_t                     smem = 0;
  uint64_t                   cap = 0;  // N = 128 outputs per antenna of max_samples
  std::vector<int32_t>       off;      // [points] raster offsets
  std::vector<uint32_t>      per;      // [points] rotation period P
  std::vector<ltephy_cell_t> res;      // [points][3] of the last run
  uint64_t                   seg_n = 0; // nof_samples the segment table was built for
  ltephy_sync_t*             sync = nullptr;
  DevBuf<float2>             d_g, d_rot, d_out;
  DevBuf<ChanSeg>            d_seg;
  DevBuf<uint8_t>            d_x;
  ~ltephy_scan() { ltephy_sync_destroy(sync); }
};

// the raster offsets of cfg into off (all of them); 0, or INVALID_INPUTS
static int scan_plan(const ltephy_scan_cfg_t* cfg, std::vector<int32_t>* off, ltephy_chan_poly_t* q)
{
  if (!cfg) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan: null configuration");
  if (cfg->center_hz % 1000) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan: center_hz %llu is not a multiple of 1 kHz", (unsigned long long)cfg->center_hz);
  if (cfg->nof_rx < 1 || cfg->nof_rx > 2) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan: %u antennas not supported", cfg->nof_rx);
  if (cfg->iq_format > LTEPHY_IQ_SC8) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan: unknown iq_format %u", cfg->iq_format);
  if (cfg->lo_hz > cfg->hi_hz) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan: lo_hz %d above hi_hz %d", cfg->lo_hz, cfg->hi_hz);
  if (cfg->max_samples > (1ull << 31)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan: max_samples above 2^31");
  if (int r = chan_geometry(cfg->fs_in, 0, SCAN_N, LTEPHY_CHAN_RATIONAL, q)) return r; // the ratio is the same at every point
  if (cfg->max_samples < 1) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan: max_samples 0, fewer than a half-frame plus a symbol");
  uint64_t lo = 0, cnt = 0, nx = 0;
  chan_range(*q, 0, cfg->max_samples, &lo, &cnt, &nx);
  if (cnt < 75ull * SCAN_N + SCAN_N)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan: max_samples %llu gives %llu N = 128 samples, fewer than a half-frame plus a symbol",
                (unsigned long long)cfg->max_samples, (unsigned long long)cnt);
  // |o| + 540 kHz <= fs_in / 2 and lo <= o <= hi, o = 100 kHz k - center
  const int64_t reach = ((int64_t)cfg->fs_in - 2 * 540000ll) / 2, all = cfg->lo_hz == 0 && cfg->hi_hz == 0;
  const int64_t lo_o = all ? -reach : std::max<int64_t>(-reach, cfg->lo_hz), hi_o = all ? reach : std::min<int64_t>(reach, cfg->hi_hz);
  const int64_t c = (int64_t)cfg->center_hz;
  off->clear();
  if (reach < 0 || lo_o > hi_o) return LTEPHY_SUCCESS;
  auto fdiv = [](int64_t a, int64_t b) { return a / b - (a % b != 0 && (a < 0) != (b < 0)); };
  for (int64_t k = -fdiv(-(lo_o + c), SCAN_RASTER); k <= fdiv(hi_o + c, SCAN_RASTER); k++) {
    const int64_t o = SCAN_RASTER * k - c;
    if (2 * (std::llabs((long long)o) + 540000ll) <= (int64_t)cfg->fs_in) off->push_back((int32_t)o);
  }
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_scan_plan(const ltephy_scan_cfg_t* cfg, int32_t* offsets, uint32_t cap, uint32_t* n)
{
  if (!n || (cap && !offsets)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_plan: null argument");
  std::vector<int32_t> off;
  ltephy_chan_poly_t   q;
  if (int r = scan_plan(cfg, &off, &q)) return r;
  std::copy(off.begin(), off.begin() + std::min<size_t>(cap, off.size()), offsets);
  *n = (uint32_t)off.size();
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_scan_create(const ltephy_scan_cfg_t* cfg, ltephy_scan_t** out)
{
  if (!out) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_create: null argument");
  std::vector<int32_t> off;
  ltephy_chan_poly_t   q;
  if (int r = scan_plan(cfg, &off, &q)) return r;
  if (off.empty()) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_create: no raster point inside the capture and the range");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(LTEPHY_ERROR, "no CUDA device: this library has no CPU path");
  CU(cudaSetDevice(cfg->device));
  std::unique_ptr<ltephy_scan, decltype(&ltephy_scan_destroy)> owner(new ltephy_scan(), ltephy_scan_destroy);
  ltephy_scan* const                                           h = owner.get();
  const uint32_t                                               P = (uint32_t)off.size(), A = cfg->nof_rx;
  h->cfg = *cfg, h->q = q, h->off = off, h->per.resize(P);
  chan_tiles(q, &h->R, &h->Q, &h->rows, &h->smem);
  uint64_t lo = 0, nx = 0;
  chan_range(q, 0, cfg->max_samples, &lo, &h->cap, &nx);
  // every point's tables, as ltephy_chan_create builds them for the carrier (o_p, 128)
  for (uint32_t p = 0; p < P; p++) {
    ltephy_chan_poly_t qp;
    chan_geometry(cfg->fs_in, off[p], SCAN_N, LTEPHY_CHAN_RATIONAL, &qp);
    h->per[p] = qp.P, h->Pmax = std::max(h->Pmax, qp.P);
  }
  const size_t        G = (size_t)q.L * q.Kp;
  std::vector<float2> g(G * P), rot((size_t)h->Pmax * P);
  for (uint32_t p = 0; p < P; p++)
    chan_design(cfg->fs_in, off[p], SCAN_N, LTEPHY_CHAN_RATIONAL, nullptr, nullptr, &g[G * p].x, &rot[(size_t)h->Pmax * p].x);
  // points per pass: the streams and the cell search's intermediates of a point (its coarse metric is 3 floats per stream sample)
  const uint64_t nh = (h->cap - SCAN_N) / (75ull * SCAN_N) + 1, bytes = (uint64_t)A * h->cap * 8 + 12 * h->cap + 12 * SYNC_BINS + 3 * nh * A * 124 * 8;
  h->chunk = cfg->max_points_per_pass ? cfg->max_points_per_pass : (uint32_t)std::max<uint64_t>(1, SCAN_BUDGET / bytes);
  h->chunk = std::min<uint32_t>(std::min<uint32_t>(h->chunk, P), 65535); // grid y of the cell search
  if (h->d_g.reserve(g.size()) || h->d_rot.reserve(rot.size()) || h->d_out.reserve((size_t)h->chunk * A * h->cap) || h->d_seg.reserve((size_t)P * A) ||
      h->d_x.reserve((size_t)A * cfg->max_samples * iq_sample_bytes(cfg->iq_format)))
    return fail(LTEPHY_ERROR, "scan_create: device allocation failed");
  CU(cudaMemcpy(h->d_g.p, g.data(), g.size() * sizeof(float2), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(h->d_rot.p, rot.data(), rot.size() * sizeof(float2), cudaMemcpyHostToDevice));
  ltephy_sync_cfg_t scfg{};
  scfg.symbol_sz = SCAN_N, scfg.nof_rx = A, scfg.max_samples = h->cap, scfg.device = cfg->device, scfg.iq_format = LTEPHY_IQ_CF32;
  if (int r = sync_create_batch(&scfg, h->chunk, &h->sync)) return r;
  *out = owner.release();
  return LTEPHY_SUCCESS;
}

extern "C" void ltephy_scan_destroy(ltephy_scan_t* h)
{
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  delete h;
}

static int scan_check(ltephy_scan_t* h, const void* iq, uint64_t n, ltephy_scan_cell_t* out, uint32_t cap, uint32_t* nof_cells)
{
  if (!h || !iq || !nof_cells || (cap && !out)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_run: null argument");
  if (n > h->cfg.max_samples) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_run: %llu samples, more than max_samples", (unsigned long long)n);
  if (n < 1) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_run: no samples, fewer than a half-frame plus a symbol");
  uint64_t lo = 0, cnt = 0, nx = 0;
  chan_range(h->q, 0, n, &lo, &cnt, &nx);
  if (cnt < 75ull * SCAN_N + SCAN_N)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_run: %llu samples give %llu N = 128 samples, fewer than a half-frame plus a symbol", (unsigned long long)n,
                (unsigned long long)cnt);
  return LTEPHY_SUCCESS;
}

static int scan_run(ltephy_scan_t* h, const void* x, uint64_t n, ltephy_scan_cell_t* out, uint32_t cap, uint32_t* nof_cells)
{
  const uint32_t     P = (uint32_t)h->off.size(), A = h->cfg.nof_rx;
  const cudaStream_t st = sync_stream(h->sync);
  uint64_t           lo = 0, cnt = 0, nx = 0;
  chan_range(h->q, 0, n, &lo, &cnt, &nx);
  const uint32_t tps = (uint32_t)((cnt + (uint64_t)h->q.L * h->R - 1) / ((uint64_t)h->q.L * h->R));
  if (h->seg_n != n) { // segment (p, a) of a pass writes row (p mod chunk) A + a of the stream buffer
    std::vector<ChanSeg> seg((size_t)P * A);
    for (uint32_t p = 0; p < P; p++)
      for (uint32_t a = 0; a < A; a++) {
        ChanSeg&       s = seg[(size_t)p * A + a];
        const uint32_t r = (p % h->chunk) * A + a;
        s.g = h->d_g.p + (size_t)p * h->q.L * h->q.Kp, s.rot = h->d_rot.p + (size_t)p * h->Pmax, s.out = h->d_out.p + (size_t)r * cnt, s.n0 = 0, s.count = cnt;
        s.phi0 = 0, s.r0 = 0, s.L = h->q.L, s.M = h->q.M, s.Kp = h->q.Kp, s.Ka = h->q.Ka, s.P = h->per[p], s.R = h->R, s.Q = h->Q, s.rows = h->rows;
        s.tile0 = r * tps, s.a = a;
      }
    h->seg_n = 0; // a failed upload leaves no table behind
    CU(cudaMemcpyAsync(h->d_seg.p, seg.data(), seg.size() * sizeof(ChanSeg), cudaMemcpyHostToDevice, st));
    h->seg_n = n;
  }
  h->res.assign((size_t)3 * P, ltephy_cell_t{});
  for (uint32_t p0 = 0; p0 < P; p0 += h->chunk) {
    const uint32_t np = std::min(h->chunk, P - p0);
    ChanArgs       g{};
    g.x = x, g.lda = n, g.first = 0, g.tps = tps, g.tab = h->d_seg.p + (size_t)p0 * A;
    int r = launch_chan(g, np * A * tps, h->smem, h->cfg.iq_format, st)
                ? fail(LTEPHY_ERROR, "scan_run: channeliser kernel failed: %s", cudaGetErrorString(cudaGetLastError()))
                : sync_run_batch(h->sync, h->d_out.p, cnt, (uint64_t)A * cnt, cnt, np, &h->res[(size_t)3 * p0]);
    if (r) {
      h->res.clear(); // a failed run leaves no points behind
      return r;
    }
  }
  uint32_t k = 0;
  for (uint32_t p = 0; p < P; p++)
    for (uint32_t i = 0; i < 3; i++) {
      const ltephy_cell_t& c = h->res[(size_t)3 * p + i];
      if (!c.detected) continue;
      if (k < cap) out[k].offset_hz = h->off[p], out[k].pad = 0, out[k].cell = c;
      k++;
    }
  *nof_cells = k;
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_scan_run(ltephy_scan_t* h, const void* iq, uint64_t nof_samples, ltephy_scan_cell_t* out, uint32_t cap, uint32_t* nof_cells)
{
  if (int r = scan_check(h, iq, nof_samples, out, cap, nof_cells)) return r;
  CU(cudaSetDevice(h->cfg.device));
  CU(cudaMemcpyAsync(h->d_x.p, iq, (size_t)h->cfg.nof_rx * nof_samples * iq_sample_bytes(h->cfg.iq_format), cudaMemcpyHostToDevice, sync_stream(h->sync)));
  return scan_run(h, h->d_x.p, nof_samples, out, cap, nof_cells);
}

extern "C" int ltephy_scan_run_device(ltephy_scan_t* h, const void* iq_dev, uint64_t nof_samples, ltephy_scan_cell_t* out, uint32_t cap, uint32_t* nof_cells)
{
  if (int r = scan_check(h, iq_dev, nof_samples, out, cap, nof_cells)) return r;
  if (iq_misaligned(iq_dev, h->cfg.iq_format))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_run_device: iq_dev not aligned to its %zu-byte samples", iq_sample_bytes(h->cfg.iq_format));
  CU(cudaSetDevice(h->cfg.device));
  return scan_run(h, iq_dev, nof_samples, out, cap, nof_cells);
}

extern "C" int ltephy_scan_points(ltephy_scan_t* h, ltephy_cell_t* out, uint32_t cap)
{
  if (!h || (cap && !out)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_points: null argument");
  if (h->res.empty()) return fail(LTEPHY_ERROR_INVALID_INPUTS, "scan_points: no run yet");
  std::copy(h->res.begin(), h->res.begin() + 3 * std::min<size_t>(cap, h->off.size()), out);
  return LTEPHY_SUCCESS;
}
