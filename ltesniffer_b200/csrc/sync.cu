// sync.cu -- host side of the cell search (include/ltephy_b200.h, DESIGN.md §2 "cell search"): tables, buffers, the two kernel stages of
// k_sync.cu and the decisions on their bit-exact results (atan2f, argmax, frame timing), in the order lteo_cell_search states them.
#include "../../include/ltephy_b200.h"
#include "k_sync.cuh"
#include "ltephy_internal.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#define SYNC_PSR_MIN 2.5f  // detection thresholds: on noise-only captures neither ratio came above 1.7 (DESIGN.md §2)
#define SYNC_SSS_MIN 1.75f // a clean cell gives about 2: an SSS shares half its elements with the SSS of another N_ID_1

struct ltephy_sync {
  ltephy_sync_cfg_t cfg{};
  uint32_t          N = 0, D = 0, A = 0, NR = 0, nhmax = 0, points = 1; // points: captures a batch may hold
  uint64_t          Jmax = 0;
  Stream            stream;
  float             ep[3]{};
  std::vector<float2> dpss; // [3][62]
  DevBuf<uint8_t>   d_x; // samples in cfg.iq_format
  DevBuf<float2>    d_rep, d_W, d_dpss, d_Y;
  DevBuf<float>     d_seq, d_m, d_fold, d_rm, d_ref, d_sss;
  DevBuf<float4>    d_c12;
  DevBuf<SyncPeak>  d_pk;
  DevBuf<SyncPt>    d_pt;
  uint64_t          launches = 0;
  bool              searched = false;
};

// 36.211 6.11.1.1: d_u(n) = exp(-j pi u m / 63), m = n (n + 1) for n < 31, (n + 1) (n + 2) above; computed in double, rounded to float
static void pss_seq(uint32_t n_id_2, float2* d)
{
  static const uint32_t ROOT[3] = {25, 29, 34};
  for (uint32_t n = 0; n < 62; n++) {
    const uint32_t m  = n < 31 ? n * (n + 1) : (n + 1) * (n + 2);
    const double   ph = -M_PI * (double)((ROOT[n_id_2] * m) % 126u) / 63.0;
    d[n]              = make_float2((float)std::cos(ph), (float)std::sin(ph));
  }
}

// d_u (d[62]) and the replica p_u[k] = (1/sqrt N) sum_n d_u(n) exp(+j 2 pi f_n k / N) (rep[N]), in double rounded to float; returns E_p = sum |p|^2
// (in double, rounded): as lteo_cell_search and lteo_track compute them.  Shared by the cell search and the tracker (track.cu).
float sync_pss_replica(uint32_t N, uint32_t u, float2* d, float2* rep)
{
  pss_seq(u, d);
  const double sc = 1.0 / std::sqrt((double)N);
  double       e  = 0.0;
  for (uint32_t k = 0; k < N; k++) {
    double re = 0.0, im = 0.0;
    for (uint32_t n = 0; n < 62; n++) {
      const int64_t  f   = n < 31 ? (int64_t)n - 31 : (int64_t)n - 30;
      const uint32_t idx = (uint32_t)(((f * (int64_t)k) % (int64_t)N + (int64_t)N) % (int64_t)N);
      const double   ph = 2.0 * M_PI * (double)idx / (double)N, c = std::cos(ph), s = std::sin(ph);
      re += (double)d[n].x * c - (double)d[n].y * s;
      im += (double)d[n].x * s + (double)d[n].y * c;
    }
    rep[k] = make_float2((float)(re * sc), (float)(im * sc));
    e += (double)rep[k].x * rep[k].x + (double)rep[k].y * rep[k].y;
  }
  return (float)e;
}

// 36.211 6.11.2.1: d[62] of subframe 0 (sf5 = 0) or 5 (sf5 = 1)
static void sss_seq(uint32_t n_id_1, uint32_t n_id_2, uint32_t sf5, float* d)
{
  int st[31], ct[31], zt[31];
  uint8_t x[3][31] = {{0, 0, 0, 0, 1}, {0, 0, 0, 0, 1}, {0, 0, 0, 0, 1}};
  for (uint32_t i = 0; i + 5 < 31; i++) {
    x[0][i + 5] = (x[0][i + 2] + x[0][i]) & 1;
    x[1][i + 5] = (x[1][i + 3] + x[1][i]) & 1;
    x[2][i + 5] = (x[2][i + 4] + x[2][i + 2] + x[2][i + 1] + x[2][i]) & 1;
  }
  for (uint32_t i = 0; i < 31; i++) st[i] = 1 - 2 * x[0][i], ct[i] = 1 - 2 * x[1][i], zt[i] = 1 - 2 * x[2][i];
  const uint32_t qp = n_id_1 / 30, q = (n_id_1 + qp * (qp + 1) / 2) / 30, mp = n_id_1 + q * (q + 1) / 2;
  const uint32_t m0 = mp % 31, m1 = (m0 + mp / 31 + 1) % 31;
  for (uint32_t n = 0; n < 31; n++) {
    const int s0 = st[(n + m0) % 31], s1 = st[(n + m1) % 31], c0 = ct[(n + n_id_2) % 31], c1 = ct[(n + n_id_2 + 3) % 31];
    const int z0 = zt[(n + m0 % 8) % 31], z1 = zt[(n + m1 % 8) % 31];
    d[2 * n]     = (float)(sf5 ? s1 * c0 : s0 * c0);
    d[2 * n + 1] = (float)(sf5 ? s0 * c1 * z1 : s1 * c1 * z0);
  }
}

// points: captures a batch holds; stage: keep a buffer for the host input of ltephy_cell_search
static int sync_create(const ltephy_sync_cfg_t* cfg, uint32_t points, bool stage, ltephy_sync_t** out)
{
  if (!cfg || !out) return fail(LTEPHY_ERROR_INVALID_INPUTS, "sync_create: null argument");
  const uint32_t N = cfg->symbol_sz, M = N % 3 ? N : N / 3;
  if (N < 128 || N > 2048 || N % 128 || (M & (M - 1)) || cfg->nof_rx < 1 || cfg->nof_rx > 2)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "sync_create: symbol size %u / %u antennas not supported", N, cfg->nof_rx);
  if (cfg->max_samples < 75ull * N + N) return fail(LTEPHY_ERROR_INVALID_INPUTS, "sync_create: max_samples below one half-frame plus a symbol");
  if (cfg->iq_format > LTEPHY_IQ_SC8)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "sync_create: iq_format %u: LTEPHY_IQ_CF32 (0), LTEPHY_IQ_SC16 (1) or LTEPHY_IQ_SC8 (2)", cfg->iq_format);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(LTEPHY_ERROR, "no CUDA device: this library has no CPU path");
  CU(cudaSetDevice(cfg->device));
  std::unique_ptr<ltephy_sync, decltype(&ltephy_sync_destroy)> owner(new ltephy_sync(), ltephy_sync_destroy);
  ltephy_sync* const                                           h = owner.get();
  h->cfg = *cfg, h->N = N, h->D = N / 128, h->A = cfg->nof_rx, h->NR = 2 * h->D - 1, h->points = points;
  h->Jmax  = (cfg->max_samples - N) / h->D + 1;
  h->nhmax = (uint32_t)((cfg->max_samples - N) / (75ull * N) + 1);
  CU(cudaStreamCreateWithFlags(&h->stream.raw, cudaStreamNonBlocking));
  // replicas p_u[k] = (1/sqrt N) sum_n d_u(n) exp(+j 2 pi f_n k / N) and E_p, in double, as lteo_cell_search computes them
  std::vector<float2> rep((size_t)3 * N), W(N);
  h->dpss.resize(3 * 62);
  for (uint32_t u = 0; u < 3; u++) h->ep[u] = sync_pss_replica(N, u, &h->dpss[62 * u], &rep[(size_t)u * N]);
  for (uint32_t i = 0; i < N; i++) {
    const double ph = -2.0 * M_PI * (double)i / (double)N;
    W[i]            = make_float2((float)std::cos(ph), (float)std::sin(ph));
  }
  std::vector<float> seq((size_t)3 * 168 * 2 * 62);
  for (uint32_t u = 0; u < 3; u++)
    for (uint32_t n1 = 0; n1 < 168; n1++)
      for (uint32_t q = 0; q < 2; q++) sss_seq(n1, u, q, &seq[((u * 168 + n1) * 2 + q) * 62]);
  const size_t P = points;
  if (h->d_rep.reserve(rep.size()) || h->d_W.reserve(N) || h->d_dpss.reserve(3 * 62) || h->d_seq.reserve(seq.size()) ||
      (stage && h->d_x.reserve((size_t)h->A * cfg->max_samples * iq_sample_bytes(cfg->iq_format))) || h->d_m.reserve(P * 3 * h->Jmax) ||
      h->d_fold.reserve(P * 3 * SYNC_BINS) || h->d_rm.reserve(P * 3 * h->nhmax * h->NR) || h->d_ref.reserve(P * 3 * h->NR) || h->d_sss.reserve(P * 3 * 336) ||
      h->d_c12.reserve(P * 3 * h->nhmax * h->A) || h->d_pk.reserve(P * 3) || h->d_Y.reserve(P * 3 * h->nhmax * h->A * 124) || h->d_pt.reserve(P))
    return fail(LTEPHY_ERROR, "sync_create: device allocation failed");
  CU(cudaMemcpy(h->d_rep.p, rep.data(), rep.size() * sizeof(float2), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(h->d_W.p, W.data(), W.size() * sizeof(float2), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(h->d_dpss.p, h->dpss.data(), h->dpss.size() * sizeof(float2), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(h->d_seq.p, seq.data(), seq.size() * sizeof(float), cudaMemcpyHostToDevice));
  *out = owner.release();
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_sync_create(const ltephy_sync_cfg_t* cfg, ltephy_sync_t** out) { return sync_create(cfg, 1, true, out); }

// the raster scan's handle searches its captures in place and stages no input of its own
int sync_create_batch(const ltephy_sync_cfg_t* cfg, uint32_t points, ltephy_sync_t** out) { return sync_create(cfg, points, false, out); }

cudaStream_t sync_stream(ltephy_sync_t* h) { return h->stream; }

extern "C" void ltephy_sync_destroy(ltephy_sync_t* h)
{
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

static int sync_check(ltephy_sync_t* h, const void* iq, uint64_t L, ltephy_cell_t* out)
{
  if (!h || !iq || !out) return fail(LTEPHY_ERROR_INVALID_INPUTS, "cell_search: null argument");
  if (L < 75ull * h->N + h->N) return fail(LTEPHY_ERROR_INVALID_INPUTS, "cell_search: %llu samples, fewer than a half-frame plus a symbol", (unsigned long long)L);
  if (L > h->cfg.max_samples) return fail(LTEPHY_ERROR_INVALID_INPUTS, "cell_search: %llu samples, more than max_samples", (unsigned long long)L);
  return LTEPHY_SUCCESS;
}

int sync_run(ltephy_sync_t* h, const void* x, uint64_t lda, uint64_t L, ltephy_cell_t* out) { return sync_run_batch(h, x, lda, 0, L, 1, out); }

int sync_run_batch(ltephy_sync_t* h, const void* x, uint64_t lda, uint64_t ps, uint64_t L, uint32_t np, ltephy_cell_t* out)
{
  if (np < 1 || np > h->points) return fail(LTEPHY_ERROR_INVALID_INPUTS, "cell_search: %u captures, not 1..%u", np, h->points);
  const uint32_t N = h->N, D = h->D, CP6 = 9 * D;
  const uint64_t HF = 75ull * N, FR = 150ull * N;
  SyncArgs       g{};
  g.x = x, g.lda = lda, g.ps = ps, g.L = L, g.J = (L - N) / D + 1, g.N = N, g.D = D, g.A = h->A, g.nh = (uint32_t)((L - N) / HF + 1);
  g.rep = h->d_rep.p, g.W = h->d_W.p;
  for (int u = 0; u < 3; u++) g.ep[u] = h->ep[u];
  if (launch_sync_pss(g, np, h->cfg.iq_format, h->d_m.p, h->d_fold.p, h->d_pk.p, h->d_rm.p, h->d_c12.p, h->d_ref.p, h->stream, &h->launches))
    return fail(LTEPHY_ERROR, "cell_search: PSS kernels failed: %s", cudaGetErrorString(cudaGetLastError()));
  std::vector<SyncPeak> pks((size_t)3 * np);
  CU(cudaMemcpyAsync(pks.data(), h->d_pk.p, pks.size() * sizeof(SyncPeak), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  std::vector<ltephy_cell_t> all((size_t)3 * np);
  std::vector<SyncPt>        pts(np);
  SyncSss                    s{};
  s.pt = h->d_pt.p, s.dpss = h->d_dpss.p, s.seq = h->d_seq.p;
  for (uint32_t p = 0; p < np; p++)
    for (uint32_t u = 0; u < 3; u++) {
      const SyncPeak* pk = &pks[3 * p];
      SyncPt&         q  = pts[p];
      ltephy_cell_t&  o  = all[3 * p + u];
      memset(&o, 0, sizeof(o));
      o.n_id_2   = (uint8_t)u;
      o.psr      = pk[u].side > 0.0f ? pk[u].peak / pk[u].side : (pk[u].peak > 0.0f ? INFINITY : 0.0f);
      o.pss_peak = pk[u].rpeak;
      o.cfo_re = pk[u].s_re, o.cfo_im = pk[u].s_im;
      o.cfo_hz   = atan2f(pk[u].s_im, pk[u].s_re) * (float)(15000.0 / M_PI);
      const double phi = 2.0 * M_PI * (double)o.cfo_hz * (double)(N + CP6) / (15000.0 * (double)N);
      q.rot[u][0] = (float)std::cos(phi), q.rot[u][1] = (float)-std::sin(phi);
      // half-frames h with the PSS window at tau + h HF inside the capture and the SSS window N + CP6 before it at or after sample 0
      const uint64_t tau = pk[u].tau;
      q.tau[u]           = tau;
      q.h0[u]            = tau < N + CP6 ? 1 : 0;
      const uint64_t last = (L - N - tau) / HF; // tau + HF > L - N cannot leave h = 0 without a PSS window
      q.nH[u]            = tau + N <= L && last >= q.h0[u] ? (uint32_t)(last - q.h0[u] + 1) : 0;
      o.nof_half_frames  = q.nH[u];
      s.nhmax            = std::max(s.nhmax, q.nH[u]);
    }
  CU(cudaMemcpyAsync(h->d_pt.p, pts.data(), pts.size() * sizeof(SyncPt), cudaMemcpyHostToDevice, h->stream));
  if (launch_sync_sss(g, np, h->cfg.iq_format, s, h->d_Y.p, h->d_sss.p, h->stream, &h->launches))
    return fail(LTEPHY_ERROR, "cell_search: SSS kernels failed: %s", cudaGetErrorString(cudaGetLastError()));
  std::vector<float> tabs((size_t)np * 3 * 336);
  CU(cudaMemcpyAsync(tabs.data(), h->d_sss.p, tabs.size() * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  for (uint32_t p = 0; p < np; p++) {
    const float*   tab = &tabs[(size_t)p * 3 * 336];
    ltephy_cell_t* res = &all[3 * p];
    for (uint32_t u = 0; u < 3; u++) {
      ltephy_cell_t& o  = res[u];
      const int64_t  st = (int64_t)pks[3 * p + u].tau - (int64_t)(13 * N / 2); // first sample of the subframe whose symbol 6 starts at tau
      if (!pts[p].nH[u]) {
        o.n_id_1 = o.pci = 0xFFFF;
        o.frame_offset   = (uint64_t)(((st % (int64_t)FR) + (int64_t)FR) % (int64_t)FR);
        continue;
      }
      const float* Au   = &tab[u * 336];
      uint32_t     best = 0;
      for (uint32_t i = 1; i < 336; i++)
        if (Au[i] > Au[best]) best = i; // ties: lowest N_ID_1, then q = 0
      float second = -INFINITY;
      for (uint32_t i = 0; i < 336; i++)
        if (i != best && Au[i] > second) second = Au[i];
      o.n_id_1       = (uint16_t)(best / 2);
      o.pci          = (uint16_t)(3 * (best / 2) + u);
      o.sss_peak     = Au[best];
      o.sss_ratio    = second > 0.0f ? Au[best] / second : (Au[best] > 0.0f ? INFINITY : 0.0f);
      const int64_t fs = (best & 1) ? st - (int64_t)HF : st; // q = 1: the half-frame at tau is subframe 5
      o.frame_offset = (uint64_t)(((fs % (int64_t)FR) + (int64_t)FR) % (int64_t)FR);
      o.detected     = o.psr >= SYNC_PSR_MIN && o.sss_ratio >= SYNC_SSS_MIN;
    }
    uint32_t ord[3] = {0, 1, 2};
    std::stable_sort(ord, ord + 3, [&](uint32_t a, uint32_t b) { return res[a].pss_peak > res[b].pss_peak; });
    for (uint32_t i = 0; i < 3; i++) out[3 * p + i] = res[ord[i]];
  }
  h->searched = true;
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_cell_search(ltephy_sync_t* h, const void* iq, uint64_t nof_samples, ltephy_cell_t out[3])
{
  if (int r = sync_check(h, iq, nof_samples, out)) return r;
  CU(cudaSetDevice(h->cfg.device));
  CU(cudaMemcpyAsync(h->d_x.p, iq, (size_t)h->A * nof_samples * iq_sample_bytes(h->cfg.iq_format), cudaMemcpyHostToDevice, h->stream));
  return sync_run(h, h->d_x.p, nof_samples, nof_samples, out);
}

extern "C" int ltephy_cell_search_device(ltephy_sync_t* h, const void* iq_dev, uint64_t nof_samples, ltephy_cell_t out[3])
{
  if (int r = sync_check(h, iq_dev, nof_samples, out)) return r;
  if (iq_misaligned(iq_dev, h->cfg.iq_format))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "cell_search_device: iq_dev not aligned to its %zu-byte samples", iq_sample_bytes(h->cfg.iq_format));
  CU(cudaSetDevice(h->cfg.device));
  return sync_run(h, iq_dev, nof_samples, nof_samples, out);
}

extern "C" int ltephy_sync_tap(ltephy_sync_t* h, int what, void* dst, size_t bytes)
{
  if (!h || !dst || !h->searched) return fail(LTEPHY_ERROR_INVALID_INPUTS, "sync_tap: bad arguments or no search yet");
  const void* src = nullptr;
  size_t      n   = 0;
  switch (what) {
    case LTEPHY_SYNC_TAP_COARSE: src = h->d_fold.p, n = 3 * SYNC_BINS * sizeof(float); break;
    case LTEPHY_SYNC_TAP_REFINED: src = h->d_ref.p, n = 3 * h->NR * sizeof(float); break;
    case LTEPHY_SYNC_TAP_SSS: src = h->d_sss.p, n = 3 * 336 * sizeof(float); break;
    case LTEPHY_SYNC_TAP_CFO: {
      SyncPeak pk[3];
      CU(cudaSetDevice(h->cfg.device));
      CU(cudaMemcpy(pk, h->d_pk.p, sizeof(pk), cudaMemcpyDeviceToHost));
      if (bytes < 6 * sizeof(float)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "sync_tap: buffer too small");
      float* f = static_cast<float*>(dst);
      for (int u = 0; u < 3; u++) f[2 * u] = pk[u].s_re, f[2 * u + 1] = pk[u].s_im;
      return LTEPHY_SUCCESS;
    }
    default: return fail(LTEPHY_ERROR_INVALID_INPUTS, "sync_tap: unknown tap %d", what);
  }
  if (bytes < n) return fail(LTEPHY_ERROR_INVALID_INPUTS, "sync_tap: buffer too small");
  CU(cudaSetDevice(h->cfg.device));
  CU(cudaMemcpy(dst, src, n, cudaMemcpyDeviceToHost));
  return LTEPHY_SUCCESS;
}
