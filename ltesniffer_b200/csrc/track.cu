// track.cu -- host side of the tracker (include/ltephy_b200.h, DESIGN.md §2 "tracking"): predicts the measurement windows of a push, runs the
// metric kernel over them, replays the rule on its bit-exact results in the order lteo_track states it (measuring a window again when the
// tracked position left the predicted one), then the CFO sums, the carrier-offset loop and the cut.  With LTEPHY_TRACK_REACQUIRE a loss
// enters the find state: the cell search (sync.cu, k_sync.cu) on one frame of the push's own device buffer at a time.
#include "../../include/ltephy_b200.h"
#include "k_sync.cuh"
#include "k_track.cuh"
#include "ltephy_internal.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#define TRACK_P      4u    // locked half-frames per timing correction
#define TRACK_ALPHA  0.05f // gain of the carrier-offset loop
#define TRACK_MISS   4u    // half-frames in a row without lock after which records are flagged lost
#define TRACK_LOCK_K 20.0f // lock: peak metric >= 20 / N; on noise-only captures no half-frame's peak came above 10.2 / N (DESIGN.md §2)

// a carrier the tracker cuts: the downlink, and with ltephy_track_set_ul the uplink, whose A antennas are cut at start + off and rotated by
// f ratio with their own factor tables
struct TrackCarrier {
  uint32_t         A     = 1;
  int32_t          off   = 0;
  double           ratio = 1.0;
  DevBuf<uint8_t>  d_x; // samples of a host push in cfg.iq_format
  DevBuf<float2>   d_cut, d_tabA, d_tabB;
  DevBuf<uint64_t> d_start;
  int              reserve(size_t nsf, uint32_t SF)
  {
    return d_cut.reserve(nsf * A * SF) || d_tabA.reserve(nsf * (SF / 128)) || d_tabB.reserve(nsf * 128) || d_start.reserve(nsf);
  }
};

struct ltephy_track {
  ltephy_track_cfg_t cfg{};
  uint32_t           N = 0, W = 0, SF = 0;
  float              ep = 0.0f, thr = 0.0f, max_ppm = 50.0f;
  Stream             stream;
  DevBuf<float2>     d_rep, d_c;
  DevBuf<float>      d_m;
  DevBuf<TrackWin>   d_win;
  DevBuf<uint64_t>   d_pos;
  TrackCarrier       car[2]; // the downlink, then the uplink
  uint32_t           nc = 1; // carriers cut: 2 once the uplink is set
  bool               pushed = false;
  // state: as lteo_track
  int64_t  s = 0;
  uint32_t k = 0;
  float    f = 0.0f, d = 0.0f, acc = 0.0f;
  uint32_t miss = 0, nhf = 0, ncor = 0, nl = 0;
  int64_t  sd = 0, sh = 0, shh = 0, shd = 0;
  int64_t  base = 0; // start of subframe 0 of the drift estimate's grid: frame_offset, after a find s' - k' SF
  // the find state (LTEPHY_TRACK_REACQUIRE): searching the window [f0, f0 + FR + N) predicted to start subframe kn
  bool           find = false, reacq = false;
  int64_t        f0 = 0;
  uint32_t       kn = 0;
  float          f_find = 0.0f; // the found carrier offset, installed at the re-acquired subframe in step 3
  std::unique_ptr<ltephy_sync_t, decltype(&ltephy_sync_destroy)> sync{nullptr, ltephy_sync_destroy};
  std::vector<ltephy_track_sf_t> sf;
  std::vector<ltephy_track_hf_t> hf;
};

// the lowest absolute sample the pending window of any carrier still needs; in the find state, from the window's first sample
static int64_t track_needed(const ltephy_track* h)
{
  const int64_t s  = h->find ? h->f0 : h->s;
  int64_t       lo = s;
  for (uint32_t c = 0; c < h->nc; c++) lo = std::min(lo, s + h->car[c].off);
  return lo;
}

// a subframe starting at s is cut only when the window of every carrier lies inside [first, end)
static bool track_fits(const ltephy_track* h, int64_t s, uint64_t first, uint64_t end)
{
  for (uint32_t c = 0; c < h->nc; c++) {
    const int64_t sc = s + h->car[c].off;
    if (!(sc >= (int64_t)first && (uint64_t)sc + h->SF <= end)) return false;
  }
  return true;
}

static bool track_symbol_ok(uint32_t N)
{
  const uint32_t M = N % 3 ? N : N / 3;
  return N >= 128 && N <= 2048 && N % 128 == 0 && !(M & (M - 1));
}

extern "C" int ltephy_track_create(const ltephy_track_cfg_t* cfg, ltephy_track_t** out)
{
  if (!cfg || !out) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_create: null argument");
  const uint32_t N = cfg->symbol_sz;
  if (!track_symbol_ok(N) || cfg->nof_rx < 1 || cfg->nof_rx > 2)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_create: symbol size %u / %u antennas not supported", N, cfg->nof_rx);
  if (cfg->pci > 503 || cfg->first_tti > 10239) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_create: pci %u / first_tti %u out of range", cfg->pci, cfg->first_tti);
  if (!(std::fabs(cfg->cfo_hz) <= 7500.0f)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_create: cfo_hz outside +-7500 Hz");
  if (!(cfg->max_ppm >= 0.0f && cfg->max_ppm <= 1000.0f)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_create: max_ppm outside 0..1000");
  if (cfg->max_subframes < 1 || cfg->max_subframes > 20000) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_create: max_subframes outside 1..20000");
  if (cfg->flags & ~(LTEPHY_TRACK_NO_CFO | LTEPHY_TRACK_REACQUIRE)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_create: unknown flags 0x%x", cfg->flags);
  if (cfg->iq_format > LTEPHY_IQ_SC8)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_create: iq_format %u: LTEPHY_IQ_CF32 (0), LTEPHY_IQ_SC16 (1) or LTEPHY_IQ_SC8 (2)", cfg->iq_format);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(LTEPHY_ERROR, "no CUDA device: this library has no CPU path");
  CU(cudaSetDevice(cfg->device));
  std::unique_ptr<ltephy_track, decltype(&ltephy_track_destroy)> owner(new ltephy_track(), ltephy_track_destroy);
  ltephy_track* const                                            h = owner.get();
  h->cfg = *cfg, h->N = N, h->car[0].A = cfg->nof_rx, h->W = 9 * N / 128, h->SF = 15 * N;
  h->max_ppm = cfg->max_ppm > 0.0f ? cfg->max_ppm : 50.0f;
  h->thr     = TRACK_LOCK_K / (float)N;
  h->s = h->base = (int64_t)cfg->frame_offset, h->f = cfg->cfo_hz;
  CU(cudaStreamCreateWithFlags(&h->stream.raw, cudaStreamNonBlocking));
  // the find's cell search: one window of a frame plus a symbol.  The handle's own sample buffer (A (150 N + N) samples, 4.9 MB at N = 2048
  // with 2 antennas) stays unused: the find reads the push's samples in place through sync_run.
  if (cfg->flags & LTEPHY_TRACK_REACQUIRE) {
    ltephy_sync_cfg_t sc{};
    sc.symbol_sz = N, sc.nof_rx = cfg->nof_rx, sc.max_samples = 151ull * N, sc.device = cfg->device, sc.iq_format = cfg->iq_format;
    ltephy_sync_t* sync = nullptr;
    if (int r = ltephy_sync_create(&sc, &sync)) return r;
    h->sync.reset(sync);
  }
  // the replica of N_ID_2 = pci mod 3 and its energy: the cell search's (sync.cu), as lteo_track_create computes them
  std::vector<float2> rep(N), d62(62);
  h->ep = sync_pss_replica(N, cfg->pci % 3, d62.data(), rep.data());
  const size_t nsf = cfg->max_subframes;
  if (h->d_rep.reserve(N) || h->car[0].reserve(nsf, h->SF) || h->d_pos.reserve(nsf / 5 + 1) || h->d_c.reserve((nsf / 5 + 1) * cfg->nof_rx * 2) ||
      h->d_win.reserve(nsf / 5 + 1))
    return fail(LTEPHY_ERROR, "track_create: device allocation failed");
  CU(cudaMemcpy(h->d_rep.p, rep.data(), N * sizeof(float2), cudaMemcpyHostToDevice));
  h->sf.reserve(nsf), h->hf.reserve(nsf / 5 + 1);
  *out = owner.release();
  return LTEPHY_SUCCESS;
}

extern "C" void ltephy_track_destroy(ltephy_track_t* h)
{
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

// the metric at the positions of the given windows, back on the host (m[w * stride + i])
static int track_metrics(ltephy_track_t* h, const TrackArgs& g, const std::vector<TrackWin>& win, std::vector<float>& m, uint32_t& stride)
{
  stride = 0;
  for (const TrackWin& w : win) stride = std::max(stride, w.cnt);
  m.assign((size_t)win.size() * stride, 0.0f);
  if (win.empty()) return LTEPHY_SUCCESS;
  if (h->d_win.reserve(win.size()) || h->d_m.reserve(m.size())) return fail(LTEPHY_ERROR, "track_push: device allocation failed");
  CU(cudaMemcpyAsync(h->d_win.p, win.data(), win.size() * sizeof(TrackWin), cudaMemcpyHostToDevice, h->stream));
  if (launch_track_metric(g, h->cfg.iq_format, h->d_win.p, (uint32_t)win.size(), stride, stride, h->d_m.p, h->stream))
    return fail(LTEPHY_ERROR, "track_push: metric kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
  CU(cudaMemcpyAsync(m.data(), h->d_m.p, m.size() * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return LTEPHY_SUCCESS;
}

// one find window (lteo_track's track_find): the cell search on the samples [f0, f0 + FR + N) of x, read in place; found: resume at the
// window's first subframe boundary with the subframe number of its SSS, otherwise step one frame on
static int track_find(ltephy_track_t* h, const void* x, uint64_t first, uint64_t n, bool& found)
{
  const uint32_t N = h->N, SF = h->SF;
  const uint64_t FR = 150ull * N;
  CU(cudaStreamSynchronize(h->stream)); // the push's copy of x runs on the tracker's stream, the search on the sync handle's
  ltephy_cell_t res[3];
  const uint8_t* w = static_cast<const uint8_t*>(x) + (uint64_t)(h->f0 - (int64_t)first) * iq_sample_bytes(h->cfg.iq_format);
  if (int r = sync_run(h->sync.get(), w, n, FR + N, res)) return r;
  const ltephy_cell_t* c = nullptr;
  for (uint32_t i = 0; i < 3; i++)
    if (res[i].n_id_2 == h->cfg.pci % 3) c = &res[i];
  found = c->detected && c->pci == h->cfg.pci;
  if (!found) {
    h->f0 += (int64_t)FR, h->kn += 10;
    return LTEPHY_SUCCESS;
  }
  const uint64_t fo   = c->frame_offset;
  const uint32_t sfno = (uint32_t)((10 - fo / SF) % 10);
  const uint32_t k    = h->kn + (sfno + 10 - (h->cfg.first_tti + h->kn) % 10) % 10;
  h->s = h->f0 + (int64_t)(fo % SF), h->k = k, h->f_find = c->cfo_hz;
  h->miss = 0, h->acc = 0.0f;
  h->nl = 0, h->sd = h->sh = h->shh = h->shd = 0, h->ncor = 0;
  h->base = h->s - (int64_t)k * SF, h->nhf = 0; // the drift d is kept: a clock does not change with a gap
  h->find = false, h->reacq = true;
  return LTEPHY_SUCCESS;
}

// x[c]: the device samples of carrier c
static int track_run(ltephy_track_t* h, const void* const* x, uint64_t first, uint64_t n, ltephy_track_out_t* out, const void** ul_iq_dev)
{
  const uint32_t N = h->N, SF = h->SF, W = h->W, A = h->car[0].A, maxsf = h->cfg.max_subframes;
  const uint64_t end = first + n;
  TrackArgs      g{};
  g.x = x[0], g.lda = n, g.N = N, g.A = A, g.rep = h->d_rep.p, g.ep = h->ep;
  // 1. predict: the subframes of this push from the state at its start (and again after a find), without corrections; each half-frame's
  //    window is the tracker's +-W plus the distance a clock max_ppm off moves the start over the predicted span, clamped to the samples fed
  std::vector<TrackWin> win;
  std::vector<uint32_t> wk; // subframe number of each window
  std::vector<float>    m;
  uint32_t              stride = 0;
  auto predict = [&]() -> int {
    win.clear(), wk.clear();
    int64_t  ps  = h->s;
    float    pac = h->acc;
    uint32_t pk = h->k, cnt = (uint32_t)h->sf.size();
    while (!h->find && cnt < maxsf && track_fits(h, ps, first, end)) {
      if ((h->cfg.first_tti + pk) % 10240 % 5 == 0) {
        const int64_t tau = ps + 13 * N / 2 - (int64_t)first;
        const int64_t M   = (int64_t)std::ceil((double)h->max_ppm * 1e-6 * (double)(ps - h->s)) + 1; // half-width W + M
        const int64_t lo = std::max<int64_t>(tau - W - M, 0), hi = std::min<int64_t>(tau + W + M, (int64_t)(n - N));
        win.push_back(TrackWin{(uint64_t)lo, (uint32_t)(hi - lo + 1), 0});
        wk.push_back(pk);
      }
      pac           = pac + h->d / 5.0f;
      const float r = roundf(pac);
      pac           = pac - r;
      ps            = ps + SF + (int64_t)r;
      pk++, cnt++;
    }
    return track_metrics(h, g, win, m, stride);
  };
  h->sf.clear(), h->hf.clear();
  if (int r = predict()) return r;
  // 2. replay the timing rule (lteo_track_push) subframe by subframe; the carrier offset waits for the sums of step 3
  std::vector<uint64_t> spos, hpos;
  std::vector<float>    fre; // the found carrier offset of each re-acquired subframe
  uint32_t              remeasured = 0, finds = 0;
  size_t                wi         = 0;
  while (h->sf.size() < maxsf) {
    if (h->find) { // a window is searched once all of its samples have been fed
      if ((uint64_t)h->f0 + 151ull * N > end) break;
      bool found = false;
      if (int r = track_find(h, x[0], first, n, found)) return r;
      finds++;
      if (found) {
        if (int r = predict()) return r;
        wi = 0;
      }
      continue;
    }
    if (!track_fits(h, h->s, first, end)) break;
    const uint32_t    tti = (h->cfg.first_tti + h->k) % 10240;
    ltephy_track_sf_t o{};
    o.start = h->s, o.tti = tti, o.index = h->k;
    o.flags = (h->miss == 0 ? LTEPHY_TRACK_LOCKED : 0) | (h->miss >= TRACK_MISS ? LTEPHY_TRACK_LOST : 0) | (h->reacq ? LTEPHY_TRACK_REACQUIRED : 0);
    if (h->reacq) fre.push_back(h->f_find), h->reacq = false;
    h->sf.push_back(o);
    spos.push_back((uint64_t)(h->s - (int64_t)first));
    bool lost_now = false;
    if (tti % 5 == 0) {
      ltephy_track_hf_t q{};
      q.tau = h->s + 13 * N / 2, q.index = h->k;
      const uint64_t tau = (uint64_t)(q.tau - (int64_t)first);
      while (wi < wk.size() && wk[wi] < h->k) wi++;
      const float* mv = nullptr;
      uint64_t     t0 = 0;
      if (wi < wk.size() && wk[wi] == h->k && win[wi].t0 + W <= tau && tau + W < win[wi].t0 + win[wi].cnt)
        mv = &m[(size_t)wi * stride], t0 = win[wi].t0;
      std::vector<float> mr;
      if (!mv) { // the tracked window left the measured one: measure it now
        std::vector<TrackWin> one{TrackWin{tau - W, 2 * W + 1, 0}};
        uint32_t              st1 = 0;
        if (int r = track_metrics(h, g, one, mr, st1)) return r;
        mv = mr.data(), t0 = tau - W, remeasured++;
      }
      int32_t best = 0;
      float   peak = mv[tau - t0];
      for (int32_t d = 1; d <= (int32_t)W; d++)
        for (int32_t sg = -1; sg <= 1; sg += 2) {
          const float v = mv[tau + sg * d - t0];
          if (v > peak) peak = v, best = sg * d;
        }
      q.delta = best, q.peak = peak;
      const int64_t hn = h->nhf++;
      if (peak >= h->thr) {
        q.flags |= LTEPHY_TRACK_LOCKED;
        h->miss = 0;
        h->nl++, h->sd += best, h->sh += hn, h->shh += hn * hn, h->shd += hn * best;
        if (h->nl == TRACK_P) {
          const int64_t P = TRACK_P, c = h->sd >= 0 ? (h->sd + P / 2) / P : -((-h->sd + P / 2) / P);
          h->s += c;
          h->ncor++;
          if (h->ncor == 1) {
            const int64_t num = P * h->shd - h->sh * h->sd, den = P * h->shh - h->sh * h->sh;
            h->d = h->d + (float)num / (float)den;
          } else {
            const int64_t moved = h->s - h->base - (int64_t)h->k * SF;
            h->d = (float)moved / ((float)h->nhf - 0.5f * (float)(P - 1));
          }
          h->nl = 0, h->sd = h->sh = h->shh = h->shd = 0;
        }
      } else
        lost_now = ++h->miss == TRACK_MISS;
      if (h->miss >= TRACK_MISS) q.flags |= LTEPHY_TRACK_LOST;
      h->hf.push_back(q);
      hpos.push_back(tau + best);
    }
    h->acc        = h->acc + h->d / 5.0f;
    const float r = roundf(h->acc);
    h->acc        = h->acc - r;
    h->s          = h->s + SF + (int64_t)r;
    h->k++;
    if (lost_now && (h->cfg.flags & LTEPHY_TRACK_REACQUIRE)) h->find = true, h->f0 = h->s, h->kn = h->k;
  }
  const uint32_t nsf = (uint32_t)h->sf.size(), nh = (uint32_t)h->hf.size();
  // 3. the CFO sums at the chosen positions, then the loop in subframe order: each subframe keeps the offset that held before its half-frame
  std::vector<float2> c((size_t)nh * A * 2);
  if (nh) {
    CU(cudaMemcpyAsync(h->d_pos.p, hpos.data(), nh * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
    if (launch_track_sums(g, h->cfg.iq_format, h->d_pos.p, nh, h->d_c.p, h->stream))
      return fail(LTEPHY_ERROR, "track_push: sum kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
    CU(cudaMemcpyAsync(c.data(), h->d_c.p, c.size() * sizeof(float2), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
  }
  for (uint32_t i = 0, j = 0, ri = 0; i < nsf; i++) {
    ltephy_track_sf_t& o = h->sf[i];
    if (o.flags & LTEPHY_TRACK_REACQUIRED) {
      if (!(h->cfg.flags & LTEPHY_TRACK_NO_CFO)) h->f = fre[ri];
      ri++;
    }
    o.cfo_hz = h->f;
    if (j < nh && h->hf[j].index == o.index) {
      ltephy_track_hf_t& q  = h->hf[j];
      float              sr = 0.0f, si = 0.0f;
      for (uint32_t a = 0; a < A; a++) {
        const float2 c1 = c[((size_t)j * A + a) * 2], c2 = c[((size_t)j * A + a) * 2 + 1];
        sr              = sr + (c2.x * c1.x + c2.y * c1.y);
        si              = si + (c2.y * c1.x - c2.x * c1.y);
      }
      q.s_re = sr, q.s_im = si;
      q.f_meas = atan2f(si, sr) * (float)(15000.0 / M_PI);
      if ((q.flags & LTEPHY_TRACK_LOCKED) && !(h->cfg.flags & LTEPHY_TRACK_NO_CFO)) h->f = h->f + TRACK_ALPHA * (q.f_meas - h->f);
      j++;
    }
  }
  // 4. the cut of each carrier: its antennas from start + off, rotated by f = (float)(cfo_hz ratio) (cfo_hz itself at ratio 1) with the factor
  //    tables exp(-j th 128 q) and exp(-j th q) of each subframe, th = 2 pi f / (15000 N), in double, rounded to float
  std::vector<float2>   tabA[2], tabB[2]; // kept until the stream is synchronised
  std::vector<uint64_t> pos[2];
  for (uint32_t ci = 0; ci < h->nc && nsf; ci++) {
    TrackCarrier& cr = h->car[ci];
    tabA[ci].resize((size_t)nsf * (SF / 128)), tabB[ci].resize((size_t)nsf * 128), pos[ci].resize(nsf);
    for (uint32_t i = 0; i < nsf; i++) {
      const double th = 2.0 * M_PI * (double)(float)((double)h->sf[i].cfo_hz * cr.ratio) / (15000.0 * (double)N);
      for (uint32_t q = 0; q < SF / 128; q++)
        tabA[ci][(size_t)i * (SF / 128) + q] = make_float2((float)std::cos(-th * 128.0 * (double)q), (float)std::sin(-th * 128.0 * (double)q));
      for (uint32_t q = 0; q < 128; q++) tabB[ci][(size_t)i * 128 + q] = make_float2((float)std::cos(-th * (double)q), (float)std::sin(-th * (double)q));
      pos[ci][i] = (uint64_t)((int64_t)spos[i] + cr.off);
    }
    TrackArgs gc = g;
    gc.x = x[ci], gc.A = cr.A;
    CU(cudaMemcpyAsync(cr.d_start.p, pos[ci].data(), nsf * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(cr.d_tabA.p, tabA[ci].data(), tabA[ci].size() * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(cr.d_tabB.p, tabB[ci].data(), tabB[ci].size() * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
    if (launch_track_cut(gc, h->cfg.iq_format, cr.d_start.p, cr.d_tabA.p, cr.d_tabB.p, nsf, cr.d_cut.p, h->stream))
      return fail(LTEPHY_ERROR, "track_push: %scut kernel failed: %s", ci ? "UL " : "", cudaGetErrorString(cudaGetLastError()));
  }
  if (nsf) CU(cudaStreamSynchronize(h->stream));
  if (ul_iq_dev) *ul_iq_dev = h->car[1].d_cut.p;
  out->nof_subframes = nsf, out->nof_half_frames = nh;
  out->sf = h->sf.data(), out->hf = h->hf.data(), out->iq_dev = h->car[0].d_cut.p;
  out->next_sample = (uint64_t)track_needed(h), out->remeasured = remeasured, out->finds = finds;
  return LTEPHY_SUCCESS;
}

// every push: the samples of the downlink (x0) and, with ul, of the uplink (xu), on the host or, with dev, on the device
static int track_push(ltephy_track_t* h, const void* x0, const void* xu, bool dev, bool ul, uint64_t first, uint64_t n, ltephy_track_out_t* out,
                      const void** ul_iq_dev)
{
  const void* x[2] = {x0, xu};
  if (ul && !xu && n) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_push_ul: null argument");
  if (!h || !out || (!x[0] && n)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_push: null argument");
  if (ul != (h->nc == 2))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, ul ? "track_push_ul: ltephy_track_set_ul has not been called" : "track_push: the uplink is set: push with ltephy_track_push_ul");
  if ((int64_t)first > track_needed(h))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_push: first_sample %llu is after the next sample needed, %lld", (unsigned long long)first,
                (long long)track_needed(h));
  h->pushed = true;
  const size_t xb = iq_sample_bytes(h->cfg.iq_format);
  if (dev && (iq_misaligned(x[0], h->cfg.iq_format) || (ul && iq_misaligned(x[1], h->cfg.iq_format))))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, ul ? "track_push_ul_device: iq_dev / iq_ul_dev not aligned to their %zu-byte samples"
                                                : "track_push_device: iq_dev not aligned to its %zu-byte samples", xb);
  CU(cudaSetDevice(h->cfg.device));
  if (dev) return track_run(h, x, first, n, out, ul_iq_dev);
  for (uint32_t c = 0; n && c < h->nc; c++)
    if (h->car[c].d_x.reserve((size_t)h->car[c].A * n * xb))
      return fail(LTEPHY_ERROR, ul ? "track_push_ul: device allocation failed" : "track_push: device allocation failed");
  for (uint32_t c = 0; n && c < h->nc; c++)
    CU(cudaMemcpyAsync(h->car[c].d_x.p, x[c], (size_t)h->car[c].A * n * xb, cudaMemcpyHostToDevice, h->stream));
  const void* xd[2] = {h->car[0].d_x.p, h->car[1].d_x.p};
  return track_run(h, xd, first, n, out, ul_iq_dev);
}

extern "C" int ltephy_track_push(ltephy_track_t* h, const void* iq, uint64_t first_sample, uint64_t nof_samples, ltephy_track_out_t* out)
{
  return track_push(h, iq, nullptr, false, false, first_sample, nof_samples, out, nullptr);
}

extern "C" int ltephy_track_push_device(ltephy_track_t* h, const void* iq_dev, uint64_t first_sample, uint64_t nof_samples, ltephy_track_out_t* out)
{
  return track_push(h, iq_dev, nullptr, true, false, first_sample, nof_samples, out, nullptr);
}

extern "C" int ltephy_track_set_ul(ltephy_track_t* h, const ltephy_track_ul_cfg_t* cfg)
{
  if (!h || !cfg) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_set_ul: null argument");
  if (h->pushed || h->nc == 2) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_set_ul: only before the first push, once");
  if (!(cfg->cfo_ratio > 0.0 && cfg->cfo_ratio <= 2.0)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_set_ul: cfo_ratio outside (0, 2]");
  const int64_t off = cfg->ul_offset;
  if ((off < 0 ? -off : off) >= (int64_t)h->SF) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_set_ul: |ul_offset| %lld >= 15 N", (long long)off);
  if ((int64_t)h->cfg.frame_offset + off < 0)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_set_ul: the first UL subframe would start before sample 0 (frame_offset + ul_offset < 0)");
  if (cfg->nof_rx > 2) return fail(LTEPHY_ERROR_INVALID_INPUTS, "track_set_ul: nof_rx %u: 0 or 1 (one UL antenna) or 2", cfg->nof_rx);
  CU(cudaSetDevice(h->cfg.device));
  TrackCarrier& u = h->car[1];
  u.A = cfg->nof_rx ? cfg->nof_rx : 1;
  if (u.reserve(h->cfg.max_subframes, h->SF)) return fail(LTEPHY_ERROR, "track_set_ul: device allocation failed");
  h->nc = 2, u.ratio = cfg->cfo_ratio, u.off = cfg->ul_offset;
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_track_push_ul(ltephy_track_t* h, const void* iq, const void* iq_ul, uint64_t first_sample, uint64_t nof_samples,
                                    ltephy_track_out_t* out, const void** ul_iq_dev)
{
  return track_push(h, iq, iq_ul, false, true, first_sample, nof_samples, out, ul_iq_dev);
}

extern "C" int ltephy_track_push_ul_device(ltephy_track_t* h, const void* iq_dev, const void* iq_ul_dev, uint64_t first_sample, uint64_t nof_samples,
                                           ltephy_track_out_t* out, const void** ul_iq_dev)
{
  return track_push(h, iq_dev, iq_ul_dev, true, true, first_sample, nof_samples, out, ul_iq_dev);
}
