// ltephy_capi.cu -- C-ABI (include/ltephy_b200.h) of the CUDA LTE PHY library: device memory, table
// caches, job construction for phase A / phase B and kernel launches on one CUDA stream.
// There is no CPU fallback: creation fails when no CUDA device can be used.
#include "../../include/ltephy_b200.h"
#include "../../include/ltephy_search.h"
#include "ltephy_internal.cuh"
#include "k_launch.cuh"
#include "../../include/lte_tables.h"
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

static std::mutex  g_h2d_mtx;
static cudaEvent_t g_h2d_last[64]; // per device: completion of the most recently issued sample upload (phase_a_common)

thread_local std::string ltephy_g_err;
// a constant table of the handle on the device; a failure is kept in h->table_err, which ltephy_create checks after the last upload
template <typename T>
static T* upload(ltephy* h, const T* src, size_t n)
{
  if (h->table_err != cudaSuccess) return nullptr;
  DevBuf<uint8_t>& b = h->tables.emplace_back();
  if ((h->table_err = cudaMalloc(&b.p, n * sizeof(T))) != cudaSuccess ||
      (h->table_err = cudaMemcpy(b.p, src, n * sizeof(T), cudaMemcpyHostToDevice)) != cudaSuccess)
    return nullptr;
  b.cap = n * sizeof(T);
  return reinterpret_cast<T*>(b.p);
}

// Small host->device transfers do not use the copy engine: a DMA queued behind another pipeline's 0.5 GB IQ copy would
// hold this stream up for ~9 ms (measured: phase A 3.9 ms alone, 8.8 ms with a concurrent H2D).  The bytes sit in pinned
// host memory (device-visible under unified addressing) and a kernel pulls them over PCIe instead.
__global__ void __launch_bounds__(256) pull_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src_host, size_t n16)
{
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) dst[i] = src_host[i];
}
void ltephy_pull(ltephy* h, void* dst_dev, const void* src_pinned, size_t bytes, cudaStream_t st)
{
  const size_t n16 = (bytes + 15) / 16;
  if (!n16) return;
  const unsigned grid = (unsigned)std::min<size_t>((n16 + 255) / 256, 592);
  pull_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<uint4*>(dst_dev), reinterpret_cast<const uint4*>(src_pinned), n16);
  h->launches++;
}
static void pull(ltephy* h, void* dst_dev, const void* src_pinned, size_t bytes) { ltephy_pull(h, dst_dev, src_pinned, bytes, h->stream); }
// copy `bytes` from pageable memory into the handle's pinned arena (16-byte slots, consecutive calls take consecutive slots)
static uint8_t* stage(ltephy* h, const void* src, size_t bytes)
{
  uint8_t* slot = h->h_stage.p + h->stage_used;
  if (bytes) memcpy(slot, src, bytes);
  h->stage_used += (bytes + 15) & ~(size_t)15;
  return slot;
}
// stage `bytes` and pull them to dst_dev
static void stage_and_pull(ltephy* h, void* dst_dev, const void* src, size_t bytes)
{
  if (bytes) pull(h, dst_dev, stage(h, src, bytes), bytes);
}

extern "C" const char* ltephy_last_error(void) { return ltephy_g_err.c_str(); }

extern "C" int ltephy_create(const ltephy_cfg_t* cfg, ltephy_t** out)
{
  if (!cfg || !out) return fail(LTEPHY_ERROR_INVALID_INPUTS, "null argument");
  if (cfg->nof_prb <= 10 || cfg->nof_prb > 100 || cfg->nof_ports < 1 || cfg->nof_ports > 2 || cfg->nof_rx < 1 || cfg->nof_rx > 2 ||
      cfg->max_subframes == 0)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "unsupported cell/batch configuration");
  if (cfg->ul_nof_rx > 2) return fail(LTEPHY_ERROR_INVALID_INPUTS, "ul_nof_rx %u: 0 or 1 (one uplink antenna) or 2", cfg->ul_nof_rx);
  if (cfg->iq_format > LTEPHY_IQ_SC8) return fail(LTEPHY_ERROR_INVALID_INPUTS, "iq_format %u: LTEPHY_IQ_CF32 (0), LTEPHY_IQ_SC16 (1) or LTEPHY_IQ_SC8 (2)", cfg->iq_format);
  // the front end puts the subframe index on gridDim.y / gridDim.z (k_frontend.cu), which stop at 65 535
  if (cfg->max_subframes > LTEPHY_MAX_BATCH_SUBFRAMES)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "max_subframes %u: at most %u subframes per batch", cfg->max_subframes, (uint32_t)LTEPHY_MAX_BATCH_SUBFRAMES);
  // 2^k or 3 * 2^k samples per symbol, wide enough for the carrier: the standard LTE rate, or what srsran_symbol_sz answers in srsRAN's default
  // build (3/4 of it: 1536 at 100 PRB, 768 at 50, 384 at 25 -- the rate LTESniffer records at)
  if (cfg->symbol_sz) {
    const uint32_t N = cfg->symbol_sz, M = N % 3 ? N : N / 3;
    if ((M & (M - 1)) || M < 128 || N > 2048 || N <= 12 * cfg->nof_prb)
      return fail(LTEPHY_ERROR_INVALID_INPUTS, "symbol size %u not supported for %u PRB (2^k or 3 * 2^k, above %u, at most 2048)", N, cfg->nof_prb, 12 * cfg->nof_prb);
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(LTEPHY_ERROR, "no CUDA device: this library has no CPU path");
  CU(cudaSetDevice(cfg->device));
  std::unique_ptr<ltephy, decltype(&ltephy_destroy)> owner(new ltephy(), ltephy_destroy); // every failing return below destroys what was created so far
  ltephy* const                                      h = owner.get();
  h->cfg    = *cfg;
  if (!h->cfg.turbo_max_iter) h->cfg.turbo_max_iter = 8;
  if (!h->cfg.max_grants) h->cfg.max_grants = 24 * cfg->max_subframes;
  if (!h->cfg.ul_nof_rx) h->cfg.ul_nof_rx = 1;
  if (cfg->phich_resources > 3 || cfg->phich_length > 1)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "phich_resources %u / phich_length %u: 0 (Ng = 1/6), 1 (1/2), 2 (1) or 3 (2); 0 normal or 1 extended", cfg->phich_resources, cfg->phich_length);
  h->cell = {cfg->nof_prb, cfg->nof_ports, cfg->cell_id, cfg->nof_rx, cfg->phich_resources, cfg->phich_length};
  if (!ltehost::build_ctrl_map(h->cell, h->cm)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "control region map failed");
  h->st = ltehost::dci_size_table(h->cell);
  memset(h->pi_fast, 0xFF, sizeof(h->pi_fast));
  h->segm_fast.assign(110000 / 8, ltehost::Segm{});
  CU(cudaStreamCreateWithFlags(&h->stream.raw, cudaStreamNonBlocking));
  for (auto& e : h->ev) CU(cudaEventCreate(&e.raw));
  CU(cudaEventCreateWithFlags(&h->ev_h2d.raw, cudaEventDisableTiming));
  for (auto& e : h->mark) CU(cudaEventCreate(&e.raw));

  DevCell& c = h->dc;
  c.nof_prb = cfg->nof_prb, c.nof_ports = cfg->nof_ports, c.cell_id = cfg->cell_id, c.nof_rx = cfg->nof_rx, c.ul_nof_rx = h->cfg.ul_nof_rx;
  c.fft = cfg->symbol_sz ? cfg->symbol_sz : ltehost::fft_size(cfg->nof_prb), c.nsc = 12 * cfg->nof_prb, c.sf_len = 15 * c.fft;
  c.sub = c.fft % 3 ? c.fft : c.fft / 3; // length of the power-of-two transforms: the whole symbol, or a third of a 3 * 2^k one
  for (c.log2n = 0; (1u << c.log2n) < c.sub; c.log2n++) {
  }
  uint32_t pos = 0;
  for (uint32_t l = 0; l < 14; l++) {
    pos += ltehost::cp_len(c.fft, l % 7);
    c.sym_off[l] = pos;
    pos += c.fft;
  }
  for (int p = 0; p < 2; p++) {
    c.crs_off[p][0] = ltehost::crs_offset(h->cell, p, 0);
    c.crs_off[p][1] = ltehost::crs_offset(h->cell, p, 4);
  }
  { // smoothing filter {4,1} (src/src/SubframeWorker.cc:379-389), evaluated exactly like the oracle
    float s = 0.0f;
    for (int i = 0; i < 5; i++) {
      c.filt[i] = (float)std::exp(-(double)((i - 2) * (i - 2)) / 2.0);
      s         = s + c.filt[i];
    }
    float s2 = 0.0f;
    for (int i = 0; i < 5; i++) {
      c.filt[i] = c.filt[i] / s;
      s2        = s2 + c.filt[i] * c.filt[i];
    }
    c.noise_corr = (1.0f - 2.0f * c.filt[2]) + s2;
    for (int j = -5; j <= 11; j++) c.interp_c[j + 5] = (float)j / 6.0f;
    for (uint32_t l = 0; l < 14; l++) {
      if (l < 4)
        c.t_ia[l] = 0, c.t_ib[l] = 1, c.t_frac[l] = (float)l / 4.0f;
      else if (l < 7)
        c.t_ia[l] = 1, c.t_ib[l] = 2, c.t_frac[l] = (float)(l - 4) / 3.0f;
      else if (l < 11)
        c.t_ia[l] = 2, c.t_ib[l] = 3, c.t_frac[l] = (float)(l - 7) / 4.0f;
      else
        c.t_ia[l] = 2, c.t_ib[l] = 3, c.t_frac[l] = (float)(l - 11) / 4.0f;
    }
  }
  { // twiddles
    std::vector<float2> tw(c.sub / 2);
    for (uint32_t k = 0; k < c.sub / 2; k++) {
      double a = -2.0 * M_PI * (double)k / (double)c.sub;
      tw[k]    = make_float2((float)std::cos(a), (float)std::sin(a));
    }
    c.tw = upload(h, tw.data(), tw.size());
    std::vector<float2> tws(c.sub, make_float2(0.0f, 0.0f)); // per-stage contiguous copies: tws[H + pos] = tw[pos * sub / (2 H)]
    for (uint32_t H = 1; H <= c.sub / 2; H *= 2)
      for (uint32_t pos = 0; pos < H; pos++) tws[H + pos] = tw[(size_t)pos * (c.sub / (2 * H))];
    c.tw_st = upload(h, tws.data(), tws.size());
    c.w3    = nullptr;
    if (c.sub != c.fft) { // radix-3 step of a 3 * 2^k symbol: w3[k] = W_N^k, w3[N + k] = W_N^(2k)
      std::vector<float2> w3((size_t)2 * c.fft);
      for (uint32_t k = 0; k < c.fft; k++)
        for (uint32_t r = 1; r < 3; r++) {
          const double a = -2.0 * M_PI * (double)((uint64_t)r * k % c.fft) / (double)c.fft;
          w3[(size_t)(r - 1) * c.fft + k] = make_float2((float)std::cos(a), (float)std::sin(a));
        }
      c.w3 = upload(h, w3.data(), w3.size());
    }
    std::vector<float2> rot(c.fft);
    for (uint32_t i = 0; i < c.fft; i++) {
      double ph = M_PI * (double)i / (double)c.fft;
      rot[i]    = make_float2((float)std::cos(ph), (float)-std::sin(ph));
    }
    c.ul_rot = upload(h, rot.data(), rot.size());
  }
  {
    auto crs = ltehost::crs_table(h->cell);
    c.crs    = reinterpret_cast<const float2*>(upload(h, crs.data(), crs.size()));
  }
  c.nsizes = (uint32_t)h->st.sizes.size();
  if (c.nsizes > LTEPHY_MAX_SIZES) return fail(LTEPHY_ERROR, "too many distinct DCI sizes");
  for (uint32_t i = 0; i < c.nsizes; i++) {
    c.sizes[i]    = h->st.sizes[i];
    auto t        = ltehost::conv_rm_table(c.sizes[i] + 16);
    c.conv_tab[i] = upload(h, t.data(), t.size());
  }
  { // PBCH: resource elements of subframe 0 (slot 1, symbols 0..3, central 72 sub-carriers minus the CRS of four ports), c(cell_id), rate matching of K = 40
    std::vector<uint32_t> re;
    const uint32_t        k0 = c.nsc / 2 - 36;
    for (uint32_t l = 7; l < 11; l++)
      for (uint32_t k = k0; k < k0 + 72; k++)
        if (!(l < 9 && k % 3 == c.cell_id % 3)) re.push_back((l << 16) | k);
    c.pbch_re = upload(h, re.data(), re.size());
    auto gw    = ltehost::gold_words(c.cell_id, 1920);
    c.pbch_scr = upload(h, gw.data(), gw.size());
    auto t40   = ltehost::conv_rm_table(40);
    c.pbch_tab = upload(h, t40.data(), t40.size());
    c.cfo_rot  = nullptr;
    c.ul_cfo_rot = nullptr;
  }
  for (uint32_t cfi = 0; cfi < 3; cfi++) {
    c.nof_cce[cfi] = h->cm.nof_cce[cfi];
    c.pdcch_idx[cfi] = upload(h, h->cm.pdcch_idx[cfi].data(), h->cm.pdcch_idx[cfi].size());
    auto                  locs = ltehost::all_locations(c.nof_cce[cfi]);
    std::vector<uint16_t> lt;
    for (auto& l : locs) lt.push_back((uint16_t)(l.ncce | (l.L << 8)));
    c.nloc[cfi]    = (uint32_t)lt.size();
    c.loc_tab[cfi] = upload(h, lt.data(), lt.size());
  }
  memcpy(c.pcfich_idx, h->cm.pcfich_idx, sizeof(c.pcfich_idx));
  {
    c.pdcch_scr_words = (LTEPHY_MAX_CCE * 72 + 31) / 32;
    std::vector<uint32_t> scr(10 * c.pdcch_scr_words);
    for (uint32_t sf = 0; sf < 10; sf++) {
      auto w = ltehost::gold_words((sf << 9) + c.cell_id, LTEPHY_MAX_CCE * 72);
      std::copy(w.begin(), w.end(), scr.begin() + sf * c.pdcch_scr_words);
      c.pcfich_scr[sf] = ltehost::gold_words((sf + 1) * (2 * c.cell_id + 1) * 512u + c.cell_id, 32)[0];
    }
    c.pdcch_scr = upload(h, scr.data(), scr.size());
  }
  c.flags = cfg->flags;
  { // Gold basis for PDSCH descrambling: up to 14*nsc*8 bits per codeword
    auto gb         = ltehost::gold_basis(14 * c.nsc * 8);
    h->gold_words   = gb.nwords;
    h->d_gold_x1    = upload(h, gb.x1.data(), gb.x1.size());
    h->d_gold_basis = upload(h, gb.basis.data(), gb.basis.size());
    auto xa = ltehost::crc24_xpow8(ltehost::CRC24A, 16384), xb = ltehost::crc24_xpow8(ltehost::CRC24B, 1024);
    h->d_xpowA = upload(h, xa.data(), xa.size());
    h->d_xpowB = upload(h, xb.data(), xb.size());
  }
  { // data-RE count and 12-bit mask per (subframe class, cfi, symbol, prb)
    const uint32_t N = c.nof_prb;
    h->re_cnt.resize((size_t)3 * 3 * 14 * N);
    std::vector<uint16_t> masks((size_t)3 * 3 * 14 * N, 0);
    const uint32_t        cls_sf[3] = {0, 5, 1};
    uint16_t              kk[12];
    for (uint32_t cls = 0; cls < 3; cls++)
      for (uint32_t cfi = 1; cfi <= 3; cfi++)
        for (uint32_t l = 0; l < 14; l++)
          for (uint32_t prb = 0; prb < N; prb++) {
            const size_t   idx = ((cls * 3 + (cfi - 1)) * 14 + l) * N + prb;
            const uint32_t n   = ltehost::pdsch_re_in_prb(h->cell, cls_sf[cls], cfi, l, prb, kk);
            h->re_cnt[idx]     = (uint8_t)n;
            for (uint32_t i = 0; i < n; i++) masks[idx] |= (uint16_t)(1u << (kk[i] - 12 * prb));
          }
    c.re_mask = upload(h, masks.data(), masks.size());
  }
  if (h->table_err != cudaSuccess) return fail(LTEPHY_ERROR, "table upload failed: %s", cudaGetErrorString(h->table_err));
  const size_t S = cfg->max_subframes, g = (size_t)14 * c.nsc;
  if (h->d_iq.reserve(S * c.nof_rx * c.sf_len * iq_sample_bytes(cfg->iq_format)) || h->d_sym.reserve(S * c.nof_rx * g) || h->d_pil.reserve(S * c.nof_ports * c.nof_rx * 4 * 2 * c.nof_prb) ||
      h->d_llr.reserve(S * LLR_STRIDE) || h->d_info.reserve(S) || h->d_cands.reserve(S * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES) || h->d_vwork.reserve(S * (LTEPHY_MAX_LOC / 2) * LTEPHY_MAX_SIZES * 2 + 16) ||
      h->h_info.reserve(S) || h->d_compact.reserve(S) || h->h_compact.reserve(S) || h->d_rm.reserve((size_t)4 << 20) || h->d_pi.reserve((size_t)188 * 6144))
    return fail(LTEPHY_ERROR, "device allocation failed");
  CU(cudaMemset(h->d_cands.p, 0, h->d_cands.cap * sizeof(ltephy_cand_t)));
  *out = owner.release();
  return LTEPHY_SUCCESS;
}

extern "C" void ltephy_destroy(ltephy_t* h)
{
  if (!h) return;
  cudaSetDevice(h->cfg.device);
  cudaDeviceSynchronize();
  {
    std::lock_guard<std::mutex> lk(g_h2d_mtx); // no later upload may wait on the event once it is destroyed
    if (g_h2d_last[h->cfg.device & 63] == h->ev_h2d) g_h2d_last[h->cfg.device & 63] = nullptr;
  }
  delete h;
}

extern "C" uint32_t ltephy_sf_len(const ltephy_t* h) { return h->dc.sf_len; }
extern "C" uint32_t ltephy_nof_cce(const ltephy_t* h, uint32_t cfi) { return cfi >= 1 && cfi <= 3 ? h->dc.nof_cce[cfi - 1] : 0; }
extern "C" uint32_t ltephy_nof_sizes(const ltephy_t* h) { return h->dc.nsizes; }
extern "C" uint32_t ltephy_dci_size(const ltephy_t* h, uint32_t f) { return f < LTEPHY_NOF_FORMATS ? h->st.sizes[h->st.index_of[f]] : 0; }
extern "C" uint32_t ltephy_size_index(const ltephy_t* h, uint32_t f) { return f < LTEPHY_NOF_FORMATS ? h->st.index_of[f] : 0; }
extern "C" uint32_t ltephy_locations(const ltephy_t* h, uint32_t cfi, uint16_t* ncce, uint8_t* L, uint32_t max)
{
  if (cfi < 1 || cfi > 3) return 0;
  auto     v = ltehost::all_locations(h->dc.nof_cce[cfi - 1]);
  uint32_t n = (uint32_t)std::min<size_t>(v.size(), max);
  for (uint32_t i = 0; i < n; i++) ncce[i] = v[i].ncce, L[i] = v[i].L;
  return n;
}
extern "C" void ltephy_cell_of(const ltephy_t* h, uint32_t* a, uint32_t* b, uint32_t* c, uint32_t* d)
{
  *a = h->cell.nof_prb, *b = h->cell.nof_ports, *c = h->cell.cell_id, *d = h->cell.nof_rx;
}
extern "C" uint32_t ltephy_phich_resources(const ltephy_t* h) { return h ? h->cell.phich_ng | (h->cell.phich_ext << 8) : 0; }
extern "C" int ltephy_mark(ltephy_t* h, int slot)
{
  if (!h || slot < 0 || slot > 1) return LTEPHY_ERROR_INVALID_INPUTS;
  CU(cudaEventRecord(h->mark[slot], h->stream));
  return LTEPHY_SUCCESS;
}
extern "C" float ltephy_mark_elapsed_ms(ltephy_t* h)
{
  float ms = -1.0f;
  if (cudaEventSynchronize(h->mark[1]) != cudaSuccess) return -1.0f;
  cudaEventElapsedTime(&ms, h->mark[0], h->mark[1]);
  return ms;
}
extern "C" int ltephy_last_turbo_work(ltephy_t* h, uint64_t* bytes, uint64_t* code_blocks, uint64_t* info_bits)
{
  uint64_t b = 0, ib = 0;
  for (auto& cb : h->pb.cbs) b += 3ull * (cb.K + 4) * 2 + cb.K / 8;
  for (auto& tb : h->pb.tbs) ib += 8ull * tb.nbytes;
  if (bytes) *bytes = b;
  if (code_blocks) *code_blocks = h->pb.cbs.size();
  if (info_bits) *info_bits = ib;
  return LTEPHY_SUCCESS;
}
extern "C" uint64_t ltephy_launch_count(const ltephy_t* h) { return h->launches; }
extern "C" int      ltephy_last_timing(ltephy_t* h, float ms[4])
{
  memcpy(ms, h->t_ms, sizeof(h->t_ms));
  return LTEPHY_SUCCESS;
}

// ---------------------------------------------------------------------------------------- phase A
// Phase A over n subframes.  iq_host != nullptr: the samples are still in (pinned) host memory and are copied first, as ONE
// transfer: splitting it into chunks with per-chunk kernels was measured and is slower with several pipelines (the chunks of
// different batches interleave on the copy engine, so every batch's front end finishes later: e2e 87-91 k -> 82 k subframes/s).
static int phase_a_common(ltephy* h, const void* iq_dev, const void* iq_host, const uint32_t* tti, uint32_t n)
{
  for (uint32_t i = 0; i < n; i++) {
    memset(&h->h_info.p[i], 0, sizeof(DevSfInfo));
    h->h_info.p[i].tti = tti[i];
  }
  pull(h, h->d_info.p, h->h_info.p, n * sizeof(DevSfInfo));
  const DevCell& c = h->dc;
  if (iq_host) {
    // Host-to-device copies of different handles are chained (each waits for the one issued before it on this device): the copy engine would
    // otherwise interleave them, and every batch would get its samples late instead of the first one getting them at full PCIe rate.
    std::lock_guard<std::mutex> lk(g_h2d_mtx);
    cudaEvent_t& last = g_h2d_last[h->cfg.device & 63];
    if (last && last != h->ev_h2d) CU(cudaStreamWaitEvent(h->stream, last, 0));
    CU(cudaMemcpyAsync(h->d_iq.p, iq_host, (size_t)n * c.nof_rx * c.sf_len * iq_sample_bytes(h->cfg.iq_format), cudaMemcpyHostToDevice, h->stream));
    CU(cudaEventRecord(h->ev_h2d, h->stream));
    last = h->ev_h2d;
  }
  launch_frontend(c, iq_dev, h->cfg.iq_format, h->d_sym.p, h->d_pil.p, h->d_llr.p, h->d_info.p, n, h->stream, &h->launches);
  launch_viterbi(c, h->d_llr.p, h->d_info.p, h->d_cands.p, h->d_vwork.p, n, h->stream, &h->launches);
  launch_compact(c, h->d_info.p, h->d_cands.p, h->d_compact.p, n, h->stream, &h->launches);
  CU(cudaEventRecord(h->ev[1], h->stream));
  CU(cudaGetLastError());
  h->n_cur = n;
  return LTEPHY_SUCCESS;
}
extern "C" int ltephy_submit_iq(ltephy_t* h, const void* iq, const uint32_t* tti, uint32_t n)
{
  if (!h || !iq || !tti || n == 0 || n > h->cfg.max_subframes) return fail(LTEPHY_ERROR_INVALID_INPUTS, "submit_iq: bad arguments");
  CU(cudaSetDevice(h->cfg.device));
  CU(cudaEventRecord(h->ev[0], h->stream));
  return phase_a_common(h, h->d_iq.p, iq, tti, n);
}
extern "C" int ltephy_submit_iq_device(ltephy_t* h, const void* iq_dev, const uint32_t* tti, uint32_t n)
{
  if (!h || !iq_dev || !tti || n == 0 || n > h->cfg.max_subframes) return fail(LTEPHY_ERROR_INVALID_INPUTS, "submit_iq_device: bad arguments");
  if (iq_misaligned(iq_dev, h->cfg.iq_format))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "submit_iq_device: iq_dev not aligned to its %zu-byte samples", iq_sample_bytes(h->cfg.iq_format));
  CU(cudaSetDevice(h->cfg.device));
  CU(cudaEventRecord(h->ev[0], h->stream));
  return phase_a_common(h, iq_dev, nullptr, tti, n); // read in place: the caller keeps the buffer alive until phase A is fetched
}
// log10f / atan2f of the bit-exact device sums are taken on the host (DESIGN.md section 2); idempotent
extern "C" void ltephy_finalize_info(ltephy_sf_info_t* info, uint32_t n, uint32_t nof_ports, uint32_t nof_rx)
{
  const float npa = (float)(nof_ports * nof_rx);
  for (uint32_t i = 0; i < n; i++) {
    DevSfInfo& s  = reinterpret_cast<DevSfInfo*>(info)[i];
    float      ns = 0.0f, ps = 0.0f;
    for (uint32_t p = 0; p < nof_ports; p++)
      for (uint32_t a = 0; a < nof_rx; a++) {
        ns = ns + s.noise[p][a];
        ps = ps + s.rsrp[p][a];
      }
    s.noise_avg = ns / npa;
    s.rsrp_avg  = ps / npa;
    s.snr_db    = 10.0f * log10f(s.rsrp_avg / s.noise_avg);
    s.cfo       = atan2f(s.cfo_im, s.cfo_re) / (2.0f * (float)M_PI * 7.5f);
  }
}
// Device-to-device copies of the raw per-subframe records and the survivor forms of the current batch, for an all-gather
// without a host round trip (a host->device DMA would queue behind the other pipelines' IQ copies).  Blocks until done.
extern "C" int ltephy_copy_phase_a_device(ltephy_t* h, void* dst_info_dev, void* dst_compact_dev)
{
  if (!h || !h->n_cur) return fail(LTEPHY_ERROR_INVALID_INPUTS, "copy_phase_a_device: nothing submitted");
  CU(cudaSetDevice(h->cfg.device));
  const uint32_t n = h->n_cur;
  if (dst_info_dev) CU(cudaMemcpyAsync(dst_info_dev, h->d_info.p, (size_t)n * sizeof(DevSfInfo), cudaMemcpyDeviceToDevice, h->stream));
  if (dst_compact_dev) CU(cudaMemcpyAsync(dst_compact_dev, h->d_compact.p, (size_t)n * sizeof(ltephy_compact_t), cudaMemcpyDeviceToDevice, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return LTEPHY_SUCCESS;
}
static int fetch_phase_a(ltephy_t* h, ltephy_sf_info_t* info, ltephy_cand_t* cands, bool compact, ltephy_compact_t* comp)
{
  if (!h || !h->n_cur) return fail(LTEPHY_ERROR_INVALID_INPUTS, "get_phase_a: nothing submitted");
  const uint32_t n = h->n_cur;
  CU(cudaMemcpyAsync(h->h_info.p, h->d_info.p, n * sizeof(DevSfInfo), cudaMemcpyDeviceToHost, h->stream));
  if (cands)
    CU(cudaMemcpyAsync(cands, h->d_cands.p, (size_t)n * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES * sizeof(ltephy_cand_t), cudaMemcpyDeviceToHost,
                       h->stream));
  if (compact) CU(cudaMemcpyAsync(comp ? comp : h->h_compact.p, h->d_compact.p, (size_t)n * sizeof(ltephy_compact_t), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  cudaEventElapsedTime(&h->t_ms[0], h->ev[0], h->ev[1]);
  ltephy_finalize_info(reinterpret_cast<ltephy_sf_info_t*>(h->h_info.p), n, h->dc.nof_ports, h->dc.nof_rx);
  if (info) memcpy(info, h->h_info.p, (size_t)n * sizeof(DevSfInfo));
  return LTEPHY_SUCCESS;
}
extern "C" int ltephy_get_phase_a(ltephy_t* h, ltephy_sf_info_t* info, ltephy_cand_t* cands) { return fetch_phase_a(h, info, cands, false, nullptr); }
extern "C" int ltephy_get_phase_a_compact(ltephy_t* h, ltephy_sf_info_t* info, ltephy_compact_t* comp) { return fetch_phase_a(h, info, nullptr, true, comp); }
extern "C" const ltephy_compact_t* ltephy_phase_a_compact_buffer(const ltephy_t* h) { return h ? h->h_compact.p : nullptr; }

// ---------------------------------------------------------------------------------------- phase B
// words of one code-block pair in the turbo pool: the three window-transposed input streams (sys, p1, p2: [32][NW] each) and the
// 12 termination words; the decoder keeps its extrinsic values in shared memory and its window-boundary metrics in per-CTA scratch
static inline size_t ltephy_pair_words(uint32_t NW) { return (size_t)3 * 32 * NW + 16; }
// Append n values to a pool of lazily built device tables and return their offset, or -1.  A full pool is reallocated to 2 * cap + n once
// the stream has drained, and its used part copied over, so every offset handed out earlier stays valid.  The upload is synchronous, so src
// may be a temporary.
template <typename T>
static int64_t pool_append(ltephy* h, DevBuf<T>& pool, size_t& used, const T* src, size_t n)
{
  if (used + n > pool.cap) {
    const size_t want = 2 * pool.cap + n;
    DevBuf<T>    grown;
    if (cudaStreamSynchronize(h->stream) != cudaSuccess || cudaMalloc(&grown.p, want * sizeof(T)) != cudaSuccess ||
        cudaMemcpy(grown.p, pool.p, used * sizeof(T), cudaMemcpyDeviceToDevice) != cudaSuccess)
      return -1;
    grown.cap = want;
    pool      = std::move(grown);
  }
  if (cudaMemcpyAsync(pool.p + used, src, n * sizeof(T), cudaMemcpyHostToDevice, h->stream) != cudaSuccess) return -1;
  cudaStreamSynchronize(h->stream);
  used += n;
  return (int64_t)(used - n);
}
// inverse rate-matching table of (K, F) in the pool (one per code-block size and filler count; the redundancy version is a rotation)
static const ltephy::RmEntry* rm_table_for(ltephy* h, uint32_t K, uint32_t F)
{
  const int ki = lte_qpp_index_ge(K);
  if (ki < 0 || lte_qpp_K((uint32_t)ki) != K) return nullptr;
  ltephy::RmEntry& e = F == 0 ? h->rm_fast[ki] : h->rm_cache[{K, F}];
  if (e.off >= 0) return &e;
  auto t = ltehost::rm_turbo_inverse(K, F);
  if ((e.off = pool_append(h, h->d_rm, h->rm_used, t.inv.data(), t.inv.size())) < 0) return nullptr;
  e.nn = t.nn;
  memcpy(e.rot, t.rot, sizeof(e.rot));
  return &e;
}
extern "C" int ltephy_rm_turbo_tables(uint32_t K, uint32_t F, uint32_t rv, uint32_t* order, uint32_t* nn, uint16_t* inv, uint32_t* rot)
{
  const int ki = lte_qpp_index_ge(K);
  if (ki < 0 || lte_qpp_K((uint32_t)ki) != K || F >= K || rv > 3 || !order || !nn || !inv || !rot)
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "rm_turbo_tables: bad arguments");
  const auto t = ltehost::rm_turbo_table(K, F, rv);
  for (uint32_t k = 0; k < t.nn; k++) order[k] = ltehost::rm_turbo_word(K, t.order[k]);
  *nn          = t.nn;
  const auto v = ltehost::rm_turbo_inverse(K, F);
  memcpy(inv, v.inv.data(), v.inv.size() * sizeof(uint16_t));
  memcpy(rot, v.rot, sizeof(v.rot));
  return LTEPHY_SUCCESS;
}
// QPP interleaver table of K in the pool, window-transposed like the turbo streams
static int pi_table_for(ltephy* h, uint32_t K, uint32_t& off)
{
  const int ki = lte_qpp_index_ge(K);
  if (ki < 0) return -1;
  if (h->pi_fast[ki] < 0) {
    uint32_t f1, f2;
    if (!ltehost::qpp_params(K, f1, f2)) return -1;
    const uint32_t        NW = (K + 31) / 32;
    std::vector<uint16_t> t((size_t)32 * NW, 0);
    for (uint64_t i = 0; i < K; i++) t[(i & 31) * NW + (i >> 5)] = (uint16_t)((f1 * i + f2 * i * i) % K);
    if ((h->pi_fast[ki] = pool_append(h, h->d_pi, h->pi_used, t.data(), t.size())) < 0) return -1;
  }
  off = (uint32_t)h->pi_fast[ki];
  return 0;
}

// transport block -> code blocks (shared by the PDSCH and PUSCH paths); pair_code_blocks puts them into turbo pairs once the batch is complete
static int add_transport_block(ltephy* h, uint32_t tbs, uint32_t G, uint32_t qm, uint32_t rv, uint32_t NL, uint64_t llr_off, uint32_t& tb_index,
                               uint32_t harq_op = LTEPHY_HARQ_NONE, uint32_t harq_slot = 0)
{
  if (tbs / 8 >= h->segm_fast.size() || (tbs & 7)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "invalid TBS %u", tbs);
  if (h->segm_fast[tbs / 8].C == 0 && !ltehost::cb_segmentation(tbs, h->segm_fast[tbs / 8])) return fail(LTEPHY_ERROR_INVALID_INPUTS, "invalid TBS %u", tbs);
  const ltehost::Segm& s = h->segm_fast[tbs / 8];
  ltephy::PhaseB&      b = h->pb;
  uint32_t             harq_gen = 0;
  if (harq_op != LTEPHY_HARQ_NONE) {
    if (harq_op > LTEPHY_HARQ_RETX || harq_slot >= h->harq_slots) return fail(LTEPHY_ERROR_INVALID_INPUTS, "HARQ slot %u outside the store (%u slots, ltephy_harq_reserve)", harq_slot, h->harq_slots);
    if (s.C > 16) return fail(LTEPHY_ERROR_INVALID_INPUTS, "transport block of %u code blocks does not fit a HARQ slot", s.C);
    harq_gen       = b.harq_uses[harq_slot]++; // a slot used again inside one batch: its rate-dematch runs in a later launch, after the earlier use
    b.harq_max_gen = std::max(b.harq_max_gen, harq_gen);
  }
  DevTb                tb{};
  tb.byte_off = (uint32_t)b.payload_bytes, tb.nbytes = tbs / 8, tb.cb_first = (uint32_t)b.cbs.size(), tb.ncb = s.C;
  b.payload_bytes += (tb.nbytes + 3 + 3) & ~3u;
  uint64_t rp   = llr_off;
  uint32_t wbit = 0;
  for (uint32_t r = 0; r < s.C; r++) {
    DevCb cb{};
    cb.K = s.K(r), cb.F = r == 0 ? s.F : 0, cb.E = ltehost::rm_turbo_E(G, s.C, r, qm, NL);
    cb.llr_off = rp;
    rp += cb.E;
    cb.shift = qm == 2 ? 0 : qm == 4 ? 1 : 2;
    cb.harq_op = harq_op, cb.harq_off = harq_op ? (uint64_t)harq_slot * (LTEPHY_HARQ_SLOT_BYTES / 2) + (uint64_t)r * 18448u : 0u, cb.harq_gen = harq_gen;
    const ltephy::RmEntry* rm = rm_table_for(h, cb.K, cb.F);
    if (!rm) return fail(LTEPHY_ERROR, "rate-matching table upload failed");
    cb.rm_tab = (uint32_t)rm->off, cb.rm_nn = rm->nn, cb.rm_rot = rm->rot[rv & 3u];
    ltephy::PhaseB::CbHalf o;
    o.tbs = tbs, o.G = G, o.crc_type = s.C > 1 ? 2 : 1, o.out_bits = cb.K - cb.F - (s.C > 1 ? 24 : 0), o.out_byte = tb.byte_off + wbit / 8;
    wbit += o.out_bits;
    b.cbs.push_back(cb);
    b.cb_half.push_back(o);
  }
  tb_index = (uint32_t)b.tbs.size();
  b.tbs.push_back(tb);
  return LTEPHY_SUCCESS;
}
// LLR and scrambling space of one codeword: G soft bits, scrambled with the first `bits` bits of the Gold sequence of c_init (PDSCH: G,
// PUSCH: 12 M Qm), whose words go on scr_seq_kernel's list; false if the scrambling basis is shorter
static bool alloc_codeword(ltephy* h, uint32_t bits, uint32_t G, uint32_t c_init, uint64_t& llr_off, uint32_t& scr_off)
{
  ltephy::PhaseB& b = h->pb;
  const uint32_t  w = (bits + 31) / 32;
  if (w > h->gold_words) return false;
  llr_off = b.pllr_elems, scr_off = (uint32_t)b.seq_words;
  b.scr.push_back(DevScr{c_init, w, scr_off});
  b.max_scr_words = std::max(b.max_scr_words, w);
  b.seq_words += w + 1; // +1: the demapper reads a 64-bit window
  b.pllr_elems += (G + 7) & ~7u;
  return true;
}

// Code blocks -> turbo pairs (two code blocks of equal K, one per 16-bit half).  A pair runs until both halves pass their CRC or reach the
// iteration limit, so it costs K x the larger of the two iteration counts, while each half's result depends on its own inputs alone.
// Blocks of one K are therefore paired in the order of their transport block's code rate TBS / G (highest first, in steps of 2^-16, then
// index): neighbours in that order tend to need similar iteration counts.  Pairs are numbered in the same order, larger K first, so each
// persistent turbo launch (one per CTA size, launch_turbo_buckets) takes its longest pairs off the queue first.  This runs on the host for every
// batch, between the DCI walk and the launch of phase B, so it is a stable counting sort of a 24-bit key (187 - QPP index of K, then
// 0xFFFF - rate), two passes of 12 bits: O(n), where a comparison sort of a cfg-2 batch's 25 000 code blocks took milliseconds.
static uint32_t turbo_pairing(uint32_t ncb, const uint32_t* K, const uint32_t* tbs, const uint32_t* G, uint32_t* pair, uint32_t* half)
{
  std::vector<uint32_t> key(ncb), ord(ncb), tmp(ncb), cnt(4097);
  for (uint32_t i = 0; i < ncb; i++) {
    const uint64_t rate = G[i] ? std::min<uint64_t>(((uint64_t)tbs[i] << 16) / G[i], 0xFFFFu) : 0xFFFFu;
    key[i] = ((187u - (uint32_t)lte_qpp_index_ge(K[i])) << 16) | (0xFFFFu - (uint32_t)rate);
    ord[i] = i;
  }
  for (uint32_t shift = 0; shift < 24; shift += 12) {
    std::fill(cnt.begin(), cnt.end(), 0u);
    for (uint32_t i = 0; i < ncb; i++) cnt[((key[i] >> shift) & 0xFFFu) + 1]++;
    for (uint32_t d = 0; d < 4096; d++) cnt[d + 1] += cnt[d];
    for (uint32_t j = 0; j < ncb; j++) tmp[cnt[(key[ord[j]] >> shift) & 0xFFFu]++] = ord[j];
    ord.swap(tmp);
  }
  uint32_t np = 0;
  for (uint32_t j = 0; j < ncb; j++) {
    const uint32_t ci = ord[j];
    const bool     second = j > 0 && half[ord[j - 1]] == 0 && K[ord[j - 1]] == K[ci];
    half[ci] = second ? 1u : 0u;
    pair[ci] = second ? np - 1 : np++;
  }
  return np;
}
extern "C" int ltephy_turbo_pairing(uint32_t ncb, const uint32_t* K, const uint32_t* tbs, const uint32_t* G, uint32_t* pair, uint32_t* half,
                                    uint32_t* npairs)
{
  if ((ncb && (!K || !tbs || !G || !pair || !half)) || !npairs) return fail(LTEPHY_ERROR_INVALID_INPUTS, "turbo_pairing: bad arguments");
  for (uint32_t i = 0; i < ncb; i++) {
    const int ki = lte_qpp_index_ge(K[i]);
    if (ki < 0 || lte_qpp_K((uint32_t)ki) != K[i]) return fail(LTEPHY_ERROR_INVALID_INPUTS, "turbo_pairing: K=%u is not a turbo block size", K[i]);
  }
  *npairs = turbo_pairing(ncb, K, tbs, G, pair, half);
  return LTEPHY_SUCCESS;
}
static int pair_code_blocks(ltephy* h)
{
  ltephy::PhaseB&       b   = h->pb;
  const uint32_t        ncb = (uint32_t)b.cbs.size();
  std::vector<uint32_t> K(ncb), tbs(ncb), G(ncb), pair(ncb), half(ncb);
  for (uint32_t i = 0; i < ncb; i++) K[i] = b.cbs[i].K, tbs[i] = b.cb_half[i].tbs, G[i] = b.cb_half[i].G;
  b.pairs.assign(turbo_pairing(ncb, K.data(), tbs.data(), G.data(), pair.data(), half.data()), DevPair{});
  for (uint32_t ci = 0; ci < ncb; ci++) {
    DevCb&                        cb = b.cbs[ci];
    DevPair&                      p  = b.pairs[pair[ci]];
    const ltephy::PhaseB::CbHalf& o  = b.cb_half[ci];
    const uint32_t                hh = half[ci];
    cb.pair = pair[ci], cb.half = hh;
    p.K = cb.K, p.ncb = std::max(p.ncb, hh + 1);
    p.crc_type[hh] = o.crc_type;
    p.out_skip[hh] = cb.F;
    p.out_bits[hh] = o.out_bits;
    p.out_byte[hh] = o.out_byte;
    p.cb_index[hh] = ci;
  }
  b.turbo_words = 0;
  b.pair_pi_off.resize(b.pairs.size());
  for (uint32_t pi = 0; pi < b.pairs.size(); pi++) {
    DevPair& p = b.pairs[pi];
    p.NW = (p.K + 31) / 32;
    ltehost::qpp_params(p.K, p.f1, p.f2);
    p.buf_off = b.turbo_words;
    b.turbo_words += ltephy_pair_words(p.NW);
    if (pi_table_for(h, p.K, b.pair_pi_off[pi])) return fail(LTEPHY_ERROR, "interleaver table upload failed");
  }
  return LTEPHY_SUCCESS;
}

static int build_jobs(ltephy* h, const ltephy_grant_t* gin, uint32_t n)
{
  const DevCell&  c = h->dc;
  const uint32_t  N = c.nof_prb;
  ltephy::PhaseB& b = h->pb;
  b.reset((size_t)n * 2);
  b.grants.reserve(n), b.cbs.reserve((size_t)n * 4), b.cb_half.reserve((size_t)n * 4), b.pairs.reserve((size_t)n * 2), b.tbs.reserve((size_t)n * 2),
      b.pair_pi_off.reserve((size_t)n * 2);
  for (uint32_t gi = 0; gi < n; gi++) {
    const ltephy_grant_t& g = gin[gi];
    if (g.sf >= h->n_cur) return fail(LTEPHY_ERROR_INVALID_INPUTS, "grant %u: subframe %u outside the batch", gi, g.sf);
    DevGrant d{};
    d.sf = g.sf, d.sf_idx = h->h_info.p[g.sf].tti % 10, d.cfi = h->h_info.p[g.sf].cfi, d.rnti = g.rnti, d.tx_scheme = g.tx_scheme;
    if (d.cfi < 1 || d.cfi > 3) return fail(LTEPHY_ERROR_INVALID_INPUTS, "grant %u: subframe has no CFI (phase A not fetched?)", gi);
    memcpy(d.prb_mask, g.prb_mask, sizeof(d.prb_mask));
    const uint32_t cls = d.sf_idx == 0 ? 0 : d.sf_idx == 5 ? 1 : 2;
    const uint8_t* cnt = &h->re_cnt[((size_t)(cls * 3 + d.cfi - 1) * 14) * N];
    uint32_t       acc = 0;
    uint8_t        plist[2][LTEPHY_MAX_PRB];
    uint32_t       pn[2] = {0, 0};
    for (uint32_t sl = 0; sl < 2; sl++)
      for (uint32_t w = 0; w < 4; w++) {
        uint32_t m = d.prb_mask[sl][w];
        while (m) {
          const uint32_t b = (uint32_t)__builtin_ctz(m);
          m &= m - 1;
          if (32 * w + b < N) plist[sl][pn[sl]++] = (uint8_t)(32 * w + b);
        }
      }
    for (uint32_t l = 0; l < 14; l++) {
      d.re_off[l] = acc;
      const uint8_t* pl = plist[l / 7];
      const uint8_t* cl = cnt + l * N;
      for (uint32_t i = 0; i < pn[l / 7]; i++) acc += cl[pl[i]];
    }
    d.cls = cls, d.np[0] = pn[0], d.np[1] = pn[1];
    memcpy(d.plist[0], plist[0], pn[0]);
    memcpy(d.plist[1], plist[1], pn[1]);
    d.re_off[14] = acc;
    d.nof_re     = acc;
    if (acc != g.nof_re) return fail(LTEPHY_ERROR_INVALID_INPUTS, "grant %u: nof_re %u does not match the PRB mask (%u)", gi, g.nof_re, acc);
    const bool two_cw = g.tx_scheme == LTEPHY_TX_CDD || (g.tx_scheme == LTEPHY_TX_SPATIALMUX && g.nof_tb == 2);
    if (g.tx_scheme == LTEPHY_TX_SPATIALMUX && (c.nof_ports != 2 || (g.nof_tb == 2 && c.nof_rx != 2) || g.pmi > 3 || (g.nof_tb == 2 && g.pmi > 1)))
      return fail(LTEPHY_ERROR_INVALID_INPUTS, "grant %u: unsupported spatial multiplexing configuration", gi);
    d.pmi = g.pmi;
    if (g.tx_scheme == LTEPHY_TX_CDD && !(c.nof_ports == 2 && c.nof_rx == 2)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "grant %u: CDD needs 2x2", gi);
    if (g.tx_scheme == LTEPHY_TX_DIVERSITY && c.nof_ports != 2) return fail(LTEPHY_ERROR_INVALID_INPUTS, "grant %u: tx diversity needs 2 ports", gi);
    // codeword of each enabled TB: srsran_ra_tb_t.cw_idx (dl_sniffer_pdsch.c:24) -- scrambling (q << 13) and the layer the
    // demapper writes follow the codeword, not the TB (DCI 2/2A swap flag)
    const uint32_t n_en = (g.tb[0].enabled ? 1u : 0u) + (g.tb[1].enabled ? 1u : 0u);
    if (n_en > (two_cw ? 2u : 1u)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "grant %u: too many transport blocks for the tx scheme", gi);
    if (n_en == 2 && (g.tb[0].cw_idx > 1 || g.tb[1].cw_idx > 1 || g.tb[0].cw_idx == g.tb[1].cw_idx))
      return fail(LTEPHY_ERROR_INVALID_INPUTS, "grant %u: transport blocks must map to distinct codewords 0 / 1", gi);
    for (int t = 0; t < 2; t++) {
      if (!g.tb[t].enabled) continue;
      const uint32_t cw = n_en == 2 ? g.tb[t].cw_idx : 0u;
      const uint32_t qm = g.tb[t].qm, G = acc * qm;
      if (qm != 2 && qm != 4 && qm != 6 && qm != 8) return fail(LTEPHY_ERROR_INVALID_INPUTS, "grant %u: bad modulation order", gi);
      d.qm[cw] = qm;
      const uint32_t c_init = (d.rnti << 14) + (cw << 13) + (d.sf_idx << 9) + c.cell_id; // 36.211 6.3.1
      if (!alloc_codeword(h, G, G, c_init, d.llr_off[cw], d.scr_off[cw])) return fail(LTEPHY_ERROR, "grant %u: codeword longer than the scrambling basis", gi);
      if (g.tb[t].tbs > 0) {
        uint32_t tbi;
        int r = add_transport_block(h, (uint32_t)g.tb[t].tbs, G, qm, g.tb[t].rv, g.tx_scheme == LTEPHY_TX_DIVERSITY ? 2 : 1, d.llr_off[cw], tbi,
                                    g.tb[t].harq_op, g.tb[t].harq_slot);
        if (r) return r;
        b.tb_slot[(size_t)gi * 2 + t] = tbi;
      }
    }
    d.ncw = n_en;
    b.grants.push_back(d);
  }
  return pair_code_blocks(h);
}

// The persistent turbo launches of h->pb.pairs, which lie in bucket order: one launch per bucket (2 * threads + ragged last window, pairs)
static int launch_turbo_buckets(ltephy* h, const std::vector<std::pair<uint32_t, uint32_t>>& buckets, uint32_t max_iter)
{
  // per-CTA scratch (k_turbo.cu), sized for the largest launch: at most 2048 resident threads per SM, 32 words per thread
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->cfg.device);
  if (h->d_tscratch.reserve((size_t)sms * 2048 * 32) || h->d_tqueue.reserve(16)) return fail(LTEPHY_ERROR, "device allocation failed");
  CU(cudaMemsetAsync(h->d_tqueue.p, 0, 16 * sizeof(uint32_t), h->stream));
  CU(cudaEventRecord(h->ev[4], h->stream));
  uint32_t first = 0, bi = 0;
  for (auto& r : buckets) {
    launch_turbo(h->d_pairs.p + first, r.second, r.first / 2, (r.first & 1u) == 0, h->d_tqueue.p + (bi++ & 15u), h->d_turbo.p, h->d_tscratch.p,
                 h->d_tscratch.cap, h->d_pi.p, h->d_pair_pi_off.p + first, h->d_xpowA, h->d_xpowB, h->d_payload.p, h->d_cb_iters.p, h->d_cb_crc.p,
                 max_iter, h->stream, &h->launches);
    first += r.second;
  }
  CU(cudaEventRecord(h->ev[5], h->stream));
  return LTEPHY_SUCCESS;
}

// The tail of every phase B, after the front kernel has written the soft bits: rate-dematch and turbo-decode the code blocks, then check
// the transport-block CRCs
static int decode_code_blocks(ltephy* h)
{
  ltephy::PhaseB& b = h->pb;
  if (b.cbs.empty()) return LTEPHY_SUCCESS;
  // pairs are launched in buckets of equal CTA size so that small code blocks do not pay for 192 threads
  // (bucket by rounded thread count; the pair order of pair_code_blocks is kept inside a bucket)
  std::map<uint32_t, std::vector<uint32_t>> buckets; // key = 2 * threads + (ragged last window)
  for (uint32_t i = 0; i < b.pairs.size(); i++) buckets[2 * (((b.pairs[i].NW + 31) / 32) * 32) + ((b.pairs[i].K & 31u) ? 1 : 0)].push_back(i);
  std::vector<DevPair>  sorted;
  std::vector<uint32_t> sorted_pi;
  std::vector<std::pair<uint32_t, uint32_t>> ranges; // (key, count)
  std::vector<uint32_t> remap(b.pairs.size());
  for (auto& bk : buckets) {
    ranges.push_back({bk.first, (uint32_t)bk.second.size()});
    for (uint32_t i : bk.second) {
      remap[i] = (uint32_t)sorted.size();
      sorted.push_back(b.pairs[i]);
      sorted_pi.push_back(b.pair_pi_off[i]);
    }
  }
  for (auto& cb : b.cbs) cb.pair = remap[cb.pair];
  b.pairs.swap(sorted);
  b.pair_pi_off.swap(sorted_pi);
  if (h->d_pairs.reserve(b.pairs.size()) || h->d_pair_pi_off.reserve(b.pairs.size()) || h->d_cbs.reserve(b.cbs.size()))
    return fail(LTEPHY_ERROR, "device allocation failed");
  stage_and_pull(h, h->d_pairs.p, b.pairs.data(), b.pairs.size() * sizeof(DevPair));
  stage_and_pull(h, h->d_pair_pi_off.p, b.pair_pi_off.data(), b.pairs.size() * 4);
  stage_and_pull(h, h->d_cbs.p, b.cbs.data(), b.cbs.size() * sizeof(DevCb));
  for (uint32_t gen = 0; gen <= b.harq_max_gen; gen++) // one launch unless a HARQ slot is used more than once in this batch
    launch_rm_turbo_rx(h->d_cbs.p, h->d_pairs.p, (uint32_t)b.pairs.size(), h->d_pllr.p, h->d_rm.p, h->d_turbo.p, h->d_harq.p, gen, h->stream, &h->launches);
  if (int r = launch_turbo_buckets(h, ranges, h->cfg.turbo_max_iter)) return r;
  launch_tb_crc(h->d_tbs.p, (uint32_t)b.tbs.size(), h->d_payload.p, h->d_cb_crc.p, h->d_cb_iters.p, h->d_xpowA, h->d_res.p, h->stream, &h->launches);
  return LTEPHY_SUCCESS;
}

// Once a submit has built its batch: reset the pinned staging arena and size it for the batch's descriptors (grant_bytes of them are the
// grants), and reserve the buffers every phase B uses.  The grant-specific buffers are the caller's.
static int reserve_phase_b(ltephy* h, size_t grant_bytes)
{
  const ltephy::PhaseB& b = h->pb;
  if (h->stage_busy) CU(cudaStreamSynchronize(h->stream)); // a phase B that was never fetched may still be pulling from the arena
  h->stage_used = 0, h->stage_busy = true;
  const size_t scr_bytes = b.scr.size() * sizeof(DevScr);
  if (h->h_stage.reserve(grant_bytes + b.tbs.size() * sizeof(DevTb) + scr_bytes + b.pairs.size() * (sizeof(DevPair) + 4) + b.cbs.size() * sizeof(DevCb) + 256))
    return fail(LTEPHY_ERROR, "pinned allocation failed");
  if (h->d_tbs.reserve(b.tbs.size() + (scr_bytes + sizeof(DevTb) - 1) / sizeof(DevTb) + 1) || h->d_seq.reserve(b.seq_words + 1) ||
      h->d_pllr.reserve(b.pllr_elems + 8) || h->d_turbo.reserve(b.turbo_words + 1) || h->d_payload.reserve(b.payload_bytes + 4) || h->d_cb_iters.reserve(b.cbs.size() + 1) || h->d_cb_crc.reserve(b.cbs.size() + 1) ||
      h->d_res.reserve(b.tbs.size() + 1) || h->h_res.reserve(b.tbs.size() + 1) || h->h_payload.reserve(b.payload_bytes + 4))
    return fail(LTEPHY_ERROR, "device allocation failed");
  return LTEPHY_SUCCESS;
}

// The start of every PDSCH / PUSCH phase B, after the caller has staged its grants: stage the transport blocks (tb_crc) and the codeword
// list (scr_seq_kernel) behind them, both into d_tbs with one pull, then write every codeword's scrambling sequence
static void stage_tbs_and_scramble(ltephy* h)
{
  static_assert(sizeof(DevTb) % 16 == 0, "the codeword list must start in the arena slot right behind the transport blocks");
  const ltephy::PhaseB& b = h->pb;
  const size_t          tb_bytes = b.tbs.size() * sizeof(DevTb), scr_bytes = b.scr.size() * sizeof(DevScr);
  uint8_t*              slot = stage(h, b.tbs.data(), tb_bytes);
  stage(h, b.scr.data(), scr_bytes);
  pull(h, h->d_tbs.p, slot, tb_bytes + scr_bytes);
  launch_scr_seq(reinterpret_cast<const DevScr*>(h->d_tbs.p + b.tbs.size()), (uint32_t)b.scr.size(), b.max_scr_words, h->d_gold_x1, h->d_gold_basis,
                 h->gold_words, h->d_seq.p, h->stream, &h->launches);
}

extern "C" int ltephy_submit_grants(ltephy_t* h, const ltephy_grant_t* gin, uint32_t n)
{
  if (!h || (!gin && n)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "submit_grants: bad arguments");
  CU(cudaSetDevice(h->cfg.device));
  if (int r = build_jobs(h, gin, n)) return r;
  if (int r = reserve_phase_b(h, n * sizeof(DevGrant))) return r;
  if (h->d_grants.reserve(n + 1)) return fail(LTEPHY_ERROR, "device allocation failed");
  const ltephy::PhaseB& b = h->pb;
  CU(cudaEventRecord(h->ev[2], h->stream));
  if (n) {
    stage_and_pull(h, h->d_grants.p, b.grants.data(), n * sizeof(DevGrant));
    stage_tbs_and_scramble(h);
    launch_pdsch_front(h->dc, h->d_grants.p, n, h->d_sym.p, h->d_pil.p, h->d_seq.p, h->d_pllr.p, h->stream, &h->launches);
    CU(cudaGetLastError()); // a front kernel that could not launch would leave the previous batch's sequences and soft bits behind
    if (int r = decode_code_blocks(h)) return r;
  }
  CU(cudaEventRecord(h->ev[3], h->stream));
  CU(cudaGetLastError());
  return LTEPHY_SUCCESS;
}

// Device-to-device copy of the raw phase-B payload buffer (TB i at the running offset sum_{j<i} ((tbs_j/8 + 6) & ~3), its 3 CRC
// bytes behind it), for callers that hand the decoded transport blocks to a collective without a host round trip.
extern "C" int ltephy_copy_phase_b_device(ltephy_t* h, void* dst_dev, size_t cap, size_t* nbytes)
{
  if (!h || !dst_dev || !nbytes) return fail(LTEPHY_ERROR_INVALID_INPUTS, "copy_phase_b_device: bad arguments");
  CU(cudaSetDevice(h->cfg.device));
  const size_t n = h->pb.payload_bytes < cap ? h->pb.payload_bytes : cap;
  if (n) CU(cudaMemcpyAsync(dst_dev, h->d_payload.p, n, cudaMemcpyDeviceToDevice, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  *nbytes = n;
  return LTEPHY_SUCCESS;
}
// Results of the last phase B, downlink or uplink: one per slot of tb_slot, the payload packed in slot order
extern "C" int ltephy_get_phase_b(ltephy_t* h, ltephy_tb_result_t* results, uint8_t* payload, size_t payload_cap)
{
  if (!h || !results) return fail(LTEPHY_ERROR_INVALID_INPUTS, "get_phase_b: bad arguments");
  const ltephy::PhaseB& b = h->pb;
  if (!b.tbs.empty()) {
    CU(cudaMemcpyAsync(h->h_res.p, h->d_res.p, b.tbs.size() * sizeof(ltephy_tb_result_t), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(h->h_payload.p, h->d_payload.p, b.payload_bytes, cudaMemcpyDeviceToHost, h->stream));
  }
  CU(cudaStreamSynchronize(h->stream));
  h->stage_busy = false;
  cudaEventElapsedTime(&h->t_ms[1], h->ev[2], h->ev[3]); // uplink: from before the H2D of its samples
  if (!b.cbs.empty()) cudaEventElapsedTime(&h->t_ms[2], h->ev[4], h->ev[5]);
  size_t wp = 0;
  for (size_t i = 0; i < b.tb_slot.size(); i++) {
    ltephy_tb_result_t o{};
    if (b.tb_slot[i] != 0xFFFFFFFFu) {
      const DevTb& tb = b.tbs[b.tb_slot[i]];
      o               = h->h_res.p[b.tb_slot[i]];
      o.payload_off   = (uint32_t)wp;
      o.payload_len   = tb.nbytes;
      if (payload) {
        if (wp + tb.nbytes > payload_cap) return fail(LTEPHY_ERROR_INVALID_INPUTS, "payload buffer too small");
        memcpy(payload + wp, h->h_payload.p + tb.byte_off, tb.nbytes);
      }
      wp += tb.nbytes;
    }
    results[i] = o;
  }
  return LTEPHY_SUCCESS;
}


// ---------------------------------------------------------------------------------------- file-mode front matter (SURVEY 8f-1)
// constant frequency-offset correction of every subframe of samples: srsran_cfo_correct(&q->file_cfo_correct, ..., file_cfo / 15000 / fft_size)
// in srsran_ue_sync's file mode (args.file_offset_freq, reference src/src/LTESniffer_Core.cc:252-257); the rotation is applied by the OFDM kernel
// the table both directions use: rot[n] = exp(-j 2 pi f n / (15000 fft)) over one subframe, in double, rounded to float (lteo_cfo_correct)
static int cfo_table(ltephy_t* h, float cfo_hz, DevBuf<float2>& buf, const float2*& ptr)
{
  CU(cudaSetDevice(h->cfg.device));
  CU(cudaStreamSynchronize(h->stream));
  if (cfo_hz == 0.0f) {
    ptr = nullptr;
    return LTEPHY_SUCCESS;
  }
  std::vector<float2> rot(h->dc.sf_len);
  for (uint32_t n = 0; n < h->dc.sf_len; n++) {
    const double ph = -2.0 * M_PI * (double)cfo_hz * (double)n / (15000.0 * (double)h->dc.fft);
    rot[n]          = make_float2((float)std::cos(ph), (float)std::sin(ph));
  }
  if (buf.reserve(rot.size())) return fail(LTEPHY_ERROR, "device allocation failed");
  CU(cudaMemcpy(buf.p, rot.data(), rot.size() * sizeof(float2), cudaMemcpyHostToDevice));
  ptr = buf.p;
  return LTEPHY_SUCCESS;
}
extern "C" int ltephy_set_cfo(ltephy_t* h, float cfo_hz)
{
  if (!h) return fail(LTEPHY_ERROR_INVALID_INPUTS, "set_cfo: bad arguments");
  return cfo_table(h, cfo_hz, h->d_cfo, h->dc.cfo_rot);
}
// the uplink's own table (DevCell::ul_cfo_rot), applied by ofdm_rx_kernel<UL> before the half-subcarrier rotation
extern "C" int ltephy_set_ul_cfo(ltephy_t* h, float cfo_hz)
{
  if (!h) return fail(LTEPHY_ERROR_INVALID_INPUTS, "set_ul_cfo: bad arguments");
  return cfo_table(h, cfo_hz, h->d_ulcfo, h->dc.ul_cfo_rot);
}
// PBCH work of one call (k_pbch.cu): pbch_llr_kernel fills frame-store rows 3.. with the soft bits of the listed subframes 0 for the port counts
// nant_first .. nant_last, then pbch_hyp_kernel decodes the hypothesis jobs; res receives {port count of the CRC mask or 0, 24 MIB bits} per job.
static int pbch_run(ltephy* h, const std::vector<uint32_t>& frame_sf, uint32_t nant_first, uint32_t nant_last, const std::vector<uint32_t>& jobs,
                    std::vector<uint32_t>& res)
{
  const size_t F = frame_sf.size(), J = jobs.size();
  if (h->d_pbch.reserve((size_t)(3 + h->cfg.max_subframes) * 960) || h->d_mib.reserve(F + 3 * J + 1)) return fail(LTEPHY_ERROR, "device allocation failed");
  const size_t R = (F + J + 1) & ~(size_t)1; // the results are uint2: an 8-byte aligned word offset
  std::vector<uint32_t> up(frame_sf);
  up.insert(up.end(), jobs.begin(), jobs.end());
  res.assign(2 * J, 0);
  if (!up.empty()) CU(cudaMemcpyAsync(h->d_mib.p, up.data(), up.size() * 4, cudaMemcpyHostToDevice, h->stream));
  launch_pbch(h->dc, h->d_sym.p, h->d_pil.p, h->d_mib.p, (uint32_t)F, nant_first - 1, nant_last - nant_first + 1, h->d_pbch.p, h->d_mib.p + F, (uint32_t)J, h->d_mib.p + R, h->stream, &h->launches);
  CU(cudaGetLastError());
  h->pbch_frames = (uint32_t)F;
  if (J) CU(cudaMemcpyAsync(res.data(), h->d_mib.p + R, res.size() * 4, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return LTEPHY_SUCCESS;
}
// job word (k_pbch.cu): bit 0 port count - 1, bits 1..2 n - 1, bits 3..4 dst, bits 5..31 the row.  Rows go up to 3 + max_subframes, far below 2^27:
// a handle's sample buffer for 2^27 subframes would take more than 2 TB, so ltephy_create fails long before
static uint32_t pbch_job(uint32_t newest_row, uint32_t nant, uint32_t n, uint32_t dst) { return (nant - 1) | (n - 1) << 1 | dst << 3 | newest_row << 5; }
// the fields of an ltephy_mib_t from the 24 MIB bits (first bit in bit 23): srsran_pbch_mib_unpack; found = 0 for a reserved bandwidth code
static ltephy_mib_t mib_unpack(uint32_t bits, uint32_t nof_ports, uint32_t sfn_offset)
{
  static const uint32_t BW[8] = {6, 15, 25, 50, 75, 100, 0, 0};
  ltephy_mib_t          m{};
  m.found = 1, m.nof_ports = (uint8_t)nof_ports, m.sfn_offset = (uint8_t)sfn_offset;
  m.nof_prb = BW[(bits >> 21) & 7u], m.phich_length = (uint8_t)((bits >> 20) & 1u), m.phich_resources = (uint8_t)((bits >> 18) & 3u);
  m.sfn = ((((bits >> 10) & 0xFFu) << 2) + sfn_offset) % 1024u; // sfn = (sfn + sfn_offset) % 1024, LTESniffer_Core.cc:392
  m.bch_payload[0] = (uint8_t)(bits >> 16), m.bch_payload[1] = (uint8_t)(bits >> 8), m.bch_payload[2] = (uint8_t)bits;
  if (!m.nof_prb) m.found = 0;
  return m;
}

// PBCH / MIB of every subframe 0 of the last phase A: srsran_ue_mib_decode + srsran_pbch_mib_unpack (LTESniffer_Core.cc:382-396), one frame at a
// time: the four one-frame hypotheses dst = 0..3 with the handle's port count; the lowest dst whose remainder is any of the three masks wins
extern "C" int ltephy_mib_decode(ltephy_t* h, ltephy_mib_t* out)
{
  if (!h || !out) return fail(LTEPHY_ERROR_INVALID_INPUTS, "mib_decode: bad arguments");
  const uint32_t n = (uint32_t)h->n_cur;
  if (!n) return fail(LTEPHY_ERROR_INVALID_INPUTS, "mib_decode: no subframes submitted");
  CU(cudaSetDevice(h->cfg.device));
  std::vector<uint32_t> frame_sf, jobs, res;
  for (uint32_t i = 0; i < n; i++)
    if (h->h_info.p[i].tti % 10 == 0) {
      for (uint32_t dst = 0; dst < 4; dst++) jobs.push_back(pbch_job(3 + (uint32_t)frame_sf.size(), h->dc.nof_ports, 1, dst));
      frame_sf.push_back(i);
    }
  if (int r = pbch_run(h, frame_sf, h->dc.nof_ports, h->dc.nof_ports, jobs, res)) return r;
  for (uint32_t i = 0, f = 0; i < n; i++) {
    out[i] = ltephy_mib_t{};
    if (h->h_info.p[i].tti % 10) continue;
    for (uint32_t dst = 0; dst < 4; dst++) {
      const uint32_t j = 4 * f + dst;
      if (res[2 * j]) {
        out[i] = mib_unpack(res[2 * j + 1], res[2 * j], dst);
        break;
      }
    }
    f++;
  }
  return LTEPHY_SUCCESS;
}

// Soft combining across the 40 ms period (DESIGN.md §2 "PBCH combining").  The hypotheses a window of frame_idx frames can try combine n
// consecutive frames of it at positions dst..dst+n-1; every such (frames, dst, port count) is one job, evaluated for all candidate windows at once.
// The walk below then replays srsRAN's sequential state machine over the results: which window each frame sees depends on earlier passes.
extern "C" int ltephy_mib_decode_combined(ltephy_t* h, uint32_t flags, ltephy_mib_comb_t* out)
{
  if (!h || !out) return fail(LTEPHY_ERROR_INVALID_INPUTS, "mib_decode_combined: bad arguments");
  if (flags & ~LTEPHY_MIB_SEARCH_PORTS) return fail(LTEPHY_ERROR_INVALID_INPUTS, "mib_decode_combined: unknown flags 0x%x", flags);
  const uint32_t n = (uint32_t)h->n_cur;
  if (!n) return fail(LTEPHY_ERROR_INVALID_INPUTS, "mib_decode_combined: no subframes submitted");
  CU(cudaSetDevice(h->cfg.device));
  const uint32_t P = h->dc.nof_ports;
  std::vector<uint32_t> tries;
  if (flags & LTEPHY_MIB_SEARCH_PORTS)
    for (uint32_t k = 1; k <= P; k++) tries.push_back(k);
  else
    tries.push_back(P);
  // frames in batch order: subframe index, SFN and run (consecutive frames ending here, the frames held before this call included)
  std::vector<uint32_t> frame_sf, sfn, run;
  for (uint32_t i = 0; i < n; i++)
    if (h->h_info.p[i].tti % 10 == 0) frame_sf.push_back(i), sfn.push_back((h->h_info.p[i].tti / 10) % 1024);
  const uint32_t F = (uint32_t)frame_sf.size();
  const bool     cont = F && h->mib_held && (int32_t)sfn[0] == (h->mib_last_sfn + 1) % 1024;
  const int32_t  held = cont ? (int32_t)h->mib_held : 0;
  for (uint32_t k = 0; k < F; k++) run.push_back(k == 0 ? (uint32_t)held + 1 : sfn[k] == (sfn[k - 1] + 1) % 1024 ? run[k - 1] + 1 : 1);
  // jobs: for every frame ordinal o (held frames are -held..-1, in rows 3 + o) as the newest of n <= min(4, run) frames, every dst <= 4 - n
  auto run_of = [&](int32_t o) { return o < 0 ? (uint32_t)(o + held + 1) : run[o]; };
  std::vector<int32_t>  jidx((size_t)(held + F) * 2 * 10, -1); // [(o + held) * 2 + nant - 1][(n, dst)]
  auto slot = [&](int32_t o, uint32_t nant, uint32_t nn, uint32_t dst) -> int32_t& {
    static const uint32_t base[5] = {0, 0, 4, 7, 9};
    return jidx[((size_t)(o + held) * 2 + nant - 1) * 10 + base[nn] + dst];
  };
  std::vector<uint32_t> jobs, res;
  for (int32_t o = -held; o < (int32_t)F; o++)
    for (uint32_t nant : tries)
      for (uint32_t nn = 1; nn <= std::min(4u, run_of(o)); nn++)
        for (uint32_t dst = 0; dst + nn <= 4; dst++) {
          slot(o, nant, nn, dst) = (int32_t)jobs.size();
          jobs.push_back(pbch_job((uint32_t)(3 + o), nant, nn, dst));
        }
  if (int r = pbch_run(h, frame_sf, 1, P, jobs, res)) return r; // every port count: the carried rows serve later calls with either flag
  for (uint32_t i = 0; i < n; i++) out[i] = ltephy_mib_comb_t{};
  uint32_t fi = (uint32_t)held;
  for (uint32_t k = 0; k < F; k++) {
    if (run[k] == 1) fi = 0; // not the frame after the last one consumed: empty the buffer first
    fi++;
    bool done = false;
    for (uint32_t t = 0; t < tries.size() && !done; t++) {
      const uint32_t nant = tries[t];
      for (uint32_t nb = 0; nb < fi && !done; nb++)
        for (uint32_t dst = 0; dst < 4 - nb && !done; dst++)
          for (uint32_t src = 0; src < fi - nb && !done; src++) {
            const int32_t  o = (int32_t)k - (int32_t)fi + 1 + (int32_t)(src + nb); // newest combined frame
            const uint32_t j = (uint32_t)slot(o, nant, nb + 1, dst);
            if (res[2 * j] != nant) continue; // the remainder must be this port count's mask
            ltephy_mib_comb_t& r = out[frame_sf[k]];
            r.mib        = mib_unpack(res[2 * j + 1], nant, dst - src + fi - 1);
            r.nof_frames = (uint8_t)(nb + 1), r.src = (uint8_t)src, r.dst = (uint8_t)dst, r.window = (uint8_t)fi;
            done = true;
          }
    }
    if (done)
      fi = 0;
    else if (fi == 4)
      fi = 3; // drop the oldest frame
  }
  // carry the frames still held into rows 3 - fi .. 2, ascending (a source row always lies above its destination)
  const int32_t first = (int32_t)F - (int32_t)fi;
  for (uint32_t r = 0; r < fi; r++) {
    const int32_t from = 3 + first + (int32_t)r, to = 3 - (int32_t)fi + (int32_t)r;
    if (from != to) CU(cudaMemcpyAsync(h->d_pbch.p + (size_t)to * 960, h->d_pbch.p + (size_t)from * 960, 960 * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
  }
  CU(cudaStreamSynchronize(h->stream));
  if (F) h->mib_held = fi, h->mib_last_sfn = (int32_t)sfn[F - 1];
  return LTEPHY_SUCCESS;
}
extern "C" int ltephy_mib_reset(ltephy_t* h)
{
  if (!h) return fail(LTEPHY_ERROR_INVALID_INPUTS, "mib_reset: bad arguments");
  h->mib_held = 0, h->mib_last_sfn = -1;
  return LTEPHY_SUCCESS;
}

// ---------------------------------------------------------------------------------------- HARQ store
extern "C" int ltephy_harq_reserve(ltephy_t* h, uint32_t nslots)
{
  if (!h || nslots == 0) return fail(LTEPHY_ERROR_INVALID_INPUTS, "harq_reserve: bad arguments");
  CU(cudaSetDevice(h->cfg.device));
  CU(cudaStreamSynchronize(h->stream));
  const size_t words = (size_t)nslots * (LTEPHY_HARQ_SLOT_BYTES / 2);
  if (h->d_harq.reserve(words)) return fail(LTEPHY_ERROR, "harq_reserve: %zu bytes of device memory not available", words * 2);
  CU(cudaMemsetAsync(h->d_harq.p, 0, words * 2, h->stream));
  h->harq_slots = nslots;
  return LTEPHY_SUCCESS;
}

// ---------------------------------------------------------------------------------------- uplink (PUSCH)
extern "C" int ltephy_set_ul_cfg(ltephy_t* h, const ltephy_ul_cfg_t* cfg)
{
  if (!h || !cfg) return fail(LTEPHY_ERROR_INVALID_INPUTS, "set_ul_cfg: bad arguments");
  if (cfg->n_dmrs1 > 7 || cfg->delta_ss > 29) return fail(LTEPHY_ERROR_INVALID_INPUTS, "set_ul_cfg: cyclicShift is 0..7, groupAssignmentPUSCH 0..29");
  h->ulcfg = *cfg, h->ulcfg_set = true;
  const uint32_t fss = ((h->cell.cell_id % 30) + cfg->delta_ss) % 30;
  auto           cw  = ltehost::gold_words((h->cell.cell_id / 30) * 32 + fss, 8 * 7 * 20 + 8);
  auto           gh  = ltehost::gold_words(h->cell.cell_id / 30, 8 * 20 + 8);
  for (uint32_t ns = 0; ns < 20; ns++) {
    uint32_t v = 0, f = 0;
    for (uint32_t i = 0; i < 8; i++) {
      const uint32_t b = 8 * 7 * ns + i, b2 = 8 * ns + i;
      v += ((cw[b >> 5] >> (b & 31)) & 1u) << i; // n_PRS(ns), 36.211 5.5.2.1.1
      f += ((gh[b2 >> 5] >> (b2 & 31)) & 1u) << i; // f_gh(ns), 36.211 5.5.1.3 (c_init = floor(cell_id / 30))
    }
    h->n_prs[ns] = v;
    h->ul_u[ns]  = ((cfg->group_hopping ? f % 30 : 0) + fss) % 30;
    h->ul_v[ns]  = (!cfg->group_hopping && cfg->seq_hopping) ? (cw[ns >> 5] >> (ns & 31)) & 1u : 0; // 36.211 5.5.1.4 (same c_init as n_PRS); used from 6 PRB on
  }
  h->ul_tab_cache.clear();
  h->ulpool_used = 0;
  return LTEPHY_SUCCESS;
}
static uint32_t largest_prime_below(uint32_t n)
{
  for (uint32_t p = n - 1; p >= 2; p--) {
    bool ok = true;
    for (uint32_t d = 2; d * d <= p; d++)
      if (p % d == 0) {
        ok = false;
        break;
      }
    if (ok) return p;
  }
  return 2;
}
// kind 0: DMRS r_{u,v}^{(alpha)} for (M, ncs, u, v); kind 1: IDFT twiddles for M
static int ul_table_for(ltephy* h, uint32_t kind, uint32_t M, uint32_t ncs, uint32_t u, uint32_t v, uint32_t& off)
{
  const uint64_t key = ((uint64_t)kind << 40) | ((uint64_t)M << 16) | (u << 9) | (v << 8) | ncs;
  auto           it  = h->ul_tab_cache.find(key);
  if (it != h->ul_tab_cache.end()) {
    off = it->second;
    return 0;
  }
  std::vector<float2> t(M);
  if (kind == 0) {
    const uint32_t Nzc = largest_prime_below(M);
    const double   qb  = (double)Nzc * (u + 1) / 31.0;
    uint32_t       q   = (uint32_t)std::floor(qb + 0.5);
    if (v) q = ((uint32_t)std::floor(2.0 * qb) & 1u) ? q - 1 : q + 1; // q = floor(qb + 1/2) + v (-1)^floor(2 qb), 36.211 5.5.1.1
    for (uint32_t n = 0; n < M; n++) {
      const uint64_t m  = n % Nzc, tt = ((uint64_t)q * m * (m + 1)) % (2ull * Nzc);
      const uint32_t a  = (ncs * n) % 12;
      const double   ph = -M_PI * (double)tt / (double)Nzc + 2.0 * M_PI * (double)a / 12.0;
      t[n]              = make_float2((float)std::cos(ph), (float)std::sin(ph));
    }
  } else {
    for (uint32_t m = 0; m < M; m++) {
      const double ph = 2.0 * M_PI * (double)m / (double)M;
      t[m]            = make_float2((float)std::cos(ph), (float)std::sin(ph));
    }
  }
  const int64_t o = pool_append(h, h->d_ulpool, h->ulpool_used, t.data(), M);
  if (o < 0) return -1;
  off = h->ul_tab_cache[key] = (uint32_t)o;
  return 0;
}

// ltephy_submit_ul / _device: iq_host is copied into d_uliq first; iq_dev is demodulated in place; both NULL re-decodes the previous symbols
static int submit_ul_common(ltephy_t* h, const void* iq_host, const void* iq_dev, const uint32_t* tti, uint32_t n, const ltephy_ul_grant_t* gin,
                            uint32_t ng)
{
  if (!h || !tti || n == 0 || n > h->cfg.max_subframes || (!gin && ng)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "submit_ul: bad arguments");
  if (!h->ulcfg_set) return fail(LTEPHY_ERROR_INVALID_INPUTS, "submit_ul: ltephy_set_ul_cfg has not been called");
  const bool have_iq = iq_host || iq_dev;
  if (!have_iq && h->n_ul != n) return fail(LTEPHY_ERROR_INVALID_INPUTS, "submit_ul: no IQ given and the previous call demodulated %u subframes, not %u", h->n_ul, n);
  if (iq_misaligned(iq_dev, h->cfg.iq_format))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "submit_ul_device: iq_ul_dev not aligned to its %zu-byte samples", iq_sample_bytes(h->cfg.iq_format));
  CU(cudaSetDevice(h->cfg.device));
  const DevCell& c = h->dc;
  const size_t   A = c.ul_nof_rx; // samples and symbols are [n][A][..]: their offsets stay 64-bit (65 535 x 2 x 14 x 1200 x 8 bytes > 2^32)
  const size_t   xb = iq_sample_bytes(h->cfg.iq_format);
  if ((iq_host && h->d_uliq.reserve((size_t)h->cfg.max_subframes * A * c.sf_len * xb)) || h->d_ulsym.reserve((size_t)h->cfg.max_subframes * A * 14 * c.nsc) ||
      h->d_ulpool.reserve((size_t)1 << 20))
    return fail(LTEPHY_ERROR, "device allocation failed");
  CU(cudaEventRecord(h->ev[2], h->stream));
  if (have_iq) { // NULL: the demodulated symbols of the previous call stay (srsran_enb_ul_fft once, then one decode per grant)
    if (iq_host) {
      CU(cudaMemcpyAsync(h->d_uliq.p, iq_host, (size_t)n * A * c.sf_len * xb, cudaMemcpyHostToDevice, h->stream));
      iq_dev = h->d_uliq.p;
    }
    launch_ul_ofdm(c, iq_dev, h->cfg.iq_format, h->d_ulsym.p, n, h->stream, &h->launches);
  }
  h->n_ul = n;
  // jobs
  ltephy::PhaseB& b = h->pb;
  b.reset(ng);
  uint32_t max_M = 36;
  for (uint32_t gi = 0; gi < ng; gi++) {
    const ltephy_ul_grant_t& g = gin[gi];
    if (g.sf >= n) return fail(LTEPHY_ERROR_INVALID_INPUTS, "UL grant %u: subframe outside the batch", gi);
    const uint32_t M = 12 * g.L_prb, n_prb1 = (g.flags & LTEPHY_UL_FLAG_SLOT1) ? g.n_prb_slot1 : g.n_prb;
    // L_prb 1 and 2 use the 30 + 30 computer-generated QPSK base sequences of 36.211 Tables 5.5.1.2-1 / -2, which this build does not carry
    if (g.L_prb < 3 || g.n_prb + g.L_prb > c.nof_prb || n_prb1 + g.L_prb > c.nof_prb || (g.qm != 2 && g.qm != 4 && g.qm != 6 && g.qm != 8) || g.tbs <= 0)
      return fail(LTEPHY_ERROR_INVALID_INPUTS, "UL grant %u: unsupported allocation / modulation", gi);
    DevUlGrant d{};
    uint32_t   rad = M;
    while (rad % 5 == 0) d.rad |= 5u << (4 * d.nrad++), rad /= 5;
    while (rad % 3 == 0) d.rad |= 3u << (4 * d.nrad++), rad /= 3;
    while (rad % 4 == 0) d.rad |= 4u << (4 * d.nrad++), rad /= 4;
    if (rad % 2 == 0) d.rad |= 2u << (4 * d.nrad++), rad /= 2;
    if (rad != 1) return fail(LTEPHY_ERROR_INVALID_INPUTS, "UL grant %u: L_prb %u is not 2^a 3^b 5^c (valid_prb_ul)", gi, g.L_prb);
    if (g.nof_ack > 2 || g.ri_len > 2) return fail(LTEPHY_ERROR_INVALID_INPUTS, "UL grant %u: more than 2 ACK / RI bits", gi);
    ltehost::UciLayout L;
    if (!ltehost::uci_layout(g.L_prb, g.qm, (uint32_t)g.tbs, g.nof_ack, g.ri_len, g.cqi_len, g.I_offset_ack, g.I_offset_ri, g.I_offset_cqi, L))
      return fail(LTEPHY_ERROR_INVALID_INPUTS, "UL grant %u: invalid TBS / reserved beta offset index", gi);
    d.sf = g.sf, d.sf_idx = tti[g.sf] % 10, d.rnti = g.rnti, d.M = M, d.k0[0] = 12 * g.n_prb, d.k0[1] = 12 * n_prb1, d.qm = g.qm;
    d.qp_ack = L.Qp_ack, d.qp_ri = L.Qp_ri, d.qp_cqi = L.Qp_cqi;
    for (uint32_t sl = 0; sl < 2; sl++) {
      static const uint8_t n_dmrs1_of[8] = {0, 2, 3, 4, 6, 8, 9, 10}; // cyclicShift of SIB2 -> n_DMRS^(1), 36.211 Table 5.5.2.1.1-2
      const uint32_t ns = 2 * d.sf_idx + sl, ncs = (n_dmrs1_of[h->ulcfg.n_dmrs1 & 7u] + g.n_dmrs2 + h->n_prs[ns]) % 12;
      if (ul_table_for(h, 0, M, ncs, h->ul_u[ns], M >= 72 ? h->ul_v[ns] : 0, d.dmrs_off[sl])) return fail(LTEPHY_ERROR, "UL table upload failed");
    }
    if (ul_table_for(h, 1, M, 0, 0, 0, d.idft_off)) return fail(LTEPHY_ERROR, "UL table upload failed");
    const uint32_t G = L.G;
    const uint32_t c_init = (d.rnti << 14) + (d.sf_idx << 9) + c.cell_id; // 36.211 5.3.1
    if (!alloc_codeword(h, 12 * M * g.qm, G, c_init, d.llr_off, d.scr_off)) return fail(LTEPHY_ERROR, "UL grant %u: codeword longer than the scrambling basis", gi);
    if (G < g.qm * 12) return fail(LTEPHY_ERROR_INVALID_INPUTS, "UL grant %u: the control information leaves no room for the transport block", gi);
    max_M = std::max(max_M, M);
    uint32_t tbi;
    int      r = add_transport_block(h, (uint32_t)g.tbs, G, g.qm, g.rv, 1, d.llr_off, tbi);
    if (r) return r;
    b.tb_slot[gi] = tbi;
    b.ulgrants.push_back(d);
  }
  if (int r = pair_code_blocks(h)) return r;
  if (int r = reserve_phase_b(h, ng * sizeof(DevUlGrant))) return r;
  if (h->d_ulgrants.reserve(ng + 1) || h->d_ulchest.reserve(ng + 1) || h->h_ulchest.reserve(ng + 1)) return fail(LTEPHY_ERROR, "device allocation failed");
  if (ng) {
    stage_and_pull(h, h->d_ulgrants.p, b.ulgrants.data(), ng * sizeof(DevUlGrant));
    stage_tbs_and_scramble(h);
    launch_pusch(c, h->d_ulgrants.p, ng, max_M, h->d_ulsym.p, h->d_ulpool.p, h->d_ulpool.p, h->d_seq.p, h->d_pllr.p, h->d_ulchest.p, h->stream, &h->launches);
    CU(cudaGetLastError()); // as in ltephy_submit_grants
    if (int r = decode_code_blocks(h)) return r;
  }
  CU(cudaEventRecord(h->ev[3], h->stream));
  CU(cudaGetLastError());
  return LTEPHY_SUCCESS;
}
extern "C" int ltephy_submit_ul(ltephy_t* h, const void* iq_ul, const uint32_t* tti, uint32_t n, const ltephy_ul_grant_t* gin, uint32_t ng)
{
  return submit_ul_common(h, iq_ul, nullptr, tti, n, gin, ng);
}
extern "C" int ltephy_submit_ul_device(ltephy_t* h, const void* iq_ul_dev, const uint32_t* tti, uint32_t n, const ltephy_ul_grant_t* gin, uint32_t ng)
{
  return submit_ul_common(h, nullptr, iq_ul_dev, tti, n, gin, ng); // read in place until ltephy_get_ul
}

extern "C" int ltephy_get_ul(ltephy_t* h, ltephy_tb_result_t* results, ltephy_ul_chest_t* chest, uint8_t* payload, size_t payload_cap)
{
  if (!h || !results) return fail(LTEPHY_ERROR_INVALID_INPUTS, "get_ul: bad arguments");
  const size_t ng = h->pb.ulgrants.size();
  if (ng) CU(cudaMemcpyAsync(h->h_ulchest.p, h->d_ulchest.p, ng * sizeof(DevUlChest), cudaMemcpyDeviceToHost, h->stream));
  if (int r = ltephy_get_phase_b(h, results, payload, payload_cap)) return r; // one transport block per grant
  for (size_t i = 0; i < ng && chest; i++) {
    const DevUlChest& dcst = h->h_ulchest.p[i];
    chest[i].noise = dcst.noise, chest[i].rsrp = dcst.rsrp;
    chest[i].snr_db = 10.0f * log10f(dcst.rsrp / dcst.noise);
    // timing offset: -arg(sum ls[n+1] conj(ls[n])) / 2 pi per slot (srsran_vec_estimate_frequency over the pilots, meas_ta_en), slot average, / 15e-3 -> us
    float ta = 0.0f;
    for (int sl = 0; sl < 2; sl++) ta = ta + (-atan2f(dcst.ci[sl], dcst.cr[sl]) / 6.28318530717958647692f) / 2.0f;
    chest[i].ta_us = std::isnormal(ta) ? ta / 15e-3f : 0.0f;
  }
  return LTEPHY_SUCCESS;
}

// ---------------------------------------------------------------------------------------- stand-alone kernels
extern "C" int ltephy_dci_sweep(ltephy_t* h, const float* llr, const uint32_t* cfi, uint32_t n, ltephy_cand_t* cands)
{
  if (!h || !llr || !cfi || !cands || n == 0 || n > h->cfg.max_subframes) return fail(LTEPHY_ERROR_INVALID_INPUTS, "dci_sweep: bad arguments");
  CU(cudaSetDevice(h->cfg.device));
  for (uint32_t i = 0; i < n; i++) {
    DevSfInfo& s = h->h_info.p[i];
    memset(&s, 0, sizeof(s));
    if (cfi[i] < 1 || cfi[i] > 3) return fail(LTEPHY_ERROR_INVALID_INPUTS, "dci_sweep: bad cfi");
    s.cfi = cfi[i], s.nof_cce = h->dc.nof_cce[cfi[i] - 1], s.nof_locations = h->dc.nloc[cfi[i] - 1];
    for (auto& p : s.cce_power) p = 1.0f;
  }
  CU(cudaMemcpyAsync(h->d_info.p, h->h_info.p, n * sizeof(DevSfInfo), cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(h->d_llr.p, llr, (size_t)n * LLR_STRIDE * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CU(cudaEventRecord(h->ev[0], h->stream));
  launch_viterbi(h->dc, h->d_llr.p, h->d_info.p, h->d_cands.p, h->d_vwork.p, n, h->stream, &h->launches);
  launch_compact(h->dc, h->d_info.p, h->d_cands.p, h->d_compact.p, n, h->stream, &h->launches);
  CU(cudaEventRecord(h->ev[1], h->stream));
  CU(cudaMemcpyAsync(cands, h->d_cands.p, (size_t)n * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES * sizeof(ltephy_cand_t), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  CU(cudaGetLastError());
  cudaEventElapsedTime(&h->t_ms[3], h->ev[0], h->ev[1]);
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_turbo_batch(ltephy_t* h, const int16_t* d, uint32_t K, uint32_t ncb, uint32_t max_iter, int crc_type, uint8_t* bits,
                                  uint8_t* iters, uint8_t* crc_ok)
{
  if (!h || !d || !bits || ncb == 0) return fail(LTEPHY_ERROR_INVALID_INPUTS, "turbo_batch: bad arguments");
  uint32_t f1, f2;
  if (!ltehost::qpp_params(K, f1, f2)) return fail(LTEPHY_ERROR_INVALID_INPUTS, "turbo_batch: K=%u is not a turbo block size", K);
  CU(cudaSetDevice(h->cfg.device));
  const uint32_t NW = (K + 31) / 32, D = K + 4, npairs = (ncb + 1) / 2;
  const size_t   pw = ltephy_pair_words(NW); // words per pair
  ltephy::PhaseB& b = h->pb;
  b.reset(0);
  uint32_t po;
  if (pi_table_for(h, K, po)) return fail(LTEPHY_ERROR, "interleaver table upload failed");
  std::vector<uint32_t> pool(pw * npairs, 0u);
  const uint32_t        out_bytes = K / 8;
  for (uint32_t p = 0; p < npairs; p++) {
    DevPair pr{};
    pr.K = K, pr.NW = NW, pr.f1 = f1, pr.f2 = f2, pr.buf_off = pw * p, pr.ncb = (2 * p + 1 < ncb) ? 2 : 1;
    for (uint32_t hh = 0; hh < pr.ncb; hh++) {
      const uint32_t cbi = 2 * p + hh;
      pr.crc_type[hh] = (uint32_t)crc_type, pr.out_skip[hh] = 0, pr.out_bits[hh] = K, pr.out_byte[hh] = cbi * out_bytes, pr.cb_index[hh] = cbi;
      short*         buf = reinterpret_cast<short*>(pool.data() + pr.buf_off);
      const int16_t* src = d + (size_t)cbi * 3 * D;
      for (uint32_t s = 0; s < 3; s++)
        for (uint32_t i = 0; i < D; i++) {
          const uint32_t word = i < K ? s * 32 * NW + (i & 31u) * NW + (i >> 5) : 3 * 32 * NW + s * 4 + (i - K);
          const int      v    = src[s * D + i]; // conditioned LLRs: the decoder's range analysis (k_turbo.cu) assumes |d| <= 255
          buf[2 * word + hh]  = (short)(v > 255 ? 255 : (v < -255 ? -255 : v));
        }
    }
    b.pairs.push_back(pr);
    b.pair_pi_off.push_back(po);
  }
  if (h->d_turbo.reserve(pool.size()) || h->d_pairs.reserve(npairs) || h->d_pair_pi_off.reserve(npairs) || h->d_payload.reserve((size_t)ncb * out_bytes) ||
      h->d_cb_iters.reserve(ncb) || h->d_cb_crc.reserve(ncb))
    return fail(LTEPHY_ERROR, "device allocation failed");
  CU(cudaMemcpyAsync(h->d_turbo.p, pool.data(), pool.size() * 4, cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(h->d_pairs.p, b.pairs.data(), npairs * sizeof(DevPair), cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(h->d_pair_pi_off.p, b.pair_pi_off.data(), npairs * 4, cudaMemcpyHostToDevice, h->stream));
  if (int r = launch_turbo_buckets(h, {{2 * NW + ((K & 31u) ? 1u : 0u), npairs}}, max_iter ? max_iter : 1)) return r; // one bucket: NW threads
  std::vector<uint8_t> packed((size_t)ncb * out_bytes), it(ncb), ok(ncb);
  CU(cudaMemcpyAsync(packed.data(), h->d_payload.p, packed.size(), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(it.data(), h->d_cb_iters.p, ncb, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(ok.data(), h->d_cb_crc.p, ncb, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  CU(cudaGetLastError());
  cudaEventElapsedTime(&h->t_ms[2], h->ev[4], h->ev[5]);
  for (size_t i = 0; i < (size_t)ncb * K; i++) bits[i] = (packed[i >> 3] >> (7 - (i & 7))) & 1;
  if (iters) memcpy(iters, it.data(), ncb);
  if (crc_ok) memcpy(crc_ok, ok.data(), ncb);
  return LTEPHY_SUCCESS;
}

// LTEPHY_TAP_TURBO_IN after a phase B: the decoder's pairs follow pair_code_blocks, but the tap lays each code block's stream out as if
// equal-K code blocks were paired in submission order (buffers in the order of their first block), so that what it shows depends on the
// grants and the soft bits alone, not on the pairing policy.
static int tap_turbo_in(ltephy* h, void* dst, size_t bytes)
{
  std::vector<uint32_t> pool(h->d_turbo.cap);
  CU(cudaStreamSynchronize(h->stream));
  CU(cudaMemcpy(pool.data(), h->d_turbo.p, pool.size() * 4, cudaMemcpyDeviceToHost));
  if (h->pb.cbs.empty()) { // ltephy_turbo_batch: the pool is already in submission order
    memcpy(dst, pool.data(), bytes);
    return LTEPHY_SUCCESS;
  }
  std::vector<uint16_t>      out(pool.size() * 2, 0);
  const uint16_t*            src = reinterpret_cast<const uint16_t*>(pool.data());
  std::map<uint32_t, size_t> open; // K -> buffer with a free high half
  size_t                     words = 0;
  for (const DevCb& cb : h->pb.cbs) {
    const size_t n = ltephy_pair_words((cb.K + 31) / 32), from = h->pb.pairs[cb.pair].buf_off;
    size_t       to;
    uint32_t     hh = 0;
    auto         it = open.find(cb.K);
    if (it != open.end()) {
      to = it->second, hh = 1;
      open.erase(it);
    } else {
      to = words, open[cb.K] = words;
      words += n;
    }
    for (size_t w = 0; w < n; w++) out[2 * (to + w) + hh] = src[2 * (from + w) + cb.half];
  }
  memcpy(dst, out.data(), bytes);
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_tap(ltephy_t* h, int what, void* dst, size_t bytes)
{
  if (!h || !dst) return fail(LTEPHY_ERROR_INVALID_INPUTS, "tap: bad arguments");
  const void* src = nullptr;
  size_t      avail = 0;
  const size_t g = (size_t)14 * h->dc.nsc, n = h->n_cur;
  switch (what) {
    case LTEPHY_TAP_SYM: src = h->d_sym.p, avail = n * h->dc.nof_rx * g * sizeof(float2); break;
    case LTEPHY_TAP_CE: // the interpolated grid is not kept (the equalisers interpolate on the fly): materialise it from the pilot grid now
      CU(cudaSetDevice(h->cfg.device));
      if (h->d_ce.reserve((size_t)h->cfg.max_subframes * h->dc.nof_ports * h->dc.nof_rx * g)) return fail(LTEPHY_ERROR, "device allocation failed");
      if (n) launch_chest_interp(h->dc, h->d_pil.p, h->d_ce.p, (uint32_t)n, h->stream, &h->launches);
      src = h->d_ce.p, avail = n * h->dc.nof_ports * h->dc.nof_rx * g * sizeof(float2);
      break;
    case LTEPHY_TAP_LLR: src = h->d_llr.p, avail = n * LLR_STRIDE * sizeof(float); break;
    case LTEPHY_TAP_PDSCH_LLR: src = h->d_pllr.p, avail = h->pb.pllr_elems * sizeof(short); break;
    case LTEPHY_TAP_TURBO_IN: src = h->d_turbo.p, avail = h->d_turbo.cap * 4; break;
    case LTEPHY_TAP_UL_SYM: src = h->d_ulsym.p, avail = (size_t)h->n_ul * h->dc.ul_nof_rx * 14 * h->dc.nsc * sizeof(float2); break;
    case LTEPHY_TAP_PBCH_LLR: src = h->pbch_frames ? h->d_pbch.p + 3 * 960 : nullptr, avail = (size_t)h->pbch_frames * 960 * sizeof(float); break;
    default: return fail(LTEPHY_ERROR_INVALID_INPUTS, "tap: unknown buffer");
  }
  if (bytes > avail) return fail(LTEPHY_ERROR_INVALID_INPUTS, "tap: %zu bytes requested, %zu available", bytes, avail);
  if (what == LTEPHY_TAP_TURBO_IN) return tap_turbo_in(h, dst, bytes);
  CU(cudaStreamSynchronize(h->stream));
  CU(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
  return LTEPHY_SUCCESS;
}
