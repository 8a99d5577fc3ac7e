// cell_chain.h -- the steps the C++ examples share, host code over the C-ABI of libltephy_b200:
//   chain_acquire (cell_search.cpp, decode_recording.cpp, decode_recording_ul.cpp): the cell search on the start of a file, then the MIB
//     soft-combined over its frames (chain_mib_host);
//   chain_print_cell (decode_recording.cpp, decode_recording_ul.cpp, decode_wideband.cpp): the cell line;
//   CellChain (decode_recording.cpp, decode_wideband.cpp): for every push of a tracker, the decoder and the DCI search on the cut subframes,
//     written to a MAC-LTE pcap and a DCI trace, with the lock counts and the summary lines;
//   UlChain (offline_ul.cpp, decode_recording_ul.cpp): the UL mode, batch by batch: the downlink's RARs and DCI-0s turned into PUSCH grants on the
//     uplink, both directions written to a MAC-LTE pcap.
#pragma once
#include "ltephy_b200.h"
#include "ltephy_search.h"
#include "ltephy_sinks.h"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

// bytes of one complex sample of an LTEPHY_IQ_* format
static inline uint32_t chain_sample_bytes(uint32_t fmt) { return fmt == LTEPHY_IQ_SC16 ? 4 : fmt == LTEPHY_IQ_SC8 ? 2 : 8; }

// removes every "fmt=cf32|sc16|sc8" argument from argv (the sample format of the input files, LTEPHY_IQ_*; cf32 without one), so that the
// positional arguments keep their places.  0, or 2 for an unknown format (message printed)
static inline int chain_take_fmt(int& argc, char** argv, uint32_t* fmt)
{
  *fmt  = LTEPHY_IQ_CF32;
  int o = 1;
  for (int i = 1; i < argc; i++) {
    if (strncmp(argv[i], "fmt=", 4)) {
      argv[o++] = argv[i];
      continue;
    }
    const char* f = argv[i] + 4;
    if (!strcmp(f, "cf32")) *fmt = LTEPHY_IQ_CF32;
    else if (!strcmp(f, "sc16")) *fmt = LTEPHY_IQ_SC16;
    else if (!strcmp(f, "sc8")) *fmt = LTEPHY_IQ_SC8;
    else {
      fprintf(stderr, "unknown %s (fmt=cf32, sc16 or sc8)\n", argv[i]);
      return 2;
    }
  }
  argc = o;
  return 0;
}

// samples [s, s + n) of every antenna, antenna-major, b bytes per complex sample, from a file holding L samples per antenna
static inline bool read_span(FILE* f, uint32_t A, uint64_t L, uint32_t b, uint64_t s, uint64_t n, std::vector<uint8_t>& out)
{
  out.resize((size_t)b * A * n);
  for (uint32_t a = 0; a < A; a++) {
    if (fseeko(f, (off_t)(b * ((uint64_t)a * L + s)), SEEK_SET) != 0) return false;
    if (fread(out.data() + (size_t)b * a * n, b, n, f) != n) return false;
  }
  return true;
}

// the MIB, soft-combined over nframes subframes 0 ([nframes][A][15 N] samples of format fmt, host memory, subframe 0 of frame f at tti 10 f) with
// the carrier offset cfo_hz corrected and the port count searched; mib->sfn is that of frame 0.  0, 1 on a library error, 3 when no MIB passed
static inline int chain_mib_host(const void* sf0, uint32_t nframes, uint32_t pci, float cfo_hz, uint32_t N, uint32_t A, uint32_t fmt, ltephy_mib_t* mib)
{
  std::vector<uint32_t> tti0(nframes);
  for (uint32_t f = 0; f < nframes; f++) tti0[f] = 10 * f;
  ltephy_cfg_t mcfg{};
  mcfg.nof_prb = 15, mcfg.nof_ports = 2, mcfg.cell_id = pci, mcfg.nof_rx = A, mcfg.max_subframes = nframes, mcfg.symbol_sz = N, mcfg.iq_format = fmt;
  ltephy_t*                      mphy = nullptr;
  std::vector<ltephy_mib_comb_t> m(nframes);
  if (ltephy_create(&mcfg, &mphy) != LTEPHY_SUCCESS || ltephy_set_cfo(mphy, cfo_hz) != LTEPHY_SUCCESS ||
      ltephy_submit_iq(mphy, sf0, tti0.data(), nframes) != LTEPHY_SUCCESS ||
      ltephy_mib_decode_combined(mphy, LTEPHY_MIB_SEARCH_PORTS, m.data()) != LTEPHY_SUCCESS) {
    fprintf(stderr, "MIB decode: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_destroy(mphy);
  *mib = ltephy_mib_t{};
  for (uint32_t f = 0; f < nframes && !mib->found; f++)
    if (m[f].mib.found) {
      *mib     = m[f].mib;
      mib->sfn = (mib->sfn + 1024 - f % 1024) % 1024; // the SFN of the frame at frame_offset
    }
  if (!mib->found) { // no window of any frame passed its CRC (too weak even combined, or a cell with four CRS ports)
    fprintf(stderr, "cell %u found, MIB not decoded\n", pci);
    return 3;
  }
  return 0;
}

// the cell of samples [0, L0) of an antenna-major file of L samples per antenna in format fmt: the cell search there, the first cell it detects, and
// that cell's MIB soft-combined over the subframes 0 of every whole frame in those samples (chain_mib_host).  0, 1 on a read or library error, 3 when
// no cell is found, no whole frame follows its first subframe 0 or no MIB passed (message printed)
static inline int chain_acquire(FILE* f, uint32_t N, uint32_t A, uint64_t L, uint64_t L0, uint32_t fmt, ltephy_cell_t* cell, ltephy_mib_t* mib)
{
  const uint32_t       SF = 15 * N, b = chain_sample_bytes(fmt);
  std::vector<uint8_t> x;
  if (!read_span(f, A, L, b, 0, L0, x)) {
    fprintf(stderr, "short read\n");
    return 1;
  }
  ltephy_sync_cfg_t scfg{};
  scfg.symbol_sz = N, scfg.nof_rx = A, scfg.max_samples = L0, scfg.iq_format = fmt;
  ltephy_sync_t* sync = nullptr;
  ltephy_cell_t  cells[3];
  if (ltephy_sync_create(&scfg, &sync) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_sync_create: %s\n", ltephy_last_error());
    return 1;
  }
  if (ltephy_cell_search(sync, x.data(), L0, cells) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_cell_search: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_sync_destroy(sync);
  const ltephy_cell_t* c = std::find_if(cells, cells + 3, [](const ltephy_cell_t& q) { return q.detected; });
  if (c == cells + 3) {
    fprintf(stderr, "no cell found\n");
    return 3;
  }
  *cell = *c;
  // the PBCH and the centre CRS do not depend on the bandwidth: chain_mib_host's 15-PRB handle reads the MIB of any cell
  const uint32_t nframes = (uint32_t)((L0 - c->frame_offset) / (10ull * SF));
  if (!nframes) {
    fprintf(stderr, "no whole frame after the first subframe 0\n");
    return 3;
  }
  std::vector<uint8_t> sf0((size_t)b * A * SF * nframes); // subframe 0 of each frame, antenna after antenna
  for (uint32_t f = 0; f < nframes; f++)
    for (uint32_t a = 0; a < A; a++)
      std::copy_n(x.data() + b * (a * L0 + c->frame_offset + (uint64_t)f * 10 * SF), (size_t)b * SF, sf0.data() + (size_t)b * ((size_t)f * A + a) * SF);
  return chain_mib_host(sf0.data(), nframes, c->pci, c->cfo_hz, N, A, fmt, mib);
}

static inline void chain_print_cell(const ltephy_cell_t& c, const ltephy_mib_t& mib)
{
  printf("pci %u frame_offset %llu cfo_hz %.9g nof_prb %u nof_ports %u phich_resources %u phich_length %u sfn %u\n", c.pci,
         (unsigned long long)c.frame_offset, c.cfo_hz, mib.nof_prb, mib.nof_ports, mib.phich_resources, mib.phich_length, mib.sfn);
}

// decoder, DCI search and sinks of one cell, fed with the pushes of its tracker
struct CellChain {
  uint32_t           N = 0, A = 0, SF = 0, B = 0;
  int                reacq = 0;
  ltephy_cell_t      cell{};
  ltephy_t*          phy    = nullptr;
  ltephy_search_t*   search = nullptr;
  ltephy_t*          mibh   = nullptr; // the MIB decoder of the fallback after a re-acquisition
  ltephy_pcap_t*     pcap   = nullptr;
  FILE*              tsv    = nullptr;
  bool               awaiting = false; // between a re-acquired subframe and the next MIB that passes: decode nothing
  uint32_t           sfn_corr = 0;     // frames added to every tti (after the MIB read again, or when the tracker started at tti 0)
  unsigned long long n_finds = 0, n_reacq = 0, n_await = 0;
  unsigned long long n_sf = 0, n_dci = 0, n_tb = 0, n_ok = 0, n_locked = 0, n_lost = 0, n_hf = 0, n_hf_locked = 0, n_remeasured = 0;
  int64_t            last_start = 0;
  float              last_cfo   = 0.0f;
  uint32_t                        max_dcis = 0;
  std::vector<uint32_t>           ttis;
  std::vector<ltephy_sf_info_t>   info;
  std::vector<ltephy_cand_t>      scratch;
  std::vector<ltephy_dci_t>       dcis;
  std::vector<ltephy_tb_result_t> tbs;
  std::vector<uint8_t>            payload;

  // the decoder and the DCI search for the cell of the MIB; batches of up to B subframes.  0 or 1 (error printed)
  int open_decoder(const ltephy_cell_t& c, const ltephy_mib_t& mib, uint32_t N_, uint32_t A_, uint32_t B_)
  {
    N = N_, A = A_, SF = 15 * N_, B = B_, cell = c, last_start = (int64_t)c.frame_offset, last_cfo = c.cfo_hz;
    ltephy_cfg_t cfg{};
    cfg.nof_prb = mib.nof_prb, cfg.nof_ports = mib.nof_ports, cfg.cell_id = c.pci, cfg.nof_rx = A, cfg.max_subframes = B, cfg.turbo_max_iter = 8;
    cfg.flags = LTEPHY_FLAG_SKIP_LOW_POWER, cfg.symbol_sz = N, cfg.phich_resources = mib.phich_resources, cfg.phich_length = mib.phich_length;
    if (ltephy_create(&cfg, &phy) != LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_create: %s\n", ltephy_last_error());
      return 1;
    }
    search = ltephy_search_create(phy, 5); // rnti_histogram_threshold default of the reference
    return 0;
  }

  // the fallback's MIB decoder (with reacquire) and the sinks.  0 or 1 (error printed)
  int open_sinks(const ltephy_mib_t& mib, int reacquire, const char* pcap_path, const char* tsv_path)
  {
    reacq = reacquire;
    // the MIB decoder of the fallback: the cell's bandwidth and ports are known, so no port search; the cut is already CFO-corrected
    if (reacq) {
      ltephy_cfg_t rcfg{};
      rcfg.nof_prb = mib.nof_prb, rcfg.nof_ports = mib.nof_ports, rcfg.cell_id = cell.pci, rcfg.nof_rx = A, rcfg.max_subframes = 1, rcfg.symbol_sz = N;
      if (ltephy_create(&rcfg, &mibh) != LTEPHY_SUCCESS) {
        fprintf(stderr, "ltephy_create: %s\n", ltephy_last_error());
        return 1;
      }
    }
    pcap = ltephy_pcap_open(pcap_path);
    tsv  = fopen(tsv_path, "w");
    if (!pcap || !tsv) {
      fprintf(stderr, "cannot open outputs\n");
      return 1;
    }
    max_dcis = 32 * B;
    ttis.resize(B), info.resize(B), scratch.resize((size_t)B * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES), dcis.resize(max_dcis);
    tbs.resize(2 * (size_t)max_dcis), payload.resize((size_t)B * 64 * 1024);
    return 0;
  }

  // one push of the cell's tracker: lock counts, the MIB fallback after a re-acquisition, decode, pcap and trace.  0 or 1 (error printed)
  int consume(const ltephy_track_out_t& o)
  {
    char line[256];
    n_remeasured += o.remeasured, n_hf += o.nof_half_frames, n_finds += o.finds;
    for (uint32_t i = 0; i < o.nof_half_frames; i++) n_hf_locked += (o.hf[i].flags & LTEPHY_TRACK_LOCKED) != 0;
    const uint32_t got = o.nof_subframes;
    if (!got) return 0;
    for (uint32_t i = 0; i < got; i++) {
      ttis[i] = (o.sf[i].tti + 10 * sfn_corr) % 10240;
      n_locked += (o.sf[i].flags & LTEPHY_TRACK_LOCKED) != 0, n_lost += (o.sf[i].flags & LTEPHY_TRACK_LOST) != 0;
    }
    last_start = o.sf[got - 1].start, last_cfo = o.sf[got - 1].cfo_hz;
    // the push as runs of subframes to decode, split where the MIB fallback starts and ends
    const size_t sf_bytes = (size_t)A * SF * 8;
    for (uint32_t i0 = 0; i0 < got;) {
      if (awaiting || (o.sf[i0].flags & LTEPHY_TRACK_REACQUIRED)) {
        if (o.sf[i0].flags & LTEPHY_TRACK_REACQUIRED) {
          if (ltephy_mib_reset(mibh) != LTEPHY_SUCCESS) {
            fprintf(stderr, "ltephy_mib_reset: %s\n", ltephy_last_error());
            return 1;
          }
          awaiting = true, n_reacq++;
        }
        n_await++;
        if (o.sf[i0].tti % 10 == 0) {
          ltephy_mib_comb_t mc{};
          if (ltephy_submit_iq_device(mibh, static_cast<const char*>(o.iq_dev) + i0 * sf_bytes, &o.sf[i0].tti, 1) != LTEPHY_SUCCESS ||
              ltephy_mib_decode_combined(mibh, 0, &mc) != LTEPHY_SUCCESS) {
            fprintf(stderr, "MIB decode: %s\n", ltephy_last_error());
            return 1;
          }
          if (mc.mib.found) {
            sfn_corr = (mc.mib.sfn + 1024 - o.sf[i0].tti / 10 % 1024) % 1024, awaiting = false;
            for (uint32_t i = i0 + 1; i < got; i++) ttis[i] = (o.sf[i].tti + 10 * sfn_corr) % 10240;
          }
        }
        i0++;
        continue;
      }
      uint32_t i1 = i0 + 1;
      while (i1 < got && !(o.sf[i1].flags & LTEPHY_TRACK_REACQUIRED)) i1++;
      const uint32_t m = i1 - i0, base = (uint32_t)(n_sf + i0);
      uint32_t       nd = 0;
      if (ltephy_decode_subframes_device(phy, search, static_cast<const char*>(o.iq_dev) + i0 * sf_bytes, ttis.data() + i0, m, LTEPHY_SEQ_NONE, info.data(),
                                         scratch.data(), dcis.data(), max_dcis, &nd, tbs.data(), payload.data(), payload.size()) != LTEPHY_SUCCESS) {
        fprintf(stderr, "ltephy_decode_subframes_device: %s\n", ltephy_last_error());
        return 1;
      }
      // timestamps: capture time, 1 ms per subframe cut (as offline_decode)
      for (uint32_t i = 0; i < nd; i++) {
        const uint32_t t = ttis[i0 + dcis[i].sf];
        const int      n = ltephy_dci_trace_line(search, &dcis[i], t, info[dcis[i].sf].cfi, tbs[2 * i].crc == 2 || tbs[2 * i + 1].crc == 2, (base + dcis[i].sf) / 1000,
                                                 ((base + dcis[i].sf) % 1000) * 1000, line, sizeof(line));
        if (n > 0) fwrite(line, 1, (size_t)n, tsv);
        for (int k = 0; k < 2; k++) n_tb += tbs[2 * i + k].payload_len > 0, n_ok += tbs[2 * i + k].crc != 0;
      }
      if (ltephy_pcap_write_dl_batch(pcap, ttis.data() + i0, dcis.data(), nd, tbs.data(), payload.data(), 0, base / 1000, (base % 1000) * 1000) < 0) {
        fprintf(stderr, "pcap write failed\n");
        return 1;
      }
      n_dci += nd;
      i0 = i1;
    }
    n_sf += got;
    return 0;
  }

  // the tracking and decode summary lines
  void print_summary() const
  {
    const long long drift = n_sf ? (long long)(last_start - (int64_t)cell.frame_offset - (int64_t)(n_sf - 1) * SF) : 0;
    printf("tracking: subframes %llu locked %llu lost %llu  half-frames %llu locked %llu remeasured %llu  timing moved %lld samples  cfo_hz %.1f\n", n_sf,
           n_locked, n_lost, n_hf, n_hf_locked, n_remeasured, drift, last_cfo);
    printf("subframes %llu  dcis %llu  transport blocks %llu  crc ok %llu\n", n_sf, n_dci, n_tb, n_ok);
    if (reacq) printf("reacquire: finds %llu reacquired %llu awaiting_mib %llu\n", n_finds, n_reacq, n_await);
  }

  void close()
  {
    if (tsv) fclose(tsv);
    if (pcap) ltephy_pcap_close(pcap);
    if (search) ltephy_search_destroy(search);
    if (phy) ltephy_destroy(phy);
    if (mibh) ltephy_destroy(mibh);
    tsv = nullptr, pcap = nullptr, search = nullptr, phy = nullptr, mibh = nullptr;
  }
};

// the UL mode of one cell (the reference's -m 1: SubframeWorker's UL branch with PDSCH_Decoder::decode_ul_mode and PUSCH_Decoder::decode), fed one
// batch at a time with the downlink and the uplink of the same ttis: the downlink decoded in UL mode (RARs and format 1 / 1A), the msg-3 grants of
// the RARs (6 subframes later) and the grants of the DCI-0s (4 later) decoded on the uplink, both directions written to a MAC-LTE pcap.  A grant
// that lands past its batch is carried into the next one, and stays carried while it lies past that one too (a short last batch).
struct UlChain {
  ltephy_t *                      dl = nullptr, *ul = nullptr;
  ltephy_search_t*                search = nullptr;
  ltephy_pcap_t*                  pcap   = nullptr;
  uint32_t                        max_dcis = 0, max_ul = 0;
  unsigned long long              n_sf = 0, n_dl_ok = 0, n_dci0 = 0, n_rar = 0, n_ul_ok = 0;
  std::vector<uint32_t>           ttis; // the caller writes the batch's ttis here before step()
  std::vector<ltephy_sf_info_t>   info;
  std::vector<ltephy_cand_t>      scratch;
  std::vector<ltephy_dci_t>       dcis;
  std::vector<ltephy_tb_result_t> tbs, ures;
  std::vector<uint8_t>            payload, upayload, reading;
  std::vector<ltephy_ul_grant_t>  grants, now, carry; // carry: grants whose subframe lies past the batch, indexed into the next one
  std::vector<uint32_t>           grant_dci;
  std::vector<ltephy_ul_chest_t>  chest;

  // the downlink and uplink decoders of cfg (batches of up to cfg.max_subframes, cfg.ul_nof_rx uplink antennas), the UL configuration and hopping offset of SIB2, the DCI
  // search in UL mode and the pcap.  0 or 1 (error printed)
  int open(const ltephy_cfg_t& cfg, const ltephy_ul_cfg_t& ucfg, uint32_t hopping_offset, const char* pcap_path)
  {
    if (ltephy_create(&cfg, &dl) != LTEPHY_SUCCESS || ltephy_create(&cfg, &ul) != LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_create: %s\n", ltephy_last_error());
      return 1;
    }
    if (ltephy_set_ul_cfg(ul, &ucfg) != LTEPHY_SUCCESS || !(search = ltephy_search_create(dl, 5))) {
      fprintf(stderr, "UL config / search: %s\n", ltephy_last_error());
      return 1;
    }
    ltephy_search_set_ul_hopping(search, hopping_offset);
    ltephy_search_set_ul_mode(search, 1, 0); // the downlink side decodes RARs and format 1 / 1A only (decode_ul_mode)
    if (!(pcap = ltephy_pcap_open(pcap_path))) {
      fprintf(stderr, "cannot open %s\n", pcap_path);
      return 1;
    }
    const uint32_t B = cfg.max_subframes;
    max_dcis = 32 * B, max_ul = 3 * max_dcis + 64;
    ttis.resize(B), info.resize(B), scratch.resize((size_t)B * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES), dcis.resize(max_dcis);
    tbs.resize(2 * (size_t)max_dcis), ures.resize(max_ul), payload.resize((size_t)B * 64 * 1024), upayload.resize((size_t)B * 64 * 1024);
    grants.resize(max_ul), grant_dci.resize(max_ul), reading.resize(max_ul), chest.resize(max_ul);
    return 0;
  }

  // one batch of got subframes at ttis[0, got): downlink [got][15 N] of one antenna and uplink [got][A][15 N] of A = cfg.ul_nof_rx antennas (one
  // when 0), samples of cfg.iq_format, in host memory or, with on_device, in device memory (a tracker's cuts, cf32).  0 or 1 (error printed)
  int step(const void* dl_iq, const void* ul_iq, bool on_device, uint32_t got)
  {
    uint32_t  nd = 0;
    const int rd = on_device ? ltephy_decode_subframes_device(dl, search, dl_iq, ttis.data(), got, LTEPHY_SEQ_NONE, info.data(), scratch.data(), dcis.data(),
                                                              max_dcis, &nd, tbs.data(), payload.data(), payload.size())
                             : ltephy_decode_subframes(dl, search, dl_iq, ttis.data(), got, LTEPHY_SEQ_NONE, info.data(), scratch.data(), dcis.data(),
                                                       max_dcis, &nd, tbs.data(), payload.data(), payload.size());
    if (rd != LTEPHY_SUCCESS) {
      fprintf(stderr, "%s: %s\n", on_device ? "ltephy_decode_subframes_device" : "ltephy_decode_subframes", ltephy_last_error());
      return 1;
    }
    const uint32_t ts_s = (uint32_t)(n_sf / 1000), ts_us = (uint32_t)((n_sf % 1000) * 1000);
    const int      wd   = ltephy_pcap_write_dl_batch(pcap, ttis.data(), dcis.data(), nd, tbs.data(), payload.data(), 0, ts_s, ts_us);
    if (wd < 0) {
      fprintf(stderr, "pcap write failed\n");
      return 1;
    }
    n_dl_ok += (unsigned)wd;
    // grants of this batch's uplink: what the previous batch left over, the msg-3 grants of the RARs (6 subframes later), the DCI-0s (4 later)
    now.swap(carry), carry.clear();
    const auto past = std::stable_partition(now.begin(), now.end(), [&](const ltephy_ul_grant_t& g) { return g.sf < got; });
    carry.assign(past, now.end()), now.erase(past, now.end());
    auto place = [&](const ltephy_ul_grant_t& g) { (g.sf < got ? now : carry).push_back(g); };
    for (uint32_t i = 0; i < nd; i++) {
      const ltephy_tb_result_t& r = tbs[2 * i];
      if (dcis[i].rnti < 1 || dcis[i].rnti > 10 || !r.crc || !r.payload_len) continue; // RA-RNTI with a decoded block (unpack_rar_response_ul_mode)
      ltephy_rar_t rars[16];
      uint32_t     nr = 0;
      if (ltephy_rar_unpack(search, payload.data() + r.payload_off, r.payload_len, rars, 16, &nr, nullptr) != LTEPHY_SUCCESS) continue;
      for (uint32_t k = 0; k < nr; k++) {
        ltephy_search_activate(search, rars[k].t_crnti, 0, LTEPHY_ACT_RAR); // rntiManager.activateAndRefresh, DL_Sniffer_PDSCH.cc:659
        n_rar++;
        if (!rars[k].valid) continue;
        rars[k].grant.sf = dcis[i].sf + 6; // ULSchedule::get_rar_ul_tti
        place(rars[k].grant);
      }
    }
    uint32_t ng = 0;
    if (ltephy_ul_grants_from_dcis(search, info.data(), dcis.data(), nd, nullptr, 0, grants.data(), grant_dci.data(), reading.data(), max_ul, &ng) !=
        LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_ul_grants_from_dcis: %s\n", ltephy_last_error());
      return 1;
    }
    for (uint32_t k = 0; k < ng; k++) {
      n_dci0 += k == 0 || grant_dci[k] != grant_dci[k - 1];
      place(grants[k]);
    }
    for (ltephy_ul_grant_t& g : carry) g.sf -= got; // index into the next batch's uplink
    if (!now.empty()) {
      if (now.size() > max_ul) now.resize(max_ul);
      const int ru = on_device ? ltephy_submit_ul_device(ul, ul_iq, ttis.data(), got, now.data(), (uint32_t)now.size())
                               : ltephy_submit_ul(ul, ul_iq, ttis.data(), got, now.data(), (uint32_t)now.size());
      if (ru != LTEPHY_SUCCESS || ltephy_get_ul(ul, ures.data(), chest.data(), upayload.data(), upayload.size()) != LTEPHY_SUCCESS) {
        fprintf(stderr, "uplink decode: %s\n", ltephy_last_error());
        return 1;
      }
      // the attempts of one DCI-0 are adjacent and in the reference's order: keep the first that passed (PUSCH_Decoder::decode stops there)
      bool passed = false;
      for (size_t k = 0; k < now.size(); k++) {
        if (k == 0 || now[k - 1].rnti != now[k].rnti || now[k - 1].sf != now[k].sf) passed = false;
        if (ures[k].crc && passed) ures[k].crc = 0;
        passed = passed || ures[k].crc != 0;
      }
      const int wu = ltephy_pcap_write_ul_batch(pcap, ttis.data(), now.data(), (uint32_t)now.size(), ures.data(), upayload.data(), 0, ts_s, ts_us);
      if (wu < 0) {
        fprintf(stderr, "pcap write failed\n");
        return 1;
      }
      n_ul_ok += (unsigned)wu;
    }
    n_sf += got;
    return 0;
  }

  void close()
  {
    if (pcap) ltephy_pcap_close(pcap);
    if (search) ltephy_search_destroy(search);
    if (dl) ltephy_destroy(dl);
    if (ul) ltephy_destroy(ul);
    pcap = nullptr, search = nullptr, dl = nullptr, ul = nullptr;
  }
};
