// decode_recording.cpp -- raw recording in, pcap out: a continuous antenna-major cf32 recording of any length, as an SDR writes it, decoded
// through the C-ABI of libltephy_b200.  Cell search on the first 40 ms (ltephy_cell_search), the MIB soft-combined over the frames there
// (ltephy_mib_decode_combined), then the tracker (ltephy_track_push) part by part, which follows the frame timing and carrier offset through a
// sampling clock that is off by a few ppm and cuts every subframe into device memory, and ltephy_decode_subframes_device on each cut.  Writes
// the MAC-LTE pcap and the DCI trace exactly as offline_decode does, and prints the cell and a lock summary.  Host code only; without a GPU
// ltephy_sync_create fails.
//
//   decode_recording <iq.cf32> <symbol_sz> <nof_rx> <out.pcap> <out_dci.tsv> [subframes_per_push=500] [max_ppm=50] [no_cfo=0] [reacquire=0]
//
// With reacquire = 1 the tracker searches a lost cell again (LTEPHY_TRACK_REACQUIRE), and the example falls back as the reference does from
// DECODE_PDSCH to DECODE_MIB (src/src/LTESniffer_Core.cc:506-524): from the re-acquired subframe on it decodes nothing and feeds every
// subframe 0 of the cut to the MIB decoder until one passes, then adds (mib.sfn - tti / 10) mod 1024 frames to every later tti, because
// after dropped samples the tracker's SFN, which continues by sample count, is wrong.
//
// File layout: antenna after antenna, each a continuous run of complex float32 samples at 15 kHz * symbol_sz (what cell_search reads).  The
// file is read one push at a time (one seek per antenna), so its length is not limited by host memory.
#include "ltephy_b200.h"
#include "ltephy_search.h"
#include "ltephy_sinks.h"
#include <cstdio>
#include <cstdlib>
#include <vector>

// samples [s, s + n) of every antenna, antenna-major, from a file holding L samples per antenna
static bool read_span(FILE* f, uint32_t A, uint64_t L, uint64_t s, uint64_t n, std::vector<float>& out)
{
  out.resize((size_t)2 * A * n);
  for (uint32_t a = 0; a < A; a++) {
    if (fseeko(f, (off_t)(8 * ((uint64_t)a * L + s)), SEEK_SET) != 0) return false;
    if (fread(out.data() + (size_t)2 * a * n, 8, n, f) != n) return false;
  }
  return true;
}

int main(int argc, char** argv)
{
  if (argc < 6) {
    fprintf(stderr, "usage: %s <iq.cf32> <symbol_sz> <nof_rx> <out.pcap> <out_dci.tsv> [subframes_per_push=500] [max_ppm=50] [no_cfo=0] [reacquire=0]\n", argv[0]);
    return 2;
  }
  const uint32_t N = (uint32_t)atoi(argv[2]), A = (uint32_t)atoi(argv[3]), SF = 15 * N;
  const uint32_t B       = argc > 6 ? (uint32_t)atoi(argv[6]) : 500;
  const float    max_ppm = argc > 7 ? (float)atof(argv[7]) : 50.0f;
  const int      no_cfo  = argc > 8 ? atoi(argv[8]) : 0;
  const int      reacq   = argc > 9 ? atoi(argv[9]) : 0;
  FILE*          in      = fopen(argv[1], "rb");
  if (!in || A < 1 || A > 2 || B < 1) {
    fprintf(stderr, "cannot open %s / bad nof_rx or subframes_per_push\n", argv[1]);
    return 2;
  }
  fseeko(in, 0, SEEK_END);
  const uint64_t L = (uint64_t)ftello(in) / (8ull * A);

  // 1. cell search on the first 40 ms
  const uint64_t     L0 = L < 40ull * SF ? L : 40ull * SF;
  std::vector<float> x;
  ltephy_sync_cfg_t  scfg{};
  scfg.symbol_sz = N, scfg.nof_rx = A, scfg.max_samples = L0;
  ltephy_sync_t* sync = nullptr;
  ltephy_cell_t  cells[3];
  if (!read_span(in, A, L, 0, L0, x)) {
    fprintf(stderr, "short read\n");
    return 1;
  }
  if (ltephy_sync_create(&scfg, &sync) != LTEPHY_SUCCESS || ltephy_cell_search(sync, x.data(), L0, cells) != LTEPHY_SUCCESS) {
    fprintf(stderr, "cell search: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_sync_destroy(sync);
  const ltephy_cell_t* c = nullptr;
  for (auto& q : cells)
    if (q.detected) {
      c = &q;
      break;
    }
  if (!c) {
    fprintf(stderr, "no cell found\n");
    return 3;
  }

  // 2. the MIB, soft-combined over the frames of those 40 ms at the found timing, with the found carrier offset (as cell_search does)
  const uint32_t nframes = (uint32_t)((L0 - c->frame_offset) / (10ull * SF));
  if (!nframes) {
    fprintf(stderr, "no whole frame after the first subframe 0\n");
    return 3;
  }
  std::vector<float>    sf0((size_t)2 * A * SF * nframes);
  std::vector<uint32_t> tti0(nframes);
  for (uint32_t f = 0; f < nframes; f++) {
    tti0[f] = 10 * f;
    for (uint32_t a = 0; a < A; a++)
      for (uint32_t n = 0; n < SF; n++) {
        const uint64_t s = c->frame_offset + (uint64_t)f * 10 * SF + n;
        const size_t   d = ((size_t)f * A + a) * SF + n;
        sf0[2 * d] = x[2 * (a * L0 + s)], sf0[2 * d + 1] = x[2 * (a * L0 + s) + 1];
      }
  }
  ltephy_cfg_t mcfg{};
  mcfg.nof_prb = 15, mcfg.nof_ports = 2, mcfg.cell_id = c->pci, mcfg.nof_rx = A, mcfg.max_subframes = nframes, mcfg.symbol_sz = N;
  ltephy_t*                      mphy = nullptr;
  std::vector<ltephy_mib_comb_t> m(nframes);
  if (ltephy_create(&mcfg, &mphy) != LTEPHY_SUCCESS || ltephy_set_cfo(mphy, c->cfo_hz) != LTEPHY_SUCCESS ||
      ltephy_submit_iq(mphy, sf0.data(), tti0.data(), nframes) != LTEPHY_SUCCESS ||
      ltephy_mib_decode_combined(mphy, LTEPHY_MIB_SEARCH_PORTS, m.data()) != LTEPHY_SUCCESS) {
    fprintf(stderr, "MIB decode: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_destroy(mphy);
  ltephy_mib_t mib{};
  for (uint32_t f = 0; f < nframes && !mib.found; f++)
    if (m[f].mib.found) {
      mib     = m[f].mib;
      mib.sfn = (mib.sfn + 1024 - f % 1024) % 1024; // the SFN of the frame at frame_offset
    }
  if (!mib.found) {
    fprintf(stderr, "cell %u found, MIB not decoded\n", c->pci);
    return 3;
  }
  printf("pci %u frame_offset %llu cfo_hz %.9g nof_prb %u nof_ports %u phich_resources %u phich_length %u sfn %u\n", c->pci,
         (unsigned long long)c->frame_offset, c->cfo_hz, mib.nof_prb, mib.nof_ports, mib.phich_resources, mib.phich_length, mib.sfn);

  // 3. decoder, DCI search and tracker for the cell
  ltephy_cfg_t cfg{};
  cfg.nof_prb = mib.nof_prb, cfg.nof_ports = mib.nof_ports, cfg.cell_id = c->pci, cfg.nof_rx = A, cfg.max_subframes = B, cfg.turbo_max_iter = 8;
  cfg.flags = LTEPHY_FLAG_SKIP_LOW_POWER, cfg.symbol_sz = N, cfg.phich_resources = mib.phich_resources, cfg.phich_length = mib.phich_length;
  ltephy_t* phy = nullptr;
  if (ltephy_create(&cfg, &phy) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_create: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_search_t*   search = ltephy_search_create(phy, 5); // rnti_histogram_threshold default of the reference
  ltephy_track_cfg_t tcfg{};
  tcfg.symbol_sz = N, tcfg.nof_rx = A, tcfg.pci = c->pci, tcfg.first_tti = 10 * mib.sfn, tcfg.frame_offset = c->frame_offset, tcfg.cfo_hz = c->cfo_hz;
  tcfg.max_ppm = max_ppm, tcfg.max_subframes = B, tcfg.flags = (no_cfo ? LTEPHY_TRACK_NO_CFO : 0) | (reacq ? LTEPHY_TRACK_REACQUIRE : 0);
  ltephy_track_t* tr = nullptr;
  if (!search || ltephy_track_create(&tcfg, &tr) != LTEPHY_SUCCESS) {
    fprintf(stderr, "search / tracker: %s\n", ltephy_last_error());
    return 1;
  }
  // the MIB decoder of the fallback: the cell's bandwidth and ports are known, so no port search; the cut is already CFO-corrected
  ltephy_t* mibh = nullptr;
  if (reacq) {
    ltephy_cfg_t rcfg{};
    rcfg.nof_prb = mib.nof_prb, rcfg.nof_ports = mib.nof_ports, rcfg.cell_id = c->pci, rcfg.nof_rx = A, rcfg.max_subframes = 1, rcfg.symbol_sz = N;
    if (ltephy_create(&rcfg, &mibh) != LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_create: %s\n", ltephy_last_error());
      return 1;
    }
  }
  bool               awaiting = false; // between a re-acquired subframe and the next MIB that passes: decode nothing
  uint32_t           sfn_corr = 0;     // frames added to every tti after the MIB read again
  unsigned long long n_finds = 0, n_reacq = 0, n_await = 0;
  ltephy_pcap_t* pcap = ltephy_pcap_open(argv[4]);
  FILE*          tsv  = fopen(argv[5], "w");
  if (!pcap || !tsv) {
    fprintf(stderr, "cannot open outputs\n");
    return 1;
  }
  const uint32_t                  max_dcis = 32 * B;
  std::vector<uint32_t>           ttis(B);
  std::vector<ltephy_sf_info_t>   info(B);
  std::vector<ltephy_cand_t>      scratch((size_t)B * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES);
  std::vector<ltephy_dci_t>       dcis(max_dcis);
  std::vector<ltephy_tb_result_t> tbs(2 * (size_t)max_dcis);
  std::vector<uint8_t>            payload((size_t)B * 64 * 1024);
  unsigned long long n_sf = 0, n_dci = 0, n_tb = 0, n_ok = 0, n_locked = 0, n_lost = 0, n_hf = 0, n_hf_locked = 0, n_remeasured = 0;
  int64_t            last_start = (int64_t)c->frame_offset;
  float              last_cfo   = c->cfo_hz;
  char               line[256];
  // 4. the recording arrives B subframes at a time; each push re-feeds from the tracker's next_sample
  uint64_t recv = 0, next = c->frame_offset;
  for (;;) {
    if (recv < L) recv = recv + (uint64_t)B * SF < L ? recv + (uint64_t)B * SF : L;
    if (next >= recv) {
      if (recv == L) break;
      continue;
    }
    if (!read_span(in, A, L, next, recv - next, x)) {
      fprintf(stderr, "short read\n");
      return 1;
    }
    ltephy_track_out_t o{};
    if (ltephy_track_push(tr, x.data(), next, recv - next, &o) != LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_track_push: %s\n", ltephy_last_error());
      return 1;
    }
    next = o.next_sample;
    n_remeasured += o.remeasured, n_hf += o.nof_half_frames, n_finds += o.finds;
    for (uint32_t i = 0; i < o.nof_half_frames; i++) n_hf_locked += (o.hf[i].flags & LTEPHY_TRACK_LOCKED) != 0;
    const uint32_t got = o.nof_subframes;
    if (!got) {
      if (recv == L) break;
      continue;
    }
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
  }
  const long long drift = n_sf ? (long long)(last_start - (int64_t)c->frame_offset - (int64_t)(n_sf - 1) * SF) : 0;
  printf("tracking: subframes %llu locked %llu lost %llu  half-frames %llu locked %llu remeasured %llu  timing moved %lld samples  cfo_hz %.1f\n", n_sf,
         n_locked, n_lost, n_hf, n_hf_locked, n_remeasured, drift, last_cfo);
  printf("subframes %llu  dcis %llu  transport blocks %llu  crc ok %llu\n", n_sf, n_dci, n_tb, n_ok);
  if (reacq) printf("reacquire: finds %llu reacquired %llu awaiting_mib %llu\n", n_finds, n_reacq, n_await);
  fclose(in), fclose(tsv);
  ltephy_pcap_close(pcap);
  ltephy_track_destroy(tr);
  ltephy_search_destroy(search);
  ltephy_destroy(phy);
  if (mibh) ltephy_destroy(mibh);
  return 0;
}
