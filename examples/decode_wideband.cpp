// decode_wideband.cpp -- one wideband recording in, one pcap per carrier out: a continuous antenna-major capture (cf32, sc16 or sc8) at any rate
// fs_in that holds one or several LTE carriers, decoded through the C-ABI of libltephy_b200.  The capture is read one span at a time and the
// channeliser (ltephy_chan_run, LTEPHY_CHAN_RATIONAL set) shifts, filters and resamples every carrier of the span to 15 kHz * N in one call.  Per carrier the chain of decode_recording follows on the carrier
// stream in device memory: cell search on its first 40 ms (ltephy_cell_search_device), the tracker (ltephy_track_push_device), the MIB
// soft-combined over the subframes 0 of the tracker's first cut, then ltephy_decode_subframes_device (cell_chain.h).  Host code only; without a
// GPU ltephy_chan_create fails.
//
//   decode_wideband <iq file> <fs_in> <nof_rx> <out_prefix> <offset_hz>:<N> [<offset_hz>:<N> ...] [subframes_per_push=500] [fmt=cf32|sc16|sc8]
//   decode_wideband <iq file> <fs_in> <nof_rx> <out_prefix> scan=<center_hz> [subframes_per_push=500] [fmt=cf32|sc16|sc8]
//
// scan=<center_hz> (the capture's absolute centre, a multiple of 1 kHz) takes the place of the carrier list: the raster scan (ltephy_scan_run)
// of the first 40 ms finds the cells.  For each reported offset the strongest cell's MIB is read on an N = 256 stream of that offset, as a
// listed carrier's is (cell search, the tracker's cut, ltephy_mib_decode_combined with LTEPHY_MIB_SEARCH_PORTS on a 15-PRB handle); the
// smallest N whose PRB count covers the MIB's nof_prb makes the carrier, and those carriers, by offset ascending, are decoded exactly as the
// same <offset_hz>:<N> list would be.  One "scan" line per reported cell: offset, PCI, psr, and its MIB or why it is not decoded (6 PRB, no MIB,
// a second cell at the offset, more than LTEPHY_CHAN_MAX_CARRIERS carriers).
//
// A single-carrier capture at any rate, e.g. a 20 Msps sc16 recording of a 20 MHz cell, decodes with the one carrier 0:2048.
// Carrier c writes <out_prefix>_<c>.pcap and <out_prefix>_<c>.tsv and prints, in carrier order, a "carrier" line, then the cell line and the
// summary lines in decode_recording's format.  The tracker starts at tti 0 on the cell search's frame timing; the MIB read from its cut gives the
// SFN, added to every tti from then on.  Subframes cut before the first push whose subframes 0 pass the MIB are not decoded.  Each span of the
// capture starts at the lowest sample any carrier's tracker still needs, so every carrier's output starts at or before what its tracker needs:
// carrier sample s needs capture samples from floor(s M / L) - Ka (ltephy_chan_design).
#include "cell_chain.h"
#include <algorithm>
#include <cstring>
#include <string>

struct Carrier {
  int32_t         offset_hz = 0;
  uint32_t        N = 0, SF = 0;
  uint32_t        Lr = 1, Mr = 1, Ka = 0; // output / capture rate L / M, and the taps before an output's own sample (ltephy_chan_design)
  bool            found = false, mib_found = false;
  ltephy_cell_t   cell{};
  ltephy_mib_t    mib{};
  ltephy_track_t* tr   = nullptr;
  ltephy_t*       mibh = nullptr; // MIB decoder on the tracker's cut (no port count known yet: searched)
  uint64_t        next = 0;       // the tracker's next_sample, in carrier samples
  CellChain       chain;
};

// The per-carrier chain on carriers car of the capture in (L samples per antenna): channeliser, cell search on the first 40 ms, tracker, MIB,
// decode.  With probe set, only the MIB is read: no decoder, no output, and a carrier stops at its MIB (or the capture at its first second).
// 0, 1 on an error of the library or the file, 2 for a carrier the channeliser refuses, 3 when a carrier had no cell or no MIB (not with probe).
static int run_carriers(FILE* in, uint32_t fs, uint32_t A, uint32_t fmt, uint64_t L, uint32_t B, const std::string& prefix, std::vector<Carrier>& car,
                        bool probe)
{
  const uint32_t bps = chain_sample_bytes(fmt);
  const uint64_t MS  = fs / 1000; // capture samples per ms
  ltephy_chan_cfg_t ccfg{};
  ccfg.fs_in = fs, ccfg.nof_rx = A, ccfg.nof_carriers = (uint32_t)car.size(), ccfg.flags = LTEPHY_CHAN_RATIONAL, ccfg.iq_format = fmt;
  for (size_t c = 0; c < car.size(); c++) ccfg.carrier[c].offset_hz = car[c].offset_hz, ccfg.carrier[c].symbol_sz = car[c].N;
  uint32_t reach = 0; // the longest filter window in capture samples (T of an integer carrier)
  for (size_t c = 0; c < car.size(); c++) {
    ltephy_chan_poly_t q;
    if (ltephy_chan_design(&ccfg, (uint32_t)c, &q, nullptr, nullptr, nullptr) != LTEPHY_SUCCESS) {
      fprintf(stderr, "carrier %zu: %s\n", c, ltephy_last_error());
      return 2;
    }
    car[c].Lr = q.L, car[c].Mr = q.M, car[c].Ka = q.Ka, reach = std::max(reach, q.Kp);
  }
  // 1. the first 40 ms of every carrier (and the filter's reach past them) in one call; cell search on each carrier stream
  const uint64_t L0   = std::min<uint64_t>(L, 40 * MS + reach);
  const uint64_t span = std::min<uint64_t>(L, std::max<uint64_t>(L0, (uint64_t)(B + 20) * MS));
  ccfg.max_samples    = span;
  ltephy_chan_t* ch   = nullptr;
  if (ltephy_chan_create(&ccfg, &ch) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_chan_create: %s\n", ltephy_last_error());
    return 1;
  }
  std::vector<uint8_t>           x;
  std::vector<ltephy_chan_out_t> out(car.size());
  uint64_t                       nx = 0;
  if (!read_span(in, A, L, bps, 0, L0, x)) {
    fprintf(stderr, "short read\n");
    return 1;
  }
  if (ltephy_chan_run(ch, x.data(), 0, L0, out.data(), &nx) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_chan_run: %s\n", ltephy_last_error());
    return 1;
  }
  int status = 0;
  for (size_t c = 0; c < car.size(); c++) {
    Carrier&          k = car[c];
    ltephy_sync_cfg_t scfg{};
    scfg.symbol_sz = k.N, scfg.nof_rx = A, scfg.max_samples = out[c].count;
    ltephy_sync_t* sync = nullptr;
    ltephy_cell_t  cells[3];
    if (out[c].count < 75ull * k.N + k.N) {
      fprintf(stderr, "carrier %zu: capture shorter than a half-frame\n", c);
      status = 3;
      continue;
    }
    if (ltephy_sync_create(&scfg, &sync) != LTEPHY_SUCCESS || ltephy_cell_search_device(sync, out[c].iq_dev, out[c].count, cells) != LTEPHY_SUCCESS) {
      fprintf(stderr, "cell search: %s\n", ltephy_last_error());
      return 1;
    }
    ltephy_sync_destroy(sync);
    for (auto& q : cells)
      if (q.detected) {
        k.cell = q, k.found = true;
        break;
      }
    if (!k.found) {
      fprintf(stderr, "carrier %zu: no cell found\n", c);
      status = 3;
      continue;
    }
    // 2. the tracker from tti 0 at the found timing, and a MIB decoder for the subframes 0 of its cut
    ltephy_track_cfg_t tcfg{};
    tcfg.symbol_sz = k.N, tcfg.nof_rx = A, tcfg.pci = k.cell.pci, tcfg.first_tti = 0, tcfg.frame_offset = k.cell.frame_offset, tcfg.cfo_hz = k.cell.cfo_hz;
    tcfg.max_ppm = 50.0f, tcfg.max_subframes = B;
    ltephy_cfg_t mcfg{};
    mcfg.nof_prb = 15, mcfg.nof_ports = 2, mcfg.cell_id = k.cell.pci, mcfg.nof_rx = A, mcfg.max_subframes = 1, mcfg.symbol_sz = k.N;
    if (ltephy_track_create(&tcfg, &k.tr) != LTEPHY_SUCCESS || ltephy_create(&mcfg, &k.mibh) != LTEPHY_SUCCESS) {
      fprintf(stderr, "tracker / MIB decoder: %s\n", ltephy_last_error());
      return 1;
    }
    k.next = k.cell.frame_offset;
  }
  // 3. the capture one span at a time, from the lowest sample any tracker still needs; every carrier's cut through its chain
  uint64_t recv = 0;
  for (;;) {
    if (recv < L) recv = recv + (uint64_t)B * MS < L ? recv + (uint64_t)B * MS : L;
    uint64_t first = UINT64_MAX;
    for (auto& k : car)
      if (k.tr) {
        const uint64_t n = (uint64_t)(((unsigned __int128)k.next * k.Mr) / k.Lr); // capture sample of carrier sample next
        first            = std::min(first, n > k.Ka ? n - k.Ka : 0);
      }
    if (first == UINT64_MAX || (probe && recv >= std::min<uint64_t>(L, 1000 * MS))) break;
    if (first >= recv) {
      if (recv == L) break;
      continue;
    }
    const uint64_t end = std::min(recv, first + span);
    if (!read_span(in, A, L, bps, first, end - first, x)) {
      fprintf(stderr, "short read\n");
      return 1;
    }
    if (ltephy_chan_run(ch, x.data(), first, end - first, out.data(), &nx) != LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_chan_run: %s\n", ltephy_last_error());
      return 1;
    }
    bool any = false;
    for (size_t c = 0; c < car.size(); c++) {
      Carrier& k = car[c];
      if (!k.tr || !out[c].count) continue;
      ltephy_track_out_t o{};
      if (ltephy_track_push_device(k.tr, out[c].iq_dev, out[c].first, out[c].count, &o) != LTEPHY_SUCCESS) {
        fprintf(stderr, "ltephy_track_push_device: %s\n", ltephy_last_error());
        return 1;
      }
      k.next = o.next_sample;
      any    = any || o.nof_subframes > 0;
      if (!k.mib_found) {
        const size_t sf_bytes = (size_t)A * k.SF * 8;
        for (uint32_t i = 0; i < o.nof_subframes && !k.mib_found; i++) {
          if (o.sf[i].tti % 10) continue;
          ltephy_mib_comb_t mc{};
          if (ltephy_submit_iq_device(k.mibh, static_cast<const char*>(o.iq_dev) + i * sf_bytes, &o.sf[i].tti, 1) != LTEPHY_SUCCESS ||
              ltephy_mib_decode_combined(k.mibh, LTEPHY_MIB_SEARCH_PORTS, &mc) != LTEPHY_SUCCESS) {
            fprintf(stderr, "MIB decode: %s\n", ltephy_last_error());
            return 1;
          }
          if (!mc.mib.found) continue;
          k.mib = mc.mib, k.mib_found = true;
          k.mib.sfn = (mc.mib.sfn + 1024 - o.sf[i].tti / 10 % 1024) % 1024; // the SFN of the frame at frame_offset
          if (probe) break;
          const std::string base = prefix + "_" + std::to_string(c);
          if (k.chain.open_decoder(k.cell, k.mib, k.N, A, B) || !k.chain.search || k.chain.open_sinks(k.mib, 0, (base + ".pcap").c_str(), (base + ".tsv").c_str()))
            return 1;
          k.chain.sfn_corr = k.mib.sfn;
        }
        if (!k.mib_found) continue;
        if (probe) { // its MIB is all this carrier was read for
          ltephy_track_destroy(k.tr), k.tr = nullptr;
          continue;
        }
      }
      if (k.chain.consume(o)) return 1;
    }
    if (!any && recv == L) break;
  }
  for (size_t c = 0; c < car.size(); c++) {
    Carrier& k = car[c];
    if (!probe) {
      printf("carrier %zu offset_hz %d symbol_sz %u\n", c, k.offset_hz, k.N);
      if (k.found && k.mib_found) {
        chain_print_cell(k.cell, k.mib);
        k.chain.print_summary();
      } else {
        printf(k.found ? "cell %u found, MIB not decoded\n" : "no cell found\n", k.cell.pci);
        status = 3;
      }
    }
    k.chain.close();
    if (k.tr) ltephy_track_destroy(k.tr);
    if (k.mibh) ltephy_destroy(k.mibh);
  }
  ltephy_chan_destroy(ch);
  return status;
}

// the smallest symbol size whose PRB count covers nof_prb (the channeliser's N -> PRB table), 0 for none
static uint32_t symbol_size_for(uint32_t nof_prb)
{
  static const uint32_t N[] = {128, 256, 384, 768, 1536}, PRB[] = {6, 15, 25, 50, 100};
  for (int i = 0; i < 5; i++)
    if (PRB[i] >= nof_prb) return N[i];
  return 0;
}

// scan=<center_hz>: the raster scan of the first 40 ms, the MIB of the strongest cell of every reported offset on an N = 256 stream, one scan
// line per reported cell, and into car the carriers to decode, by offset ascending.  0, 1 on an error of the library or the file, 2 for a
// configuration the scan refuses.
static int scan_carriers(FILE* in, uint32_t fs, uint32_t A, uint32_t fmt, uint64_t L, uint64_t center, uint32_t B, std::vector<Carrier>& car)
{
  ltephy_scan_cfg_t cfg{};
  cfg.fs_in = fs, cfg.nof_rx = A, cfg.iq_format = fmt, cfg.center_hz = center, cfg.max_samples = std::min<uint64_t>(L, 40ull * (fs / 1000));
  uint32_t       np = 0, nc = 0;
  ltephy_scan_t* sc = nullptr;
  int r = ltephy_scan_plan(&cfg, nullptr, 0, &np);
  if (r == LTEPHY_SUCCESS) r = ltephy_scan_create(&cfg, &sc);
  if (r != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_scan_create: %s\n", ltephy_last_error());
    return r == LTEPHY_ERROR_INVALID_INPUTS ? 2 : 1;
  }
  std::vector<uint8_t>            x;
  std::vector<ltephy_scan_cell_t> cells(3 * (size_t)np);
  if (!read_span(in, A, L, chain_sample_bytes(fmt), 0, cfg.max_samples, x)) {
    fprintf(stderr, "short read\n");
    return 1;
  }
  r = ltephy_scan_run(sc, x.data(), cfg.max_samples, cells.data(), (uint32_t)cells.size(), &nc);
  ltephy_scan_destroy(sc);
  if (r != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_scan_run: %s\n", ltephy_last_error());
    return 1;
  }
  cells.resize(nc);
  // one N = 256 carrier per reported offset whose N = 256 band fits the capture, LTEPHY_CHAN_MAX_CARRIERS to a channeliser handle
  std::vector<Carrier> probe;
  for (const auto& c : cells) {
    if (!probe.empty() && probe.back().offset_hz == c.offset_hz) continue;
    ltephy_chan_cfg_t ccfg{};
    ltephy_chan_poly_t q;
    ccfg.fs_in = fs, ccfg.nof_rx = A, ccfg.nof_carriers = 1, ccfg.flags = LTEPHY_CHAN_RATIONAL, ccfg.carrier[0].offset_hz = c.offset_hz, ccfg.carrier[0].symbol_sz = 256;
    if (ltephy_chan_design(&ccfg, 0, &q, nullptr, nullptr, nullptr) != LTEPHY_SUCCESS) continue;
    Carrier k;
    k.offset_hz = c.offset_hz, k.N = 256, k.SF = 15 * 256;
    probe.push_back(std::move(k));
  }
  for (size_t g = 0; g < probe.size(); g += LTEPHY_CHAN_MAX_CARRIERS) {
    std::vector<Carrier> part(std::make_move_iterator(probe.begin() + g),
                              std::make_move_iterator(probe.begin() + std::min<size_t>(probe.size(), g + LTEPHY_CHAN_MAX_CARRIERS)));
    const int s = run_carriers(in, fs, A, fmt, L, B, "", part, true);
    if (s == 1 || s == 2) return s;
    for (size_t i = 0; i < part.size(); i++) probe[g + i].mib_found = part[i].mib_found, probe[g + i].mib = part[i].mib;
  }
  for (size_t i = 0; i < cells.size(); i++) {
    const ltephy_scan_cell_t& c = cells[i];
    printf("scan offset_hz %d pci %u psr %.3f ", c.offset_hz, c.cell.pci, c.cell.psr);
    const Carrier* k = nullptr;
    for (const auto& p : probe)
      if (p.offset_hz == c.offset_hz) k = &p;
    const uint32_t N = k && k->mib_found ? symbol_size_for(k->mib.nof_prb) : 0;
    ltephy_chan_cfg_t  ccfg{};
    ltephy_chan_poly_t q;
    ccfg.fs_in = fs, ccfg.nof_rx = A, ccfg.nof_carriers = 1, ccfg.flags = LTEPHY_CHAN_RATIONAL, ccfg.carrier[0].offset_hz = c.offset_hz, ccfg.carrier[0].symbol_sz = N;
    if (i > 0 && cells[i - 1].offset_hz == c.offset_hz) {
      printf("not decoded: a stronger cell at this offset\n");
      continue;
    }
    if (!k || !k->mib_found) {
      printf("not decoded: no MIB\n");
      continue;
    }
    printf("nof_prb %u nof_ports %u ", k->mib.nof_prb, k->mib.nof_ports);
    if (k->mib.nof_prb <= 6)
      printf("not decoded: %u PRB\n", k->mib.nof_prb);
    else if (!N || ltephy_chan_design(&ccfg, 0, &q, nullptr, nullptr, nullptr) != LTEPHY_SUCCESS)
      printf("not decoded: no symbol size for it inside the capture\n");
    else if (car.size() == LTEPHY_CHAN_MAX_CARRIERS)
      printf("not decoded: more than %d carriers\n", LTEPHY_CHAN_MAX_CARRIERS);
    else {
      printf("carrier %zu symbol_sz %u\n", car.size(), N);
      Carrier d;
      d.offset_hz = c.offset_hz, d.N = N, d.SF = 15 * N;
      car.push_back(std::move(d));
    }
  }
  return 0;
}

int main(int argc, char** argv)
{
  uint32_t fmt = LTEPHY_IQ_CF32;
  if (int r = chain_take_fmt(argc, argv, &fmt)) return r;
  if (argc < 6) {
    fprintf(stderr,
            "usage: %s <iq file> <fs_in> <nof_rx> <out_prefix> <offset_hz>:<N> [<offset_hz>:<N> ...] | scan=<center_hz> [subframes_per_push=500] "
            "[fmt=cf32|sc16|sc8]\n",
            argv[0]);
    return 2;
  }
  const uint32_t       fs = (uint32_t)strtoul(argv[2], nullptr, 10), A = (uint32_t)atoi(argv[3]);
  const std::string    prefix = argv[4];
  std::vector<Carrier> car;
  uint32_t             B = 500;
  bool                 scan = false;
  uint64_t             center = 0;
  for (int i = 5; i < argc; i++) {
    if (!strncmp(argv[i], "scan=", 5)) {
      scan = true, center = strtoull(argv[i] + 5, nullptr, 10);
      continue;
    }
    const char* colon = strchr(argv[i], ':');
    if (!colon) {
      B = (uint32_t)atoi(argv[i]);
      continue;
    }
    Carrier k;
    k.offset_hz = (int32_t)strtol(argv[i], nullptr, 10), k.N = (uint32_t)atoi(colon + 1), k.SF = 15 * k.N;
    car.push_back(std::move(k));
  }
  FILE* in = fopen(argv[1], "rb");
  if (!in || A < 1 || A > 2 || B < 1 || car.empty() == !scan || car.size() > LTEPHY_CHAN_MAX_CARRIERS || fs % 1000) {
    fprintf(stderr, "cannot open %s / bad nof_rx, carriers (or scan= instead of them), fs_in or subframes_per_push\n", argv[1]);
    return 2;
  }
  const uint64_t L = [&] {
    fseeko(in, 0, SEEK_END);
    return (uint64_t)ftello(in) / ((uint64_t)chain_sample_bytes(fmt) * A);
  }();
  int status = scan ? scan_carriers(in, fs, A, fmt, L, center, B, car) : 0;
  if (status == 0) status = car.empty() ? 3 : run_carriers(in, fs, A, fmt, L, B, prefix, car, false);
  fclose(in);
  return status;
}
