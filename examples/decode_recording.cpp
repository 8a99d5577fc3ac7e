// decode_recording.cpp -- raw recording in, pcap out: a continuous antenna-major recording of any length, as an SDR writes it, decoded
// through the C-ABI of libltephy_b200.  Cell search on the first 40 ms (ltephy_cell_search), the MIB soft-combined over the frames there
// (ltephy_mib_decode_combined), then the tracker (ltephy_track_push) part by part, which follows the frame timing and carrier offset through a
// sampling clock that is off by a few ppm and cuts every subframe into device memory, and ltephy_decode_subframes_device on each cut.  Writes
// the MAC-LTE pcap and the DCI trace exactly as offline_decode does, and prints the cell and a lock summary.  Host code only; without a GPU
// ltephy_sync_create fails.
//
//   decode_recording <iq file> <symbol_sz> <nof_rx> <out.pcap> <out_dci.tsv> [subframes_per_push=500] [max_ppm=50] [no_cfo=0] [reacquire=0]
//                    [fmt=cf32|sc16|sc8]
//
// With reacquire = 1 the tracker searches a lost cell again (LTEPHY_TRACK_REACQUIRE), and the example falls back as the reference does from
// DECODE_PDSCH to DECODE_MIB (src/src/LTESniffer_Core.cc:506-524): from the re-acquired subframe on it decodes nothing and feeds every
// subframe 0 of the cut to the MIB decoder until one passes, then adds (mib.sfn - tti / 10) mod 1024 frames to every later tti, because
// after dropped samples the tracker's SFN, which continues by sample count, is wrong.
//
// File layout: antenna after antenna, each a continuous run of complex samples at 15 kHz * symbol_sz (what cell_search reads): float32 (cf32, the
// default) or int16 / int8 I/Q pairs (sc16 / sc8), which the search and the tracker take as they are.  The file is read one push at a time (one
// seek per antenna), so its length is not limited by host memory.
#include "cell_chain.h"

int main(int argc, char** argv)
{
  uint32_t fmt = LTEPHY_IQ_CF32;
  if (int r = chain_take_fmt(argc, argv, &fmt)) return r;
  if (argc < 6) {
    fprintf(stderr, "usage: %s <iq file> <symbol_sz> <nof_rx> <out.pcap> <out_dci.tsv> [subframes_per_push=500] [max_ppm=50] [no_cfo=0] [reacquire=0] [fmt=cf32|sc16|sc8]\n",
            argv[0]);
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
  const uint32_t b = chain_sample_bytes(fmt);
  const uint64_t L = (uint64_t)ftello(in) / ((uint64_t)b * A);

  // 1. cell search on the first 40 ms, and the MIB soft-combined over the frames there at the found timing, with the found carrier offset
  ltephy_cell_t c{};
  ltephy_mib_t  mib{};
  if (int r = chain_acquire(in, N, A, L, L < 40ull * SF ? L : 40ull * SF, fmt, &c, &mib)) return r;
  chain_print_cell(c, mib);

  // 2. decoder, DCI search and tracker for the cell
  CellChain chain;
  if (chain.open_decoder(c, mib, N, A, B)) return 1;
  ltephy_track_cfg_t tcfg{};
  tcfg.symbol_sz = N, tcfg.nof_rx = A, tcfg.pci = c.pci, tcfg.first_tti = 10 * mib.sfn, tcfg.frame_offset = c.frame_offset, tcfg.cfo_hz = c.cfo_hz;
  tcfg.max_ppm = max_ppm, tcfg.max_subframes = B, tcfg.flags = (no_cfo ? LTEPHY_TRACK_NO_CFO : 0) | (reacq ? LTEPHY_TRACK_REACQUIRE : 0);
  tcfg.iq_format = fmt; // the cut it hands the decoder is cf32 whatever the file holds
  ltephy_track_t* tr = nullptr;
  if (!chain.search || ltephy_track_create(&tcfg, &tr) != LTEPHY_SUCCESS) {
    fprintf(stderr, "search / tracker: %s\n", ltephy_last_error());
    return 1;
  }
  if (chain.open_sinks(mib, reacq, argv[4], argv[5])) return 1;
  // 3. the recording arrives B subframes at a time; each push re-feeds from the tracker's next_sample
  std::vector<uint8_t> x;
  uint64_t             recv = 0, next = c.frame_offset;
  for (;;) {
    if (recv < L) recv = recv + (uint64_t)B * SF < L ? recv + (uint64_t)B * SF : L;
    if (next >= recv) {
      if (recv == L) break;
      continue;
    }
    if (!read_span(in, A, L, b, next, recv - next, x)) {
      fprintf(stderr, "short read\n");
      return 1;
    }
    ltephy_track_out_t o{};
    if (ltephy_track_push(tr, x.data(), next, recv - next, &o) != LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_track_push: %s\n", ltephy_last_error());
      return 1;
    }
    next = o.next_sample;
    if (chain.consume(o)) return 1;
    if (!o.nof_subframes && recv == L) break;
  }
  chain.print_summary();
  fclose(in);
  ltephy_track_destroy(tr);
  chain.close();
  return 0;
}
