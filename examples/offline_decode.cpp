// offline_decode.cpp -- the reference's offline mode (LTESniffer -i file.cf32: src/src/LTESniffer_Core.cc:365-444 feeding
// SubframeWorker::work, results to LTESniffer_pcap_writer and DCIToFile) written against the C-ABI of libltephy_b200 from C++,
// the way a maintainer would call it: read a capture in batches, ltephy_decode_subframes, write the MAC-LTE pcap and the
// DCI trace.  Host code only; every computation happens in the library (there is no CPU fallback: without a GPU ltephy_create fails).
//
//   offline_decode <iq.cf32> <nof_prb> <nof_ports> <cell_id> <nof_rx> <out.pcap> <out_dci.tsv> [batch=500] [first_tti=0] [speculate_256qam=0]
//                  [phich_resources=0] [phich_length=0]      (the MIB's PHICH configuration; the reference's file mode presets 1/6, normal)
//                  [fmt=cf32|sc16|sc8]
//
// File layout: subframe after subframe, antenna after antenna, lte sf_len complex samples each (what srsran_filesource_read_multi hands
// SubframeWorker, src/src/SubframeWorker.cc:89): float32 (cf32, the default) or int16 / int8 I/Q pairs (sc16 / sc8), handed to the library as
// read, so the host-to-device copy moves a half or a quarter of the bytes.
#include "cell_chain.h"

int main(int argc, char** argv)
{
  uint32_t fmt = LTEPHY_IQ_CF32;
  if (int r = chain_take_fmt(argc, argv, &fmt)) return r;
  if (argc < 8) {
    fprintf(stderr, "usage: %s <iq.cf32> <nof_prb> <nof_ports> <cell_id> <nof_rx> <out.pcap> <out_dci.tsv> [batch] [first_tti] [speculate_256qam]\n", argv[0]);
    return 2;
  }
  const char*    iq_path = argv[1];
  ltephy_cfg_t   cfg{};
  cfg.nof_prb = (uint32_t)atoi(argv[2]), cfg.nof_ports = (uint32_t)atoi(argv[3]), cfg.cell_id = (uint32_t)atoi(argv[4]), cfg.nof_rx = (uint32_t)atoi(argv[5]);
  const uint32_t B         = argc > 8 ? (uint32_t)atoi(argv[8]) : 500;
  uint32_t       tti       = argc > 9 ? (uint32_t)atoi(argv[9]) : 0;
  const int      speculate = argc > 10 ? atoi(argv[10]) : 0;
  cfg.max_subframes = B, cfg.turbo_max_iter = 8, cfg.flags = LTEPHY_FLAG_SKIP_LOW_POWER, cfg.iq_format = fmt;
  cfg.phich_resources = argc > 11 ? (uint32_t)atoi(argv[11]) : 0, cfg.phich_length = argc > 12 ? (uint32_t)atoi(argv[12]) : 0;

  ltephy_t* phy = nullptr;
  if (ltephy_create(&cfg, &phy) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_create: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_search_t* search = ltephy_search_create(phy, 5); // rnti_histogram_threshold default of the reference
  ltephy_search_speculate_256qam(search, speculate);
  ltephy_pcap_t* pcap = ltephy_pcap_open(argv[6]);
  FILE*          tsv  = fopen(argv[7], "w");
  FILE*          in   = fopen(iq_path, "rb");
  if (!search || !pcap || !tsv || !in) {
    fprintf(stderr, "cannot open inputs / outputs\n");
    return 1;
  }
  const size_t sf_bytes = (size_t)chain_sample_bytes(fmt) * cfg.nof_rx * ltephy_sf_len(phy);
  const uint32_t max_dcis = 32 * B;
  std::vector<uint8_t>             iq(sf_bytes * B);
  std::vector<uint32_t>            ttis(B);
  std::vector<ltephy_sf_info_t>    info(B);
  std::vector<ltephy_cand_t>       scratch((size_t)B * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES);
  std::vector<ltephy_dci_t>        dcis(max_dcis);
  std::vector<ltephy_tb_result_t>  tbs(2 * (size_t)max_dcis);
  std::vector<uint8_t>             payload((size_t)B * 64 * 1024);
  unsigned long long n_sf = 0, n_dci = 0, n_tb = 0, n_ok = 0;
  char               line[256];
  for (;;) {
    const size_t got = fread(iq.data(), sf_bytes, B, in);
    if (!got) break;
    for (size_t i = 0; i < got; i++) ttis[i] = (tti + (uint32_t)i) % 10240;
    uint32_t nd = 0;
    if (ltephy_decode_subframes(phy, search, iq.data(), ttis.data(), (uint32_t)got, LTEPHY_SEQ_NONE, info.data(), scratch.data(), dcis.data(), max_dcis, &nd,
                                tbs.data(), payload.data(), payload.size()) != LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_decode_subframes: %s\n", ltephy_last_error());
      return 1;
    }
    // timestamps: the reference stamps wall-clock time of decoding; an offline run uses capture time (1 ms per subframe)
    for (uint32_t i = 0; i < nd; i++) {
      const uint32_t t = ttis[dcis[i].sf];
      const int      n = ltephy_dci_trace_line(search, &dcis[i], t, info[dcis[i].sf].cfi, tbs[2 * i].crc == 2 || tbs[2 * i + 1].crc == 2, (uint32_t)((n_sf + dcis[i].sf) / 1000),
                                               (uint32_t)(((n_sf + dcis[i].sf) % 1000) * 1000), line, sizeof(line));
      if (n > 0) fwrite(line, 1, (size_t)n, tsv);
      for (int k = 0; k < 2; k++) n_tb += tbs[2 * i + k].payload_len > 0, n_ok += tbs[2 * i + k].crc != 0;
    }
    const int w = ltephy_pcap_write_dl_batch(pcap, ttis.data(), dcis.data(), nd, tbs.data(), payload.data(), 0, (uint32_t)(n_sf / 1000), (uint32_t)((n_sf % 1000) * 1000));
    if (w < 0) {
      fprintf(stderr, "pcap write failed\n");
      return 1;
    }
    n_sf += got, n_dci += nd, tti = (tti + (uint32_t)got) % 10240;
  }
  printf("subframes %llu  dcis %llu  transport blocks %llu  crc ok %llu\n", n_sf, n_dci, n_tb, n_ok);
  fclose(in), fclose(tsv);
  ltephy_pcap_close(pcap);
  ltephy_search_destroy(search);
  ltephy_destroy(phy);
  return 0;
}
