// decode_recording_ul.cpp -- the reference's UL mode (LTESniffer -m 1) on two raw recordings of one radio: channel 0 on the downlink, channel 1 on
// the uplink (src/src/LTESniffer_Core.cc:174-181), the same sample clock and the same first sample.  The downlink file holds one antenna; the uplink
// file holds ul_rx antennas, antenna-major (all of antenna 0, then all of antenna 1), and with ul_rx = 2 the PUSCH is combined over both (DESIGN.md
// §2, "uplink receive diversity").  Both carriers are cut at the
// timing the tracker follows on the downlink PSS (ltephy_track_push_ul: what srsran_ue_sync_zerocopy does to both channels, :365), so a sampling
// clock a few ppm off and a carrier offset do not lose the uplink.  In order:
//   1. cell search and the combined MIB on the first 40 ms of the downlink, as decode_recording does;
//   2. both files pushed part by part through the tracker, which cuts every subframe of both carriers into device memory;
//   3. the downlink cut decoded with ltephy_decode_subframes_device in UL mode (RARs and format 1 / 1A);
//   4. DCI-0s (4 subframes later) and RARs (6 later) turned into PUSCH grants, carrying grants that land in a later push;
//   5. those grants decoded with ltephy_submit_ul_device on the uplink cut (3 to 5: UlChain of cell_chain.h, as in offline_ul);
// and one summary line.  Writes a MAC-LTE pcap with both directions.  Host code only; without a GPU ltephy_sync_create fails.
//
//   decode_recording_ul <dl file> <ul file> <symbol_sz> <out.pcap> [cfo_ratio=1] [ul_offset=0] [cyclic_shift=0] [group_assignment=0]
//                       [hopping_offset=0] [ul_rx=1] [fmt=cf32|sc16|sc8]
//
// cfo_ratio = f_UL / f_DL scales the tracked carrier offset for the uplink (1 applies the downlink's, as srsRAN does); ul_offset is the number of
// samples the uplink subframe starts after the downlink one.  cyclic_shift / group_assignment / hopping_offset are SIB2's values, as for offline_ul.
// ul_rx (1 or 2) is the number of uplink antennas in <ul file>.  fmt is the sample format of both files: complex float32 (the default) or int16 /
// int8 I/Q pairs, which the search and the tracker take as they are (the cuts the decoders read are cf32).
#include "cell_chain.h"

static const uint32_t B = 200; // subframes per push

int main(int argc, char** argv)
{
  uint32_t fmt = LTEPHY_IQ_CF32;
  if (int r = chain_take_fmt(argc, argv, &fmt)) return r;
  if (argc < 5) {
    fprintf(stderr, "usage: %s <dl file> <ul file> <symbol_sz> <out.pcap> [cfo_ratio=1] [ul_offset=0] [cyclic_shift] [group_assignment] [hopping_offset] [ul_rx=1] [fmt=cf32|sc16|sc8]\n",
            argv[0]);
    return 2;
  }
  auto           arg = [&](int i, uint32_t dflt) { return argc > i ? (uint32_t)atoi(argv[i]) : dflt; };
  const uint32_t N = (uint32_t)atoi(argv[3]), SF = 15 * N;
  const double   cfo_ratio = argc > 5 ? atof(argv[5]) : 1.0;
  const int32_t  ul_offset = argc > 6 ? atoi(argv[6]) : 0;
  const uint32_t ul_rx     = arg(10, 1);
  if (ul_rx < 1 || ul_rx > 2) {
    fprintf(stderr, "ul_rx %u: 1 or 2 uplink antennas\n", ul_rx);
    return 2;
  }
  FILE *         fd = fopen(argv[1], "rb"), *fu = fopen(argv[2], "rb");
  if (!fd || !fu) {
    fprintf(stderr, "cannot open %s / %s\n", argv[1], argv[2]);
    return 2;
  }
  fseeko(fd, 0, SEEK_END), fseeko(fu, 0, SEEK_END);
  const uint32_t b  = chain_sample_bytes(fmt);
  const uint64_t Ld = (uint64_t)ftello(fd) / b, Lu = (uint64_t)ftello(fu) / b / ul_rx, L = Ld < Lu ? Ld : Lu; // Lu: samples per UL antenna

  // 1. cell search and the MIB on the first 40 ms of the downlink
  ltephy_cell_t c{};
  ltephy_mib_t  mib{};
  if (int r = chain_acquire(fd, N, 1, Ld, L < 40ull * SF ? L : 40ull * SF, fmt, &c, &mib)) return r;
  chain_print_cell(c, mib);

  // 2. decoders, DCI search in UL mode and the tracker with the uplink; the tracking starts at the first subframe whose UL window is recorded
  ltephy_cfg_t cfg{};
  cfg.nof_prb = mib.nof_prb, cfg.nof_ports = mib.nof_ports, cfg.cell_id = c.pci, cfg.nof_rx = 1, cfg.max_subframes = B, cfg.turbo_max_iter = 8;
  cfg.flags = LTEPHY_FLAG_SKIP_LOW_POWER, cfg.symbol_sz = N, cfg.phich_resources = mib.phich_resources, cfg.phich_length = mib.phich_length;
  cfg.ul_nof_rx = ul_rx;
  UlChain u;
  if (u.open(cfg, ltephy_ul_cfg_t{arg(7, 0), arg(8, 0), 0, 0}, arg(9, 0), argv[4])) return 1;
  uint64_t fo  = c.frame_offset;
  uint32_t tti = 10 * mib.sfn;
  while ((int64_t)fo + ul_offset < 0) fo += SF, tti = (tti + 1) % 10240;
  ltephy_track_cfg_t tcfg{};
  tcfg.symbol_sz = N, tcfg.nof_rx = 1, tcfg.pci = c.pci, tcfg.first_tti = tti, tcfg.frame_offset = fo, tcfg.cfo_hz = c.cfo_hz;
  tcfg.max_ppm = 50.0f, tcfg.max_subframes = B, tcfg.iq_format = fmt;
  ltephy_track_ul_cfg_t tul{};
  tul.cfo_ratio = cfo_ratio, tul.ul_offset = ul_offset, tul.nof_rx = ul_rx; // the UL cut is [got][ul_rx][15 N], what the UL decoder of cfg takes
  ltephy_track_t* tr = nullptr;
  if (ltephy_track_create(&tcfg, &tr) != LTEPHY_SUCCESS || ltephy_track_set_ul(tr, &tul) != LTEPHY_SUCCESS) {
    fprintf(stderr, "tracker: %s\n", ltephy_last_error());
    return 1;
  }
  // 3. the recordings arrive B subframes at a time; each push re-feeds both from the tracker's next_sample
  std::vector<uint8_t> x, xu;
  unsigned long long   n_lost = 0;
  uint64_t             recv = 0, next = (int64_t)fo + ul_offset < (int64_t)fo ? fo + ul_offset : fo;
  for (;;) {
    if (recv < L) recv = recv + (uint64_t)B * SF < L ? recv + (uint64_t)B * SF : L;
    if (next >= recv) {
      if (recv == L) break;
      continue;
    }
    if (!read_span(fd, 1, Ld, b, next, recv - next, x) || !read_span(fu, ul_rx, Lu, b, next, recv - next, xu)) {
      fprintf(stderr, "short read\n");
      return 1;
    }
    ltephy_track_out_t o{};
    const void*        ul_dev = nullptr;
    if (ltephy_track_push_ul(tr, x.data(), xu.data(), next, recv - next, &o, &ul_dev) != LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_track_push_ul: %s\n", ltephy_last_error());
      return 1;
    }
    next = o.next_sample;
    const uint32_t got = o.nof_subframes;
    if (!got) {
      if (recv == L) break;
      continue;
    }
    // 4. the downlink cut decoded in UL mode, its RARs and DCI-0s turned into grants, and the uplink cut decoded where it lies
    for (uint32_t i = 0; i < got; i++) u.ttis[i] = o.sf[i].tti, n_lost += (o.sf[i].flags & LTEPHY_TRACK_LOST) != 0;
    if (u.step(o.iq_dev, ul_dev, true, got)) return 1;
  }
  printf("subframes %llu  lost %llu  dl blocks %llu  dci0 %llu  rar %llu  ul blocks %llu  ul grants beyond the recording %zu\n", u.n_sf, n_lost,
         u.n_dl_ok, u.n_dci0, u.n_rar, u.n_ul_ok, u.carry.size());
  fclose(fd), fclose(fu);
  ltephy_track_destroy(tr);
  u.close();
  return 0;
}
