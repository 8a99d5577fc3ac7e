// offline_ul.cpp -- the reference's UL mode (LTESniffer -m 1: SubframeWorker's UL branch, src/src/SubframeWorker.cc:236-345, with PDSCH_Decoder::decode_ul_mode
// and PUSCH_Decoder::decode) written against the C-ABI of libltephy_b200 from C++, for two recorded carriers: the downlink capture is searched for DCI-0s and
// Random Access Responses, the uplink capture is decoded with the grants they carry -- 4 subframes after a DCI-0, 6 after a RAR (UlChain of cell_chain.h,
// batch by batch; a grant past a batch is carried into a later one).  Host code only; every computation happens in the library (no CPU fallback: without a
// GPU ltephy_create fails).
//
//   offline_ul <dl file> <ul file> <nof_prb> <nof_ports> <cell_id> <out.pcap> [batch=200] [first_tti=0] [cyclic_shift=0] [group_assignment=0] [hopping_offset=0]
//              [phich_resources=0] [fmt=cf32|sc16|sc8]
//
// dl file: subframe after subframe, one antenna (the UL mode gives the downlink one antenna, README.md:57-58); ul file: the uplink carrier, same framing and
// the same first tti.  Both hold complex float32 samples (cf32, the default) or int16 / int8 I/Q pairs (sc16 / sc8), handed to the library as read.  cyclic_shift / group_assignment / hopping_offset are SIB2's values (ULSchedule::set_config, src/src/ULSchedule.cc:140-158), which the
// reference reads from the air before it starts; here they are arguments.
#include "cell_chain.h"

int main(int argc, char** argv)
{
  uint32_t fmt = LTEPHY_IQ_CF32;
  if (int r = chain_take_fmt(argc, argv, &fmt)) return r;
  if (argc < 7) {
    fprintf(stderr, "usage: %s <dl file> <ul file> <nof_prb> <nof_ports> <cell_id> <out.pcap> [batch] [first_tti] [cyclic_shift] [group_assignment] [hopping_offset] [phich_resources] [fmt=cf32|sc16|sc8]\n",
            argv[0]);
    return 2;
  }
  auto           arg = [&](int i, uint32_t dflt) { return argc > i ? (uint32_t)atoi(argv[i]) : dflt; };
  const uint32_t B = arg(7, 200);
  uint32_t       tti0 = arg(8, 0);
  ltephy_cfg_t   cfg{};
  cfg.nof_prb = (uint32_t)atoi(argv[3]), cfg.nof_ports = (uint32_t)atoi(argv[4]), cfg.cell_id = (uint32_t)atoi(argv[5]), cfg.nof_rx = 1;
  cfg.max_subframes = B, cfg.turbo_max_iter = 8, cfg.flags = LTEPHY_FLAG_SKIP_LOW_POWER, cfg.phich_resources = arg(12, 0);
  cfg.iq_format = fmt;
  UlChain u;
  if (u.open(cfg, ltephy_ul_cfg_t{arg(9, 0), arg(10, 0), 0, 0}, arg(11, 0), argv[6])) return 1;
  FILE *fd = fopen(argv[1], "rb"), *fu = fopen(argv[2], "rb");
  if (!fd || !fu) {
    fprintf(stderr, "cannot open %s / %s\n", argv[1], argv[2]);
    return 1;
  }
  const size_t         sf_bytes = (size_t)chain_sample_bytes(fmt) * ltephy_sf_len(u.dl);
  std::vector<uint8_t> iq_d(sf_bytes * B), iq_u(sf_bytes * B);
  for (;;) {
    const uint32_t got = (uint32_t)fread(iq_d.data(), sf_bytes, B, fd);
    if (!got || fread(iq_u.data(), sf_bytes, got, fu) != got) break;
    for (uint32_t i = 0; i < got; i++) u.ttis[i] = (tti0 + i) % 10240;
    if (u.step(iq_d.data(), iq_u.data(), false, got)) return 1;
    tti0 = (tti0 + got) % 10240;
  }
  printf("subframes %llu  dl blocks %llu  dci0 %llu  rar %llu  ul blocks %llu\n", u.n_sf, u.n_dl_ok, u.n_dci0, u.n_rar, u.n_ul_ok);
  fclose(fd), fclose(fu);
  u.close();
  return 0;
}
