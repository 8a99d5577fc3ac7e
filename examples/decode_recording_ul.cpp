// decode_recording_ul.cpp -- the reference's UL mode (LTESniffer -m 1) on two raw recordings of one radio: channel 0 on the downlink, channel 1 on
// the uplink (src/src/LTESniffer_Core.cc:174-181), one antenna each, the same sample clock and the same first sample.  Both carriers are cut at the
// timing the tracker follows on the downlink PSS (ltephy_track_push_ul: what srsran_ue_sync_zerocopy does to both channels, :365), so a sampling
// clock a few ppm off and a carrier offset do not lose the uplink.  In order:
//   1. cell search and the combined MIB on the first 40 ms of the downlink, as decode_recording does;
//   2. both files pushed part by part through the tracker, which cuts every subframe of both carriers into device memory;
//   3. the downlink cut decoded with ltephy_decode_subframes_device in UL mode (RARs and format 1 / 1A);
//   4. DCI-0s (4 subframes later) and RARs (6 later) turned into PUSCH grants, carrying grants that land in the next push, as offline_ul does;
//   5. those grants decoded with ltephy_submit_ul_device on the uplink cut;
// and one summary line.  Writes a MAC-LTE pcap with both directions.  Host code only; without a GPU ltephy_sync_create fails.
//
//   decode_recording_ul <dl.cf32> <ul.cf32> <symbol_sz> <out.pcap> [cfo_ratio=1] [ul_offset=0] [cyclic_shift=0] [group_assignment=0]
//                       [hopping_offset=0]
//
// cfo_ratio = f_UL / f_DL scales the tracked carrier offset for the uplink (1 applies the downlink's, as srsRAN does); ul_offset is the number of
// samples the uplink subframe starts after the downlink one.  cyclic_shift / group_assignment / hopping_offset are SIB2's values, as for offline_ul.
#include "ltephy_b200.h"
#include "ltephy_search.h"
#include "ltephy_sinks.h"
#include <cstdio>
#include <cstdlib>
#include <vector>

static const uint32_t B = 200; // subframes per push

// samples [s, s + n) of a one-antenna file
static bool read_span(FILE* f, uint64_t s, uint64_t n, std::vector<float>& out)
{
  out.resize((size_t)2 * n);
  return fseeko(f, (off_t)(8 * s), SEEK_SET) == 0 && fread(out.data(), 8, n, f) == n;
}

int main(int argc, char** argv)
{
  if (argc < 5) {
    fprintf(stderr, "usage: %s <dl.cf32> <ul.cf32> <symbol_sz> <out.pcap> [cfo_ratio=1] [ul_offset=0] [cyclic_shift] [group_assignment] [hopping_offset]\n",
            argv[0]);
    return 2;
  }
  auto           arg = [&](int i, uint32_t dflt) { return argc > i ? (uint32_t)atoi(argv[i]) : dflt; };
  const uint32_t N = (uint32_t)atoi(argv[3]), SF = 15 * N;
  const double   cfo_ratio = argc > 5 ? atof(argv[5]) : 1.0;
  const int32_t  ul_offset = argc > 6 ? atoi(argv[6]) : 0;
  FILE *         fd = fopen(argv[1], "rb"), *fu = fopen(argv[2], "rb");
  if (!fd || !fu) {
    fprintf(stderr, "cannot open %s / %s\n", argv[1], argv[2]);
    return 2;
  }
  fseeko(fd, 0, SEEK_END), fseeko(fu, 0, SEEK_END);
  const uint64_t Ld = (uint64_t)ftello(fd) / 8, Lu = (uint64_t)ftello(fu) / 8, L = Ld < Lu ? Ld : Lu;

  // 1. cell search and the MIB on the first 40 ms of the downlink
  const uint64_t     L0 = L < 40ull * SF ? L : 40ull * SF;
  std::vector<float> x, xu;
  ltephy_sync_cfg_t  scfg{};
  scfg.symbol_sz = N, scfg.nof_rx = 1, scfg.max_samples = L0;
  ltephy_sync_t* sync = nullptr;
  ltephy_cell_t  cells[3];
  if (!read_span(fd, 0, L0, x)) {
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
  const uint32_t nframes = (uint32_t)((L0 - c->frame_offset) / (10ull * SF));
  if (!nframes) {
    fprintf(stderr, "no whole frame after the first subframe 0\n");
    return 3;
  }
  std::vector<float>    sf0((size_t)2 * SF * nframes);
  std::vector<uint32_t> tti0(nframes);
  for (uint32_t f = 0; f < nframes; f++) {
    tti0[f] = 10 * f;
    for (uint32_t n = 0; n < 2 * SF; n++) sf0[(size_t)2 * f * SF + n] = x[2 * (c->frame_offset + (uint64_t)f * 10 * SF) + n];
  }
  ltephy_cfg_t mcfg{};
  mcfg.nof_prb = 15, mcfg.nof_ports = 2, mcfg.cell_id = c->pci, mcfg.nof_rx = 1, mcfg.max_subframes = nframes, mcfg.symbol_sz = N;
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
      mib.sfn = (mib.sfn + 1024 - f % 1024) % 1024;
    }
  if (!mib.found) {
    fprintf(stderr, "cell %u found, MIB not decoded\n", c->pci);
    return 3;
  }
  printf("pci %u frame_offset %llu cfo_hz %.9g nof_prb %u nof_ports %u phich_resources %u phich_length %u sfn %u\n", c->pci,
         (unsigned long long)c->frame_offset, c->cfo_hz, mib.nof_prb, mib.nof_ports, mib.phich_resources, mib.phich_length, mib.sfn);

  // 2. decoders, DCI search in UL mode and the tracker with the uplink; the tracking starts at the first subframe whose UL window is recorded
  ltephy_cfg_t cfg{};
  cfg.nof_prb = mib.nof_prb, cfg.nof_ports = mib.nof_ports, cfg.cell_id = c->pci, cfg.nof_rx = 1, cfg.max_subframes = B, cfg.turbo_max_iter = 8;
  cfg.flags = LTEPHY_FLAG_SKIP_LOW_POWER, cfg.symbol_sz = N, cfg.phich_resources = mib.phich_resources, cfg.phich_length = mib.phich_length;
  ltephy_t *dl = nullptr, *ul = nullptr;
  if (ltephy_create(&cfg, &dl) != LTEPHY_SUCCESS || ltephy_create(&cfg, &ul) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_create: %s\n", ltephy_last_error());
    return 1;
  }
  const ltephy_ul_cfg_t ucfg{arg(7, 0), arg(8, 0), 0, 0};
  ltephy_search_t*      search = ltephy_search_create(dl, 5);
  if (ltephy_set_ul_cfg(ul, &ucfg) != LTEPHY_SUCCESS || !search) {
    fprintf(stderr, "UL config / search: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_search_set_ul_hopping(search, arg(9, 0));
  ltephy_search_set_ul_mode(search, 1, 0);
  uint64_t fo  = c->frame_offset;
  uint32_t tti = 10 * mib.sfn;
  while ((int64_t)fo + ul_offset < 0) fo += SF, tti = (tti + 1) % 10240;
  ltephy_track_cfg_t tcfg{};
  tcfg.symbol_sz = N, tcfg.nof_rx = 1, tcfg.pci = c->pci, tcfg.first_tti = tti, tcfg.frame_offset = fo, tcfg.cfo_hz = c->cfo_hz;
  tcfg.max_ppm = 50.0f, tcfg.max_subframes = B;
  ltephy_track_ul_cfg_t tul{};
  tul.cfo_ratio = cfo_ratio, tul.ul_offset = ul_offset;
  ltephy_track_t* tr = nullptr;
  if (ltephy_track_create(&tcfg, &tr) != LTEPHY_SUCCESS || ltephy_track_set_ul(tr, &tul) != LTEPHY_SUCCESS) {
    fprintf(stderr, "tracker: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_pcap_t* pcap = ltephy_pcap_open(argv[4]);
  if (!pcap) {
    fprintf(stderr, "cannot open %s\n", argv[4]);
    return 1;
  }
  const uint32_t                  max_dcis = 32 * B, max_ul = 3 * max_dcis + 64;
  std::vector<uint32_t>           ttis(B);
  std::vector<ltephy_sf_info_t>   info(B);
  std::vector<ltephy_cand_t>      scratch((size_t)B * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES);
  std::vector<ltephy_dci_t>       dcis(max_dcis);
  std::vector<ltephy_tb_result_t> tbs(2 * (size_t)max_dcis), ures(max_ul);
  std::vector<uint8_t>            payload((size_t)B * 64 * 1024), upayload((size_t)B * 64 * 1024);
  std::vector<ltephy_ul_grant_t>  grants(max_ul), now, carry; // carry: grants whose subframe lies in the next push
  std::vector<uint32_t>           grant_dci(max_ul);
  std::vector<uint8_t>            reading(max_ul);
  std::vector<ltephy_ul_chest_t>  chest(max_ul);
  unsigned long long              n_sf = 0, n_dci0 = 0, n_rar = 0, n_ul_ok = 0, n_dl_ok = 0, n_lost = 0;
  // 3. the recordings arrive B subframes at a time; each push re-feeds both from the tracker's next_sample
  uint64_t recv = 0, next = (int64_t)fo + ul_offset < (int64_t)fo ? fo + ul_offset : fo;
  for (;;) {
    if (recv < L) recv = recv + (uint64_t)B * SF < L ? recv + (uint64_t)B * SF : L;
    if (next >= recv) {
      if (recv == L) break;
      continue;
    }
    if (!read_span(fd, next, recv - next, x) || !read_span(fu, next, recv - next, xu)) {
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
    for (uint32_t i = 0; i < got; i++) ttis[i] = o.sf[i].tti, n_lost += (o.sf[i].flags & LTEPHY_TRACK_LOST) != 0;
    uint32_t nd = 0;
    if (ltephy_decode_subframes_device(dl, search, o.iq_dev, ttis.data(), got, LTEPHY_SEQ_NONE, info.data(), scratch.data(), dcis.data(), max_dcis, &nd,
                                       tbs.data(), payload.data(), payload.size()) != LTEPHY_SUCCESS) {
      fprintf(stderr, "ltephy_decode_subframes_device: %s\n", ltephy_last_error());
      return 1;
    }
    const uint32_t ts_s = (uint32_t)(n_sf / 1000), ts_us = (uint32_t)((n_sf % 1000) * 1000);
    const int      wd   = ltephy_pcap_write_dl_batch(pcap, ttis.data(), dcis.data(), nd, tbs.data(), payload.data(), 0, ts_s, ts_us);
    if (wd < 0) return 1;
    n_dl_ok += (unsigned)wd;
    // 4. grants of this push's uplink: what the previous push left over, the msg-3 grants of the RARs (6 subframes later), the DCI-0s (4 later).
    //    A carried grant can land beyond a short push (the last one of the recording): it stays carried.
    now.swap(carry), carry.clear();
    {
      size_t w = 0;
      for (size_t k = 0; k < now.size(); k++) {
        if (now[k].sf < got)
          now[w++] = now[k];
        else
          carry.push_back(now[k]);
      }
      now.resize(w);
    }
    for (uint32_t i = 0; i < nd; i++) {
      const ltephy_tb_result_t& r = tbs[2 * i];
      if (dcis[i].rnti < 1 || dcis[i].rnti > 10 || !r.crc || !r.payload_len) continue; // RA-RNTI with a decoded block
      ltephy_rar_t rars[16];
      uint32_t     nr = 0;
      if (ltephy_rar_unpack(search, payload.data() + r.payload_off, r.payload_len, rars, 16, &nr, nullptr) != LTEPHY_SUCCESS) continue;
      for (uint32_t k = 0; k < nr; k++) {
        ltephy_search_activate(search, rars[k].t_crnti, 0, LTEPHY_ACT_RAR);
        n_rar++;
        if (!rars[k].valid) continue;
        rars[k].grant.sf = dcis[i].sf + 6;
        (rars[k].grant.sf < got ? now : carry).push_back(rars[k].grant);
      }
    }
    uint32_t ng = 0;
    if (ltephy_ul_grants_from_dcis(search, info.data(), dcis.data(), nd, nullptr, 0, grants.data(), grant_dci.data(), reading.data(), max_ul, &ng) != LTEPHY_SUCCESS)
      return 1;
    for (uint32_t k = 0; k < ng; k++) {
      n_dci0 += k == 0 || grant_dci[k] != grant_dci[k - 1];
      (grants[k].sf < got ? now : carry).push_back(grants[k]);
    }
    for (ltephy_ul_grant_t& g : carry) g.sf -= got; // index into the next push's uplink
    // 5. the uplink cut, decoded where it lies
    if (!now.empty()) {
      if (now.size() > max_ul) now.resize(max_ul);
      if (ltephy_submit_ul_device(ul, ul_dev, ttis.data(), got, now.data(), (uint32_t)now.size()) != LTEPHY_SUCCESS ||
          ltephy_get_ul(ul, ures.data(), chest.data(), upayload.data(), upayload.size()) != LTEPHY_SUCCESS) {
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
      if (wu < 0) return 1;
      n_ul_ok += (unsigned)wu;
    }
    n_sf += got;
  }
  printf("subframes %llu  lost %llu  dl blocks %llu  dci0 %llu  rar %llu  ul blocks %llu  ul grants beyond the recording %zu\n", n_sf, n_lost, n_dl_ok,
         n_dci0, n_rar, n_ul_ok, carry.size());
  fclose(fd), fclose(fu);
  ltephy_pcap_close(pcap);
  ltephy_track_destroy(tr);
  ltephy_search_destroy(search);
  ltephy_destroy(dl), ltephy_destroy(ul);
  return 0;
}
