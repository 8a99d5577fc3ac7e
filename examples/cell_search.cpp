// cell_search.cpp -- what a recording needs before offline_decode can read it: find the cell in a continuous cf32 capture with
// ltephy_cell_search (PCI, frame timing, carrier offset), then decode its MIB (bandwidth, ports, PHICH, SFN) at that timing with the
// offset corrected, the PSS / SSS search and MIB decode of rf_search_and_decode_mib (reference src/src/LTESniffer_Core.cc:193-204).  The MIB is
// decoded with soft combining across the 40 ms period and a search over the port count, over every frame of the capture.
// Host code only; without a GPU ltephy_sync_create fails.
//
//   cell_search <iq.cf32> <symbol_sz> <nof_rx>
//
// File layout: antenna after antenna, each a continuous run of complex float32 samples at 15 kHz * symbol_sz.  Prints one line:
//   pci <pci> frame_offset <samples> cfo_hz <Hz> nof_prb <n> nof_ports <n> phich_resources <r> phich_length <l> sfn <sfn>
// where frame_offset is the first sample of a subframe 0 and sfn that frame's number: offline_decode takes the file from there on,
// with first_tti = 10 * sfn, after the carrier offset is removed.
#include "ltephy_b200.h"
#include <cstdio>
#include <cstdlib>
#include <vector>

int main(int argc, char** argv)
{
  if (argc < 4) {
    fprintf(stderr, "usage: %s <iq.cf32> <symbol_sz> <nof_rx>\n", argv[0]);
    return 2;
  }
  const uint32_t N = (uint32_t)atoi(argv[2]), A = (uint32_t)atoi(argv[3]);
  FILE*          in = fopen(argv[1], "rb");
  if (!in || A < 1 || A > 2) {
    fprintf(stderr, "cannot open %s / bad nof_rx\n", argv[1]);
    return 2;
  }
  fseek(in, 0, SEEK_END);
  const uint64_t L = (uint64_t)ftell(in) / (8ull * A);
  fseek(in, 0, SEEK_SET);
  std::vector<float> iq((size_t)2 * A * L);
  if (fread(iq.data(), 8, (size_t)A * L, in) != (size_t)A * L) {
    fprintf(stderr, "short read\n");
    return 1;
  }
  fclose(in);

  ltephy_sync_cfg_t scfg{};
  scfg.symbol_sz = N, scfg.nof_rx = A, scfg.max_samples = L;
  ltephy_sync_t* sync = nullptr;
  if (ltephy_sync_create(&scfg, &sync) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_sync_create: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_cell_t cells[3];
  if (ltephy_cell_search(sync, iq.data(), L, cells) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_cell_search: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_sync_destroy(sync);
  const ltephy_cell_t* c = nullptr;
  for (auto& x : cells)
    if (x.detected) {
      c = &x;
      break;
    }
  if (!c) {
    fprintf(stderr, "no cell found\n");
    return 3;
  }

  // the PBCH and the centre CRS do not depend on the bandwidth: a 15-PRB handle with the found PCI reads the MIB of any cell
  const uint32_t sf_len = 15 * N, nframes = (uint32_t)((L - c->frame_offset) / (10ull * sf_len));
  if (!nframes) {
    fprintf(stderr, "no whole frame after the first subframe 0\n");
    return 3;
  }
  std::vector<float>    sf((size_t)2 * A * sf_len * nframes);
  std::vector<uint32_t> tti(nframes);
  for (uint32_t f = 0; f < nframes; f++) { // subframe 0 of each frame, antenna after antenna
    tti[f] = 10 * f;
    for (uint32_t a = 0; a < A; a++)
      for (uint64_t n = 0; n < sf_len; n++) {
        const uint64_t s = c->frame_offset + (uint64_t)f * 10 * sf_len + n;
        const size_t   d = ((size_t)f * A + a) * sf_len + n;
        sf[2 * d] = iq[2 * (a * L + s)], sf[2 * d + 1] = iq[2 * (a * L + s) + 1];
      }
  }
  // one 2-port handle reads both port counts: port 0 is equalised alone for 1 port and with port 1 (SFBC) for 2.  The combining decoder keeps the
  // soft bits of up to four consecutive frames, so a MIB too weak to decode from one frame is still read from the frames after it.
  ltephy_cfg_t cfg{};
  cfg.nof_prb = 15, cfg.nof_ports = 2, cfg.cell_id = c->pci, cfg.nof_rx = A, cfg.max_subframes = nframes, cfg.symbol_sz = N;
  ltephy_t* phy = nullptr;
  if (ltephy_create(&cfg, &phy) != LTEPHY_SUCCESS) {
    fprintf(stderr, "ltephy_create: %s\n", ltephy_last_error());
    return 1;
  }
  std::vector<ltephy_mib_comb_t> m(nframes);
  if (ltephy_set_cfo(phy, c->cfo_hz) != LTEPHY_SUCCESS || ltephy_submit_iq(phy, sf.data(), tti.data(), nframes) != LTEPHY_SUCCESS ||
      ltephy_mib_decode_combined(phy, LTEPHY_MIB_SEARCH_PORTS, m.data()) != LTEPHY_SUCCESS) {
    fprintf(stderr, "MIB decode: %s\n", ltephy_last_error());
    return 1;
  }
  ltephy_destroy(phy);
  ltephy_mib_t mib{};
  uint32_t     ports = 0;
  for (uint32_t f = 0; f < nframes && !ports; f++)
    if (m[f].mib.found) {
      mib = m[f].mib, ports = mib.nof_ports;
      mib.sfn = (mib.sfn + 1024 - f % 1024) % 1024; // the SFN of frame f, counted back to the frame at frame_offset
    }
  if (!ports) { // no window of any frame passed its CRC (too weak even combined, or a cell with four CRS ports)
    fprintf(stderr, "cell %u found, MIB not decoded\n", c->pci);
    return 3;
  }
  printf("pci %u frame_offset %llu cfo_hz %.1f nof_prb %u nof_ports %u phich_resources %u phich_length %u sfn %u\n", c->pci,
         (unsigned long long)c->frame_offset, c->cfo_hz, mib.nof_prb, ports, mib.phich_resources, mib.phich_length, mib.sfn);
  return 0;
}
