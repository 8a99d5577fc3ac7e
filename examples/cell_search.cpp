// cell_search.cpp -- what a recording needs before offline_decode can read it: find the cell in a continuous capture with
// ltephy_cell_search (PCI, frame timing, carrier offset), then decode its MIB (bandwidth, ports, PHICH, SFN) at that timing with the
// offset corrected, the PSS / SSS search and MIB decode of rf_search_and_decode_mib (reference src/src/LTESniffer_Core.cc:193-204).  The MIB is
// decoded with soft combining across the 40 ms period and a search over the port count, over every frame of the capture.
// Host code only; without a GPU ltephy_sync_create fails.
//
//   cell_search <iq file> <symbol_sz> <nof_rx> [fmt=cf32|sc16|sc8]
//
// File layout: antenna after antenna, each a continuous run of complex samples at 15 kHz * symbol_sz: float32 (cf32, the default) or int16 / int8
// I/Q pairs (sc16 / sc8, what a USRP records), read as they are.  Prints one line:
//   pci <pci> frame_offset <samples> cfo_hz <Hz> nof_prb <n> nof_ports <n> phich_resources <r> phich_length <l> sfn <sfn>
// where frame_offset is the first sample of a subframe 0 and sfn that frame's number: offline_decode takes the file from there on,
// with first_tti = 10 * sfn, after the carrier offset is removed.
#include "cell_chain.h"

int main(int argc, char** argv)
{
  uint32_t fmt = LTEPHY_IQ_CF32;
  if (int r = chain_take_fmt(argc, argv, &fmt)) return r;
  if (argc < 4) {
    fprintf(stderr, "usage: %s <iq file> <symbol_sz> <nof_rx> [fmt=cf32|sc16|sc8]\n", argv[0]);
    return 2;
  }
  const uint32_t N = (uint32_t)atoi(argv[2]), A = (uint32_t)atoi(argv[3]);
  FILE*          in = fopen(argv[1], "rb");
  if (!in || A < 1 || A > 2) {
    fprintf(stderr, "cannot open %s / bad nof_rx\n", argv[1]);
    return 2;
  }
  fseeko(in, 0, SEEK_END);
  const uint64_t L = (uint64_t)ftello(in) / ((uint64_t)chain_sample_bytes(fmt) * A);
  // the search and the MIB over the whole capture: one 2-port handle reads both port counts (port 0 is equalised alone for 1 port and with port 1,
  // SFBC, for 2), and the combining decoder keeps the soft bits of up to four consecutive frames, so a MIB too weak to decode from one frame is
  // still read from the frames after it
  ltephy_cell_t c{};
  ltephy_mib_t  mib{};
  const int     r = chain_acquire(in, N, A, L, L, fmt, &c, &mib);
  fclose(in);
  if (r) return r;
  printf("pci %u frame_offset %llu cfo_hz %.1f nof_prb %u nof_ports %u phich_resources %u phich_length %u sfn %u\n", c.pci,
         (unsigned long long)c.frame_offset, c.cfo_hz, mib.nof_prb, mib.nof_ports, mib.phich_resources, mib.phich_length, mib.sfn);
  return 0;
}
