// compat_check.cpp -- drives the tier-2 shim (the srsRAN-compatible header tree compat/srsran/..., libltephy_srsran_compat.so) the way the reference's SubframeWorker / DCISearch /
// PDSCH_Decoder drive srsRAN, and dumps what it gets so that tests/test_compat_shim.py and tests/test_gpu_compat_matrix.py can compare it with the tier-1 results:
//   per subframe: srsran_ue_dl_decode_fft_estimate (or _noguru); cfi, snr_db, FNV-1a of sf_symbols / ce, the PDCCH LLRs;
//                 srsran_pdcch_dci_decode for every (location, payload size) given on the command line;
//                 srsran_ue_dl_decode_pdsch (or srsran_pdsch_decode) for the grants of that subframe read from <grants.bin>.
//   compat_check [options] <iq.cf32> <nof_prb> <nof_ports> <cell_id> <nof_rx> <n_sf> <first_tti> <grants.bin> <out.bin> <nof_bits>...
// options:
//   --rate34            leave srsRAN's 3/4-rate symbol size (the capture is sampled at 23.04 Msps at 100 PRB); default: srsran_use_standard_symbol_size(true)
//   --noguru            odd subframes go through srsran_ue_dl_decode_fft_estimate_noguru from a second set of antenna buffers
//   --pdsch-decode      srsran_pdsch_decode(&q.pdsch, ...) instead of srsran_ue_dl_decode_pdsch
//   --phich=<r>,<len>   cell.phich_resources (0: 1/6 .. 3: 2) and cell.phich_length (0 normal, 1 extended)
//   --pre-cell=<prb>,<ports>,<id>  srsran_ue_dl_set_cell with this cell first and decode one empty subframe with it, then set the real cell
//   --harq-slots=<n>    ltephy_compat_harq_slots
//   --harq              each grant record is followed by the soft-buffer operation of each TB (DL_Sniffer_PDSCH.cc:955-990), see SbOp
#include "ltephy_b200.h"
#include "ltephy_compat_ext.h"
#include "srsran/srsran.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <vector>

static uint64_t fnv(const void* p, size_t n)
{
  const uint8_t* b = static_cast<const uint8_t*>(p);
  uint64_t       h = 1469598103934665603ull;
  for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 1099511628211ull;
  return h;
}
template <class T> static void put(FILE* f, const T& v) { fwrite(&v, sizeof(T), 1, f); }

struct GrantRec {
  uint32_t       sf, rnti;
  ltephy_grant_t g;
};
// what pdsch_cfg->softbuffers.rx[t] is for one TB
enum SbOp : uint8_t {
  SB_NULL    = 0, // no soft buffer
  SB_SCRATCH = 1, // buffer[t] with reset_tbs: the reference without HARQ mode, and its FULL_BUFFER / BUSY / default cases
  SB_NEW     = 2, // HARQ buffer with reset_tbs: DL_SNIFFER_NEW_TX
  SB_RETX    = 3, // HARQ buffer, no reset: DL_SNIFFER_RE_TX
  SB_DECODED = 4, // TB disabled: DL_SNIFFER_DECODED (softbuffers.rx[t] keeps whatever an earlier grant left there)
  SB_RESET   = 5, // HARQ buffer after srsran_softbuffer_rx_reset
  SB_REINIT  = 6, // HARQ buffer freed and initialised again at the same address, no reset
};
struct HarqRec {
  uint8_t  op[2];
  uint16_t buf[2]; // which HARQ buffer (the caller's (rnti, pid, tb) key)
};

int main(int argc, char** argv)
{
  bool     rate34 = false, noguru = false, pdsch_decode = false, harq = false;
  uint32_t phich_r = 0, phich_len = 0, harq_slots = 0, pre[3] = {0, 0, 0};
  std::vector<char*> pos;
  for (int i = 1; i < argc; i++) {
    if (!strcmp(argv[i], "--rate34")) rate34 = true;
    else if (!strcmp(argv[i], "--noguru")) noguru = true;
    else if (!strcmp(argv[i], "--pdsch-decode")) pdsch_decode = true;
    else if (!strcmp(argv[i], "--harq")) harq = true;
    else if (sscanf(argv[i], "--phich=%u,%u", &phich_r, &phich_len) == 2) {}
    else if (sscanf(argv[i], "--pre-cell=%u,%u,%u", &pre[0], &pre[1], &pre[2]) == 3) {}
    else if (sscanf(argv[i], "--harq-slots=%u", &harq_slots) == 1) {}
    else if (!strncmp(argv[i], "--", 2)) return 2;
    else pos.push_back(argv[i]);
  }
  if (pos.size() < 10) return 2;
  srsran_cell_t cell{};
  cell.nof_prb = (uint32_t)atoi(pos[1]), cell.nof_ports = (uint32_t)atoi(pos[2]), cell.id = (uint32_t)atoi(pos[3]), cell.cp = SRSRAN_CP_NORM;
  cell.phich_resources = (srsran_phich_r_t)phich_r, cell.phich_length = (srsran_phich_length_t)phich_len;
  const uint32_t nof_rx = (uint32_t)atoi(pos[4]), n_sf = (uint32_t)atoi(pos[5]), tti0 = (uint32_t)atoi(pos[6]);
  std::vector<uint32_t> sizes;
  for (size_t i = 9; i < pos.size(); i++) sizes.push_back((uint32_t)atoi(pos[i]));
  FILE* in = fopen(pos[0], "rb");
  FILE* gf = fopen(pos[7], "rb");
  FILE* out = fopen(pos[8], "wb");
  if (!in || !gf || !out) return 1;
  std::vector<GrantRec> grants;
  std::vector<HarqRec>  hops;
  GrantRec              gr;
  HarqRec               hr{};
  while (fread(&gr, sizeof(gr), 1, gf) == 1) {
    if (harq && fread(&hr, sizeof(hr), 1, gf) != 1) return 1;
    grants.push_back(gr), hops.push_back(hr);
  }

  // the capture handed to this program is sampled at the standard LTE rate (30.72 Msps at 100 PRB) unless --rate34
  if (!rate34) srsran_use_standard_symbol_size(true);
  const uint32_t sf_len = SRSRAN_SF_LEN_PRB(cell.nof_prb);
  std::vector<cf_t> buf[2], buf2[2];
  cf_t*             in_buffer[SRSRAN_MAX_PORTS] = {};
  cf_t*             in_buffer2[SRSRAN_MAX_PORTS] = {};
  for (uint32_t a = 0; a < nof_rx; a++) { // SubframeBuffer over-allocates (src/src/SubframeBuffer.cc:25)
    buf[a].resize(3 * SRSRAN_SF_LEN_PRB(SRSRAN_MAX_PRB)), in_buffer[a] = buf[a].data();
    buf2[a].resize(3 * SRSRAN_SF_LEN_PRB(SRSRAN_MAX_PRB)), in_buffer2[a] = buf2[a].data();
  }
  srsran_ue_dl_t q;
  if (srsran_ue_dl_init(&q, in_buffer, SRSRAN_MAX_PRB, nof_rx)) return 1;
  if (harq_slots && ltephy_compat_harq_slots(&q, harq_slots)) return 1;
  if (pre[0]) { // another cell on the same object first: one subframe of silence through it
    srsran_cell_t c0 = cell;
    c0.nof_prb = pre[0], c0.nof_ports = pre[1], c0.id = pre[2], c0.phich_resources = SRSRAN_PHICH_R_1, c0.phich_length = SRSRAN_PHICH_NORM;
    srsran_dl_sf_cfg_t sf{};
    srsran_ue_dl_cfg_t cfg{};
    if (srsran_ue_dl_set_cell(&q, c0) || srsran_ue_dl_decode_fft_estimate(&q, &sf, &cfg) != SRSRAN_SUCCESS) {
      fprintf(stderr, "first cell failed: %s\n", ltephy_last_error());
      return 1;
    }
  }
  if (srsran_ue_dl_set_cell(&q, cell)) {
    fprintf(stderr, "init failed: %s\n", ltephy_last_error());
    return 1;
  }
  // soft buffers: scratch buffer[i] (DL_Sniffer_PDSCH.cc:43,62) and the HARQ buffers of HARQ.cc:54, allocated on first use
  srsran_softbuffer_rx_t scratch[SRSRAN_MAX_CODEWORDS];
  for (auto& s : scratch) srsran_softbuffer_rx_init(&s, cell.nof_prb);
  std::map<uint16_t, std::unique_ptr<srsran_softbuffer_rx_t>> hbuf;
  auto harq_buffer = [&](uint16_t k) {
    auto& b = hbuf[k];
    if (!b) b.reset(new srsran_softbuffer_rx_t), srsran_softbuffer_rx_init(b.get(), SRSRAN_MAX_PRB);
    return b.get();
  };
  srsran_pdsch_cfg_t pc{}; // one object for every grant, as PDSCH_Decoder keeps it
  const uint32_t     g = 14 * 12 * cell.nof_prb;
  for (uint32_t i = 0; i < n_sf; i++) {
    const bool ng = noguru && (i & 1);
    for (uint32_t a = 0; a < nof_rx; a++)
      if (fread((ng ? buf2 : buf)[a].data(), sizeof(cf_t), sf_len, in) != sf_len) return 1;
    srsran_dl_sf_cfg_t sf{};
    srsran_ue_dl_cfg_t cfg{};
    sf.tti = tti0 + i;
    const int rc = ng ? srsran_ue_dl_decode_fft_estimate_noguru(&q, &sf, &cfg, in_buffer2) : srsran_ue_dl_decode_fft_estimate(&q, &sf, &cfg);
    if (rc != SRSRAN_SUCCESS) return 1;
    put(out, sf.cfi), put(out, q.chest_res.snr_db), put(out, q.chest_res.noise_estimate), put(out, q.chest_res.cfo);
    uint64_t hs = 0, hc = 0;
    for (uint32_t a = 0; a < nof_rx; a++) hs ^= fnv(q.sf_symbols[a], g * sizeof(cf_t)) * (a + 1);
    for (uint32_t p = 0; p < cell.nof_ports; p++)
      for (uint32_t a = 0; a < nof_rx; a++) hc ^= fnv(q.chest_res.ce[p][a], g * sizeof(cf_t)) * (p * 2 + a + 1);
    put(out, hs), put(out, hc);
    const uint32_t ncce = q.pdcch.nof_cce[sf.cfi - 1];
    put(out, ncce);
    fwrite(q.pdcch.llr, sizeof(float), 72 * ncce, out);
    // every location x size, in srsran_pdcch_ue_locations_all_map order (falcon_pdcch.c:321-356)
    const uint32_t lim = ncce < 84 ? ncce : 84;
    for (int L = 3; L >= 0; L--)
      for (uint32_t k = 0; k < lim >> L; k++)
        for (uint32_t nb : sizes) {
          uint8_t  data[SRSRAN_DCI_MAX_BITS];
          uint16_t crc = 0;
          if (srsran_pdcch_dci_decode(&q.pdcch, &q.pdcch.llr[72 * (k << L)], data, 72u << L, nb, &crc) != SRSRAN_SUCCESS) return 1;
          uint64_t bits = 0;
          for (uint32_t b = 0; b < nb; b++) bits |= (uint64_t)(data[b] & 1u) << (63 - b);
          put(out, crc), put(out, bits);
        }
    for (size_t gi = 0; gi < grants.size(); gi++) {
      const GrantRec& r = grants[gi];
      if (r.sf != i) continue;
      pc.rnti = (uint16_t)r.rnti;
      pc.grant = srsran_pdsch_grant_t{};
      srsran_pdsch_grant_t& s = pc.grant;
      s.tx_scheme = r.g.tx_scheme == LTEPHY_TX_PORT0       ? SRSRAN_TXSCHEME_PORT0
                    : r.g.tx_scheme == LTEPHY_TX_DIVERSITY ? SRSRAN_TXSCHEME_DIVERSITY
                    : r.g.tx_scheme == LTEPHY_TX_CDD       ? SRSRAN_TXSCHEME_CDD
                                                           : SRSRAN_TXSCHEME_SPATIALMUX;
      s.pmi = r.g.pmi, s.nof_re = r.g.nof_re, s.nof_tb = r.g.nof_tb;
      for (int sl = 0; sl < 2; sl++)
        for (uint32_t prb = 0; prb < cell.nof_prb; prb++) s.prb_idx[sl][prb] = (r.g.prb_mask[sl][prb >> 5] >> (prb & 31)) & 1u, s.nof_prb += sl == 0 && s.prb_idx[sl][prb];
      for (int t = 0; t < 2; t++) {
        s.tb[t].enabled = r.g.tb[t].enabled, s.tb[t].tbs = r.g.tb[t].tbs, s.tb[t].rv = r.g.tb[t].rv, s.tb[t].cw_idx = r.g.tb[t].cw_idx;
        s.tb[t].mod = r.g.tb[t].qm == 2 ? SRSRAN_MOD_QPSK : r.g.tb[t].qm == 4 ? SRSRAN_MOD_16QAM : r.g.tb[t].qm == 6 ? SRSRAN_MOD_64QAM : SRSRAN_MOD_256QAM;
        if (!harq || !s.tb[t].enabled) continue;
        const uint32_t tbs = (uint32_t)s.tb[t].tbs;
        srsran_softbuffer_rx_t* hb = nullptr;
        switch (hops[gi].op[t]) {
          case SB_NULL: pc.softbuffers.rx[t] = nullptr; break;
          case SB_SCRATCH: pc.softbuffers.rx[t] = &scratch[t], srsran_softbuffer_rx_reset_tbs(&scratch[t], tbs); break;
          case SB_NEW: pc.softbuffers.rx[t] = hb = harq_buffer(hops[gi].buf[t]), srsran_softbuffer_rx_reset_tbs(hb, tbs); break;
          case SB_RETX: pc.softbuffers.rx[t] = harq_buffer(hops[gi].buf[t]); break;
          case SB_DECODED: s.tb[t].enabled = false; break;
          case SB_RESET: pc.softbuffers.rx[t] = hb = harq_buffer(hops[gi].buf[t]), srsran_softbuffer_rx_reset(hb); break;
          case SB_REINIT:
            hb = harq_buffer(hops[gi].buf[t]), srsran_softbuffer_rx_free(hb), srsran_softbuffer_rx_init(hb, SRSRAN_MAX_PRB), pc.softbuffers.rx[t] = hb;
            break;
          default: return 2;
        }
      }
      std::vector<uint8_t> pl0(16000), pl1(16000); // srsran_vec_u8_malloc(2000 * 8), DL_Sniffer_PDSCH.cc:47
      srsran_pdsch_res_t   res[SRSRAN_MAX_CODEWORDS]{};
      res[0].payload = pl0.data(), res[1].payload = pl1.data();
      if (s.tb[0].enabled || s.tb[1].enabled) { // DL_Sniffer_PDSCH.cc:994
        const int rc = pdsch_decode ? srsran_pdsch_decode(&q.pdsch, &sf, &pc, &q.chest_res, q.sf_symbols, res) : srsran_ue_dl_decode_pdsch(&q, &sf, &pc, res);
        if (rc != SRSRAN_SUCCESS) {
          fprintf(stderr, "decode failed: %s\n", ltephy_last_error());
          return 1;
        }
      }
      for (int t = 0; t < 2; t++) {
        const uint32_t nby = s.tb[t].enabled && s.tb[t].tbs > 0 ? (uint32_t)s.tb[t].tbs / 8 : 0;
        put(out, (uint8_t)res[t].crc), put(out, nby);
        fwrite(t ? pl1.data() : pl0.data(), 1, nby, out);
      }
    }
  }
  srsran_ue_dl_free(&q);
  for (auto& s : scratch) srsran_softbuffer_rx_free(&s);
  for (auto& kv : hbuf) srsran_softbuffer_rx_free(kv.second.get());
  fclose(out);
  return 0;
}
