// compat_ul_check.cpp -- drives the uplink half of the tier-2 shim (libltephy_srsran_compat.so) the way the reference's SubframeWorker
// (src/src/SubframeWorker.cc:79,261) and PUSCH_Decoder (src/src/UL_Sniffer_PUSCH.cc:256,262,392) drive srsRAN, and dumps what it gets so
// that tests/test_gpu_compat_matrix.py can compare it with ltephy_submit_ul / ltephy_get_ul and the CPU oracle:
//   srsran_enb_ul_init, srsran_enb_ul_set_cell with the SIB2 DMRS configuration; per subframe one srsran_enb_ul_fft, then per grant record
//   srsran_chest_ul_estimate_pusch and / or srsran_pusch_decode.
//   compat_ul_check [--rate34] <iq_ul.cf32> <nof_prb> <cell_id> <n_sf> <first_tti> <cyclic_shift> <delta_ss> <group_hopping> <seq_hopping>
//                   <grants.bin> <out.bin>
// grants.bin: UlRec records in subframe order.  mode 0: estimate, then decode with the same configuration; mode 1: estimate only; mode 2:
// decode only (so a mode-1 record followed by a mode-2 record decodes a configuration other than the one just estimated).
// out.bin, per record: u32 cqi_len (srsran_cqi_size); modes 0 / 1: f32 noise_estimate, noise_estimate_dbm, rsrp, snr_db, snr, ta_us;
// modes 0 / 2: u8 crc, u32 nby, nby payload bytes.
#include "ltephy_b200.h"
#include "srsran/srsran.h"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

template <class T> static void put(FILE* f, const T& v) { fwrite(&v, sizeof(T), 1, f); }

struct UlRec {
  uint32_t sf, mode, rnti, qm, rv, L_prb, n_prb[2], n_dmrs, tbs;
  uint32_t nof_ack, ri_len, cqi_enable, cqi_type, cqi_N, cqi_L, cqi_rank, I_offset_ack, I_offset_cqi, I_offset_ri;
};

int main(int argc, char** argv)
{
  bool               rate34 = false;
  std::vector<char*> pos;
  for (int i = 1; i < argc; i++) {
    if (!strcmp(argv[i], "--rate34")) rate34 = true;
    else if (!strncmp(argv[i], "--", 2)) return 2;
    else pos.push_back(argv[i]);
  }
  if (pos.size() != 11) return 2;
  srsran_cell_t cell{};
  cell.nof_prb = (uint32_t)atoi(pos[1]), cell.id = (uint32_t)atoi(pos[2]), cell.nof_ports = 1, cell.cp = SRSRAN_CP_NORM;
  const uint32_t n_sf = (uint32_t)atoi(pos[3]), tti0 = (uint32_t)atoi(pos[4]);
  srsran_refsignal_dmrs_pusch_cfg_t dmrs{}; // ULSchedule::set_config (src/src/ULSchedule.cc:143-146)
  dmrs.cyclic_shift = (uint32_t)atoi(pos[5]), dmrs.delta_ss = (uint32_t)atoi(pos[6]);
  dmrs.group_hopping_en = atoi(pos[7]) != 0, dmrs.sequence_hopping_en = atoi(pos[8]) != 0;
  FILE* in = fopen(pos[0], "rb");
  FILE* gf = fopen(pos[9], "rb");
  FILE* out = fopen(pos[10], "wb");
  if (!in || !gf || !out) return 1;
  std::vector<UlRec> recs;
  UlRec              r;
  while (fread(&r, sizeof(r), 1, gf) == 1) recs.push_back(r);

  if (!rate34) srsran_use_standard_symbol_size(true);
  const uint32_t    sf_len = SRSRAN_SF_LEN_PRB(cell.nof_prb);
  std::vector<cf_t> buf(3 * SRSRAN_SF_LEN_PRB(SRSRAN_MAX_PRB)); // antenna buffer 1 of the SubframeBuffer (UL_Sniffer_PUSCH.cc:391)
  srsran_enb_ul_t   q;
  if (srsran_enb_ul_init(&q, buf.data(), SRSRAN_MAX_PRB) || srsran_enb_ul_set_cell(&q, cell, &dmrs, nullptr)) {
    fprintf(stderr, "init failed: %s\n", ltephy_last_error());
    return 1;
  }
  srsran_chest_ul_res_init(&q.chest_res, cell.nof_prb);
  srsran_softbuffer_rx_t sb; // one buffer, never reset (UL_Sniffer_PUSCH.cc:37-44)
  srsran_softbuffer_rx_init(&sb, cell.nof_prb);
  std::vector<uint8_t> data(16000);
  for (uint32_t i = 0; i < n_sf; i++) {
    if (fread(buf.data(), sizeof(cf_t), sf_len, in) != sf_len) return 1;
    srsran_ul_sf_cfg_t sf{};
    sf.tti = tti0 + i;
    srsran_enb_ul_fft(&q);
    for (const UlRec& u : recs) {
      if (u.sf != i) continue;
      srsran_pusch_cfg_t cfg{};
      cfg.rnti = (uint16_t)u.rnti, cfg.meas_ta_en = true, cfg.softbuffers.rx = &sb, cfg.max_nof_iterations = 8;
      srsran_pusch_grant_t& g = cfg.grant;
      g.tb.mod = u.qm == 2 ? SRSRAN_MOD_QPSK : u.qm == 4 ? SRSRAN_MOD_16QAM : u.qm == 6 ? SRSRAN_MOD_64QAM : SRSRAN_MOD_256QAM;
      g.tb.rv = (int)u.rv, g.tb.tbs = (int)u.tbs, g.tb.enabled = true, g.L_prb = u.L_prb, g.n_prb[0] = u.n_prb[0], g.n_prb[1] = u.n_prb[1];
      g.n_dmrs = u.n_dmrs, g.freq_hopping = u.n_prb[0] != u.n_prb[1];
      cfg.uci_cfg.ack[0].nof_acks = u.nof_ack, cfg.uci_cfg.cqi.ri_len = u.ri_len;
      srsran_cqi_cfg_t& c = cfg.uci_cfg.cqi;
      c.data_enable = u.cqi_enable != 0, c.type = (srsran_cqi_type_t)u.cqi_type, c.N = u.cqi_N, c.L = u.cqi_L, c.rank_is_not_one = u.cqi_rank != 0;
      cfg.uci_offset.I_offset_ack = u.I_offset_ack, cfg.uci_offset.I_offset_cqi = u.I_offset_cqi, cfg.uci_offset.I_offset_ri = u.I_offset_ri;
      put(out, (uint32_t)srsran_cqi_size(&c));
      if (u.mode != 2) {
        if (srsran_chest_ul_estimate_pusch(&q.chest, &sf, &cfg, q.sf_symbols, &q.chest_res) != SRSRAN_SUCCESS) {
          fprintf(stderr, "estimate failed: %s\n", ltephy_last_error());
          return 1;
        }
        const srsran_chest_ul_res_t& e = q.chest_res;
        put(out, e.noise_estimate), put(out, e.noise_estimate_dbm), put(out, e.rsrp), put(out, e.snr_db), put(out, e.snr), put(out, e.ta_us);
      }
      if (u.mode != 1) {
        srsran_pusch_res_t res{};
        std::fill(data.begin(), data.end(), 0);
        res.data = data.data();
        if (srsran_pusch_decode(&q.pusch, &sf, &cfg, &q.chest_res, q.sf_symbols, &res) != SRSRAN_SUCCESS) {
          fprintf(stderr, "decode failed: %s\n", ltephy_last_error());
          return 1;
        }
        const uint32_t nby = u.tbs / 8;
        put(out, (uint8_t)res.crc), put(out, nby);
        fwrite(data.data(), 1, nby, out);
      }
    }
  }
  srsran_softbuffer_rx_free(&sb);
  srsran_chest_ul_res_free(&q.chest_res);
  srsran_enb_ul_free(&q);
  fclose(out);
  return 0;
}
