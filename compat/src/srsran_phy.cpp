// srsran_phy.cpp -- signal-processing part of libltephy_srsran_compat: the srsRAN objects of the hot path (srsran_ue_dl_t,
// srsran_enb_ul_t) on top of the tier-1 C-ABI of libltephy_b200 with a batch of one subframe.  No arithmetic happens here: every
// call stages buffers, runs the GPU path and mirrors the results into the fields the reference reads.
#include "../ltephy_compat_ext.h"
#include "srsran/srsran.h"
#include "../../include/ltephy_b200.h"
#include "../../include/ltephy_search.h"
#include "../../ltesniffer_b200/csrc/lte_host.hpp"
#include <cmath>
#include <cstddef>
#include <cstring>
#include <unordered_map>
#include <vector>

namespace {
typedef struct { float re, im; } cfx_t; // layout of cf_t
// One slot of the handle's HARQ store per soft-buffer object: the slot holds the soft values of the transmissions decoded into the
// buffer since its identity (b200_id, renewed by every reset) last changed.
struct HarqSlot {
  const srsran_softbuffer_rx_t* buf;
  uint64_t                      id;       // b200_id of the last decode into this slot
  uint64_t                      last_use; // for least-recently-used replacement when every slot is taken
};
struct DlPriv {
  ltephy_t*                  phy = nullptr;
  cf_t*                      in[SRSRAN_MAX_PORTS]{};
  uint32_t                   sf_len = 0, g = 0, symbol_sz = 0;
  std::vector<float>         iq;                    // [rx][sf_len] cf32, contiguous staging of the caller's antenna buffers
  std::vector<cfx_t>         sym, ce;               // host mirrors handed out through q->sf_symbols / q->chest_res.ce
  std::vector<float>         llr;
  std::vector<ltephy_cand_t> table;                 // T[location][size] of the current subframe
  ltephy_sf_info_t           info{};
  int16_t                    loc_of[3][4][LTEPHY_MAX_CCE]; // [cfi-1][L][ncce] -> location index
  ltehost::SizeTable         st;
  uint32_t                   cur_cfi = 0;
  bool                       injected = false;
  ltephy_sf_info_t           inj_info{};
  uint32_t                   harq_cap = LTEPHY_COMPAT_HARQ_SLOTS;
  bool                       harq_reserved = false; // the store of phy holds harq_cap slots
  std::vector<HarqSlot>      harq;                  // slots in use, by slot index
  std::unordered_map<const srsran_softbuffer_rx_t*, uint32_t> harq_of;
  uint64_t                   harq_clock = 0;
  void clear_harq() { harq.clear(), harq_of.clear(), harq_clock = 0; }
};
DlPriv* P(srsran_ue_dl_t* q) { return q ? static_cast<DlPriv*>(q->b200) : nullptr; }

struct UlPriv {
  ltephy_t*          phy = nullptr;
  uint32_t           sf_len = 0, g = 0;
  std::vector<cfx_t> sym;
  std::vector<uint8_t> payload;
  // result of the last srsran_chest_ul_estimate_pusch (the GPU decodes the grant in the same pass)
  bool               have = false, fft_done = false;
  ltephy_ul_grant_t  grant{};
  uint32_t           tti = 0;
  ltephy_tb_result_t res{};
  ltephy_ul_chest_t  chest{};
  srsran_refsignal_dmrs_pusch_cfg_t dmrs{};
};
} // namespace

extern "C" {

// ---------------------------------------------------------------------------------------------------- downlink
int srsran_ue_dl_init(srsran_ue_dl_t* q, cf_t* in_buffer[SRSRAN_MAX_PORTS], uint32_t max_prb, uint32_t nof_rx_antennas)
{
  if (!q || !in_buffer || nof_rx_antennas < 1 || nof_rx_antennas > 2 || max_prb > SRSRAN_MAX_PRB) return SRSRAN_ERROR_INVALID_INPUTS;
  memset((void*)q, 0, sizeof(*q));
  DlPriv* p = new DlPriv();
  for (uint32_t a = 0; a < nof_rx_antennas; a++) p->in[a] = in_buffer[a];
  q->nof_rx_antennas = nof_rx_antennas;
  q->b200            = p;
  return SRSRAN_SUCCESS;
}
int srsran_ue_dl_set_cell(srsran_ue_dl_t* q, srsran_cell_t cell)
{
  DlPriv* p = P(q);
  if (!p || cell.cp != SRSRAN_CP_NORM || cell.nof_prb < 15 || cell.nof_prb > 100 || cell.nof_ports < 1 || cell.nof_ports > 2) return SRSRAN_ERROR_INVALID_INPUTS;
  if ((uint32_t)cell.phich_length > 1 || (uint32_t)cell.phich_resources > 3) return SRSRAN_ERROR_INVALID_INPUTS;
  if (p->phy) ltephy_destroy(p->phy), p->phy = nullptr;
  p->harq_reserved = false, p->clear_harq(); // the store went with the handle: every soft buffer starts empty again
  // geometry from the host tables only: the CUDA handle is created with the first subframe that is really decoded, so a search
  // fed with ltephy_compat_inject needs no GPU
  const ltehost::Cell hc{cell.nof_prb, cell.nof_ports, cell.id, q->nof_rx_antennas, (uint32_t)cell.phich_resources, (uint32_t)cell.phich_length};
  ltehost::CtrlMap    cm;
  if (!ltehost::build_ctrl_map(hc, cm)) return SRSRAN_ERROR;
  p->st     = ltehost::dci_size_table(hc);
  q->cell   = cell;
  p->symbol_sz = (uint32_t)srsran_symbol_sz(cell.nof_prb);
  p->sf_len = 15 * p->symbol_sz, p->g = 14 * 12 * cell.nof_prb;
  p->iq.assign((size_t)2 * q->nof_rx_antennas * p->sf_len, 0.0f);
  p->sym.assign((size_t)q->nof_rx_antennas * p->g, cfx_t{0, 0});
  p->ce.assign((size_t)cell.nof_ports * q->nof_rx_antennas * p->g, cfx_t{0, 0});
  p->llr.assign((size_t)72 * LTEPHY_MAX_CCE, 0.0f);
  p->table.assign((size_t)LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES, ltephy_cand_t{});
  for (uint32_t a = 0; a < q->nof_rx_antennas; a++) q->sf_symbols[a] = reinterpret_cast<cf_t*>(p->sym.data() + (size_t)a * p->g);
  for (uint32_t pt = 0; pt < cell.nof_ports; pt++)
    for (uint32_t a = 0; a < q->nof_rx_antennas; a++)
      q->chest_res.ce[pt][a] = reinterpret_cast<cf_t*>(p->ce.data() + ((size_t)pt * q->nof_rx_antennas + a) * p->g);
  q->chest_res.nof_re = p->g;
  q->pdcch.llr = p->llr.data(), q->pdcch.cell = cell, q->pdcch.nof_rx_antennas = q->nof_rx_antennas, q->pdcch.b200 = q;
  memset(p->loc_of, 0xFF, sizeof(p->loc_of));
  for (uint32_t cfi = 1; cfi <= 3; cfi++) {
    q->pdcch.nof_cce[cfi - 1] = cm.nof_cce[cfi - 1], q->pdcch.nof_regs[cfi - 1] = 9 * cm.nof_cce[cfi - 1];
    const auto locs = ltehost::all_locations(cm.nof_cce[cfi - 1]);
    for (size_t i = 0; i < locs.size(); i++) p->loc_of[cfi - 1][locs[i].L][locs[i].ncce] = (int16_t)i;
  }
  q->pdcch.max_bits = 72 * LTEPHY_MAX_CCE;
  q->pdsch.cell = cell, q->pdsch.nof_rx_antennas = q->nof_rx_antennas, q->pdsch.b200 = q;
  p->cur_cfi = 0;
  return SRSRAN_SUCCESS;
}
void srsran_ue_dl_free(srsran_ue_dl_t* q)
{
  DlPriv* p = P(q);
  if (!p) return;
  if (p->phy) ltephy_destroy(p->phy);
  delete p;
  memset((void*)q, 0, sizeof(*q));
}
void srsran_ue_dl_set_rnti(srsran_ue_dl_t* q, uint16_t rnti) { if (q) q->pregen_rnti = rnti; }
ltephy_t* ltephy_compat_phy(srsran_ue_dl_t* q) { return P(q) ? P(q)->phy : nullptr; }
int ltephy_compat_harq_slots(srsran_ue_dl_t* q, uint32_t nslots)
{
  DlPriv* p = P(q);
  if (!p || nslots == 0) return SRSRAN_ERROR_INVALID_INPUTS;
  p->harq_cap = nslots, p->harq_reserved = false, p->clear_harq();
  return SRSRAN_SUCCESS;
}
// LTEPHY_HARQ_* for soft buffer b of one TB, and the slot it uses; see ltephy_compat_ext.h for the rules
static uint8_t harq_slot_of(DlPriv* p, const srsran_softbuffer_rx_t* b, uint32_t* slot)
{
  if (!b) return LTEPHY_HARQ_NONE;
  auto     it = p->harq_of.find(b);
  uint32_t s;
  uint8_t  op = LTEPHY_HARQ_NEW;
  if (it != p->harq_of.end()) {
    s = it->second;
    if (p->harq[s].id == b->b200_id) op = LTEPHY_HARQ_RETX;
  } else if (p->harq.size() < p->harq_cap) {
    s = (uint32_t)p->harq.size(), p->harq.push_back(HarqSlot{});
  } else { // every slot taken: the least recently decoded buffer gives its slot up and starts empty at its next decode
    s = 0;
    for (uint32_t i = 1; i < p->harq.size(); i++)
      if (p->harq[i].last_use < p->harq[s].last_use) s = i;
    p->harq_of.erase(p->harq[s].buf);
  }
  p->harq_of[b] = s, p->harq[s] = HarqSlot{b, b->b200_id, ++p->harq_clock};
  *slot = s;
  return op;
}

static void publish(srsran_ue_dl_t* q, DlPriv* p, srsran_dl_sf_cfg_t* sf)
{
  sf->cfi                     = p->info.cfi;
  q->chest_res.noise_estimate = p->info.noise_avg, q->chest_res.snr_db = p->info.snr_db, q->chest_res.cfo = p->info.cfo, q->chest_res.rsrp = p->info.rsrp_avg;
  q->chest_res.noise_estimate_dbm = 10.0f * log10f(p->info.noise_avg) + 30.0f, q->chest_res.rsrp_dbm = 10.0f * log10f(p->info.rsrp_avg) + 30.0f;
  for (uint32_t pt = 0; pt < q->cell.nof_ports && pt < 2; pt++)
    for (uint32_t a = 0; a < q->nof_rx_antennas && a < 2; a++)
      q->chest_res.snr_ant_port_db[a][pt] = 10.0f * log10f(p->info.rsrp[pt][a] / p->info.noise[pt][a]);
  p->cur_cfi = (p->info.cfi >= 1 && p->info.cfi <= 3) ? p->info.cfi : 0;
}
int ltephy_compat_inject(srsran_ue_dl_t* q, const ltephy_sf_info_t* info, const ltephy_cand_t* table, const float* llr)
{
  DlPriv* p = P(q);
  if (!p || !info || !table || p->table.empty()) return SRSRAN_ERROR_INVALID_INPUTS;
  p->inj_info = *info;
  memcpy(p->table.data(), table, p->table.size() * sizeof(ltephy_cand_t));
  std::fill(p->llr.begin(), p->llr.end(), 0.0f);
  if (llr) memcpy(p->llr.data(), llr, sizeof(float) * 72 * std::min<uint32_t>(info->nof_cce, LTEPHY_MAX_CCE));
  p->injected = true;
  return SRSRAN_SUCCESS;
}
// srsran_ue_dl_decode_fft_estimate (src/src/DCISearch.cc:562): phase A for this subframe
int srsran_ue_dl_decode_fft_estimate(srsran_ue_dl_t* q, srsran_dl_sf_cfg_t* sf, srsran_ue_dl_cfg_t* cfg)
{
  (void)cfg; // estimator settings are those the reference configures (src/src/SubframeWorker.cc:376-400); see DESIGN.md section 2
  DlPriv* p = P(q);
  if (!p || !sf || p->table.empty()) return SRSRAN_ERROR_INVALID_INPUTS;
  if (p->injected) {
    p->injected = false;
    p->info     = p->inj_info;
    publish(q, p, sf);
    return SRSRAN_SUCCESS;
  }
  if (!p->phy) {
    ltephy_cfg_t c{};
    c.nof_prb = q->cell.nof_prb, c.nof_ports = q->cell.nof_ports, c.cell_id = q->cell.id, c.nof_rx = q->nof_rx_antennas;
    c.phich_resources = (uint32_t)q->cell.phich_resources, c.phich_length = (uint32_t)q->cell.phich_length;
    c.max_subframes = 1, c.turbo_max_iter = 8, c.flags = 0; // every location is decoded: the caller decides which ones it asks for
    c.symbol_sz = p->symbol_sz;                             // what srsran_symbol_sz() says (standard or 3/4 rate)
    if (ltephy_create(&c, &p->phy) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
    if (ltephy_sf_len(p->phy) != p->sf_len) return SRSRAN_ERROR;
  }
  for (uint32_t a = 0; a < q->nof_rx_antennas; a++) memcpy(p->iq.data() + (size_t)2 * a * p->sf_len, (const void*)p->in[a], (size_t)p->sf_len * sizeof(cf_t));
  const uint32_t tti = sf->tti;
  if (ltephy_submit_iq(p->phy, p->iq.data(), &tti, 1) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
  if (ltephy_get_phase_a(p->phy, &p->info, p->table.data()) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
  if (ltephy_tap(p->phy, LTEPHY_TAP_SYM, p->sym.data(), p->sym.size() * sizeof(cfx_t)) || ltephy_tap(p->phy, LTEPHY_TAP_CE, p->ce.data(), p->ce.size() * sizeof(cfx_t)) ||
      ltephy_tap(p->phy, LTEPHY_TAP_LLR, p->llr.data(), p->llr.size() * sizeof(float)))
    return SRSRAN_ERROR;
  publish(q, p, sf);
  return SRSRAN_SUCCESS;
}
int srsran_ue_dl_decode_fft_estimate_noguru(srsran_ue_dl_t* q, srsran_dl_sf_cfg_t* sf, srsran_ue_dl_cfg_t* cfg, cf_t* input[SRSRAN_MAX_PORTS])
{
  DlPriv* p = P(q);
  if (!p || !input) return SRSRAN_ERROR_INVALID_INPUTS;
  // input serves this call only: the next srsran_ue_dl_decode_fft_estimate reads the buffers of srsran_ue_dl_init again
  cf_t* keep[SRSRAN_MAX_PORTS];
  memcpy(keep, p->in, sizeof(keep));
  for (uint32_t a = 0; a < q->nof_rx_antennas; a++) p->in[a] = input[a];
  const int r = srsran_ue_dl_decode_fft_estimate(q, sf, cfg);
  memcpy(p->in, keep, sizeof(keep));
  return r;
}
// srsran_pdcch_dci_decode (lib/src/phy/falcon_phch/falcon_pdcch.c:142): (location, payload size) -> entry of the GPU's table
int srsran_pdcch_dci_decode(srsran_pdcch_t* pd, float* e, uint8_t* data, uint32_t E, uint32_t nof_bits, uint16_t* crc)
{
  if (!pd || !e || !data || !pd->b200) return SRSRAN_ERROR_INVALID_INPUTS;
  srsran_ue_dl_t* q = static_cast<srsran_ue_dl_t*>(pd->b200);
  DlPriv*         p = P(q);
  if (!p || p->cur_cfi == 0) return SRSRAN_ERROR_INVALID_INPUTS;
  const ptrdiff_t d = e - pd->llr;
  uint32_t        L = 0;
  while (L < 4 && (72u << L) != E) L++;
  if (d < 0 || d % 72 || L > 3 || (size_t)d / 72 >= LTEPHY_MAX_CCE) return SRSRAN_ERROR_INVALID_INPUTS;
  const int li = p->loc_of[p->cur_cfi - 1][L][d / 72];
  int       si = -1;
  for (size_t i = 0; i < p->st.sizes.size(); i++)
    if (p->st.sizes[i] == nof_bits) si = (int)i;
  if (li < 0 || si < 0) return SRSRAN_ERROR_INVALID_INPUTS; // not one of the blind-search locations / payload sizes
  const ltephy_cand_t& c = p->table[(size_t)li * LTEPHY_MAX_SIZES + si];
  for (uint32_t i = 0; i < nof_bits; i++) data[i] = c.valid ? (uint8_t)((c.bits >> (63 - i)) & 1u) : 0;
  if (crc) *crc = c.valid ? c.rnti : 0;
  return SRSRAN_SUCCESS;
}
int srsran_pdcch_extract_llr(srsran_pdcch_t*, srsran_dl_sf_cfg_t*, srsran_chest_dl_res_t*, cf_t**) { return SRSRAN_SUCCESS; } // part of decode_fft_estimate here

static const uint8_t QM_OF[5] = {1, 2, 4, 6, 8};
// srsran_ue_dl_decode_pdsch (src/src/DL_Sniffer_PDSCH.cc:997): phase B for one grant of the current subframe
int srsran_ue_dl_decode_pdsch(srsran_ue_dl_t* q, srsran_dl_sf_cfg_t* sf, srsran_pdsch_cfg_t* cfg, srsran_pdsch_res_t data[SRSRAN_MAX_CODEWORDS])
{
  (void)sf;
  DlPriv* p = P(q);
  if (!p || !p->phy || !cfg || !data) return SRSRAN_ERROR_INVALID_INPUTS;
  const srsran_pdsch_grant_t& s = cfg->grant;
  ltephy_grant_t              g{};
  g.sf = 0, g.rnti = cfg->rnti, g.nof_tb = (uint8_t)s.nof_tb, g.nof_re = s.nof_re, g.pmi = s.pmi;
  g.tx_scheme = s.tx_scheme == SRSRAN_TXSCHEME_PORT0       ? LTEPHY_TX_PORT0
                : s.tx_scheme == SRSRAN_TXSCHEME_DIVERSITY ? LTEPHY_TX_DIVERSITY
                : s.tx_scheme == SRSRAN_TXSCHEME_CDD       ? LTEPHY_TX_CDD
                                                           : LTEPHY_TX_SPATIALMUX;
  for (int sl = 0; sl < 2; sl++)
    for (uint32_t prb = 0; prb < q->cell.nof_prb; prb++)
      if (s.prb_idx[sl][prb]) g.prb_mask[sl][prb >> 5] |= 1u << (prb & 31);
  for (int t = 0; t < SRSRAN_MAX_CODEWORDS; t++) {
    g.tb[t].enabled = s.tb[t].enabled, g.tb[t].tbs = s.tb[t].enabled ? s.tb[t].tbs : 0, g.tb[t].rv = (uint8_t)s.tb[t].rv;
    g.tb[t].qm = (unsigned)s.tb[t].mod < 5 ? QM_OF[s.tb[t].mod] : 0;
    data[t].crc = false, data[t].avg_iterations_block = 0.0f;
  }
  if (s.tb[0].enabled && s.tb[1].enabled) // srsran_ra_tb_t.cw_idx (dl_sniffer_pdsch.c:24): DCI 2/2A swap flag
    g.tb[0].cw_idx = (uint8_t)(s.tb[0].cw_idx & 1u), g.tb[1].cw_idx = (uint8_t)(s.tb[1].cw_idx & 1u);
  // soft buffers of the enabled TBs (a disabled TB's pointer may be left over from an earlier grant, DL_Sniffer_PDSCH.cc:968-970)
  const srsran_softbuffer_rx_t* sb[2] = {s.tb[0].enabled ? cfg->softbuffers.rx[0] : nullptr, s.tb[1].enabled ? cfg->softbuffers.rx[1] : nullptr};
  if (sb[1] == sb[0]) sb[1] = nullptr; // one buffer cannot hold both TBs: the second decodes without combining
  if ((sb[0] || sb[1]) && !p->harq_reserved) {
    if (ltephy_harq_reserve(p->phy, p->harq_cap) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
    p->harq_reserved = true, p->clear_harq();
  }
  for (int t = 0; t < 2; t++) {
    uint32_t slot = 0;
    g.tb[t].harq_op = harq_slot_of(p, sb[t], &slot), g.tb[t].harq_slot = slot;
  }
  if (ltephy_submit_grants(p->phy, &g, 1) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
  ltephy_tb_result_t   r[2]{};
  std::vector<uint8_t> pl(2 * 16000);
  if (ltephy_get_phase_b(p->phy, r, pl.data(), pl.size()) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
  for (int t = 0; t < SRSRAN_MAX_CODEWORDS; t++) {
    if (!r[t].payload_len) continue;
    data[t].crc = r[t].crc != 0, data[t].avg_iterations_block = (float)r[t].avg_iters;
    if (data[t].payload) memcpy(data[t].payload, pl.data() + r[t].payload_off, r[t].payload_len);
    if (sb[t]) cfg->softbuffers.rx[t]->tb_crc = data[t].crc;
  }
  return SRSRAN_SUCCESS;
}
int srsran_pdsch_decode(srsran_pdsch_t* q, srsran_dl_sf_cfg_t* sf, srsran_pdsch_cfg_t* cfg, srsran_chest_dl_res_t*, cf_t**, srsran_pdsch_res_t data[SRSRAN_MAX_CODEWORDS])
{
  if (!q || !q->b200) return SRSRAN_ERROR_INVALID_INPUTS;
  return srsran_ue_dl_decode_pdsch(static_cast<srsran_ue_dl_t*>(q->b200), sf, cfg, data);
}

// ---------------------------------------------------------------------------------------------------- uplink
static UlPriv* U(srsran_enb_ul_t* q) { return q ? static_cast<UlPriv*>(q->b200) : nullptr; }
int srsran_enb_ul_init(srsran_enb_ul_t* q, cf_t* in_buffer, uint32_t max_prb)
{
  if (!q || max_prb > SRSRAN_MAX_PRB) return SRSRAN_ERROR_INVALID_INPUTS;
  memset((void*)q, 0, sizeof(*q));
  q->in_buffer = in_buffer;
  q->b200      = new UlPriv();
  return SRSRAN_SUCCESS;
}
void srsran_enb_ul_free(srsran_enb_ul_t* q)
{
  UlPriv* u = U(q);
  if (!u) return;
  if (u->phy) ltephy_destroy(u->phy);
  delete u;
  memset((void*)q, 0, sizeof(*q));
}
// srsran_enb_ul_set_cell (src/src/SubframeWorker.cc:79,261): cell + the DMRS configuration of SIB2 (ULSchedule::set_config)
int srsran_enb_ul_set_cell(srsran_enb_ul_t* q, srsran_cell_t cell, srsran_refsignal_dmrs_pusch_cfg_t* pusch_cfg, srsran_refsignal_srs_cfg_t* srs_cfg)
{
  (void)srs_cfg;
  UlPriv* u = U(q);
  if (!u || cell.cp != SRSRAN_CP_NORM) return SRSRAN_ERROR_INVALID_INPUTS;
  if (u->phy) ltephy_destroy(u->phy), u->phy = nullptr;
  ltephy_cfg_t c{};
  c.nof_prb = cell.nof_prb, c.nof_ports = cell.nof_ports ? cell.nof_ports : 1, c.cell_id = cell.id, c.nof_rx = 1, c.max_subframes = 1, c.turbo_max_iter = 8;
  c.symbol_sz = (uint32_t)srsran_symbol_sz(cell.nof_prb);
  if (ltephy_create(&c, &u->phy) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
  q->cell = cell, q->chest.cell = cell, q->pusch.cell = cell, q->chest.b200 = q, q->pusch.b200 = q;
  u->sf_len = ltephy_sf_len(u->phy), u->g = 14 * 12 * cell.nof_prb;
  u->sym.assign(u->g, cfx_t{0, 0});
  u->payload.assign(16384, 0);
  q->sf_symbols = reinterpret_cast<cf_t*>(u->sym.data());
  if (pusch_cfg) u->dmrs = *pusch_cfg;
  ltephy_ul_cfg_t uc{};
  uc.n_dmrs1 = u->dmrs.cyclic_shift, uc.delta_ss = u->dmrs.delta_ss, uc.group_hopping = u->dmrs.group_hopping_en, uc.seq_hopping = u->dmrs.sequence_hopping_en;
  if (ltephy_set_ul_cfg(u->phy, &uc) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
  return SRSRAN_SUCCESS;
}
// srsran_enb_ul_fft (src/src/UL_Sniffer_PUSCH.cc:392): UL OFDM demodulation of the subframe in q->in_buffer (7.5 kHz shift removed)
void srsran_enb_ul_fft(srsran_enb_ul_t* q)
{
  UlPriv* u = U(q);
  if (!u || !u->phy || !q->in_buffer) return;
  const uint32_t tti = 0;
  u->have = u->fft_done = false;
  if (ltephy_submit_ul(u->phy, reinterpret_cast<const float*>(q->in_buffer), &tti, 1, nullptr, 0) != LTEPHY_SUCCESS) return;
  u->fft_done = true;
  ltephy_tb_result_t r{};
  ltephy_get_ul(u->phy, &r, nullptr, nullptr, 0);
  ltephy_tap(u->phy, LTEPHY_TAP_UL_SYM, u->sym.data(), u->sym.size() * sizeof(cfx_t));
}
static ltephy_ul_grant_t ul_grant_of(const srsran_pusch_cfg_t* cfg)
{
  const srsran_pusch_grant_t& s = cfg->grant;
  static const uint8_t dmrs2_map[8] = {0, 6, 3, 4, 2, 8, 10, 9}; // 36.211 Table 5.5.2.1.1-1
  ltephy_ul_grant_t    g{};
  g.sf = 0, g.rnti = cfg->rnti, g.qm = (unsigned)s.tb.mod < 5 ? QM_OF[s.tb.mod] : 0, g.rv = (uint8_t)(s.tb.rv & 3);
  g.L_prb = s.L_prb, g.n_prb = s.n_prb[0], g.n_prb_slot1 = s.n_prb[1], g.flags = LTEPHY_UL_FLAG_SLOT1, g.n_dmrs2 = dmrs2_map[s.n_dmrs & 7], g.tbs = s.tb.tbs;
  g.nof_ack = cfg->uci_cfg.ack[0].nof_acks, g.cqi_len = 0, g.ri_len = cfg->uci_cfg.cqi.ri_len;
  g.I_offset_ack = cfg->uci_offset.I_offset_ack, g.I_offset_cqi = cfg->uci_offset.I_offset_cqi, g.I_offset_ri = cfg->uci_offset.I_offset_ri;
  srsran_cqi_cfg_t cqi = cfg->uci_cfg.cqi;
  if (cqi.data_enable) g.cqi_len = (uint32_t)srsran_cqi_size(&cqi);
  return g;
}
static int run_pusch(srsran_enb_ul_t* q, UlPriv* u, srsran_ul_sf_cfg_t* sf, srsran_pusch_cfg_t* cfg)
{
  const ltephy_ul_grant_t g   = ul_grant_of(cfg);
  const uint32_t          tti = sf ? sf->tti : 0;
  // the symbols of srsran_enb_ul_fft stay on the device: only the grant travels
  if (ltephy_submit_ul(u->phy, u->fft_done ? nullptr : reinterpret_cast<const float*>(q->in_buffer), &tti, 1, &g, 1) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
  u->fft_done = true;
  if (ltephy_get_ul(u->phy, &u->res, &u->chest, u->payload.data(), u->payload.size()) != LTEPHY_SUCCESS) return SRSRAN_ERROR;
  u->grant = g, u->tti = tti, u->have = true;
  return SRSRAN_SUCCESS;
}
// srsran_chest_ul_estimate_pusch (UL_Sniffer_PUSCH.cc:256): DMRS estimate of the grant; the GPU pass that produces it also decodes the
// grant, srsran_pusch_decode (UL_Sniffer_PUSCH.cc:262) then returns that result
int srsran_chest_ul_estimate_pusch(srsran_chest_ul_t* c, srsran_ul_sf_cfg_t* sf, srsran_pusch_cfg_t* cfg, cf_t* input, srsran_chest_ul_res_t* res)
{
  (void)input;
  if (!c || !c->b200 || !cfg || !res) return SRSRAN_ERROR_INVALID_INPUTS;
  srsran_enb_ul_t* q = static_cast<srsran_enb_ul_t*>(c->b200);
  UlPriv*          u = U(q);
  if (!u || !u->phy) return SRSRAN_ERROR_INVALID_INPUTS;
  if (run_pusch(q, u, sf, cfg) != SRSRAN_SUCCESS) return SRSRAN_ERROR;
  res->noise_estimate = u->chest.noise, res->noise_estimate_dbm = 10.0f * log10f(u->chest.noise) + 30.0f, res->rsrp = u->chest.rsrp;
  res->snr_db = u->chest.snr_db, res->snr = powf(10.0f, u->chest.snr_db / 10.0f), res->ta_us = u->chest.ta_us, res->nof_re = 12 * cfg->grant.L_prb * 12;
  return SRSRAN_SUCCESS;
}
// the estimate's pass decoded exactly the grant run_pusch would build for cfg, in the same TTI
static_assert(sizeof(ltephy_ul_grant_t) == 36, "ltephy_ul_grant_t has padding: same_grant cannot memcmp it");
static bool same_grant(const UlPriv* u, const srsran_ul_sf_cfg_t* sf, const srsran_pusch_cfg_t* cfg)
{
  const ltephy_ul_grant_t g = ul_grant_of(cfg); // value-initialised and free of padding: memcmp compares every field
  return u->tti == (sf ? sf->tti : 0) && memcmp(&g, &u->grant, sizeof(g)) == 0;
}
int srsran_pusch_decode(srsran_pusch_t* pq, srsran_ul_sf_cfg_t* sf, srsran_pusch_cfg_t* cfg, srsran_chest_ul_res_t* channel, cf_t* sf_symbols, srsran_pusch_res_t* data)
{
  (void)channel, (void)sf_symbols;
  if (!pq || !pq->b200 || !cfg || !data) return SRSRAN_ERROR_INVALID_INPUTS;
  srsran_enb_ul_t* q = static_cast<srsran_enb_ul_t*>(pq->b200);
  UlPriv*          u = U(q);
  if (!u || !u->phy) return SRSRAN_ERROR_INVALID_INPUTS;
  if (!u->have || !same_grant(u, sf, cfg))
    if (run_pusch(q, u, sf, cfg) != SRSRAN_SUCCESS) return SRSRAN_ERROR;
  data->crc = u->res.crc != 0, data->avg_iterations_block = (float)u->res.avg_iters;
  if (data->data && u->res.payload_len) memcpy(data->data, u->payload.data() + u->res.payload_off, u->res.payload_len);
  if (cfg->softbuffers.rx) cfg->softbuffers.rx->tb_crc = data->crc;
  return SRSRAN_SUCCESS;
}
int  srsran_chest_ul_res_init(srsran_chest_ul_res_t* q, uint32_t) { if (q) memset((void*)q, 0, sizeof(*q)); return SRSRAN_SUCCESS; }
void srsran_chest_ul_res_free(srsran_chest_ul_res_t*) {}
// CQI payload size on PUSCH (36.212 5.2.2.6.1-3), wideband and higher-layer sub-band reports without PMI
int srsran_cqi_size(srsran_cqi_cfg_t* cfg)
{
  if (!cfg->data_enable) return 0;
  switch (cfg->type) {
    case SRSRAN_CQI_TYPE_WIDEBAND: return 4;
    case SRSRAN_CQI_TYPE_SUBBAND_HL: return 4 + (cfg->rank_is_not_one ? 4 : 0) + 2 * (int)cfg->N * (cfg->rank_is_not_one ? 2 : 1);
    case SRSRAN_CQI_TYPE_SUBBAND_UE: return 4 + 2 + (int)cfg->L;
    default: return 4 + 3;
  }
}

} // extern "C"
