/*
 * ltephy_search.h -- host half of the drop-in path (C-ABI, no GPU types): FALCON's blind-search
 * acceptance walk over the GPU candidate table, RNTI history, DCI -> PDSCH grant, and the one-call
 * batched pipeline.  Replaces, for this path:
 *   DCISearch::search / recursive_blind_dci_search / inspect_dci_location_recursively
 *                                       (reference src/src/DCISearch.cc:102-578)
 *   RNTIManager (lib/src/util/RNTIManager.cc) -- a faithful restatement kept private to the search
 *       object; a deployment that keeps the reference's own RNTIManager can instead run
 *       DCISearch.cc unchanged on top of the tier-2 shim (INTEGRATION.md)
 *   DCIMetaFormats::update_formats      (src/src/MetaFormats.cc:41-89)
 *   srsran_pdcch_validate_location      (lib/src/phy/falcon_phch/falcon_pdcch.c:223-250)
 *   srsran_dci_msg_to_trace_timestamp -> dl_sniffer_ra_dl_dci_to_grant + dl_sniffer_config_mimo
 *                                       (falcon_dci.c:148-352, dl_sniffer_pdsch.c:14-276)
 *   SubframeWorker::work                (src/src/SubframeWorker.cc:142-207) == ltephy_decode_subframes
 */
#ifndef LTEPHY_SEARCH_H
#define LTEPHY_SEARCH_H
#include "ltephy_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct ltephy_search ltephy_search_t;

/* DCIBlindSearchStats, src/include/PhyCommon.h:11-25 */
typedef struct {
  uint32_t nof_decoded_locations, nof_cce, nof_missed_cce, nof_subframes, nof_subframe_collisions_dw, nof_subframe_collisions_up,
      nof_locations;
} ltephy_search_stats_t;

/* unpacked DCI fields (subset of srsran_dci_dl_t the grant conversion needs) */
typedef struct {
  uint16_t rnti;
  uint8_t  format, alloc_type;
  uint8_t  mcs[2], rv[2], ndi[2];
  uint8_t  harq_pid, tpc, tb_cw_swap, pinfo;
  uint32_t nof_prb;
} ltephy_dci_fields_t;

#define LTEPHY_MIMO_NOT_SUPPORT -10 /* DL_SNIFFER_MIMO_NOT_SUPPORT */
#define LTEPHY_MIMO_PMI_WRONG -11   /* DL_SNIFFER_PMI_WRONG */
#define LTEPHY_MIMO_LAYER_WRONG -12 /* DL_SNIFFER_LAYER_WRONG */
#define LTEPHY_SEQ_NONE (~0ull)

/* activation reasons: rnti_manager_activation_reason_t, lib/include/falcon/util/rnti_manager_c.h */
enum { LTEPHY_ACT_UNSET = 0, LTEPHY_ACT_EVERGREEN, LTEPHY_ACT_RAR, LTEPHY_ACT_SHORTCUT, LTEPHY_ACT_HISTOGRAM, LTEPHY_ACT_OTHER };

/* geometry helper used by the search (implemented next to the PHY handle) */
void ltephy_cell_of(const ltephy_t* h, uint32_t* nof_prb, uint32_t* nof_ports, uint32_t* cell_id, uint32_t* nof_rx);
uint32_t ltephy_phich_resources(const ltephy_t* h); /* phich_resources | phich_length << 8 of the handle's configuration */
/* the control region as the PHY maps it: pdcch_idx[nof_cce * 36] = grid index l * 12 nof_prb + k of every RE of the PDCCH in CCE order for this CFI (what
 * srsran_pdcch_extract_llr walks; 36.211 6.8.5), pcfich_idx[16] the PCFICH REs; either may be NULL.  cap = room in pdcch_idx (uint16 elements).
 * phich_resources as for ltephy_search_create_cell_ng (| phich_length << 8). */
int ltephy_ctrl_region_map(uint32_t nof_prb, uint32_t nof_ports, uint32_t cell_id, uint32_t phich_resources, uint32_t cfi, uint16_t* pdcch_idx, uint32_t cap,
                           uint32_t* nof_cce, uint16_t* pcfich_idx);

/* histogram_threshold: DEFAULT_RNTI_HISTOGRAM_THRESHOLD = 5 (src/include/Settings.h:57).  The evergreen
 * (RA-RNTI, P/SI-RNTI for formats 1A and 1C) and forbidden (RNTI 0) ranges are seeded as
 * LTESniffer_Core.cc:398-417 does after the MIB. */
ltephy_search_t* ltephy_search_create(const ltephy_t* h, uint32_t histogram_threshold);
/* same without a GPU handle (host-only use: unit tests, or a search running beside a remote PHY) */
ltephy_search_t* ltephy_search_create_cell(uint32_t nof_prb, uint32_t nof_ports, uint32_t cell_id, uint32_t nof_rx, uint32_t histogram_threshold);
/* same for a cell whose MIB announces another PHICH configuration than Ng = 1/6, normal duration: the CCE counts per CFI follow from it.
 * phich_resources: ltephy_cfg_t.phich_resources | ltephy_cfg_t.phich_length << 8 */
ltephy_search_t* ltephy_search_create_cell_ng(uint32_t nof_prb, uint32_t nof_ports, uint32_t cell_id, uint32_t nof_rx, uint32_t phich_resources,
                                              uint32_t histogram_threshold);
void             ltephy_search_destroy(ltephy_search_t* s);
/* shortcut discovery on/off (DCISearch::setShortcutDiscovery), -m skip_secondary_meta_formats,
 * dci_format_split_update_interval_ms (0 = never re-split) */
void ltephy_search_config(ltephy_search_t* s, int shortcut, int skip_secondary, uint32_t update_interval);
/* MCS table of C-RNTI grants unknown (no MCSTracking answer yet): ltephy_grants_from_dcis then emits BOTH readings of such a DCI
 * -- 36.213 Table 7.1.7.1-1 first, Table 7.1.7.1-1A (256QAM) second, flagged with LTEPHY_GRANT_ALT_TABLE in grant_dci[] -- when
 * they differ, and ltephy_decode_subframes reports the first reading unless only the second passes a CRC (then crc = 2): the
 * batched form of "try the 64QAM table, then the 256QAM table" (src/src/DL_Sniffer_PDSCH.cc:1089-1210).  Off by default. */
void ltephy_search_speculate_256qam(ltephy_search_t* s, int on);
/* UL mode (-m 1): the downlink side only decodes what the uplink side needs.  ltephy_grants_from_dcis then selects as PDSCH_Decoder::decode_ul_mode does
 * (src/src/DL_Sniffer_PDSCH.cc:362-457) instead of decode_dl_mode: every RA-RNTI DCI (the Random Access Responses -> ltephy_rar_unpack), and the
 * format 1 / 1A DCIs of any RNTI but the SI-RNTI (target_rnti as ULSchedule::get_rnti, 0 = none), read with the 64QAM table only. */
void ltephy_search_set_ul_mode(ltephy_search_t* s, int on, uint16_t target_rnti);
/* rv of a format-1C SI-RNTI transmission at tti as PDSCH_Decoder::decode_SIB computes it (DL_Sniffer_PDSCH.cc:505-511: k = (SFN / 2) % 4, ceil(1.5 k) % 4);
 * ltephy_dci_to_grant itself writes 0 for format 1C as decode_dl_mode does (:891-898).  For a caller acquiring SIBs: grant.tb[0].rv = this. */
uint32_t ltephy_si_format1c_rv(uint32_t tti);
/* HARQ mode (-h): ltephy_grants_from_dcis keeps the C-RNTI grants whose first block has a reserved MCS (29-31; 28-31 of the 256QAM table; tbs = 0)
 * instead of applying decode_dl_mode's "tbs > 0" rule to them; ltephy_harq_prepare_grant then gives the block the size of its process' last
 * transmission as DCICollection::addCandidate does before that rule (src/src/DCICollection.cc:236-252).  Off by default. */
void ltephy_search_keep_reserved_mcs(ltephy_search_t* s, int on);
/* pusch-HoppingOffset of SIB2 (hopping_cfg.n_rb_ho, src/src/DCICollection.cc:166-168), used by ltephy_ul_dci_to_grant for type-1 hopping grants; default 0 */
void ltephy_search_set_ul_hopping(ltephy_search_t* s, uint32_t n_rb_ho);
#define LTEPHY_GRANT_ALT_TABLE 0x80000000u
void ltephy_search_add_evergreen(ltephy_search_t* s, uint16_t rnti_start, uint16_t rnti_end, uint32_t format_idx);
void ltephy_search_add_forbidden(ltephy_search_t* s, uint16_t rnti_start, uint16_t rnti_end, uint32_t format_idx);
/* rntiManager.activateAndRefresh, e.g. for T-CRNTIs found in a RAR (src/src/DL_Sniffer_PDSCH.cc:659,794) */
void ltephy_search_activate(ltephy_search_t* s, uint16_t rnti, uint32_t format_idx, int reason);

/* One subframe (must be called in subframe order).  cands: [LTEPHY_MAX_LOC][LTEPHY_MAX_SIZES] of this
 * subframe.  Writes the accepted DCIs in the order DCICollection::addCandidate would receive them. */
int ltephy_search_subframe(ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_cand_t* cands, uint32_t sf_in_batch, ltephy_dci_t* out,
                           uint32_t max_out, uint32_t* n_out);
/* same walk over the survivor form of the table (ltephy_compact_t); LTEPHY_NEED_FULL_TABLE if it cannot serve */
int ltephy_search_subframe_compact(ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_compact_t* comp, uint32_t sf_in_batch, ltephy_dci_t* out,
                                   uint32_t max_out, uint32_t* n_out);
/* host restatement of the GPU's survivor selection: full table of one subframe -> survivor form (tests, and callers
 * that obtained the table elsewhere) */
int ltephy_compact_from_table(const ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_cand_t* cands, ltephy_compact_t* out);
void ltephy_search_get_stats(const ltephy_search_t* s, ltephy_search_stats_t* st);
uint32_t ltephy_search_validate_location(uint32_t nof_cce, uint32_t ncce, uint32_t L, uint32_t sf_idx, uint16_t rnti);

/* RNTI-history taps (same semantics as the reference's rnti_manager_* C wrappers) */
int      ltephy_search_rnti_validate_and_refresh(ltephy_search_t* s, uint16_t rnti, uint32_t format_idx);
void     ltephy_search_rnti_add_candidate(ltephy_search_t* s, uint16_t rnti, uint32_t format_idx);
void     ltephy_search_rnti_step_time(ltephy_search_t* s);
uint32_t ltephy_search_rnti_frequency(const ltephy_search_t* s, uint16_t rnti, uint32_t format_idx);
uint32_t ltephy_search_rnti_assoc_format(const ltephy_search_t* s, uint16_t rnti);
int      ltephy_search_rnti_reason(const ltephy_search_t* s, uint16_t rnti);
int      ltephy_search_rnti_is_forbidden(const ltephy_search_t* s, uint16_t rnti, uint32_t format_idx);
int      ltephy_search_rnti_is_evergreen(const ltephy_search_t* s, uint16_t rnti, uint32_t format_idx);

/* DCI bits -> grant.  use_256qam_table: 0 = 36.213 Table 7.1.7.1-1, 1 = Table 7.1.7.1-1A.
 * Returns 0, LTEPHY_ERROR (unpack / allocation / TBS failure: the reference zeroes the RNTI,
 * falcon_dci.c:286-305) or LTEPHY_MIMO_*. */
int ltephy_dci_to_grant(const ltephy_search_t* s, const ltephy_dci_t* dci, uint32_t sf_idx, uint32_t cfi, int use_256qam_table, ltephy_grant_t* grant,
                        ltephy_dci_fields_t* fields);

/* ---- HARQ bookkeeping (host): the decisions of HARQ::is_retransmission / updateHARQRNTI (reference src/src/HARQ.cc:71-188) -------------- */
typedef struct ltephy_harq ltephy_harq_t;
#define LTEPHY_HARQ_NEW_TX 0      /* DL_SNIFFER_NEW_TX */
#define LTEPHY_HARQ_RE_TX 1       /* DL_SNIFFER_RE_TX */
#define LTEPHY_HARQ_FULL_BUFFER 2 /* DL_SNIFFER_HARQ_FULL_BUFFER: no entity left for this RNTI, decode without a store */
#define LTEPHY_HARQ_DECODED 3     /* DL_SNIFFER_DECODED: the block was already decoded, the reference disables the TB */
ltephy_harq_t* ltephy_harq_create(uint32_t max_rnti); /* DL_SNIFFER_MAX_HARQ_SIZE = 150 in the reference */
void           ltephy_harq_destroy(ltephy_harq_t* q);
/* classification of transport block tb (0 / 1) of a C-RNTI DCI seen at tti; *slot = (entity * 8 + pid) * 2 + tb for NEW_TX / RE_TX */
int ltephy_harq_classify(ltephy_harq_t* q, uint16_t rnti, uint32_t pid, uint32_t tb, uint32_t ndi, int32_t tbs, uint32_t tti, uint32_t* slot);
/* after the decode (only for NEW_TX / RE_TX, as at DL_Sniffer_PDSCH.cc:1015-1018) */
void ltephy_harq_update(ltephy_harq_t* q, uint16_t rnti, uint32_t pid, uint32_t tb, uint32_t ndi, uint32_t rv, int32_t tbs, uint32_t tti, int decoded);
/* HARQ::getlastTbs (src/src/HARQ.cc:262-274): size of the last recorded transmission of (rnti, pid, tb), 0 if none */
int32_t ltephy_harq_last_tbs(ltephy_harq_t* q, uint16_t rnti, uint32_t pid, uint32_t tb);
/* classify + fill grant->tb[t].harq_op / harq_slot of a C-RNTI grant from its DCI fields; DECODED disables the TB as the reference does.  A block with a reserved MCS (tbs = 0 after ltephy_dci_to_grant) first gets
 * the size of the process' last transmission (DCICollection.cc:236-252); it stays undecoded when there is none. */
int ltephy_harq_prepare_grant(ltephy_harq_t* q, const ltephy_dci_fields_t* f, uint32_t tti, ltephy_grant_t* grant, int status[2]);

/* DCI format 0 -> PUSCH grant (srsran_ra_ul_dci_to_grant as used at falcon_dci.c:222, and ulsniffer_ra_ul_dci_to_grant_256,
 * lib/src/phy/falcon_phch/ul_sniffer_pusch.c:138-172; type-1 hopping per ul_sniffer_ra_ul_grant_to_grant_prb_allocation, same file :20-87, with the
 * offset of ltephy_search_set_ul_hopping; a type-2 grant keeps the slot-0 PRBs in both slots as the reference does).  enable_64qam selects the MCS interpretation, i.e. one of the
 * three attempts of PUSCH_Decoder::decode (src/src/UL_Sniffer_PUSCH.cc:498-521): 0 = Table 8.6.1-1 capped at 16QAM, 1 = Table
 * 8.6.1-1 as is (64QAM), 2 = Table 8.6.1-3 (256QAM, Qm up to 8, MCS 26 -> TBS row 32A).  A caller that does not know the UE's
 * table submits the alternatives as separate grants of one ltephy_submit_ul batch and keeps the one whose CRC passes.
 * Returns 0, or LTEPHY_ERROR for an invalid hop / retransmission MCS / invalid RIV / L_prb outside the DFT set or < 3 / no TBS. */
int ltephy_ul_dci_to_grant(const ltephy_search_t* s, const ltephy_dci_t* dci, int enable_64qam, ltephy_ul_grant_t* grant);

/* What MCSTracking knows about the UE's uplink table (ul_sniffer_mod_tracking_t, lib/include/falcon/phy/falcon_phch/falcon_dci.h:115-122) */
#define LTEPHY_UL_MOD_16QAM_MAX 0
#define LTEPHY_UL_MOD_64QAM_MAX 1
#define LTEPHY_UL_MOD_256QAM_MAX 2
#define LTEPHY_UL_MOD_UNKNOWN 3
/* The decode attempts of PUSCH_Decoder::decode for one accepted format-0 DCI, in the reference's order (src/src/UL_Sniffer_PUSCH.cc:417-570), after its
 * investigate_valid_ul_grant filter (:894-918): MCS 21-28 -> the known table's reading, or 16QAM, 64QAM, 256QAM when unknown; MCS 0-20 -> 16QAM (= 64QAM)
 * or 256QAM, or both when unknown.  grants[3] / reading[3] (the enable_64qam value of each) are filled; returns their number (0: the reference does not
 * decode this DCI) or LTEPHY_ERROR_INVALID_INPUTS.  The reference stops at the first attempt whose CRC passes; submit all of them in one ltephy_submit_ul
 * batch and keep the first passing one in this order. */
int ltephy_ul_decode_plan(const ltephy_search_t* s, const ltephy_dci_t* dci, int mcs_mod, ltephy_ul_grant_t* grants, uint8_t* reading);

/* One MAC RAR of a Random Access Response PDU (decoded PDSCH of an RA-RNTI) with the msg-3 PUSCH grant it carries, as
 * PDSCH_Decoder::unpack_rar_response_ul_mode builds it (src/src/DL_Sniffer_PDSCH.cc:632-665) */
typedef struct {
  uint16_t t_crnti;       /* temporary C-RNTI: activate it on the search (ltephy_search_activate, DL_Sniffer_PDSCH.cc:659) */
  uint16_t ta;            /* 11-bit timing advance command */
  uint8_t  rapid;         /* preamble index of the subheader */
  uint8_t  hopping_flag, tpc, ul_delay, cqi_request; /* the other fields of the 20-bit grant (ul_sniffer_dci_rar_unpack, falcon_dci.c:648-657) */
  uint8_t  valid;         /* 1: grant below is usable (the allocation fits, L_prb is a DFT size >= 3, the MCS has a size) */
  ltephy_ul_grant_t grant; /* Table 8.6.1-1 reading; sf = 0: the PUSCH is on the air 6 subframes after the RAR (ULSchedule::get_rar_ul_tti,
                              src/src/ULSchedule.cc:126-138) and is decoded with the 16QAM reading only (UL_Sniffer_PUSCH.cc:531-569 with an empty 256QAM grant) */
} ltephy_rar_t;
/* pdu[len] -> out[*n_out]; *backoff = the backoff indicator if the PDU carries one, else -1 (backoff may be NULL).
 * LTEPHY_ERROR: malformed PDU; LTEPHY_ERROR_INVALID_INPUTS: null argument or more than max_out RARs. */
int ltephy_rar_unpack(const ltephy_search_t* s, const uint8_t* pdu, uint32_t len, ltephy_rar_t* out, uint32_t max_out, uint32_t* n_out, int* backoff);

/* The control-information layout ltephy_submit_ul uses for this grant (36.212 5.2.2.6 as srsRAN evaluates it, in float): modulation symbols Q' of HARQ-ACK,
 * rank indication and CQI / PMI, and the UL-SCH bits G left for the transport block.  Any output pointer may be NULL.  LTEPHY_ERROR_INVALID_INPUTS for a
 * grant without a size or with a reserved beta-offset index. */
int ltephy_ul_uci_layout(const ltephy_ul_grant_t* grant, uint32_t* qp_ack, uint32_t* qp_ri, uint32_t* qp_cqi, uint32_t* G);

/* Bits of the aperiodic CQI report as the reference configures it (UL_Sniffer_PUSCH.cc:434-445; no PMI, rank 1): cqi_type = srsran_cqi_type_t,
 * 0 wideband -> 4, 3 subbands configured by higher layers (the default, MCSTracking.cc:1538) -> 4 + 2 N with N = ul_sniffer_cqi_hl_get_no_subbands
 * (lib/src/phy/falcon_phch/dl_sniffer_pdsch.c:277-302).  Other types / nof_prb < 7: LTEPHY_ERROR_INVALID_INPUTS. */
int ltephy_ul_cqi_len(uint32_t nof_prb, int cqi_type);

/* What the reference keeps per RNTI for the uplink (MCSTracking::get_ue_config_rnti / find_tracking_info_RNTI_ul, used at UL_Sniffer_PUSCH.cc:433-452) */
typedef struct {
  uint16_t rnti;      /* 0: the default entry, for every RNTI without its own */
  uint8_t  mcs_mod;   /* LTEPHY_UL_MOD_* */
  uint8_t  I_offset_ack, I_offset_cqi, I_offset_ri; /* ue_config.uci_config; SubframeWorker::setup_default_ul_cfg: 10 / 8 / 11 */
  uint16_t cqi_len;   /* srsran_cqi_size of the aperiodic report this UE sends when a DCI-0 requests one; 0: the reference's default report type,
                         ltephy_ul_cqi_len(nof_prb, 3) */
} ltephy_ul_ue_cfg_t;
/* UL mode, whole batch: the accepted DCIs of a batch of downlink subframes -> the PUSCH decode attempts to submit 4 subframes later
 * (SubframeWorker.cc:296-345: nof_ack from the downlink DCIs of the same RNTI and subframe; ULSchedule's n + 4; UL_Sniffer_PUSCH.cc:417-570: validity
 * filter, CSI request, attempt order).  grants[k].sf = dcis[grant_dci[k]].sf + 4 (indices >= the batch length belong to the next uplink batch);
 * reading[k] = the enable_64qam value of attempt k; the attempts of one DCI are adjacent and in the reference's order -- keep the first whose CRC passes.
 * dcis[] as the search returns them (the DCIs of one subframe adjacent). */
int ltephy_ul_grants_from_dcis(const ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_dci_t* dcis, uint32_t nd, const ltephy_ul_ue_cfg_t* ue,
                               uint32_t n_ue, ltephy_ul_grant_t* grants, uint32_t* grant_dci, uint8_t* reading, uint32_t max_grants, uint32_t* n_grants);

/* Whole batch: IQ in host memory, in the handle's iq_format -> accepted DCIs + transport blocks.  seq orders concurrent calls on
 * different PHY handles that share one search object (the search runs strictly in seq order, starting
 * at 0); pass LTEPHY_SEQ_NONE for a single pipeline.  A call that fails, argument checks included, still passes its turn on.  A seq
 * whose turn is over (reused, or a restart from 0 on a search that has walked), or that another call on this search object is decoding,
 * returns LTEPHY_ERROR_INVALID_INPUTS at once and consumes no turn.
 *   info[n], cand_scratch[n*LTEPHY_MAX_LOC*LTEPHY_MAX_SIZES] (caller-owned, pinned if possible),
 *   dcis[max_dcis], tbs[2*max_dcis] (tbs[2*i+t] belongs to dcis[i]), payload. */
int ltephy_decode_subframes(ltephy_t* h, ltephy_search_t* s, const void* iq, const uint32_t* tti, uint32_t n, uint64_t seq, ltephy_sf_info_t* info,
                            ltephy_cand_t* cand_scratch, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis, ltephy_tb_result_t* tbs,
                            uint8_t* payload, size_t payload_cap);

/* same, with the IQ samples already resident in device memory (kernel-side throughput measurements) */
int ltephy_decode_subframes_device(ltephy_t* h, ltephy_search_t* s, const void* iq_dev, const uint32_t* tti, uint32_t n, uint64_t seq,
                                   ltephy_sf_info_t* info, ltephy_cand_t* cand_scratch, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis,
                                   ltephy_tb_result_t* tbs, uint8_t* payload, size_t payload_cap);

/* host wall time of the phases of the last decode call (ms): submit A, wait+fetch A, search, grants, submit B, wait+fetch B */
void ltephy_last_host_timing(double* ms8);

/* building blocks of the call above, exposed for sharded (multi-GPU) operation: every rank runs phase A on
 * its subframes, candidate tables are all-gathered, each rank replays the walk over ALL subframes in order
 * and keeps the grants of the subframes it owns (sf % mod == rem; grant.sf becomes sf / mod). */
int ltephy_search_batch(ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_cand_t* cands, uint32_t n, ltephy_dci_t* dcis, uint32_t max_dcis,
                        uint32_t* n_dcis);
int ltephy_search_batch_compact(ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_compact_t* comp, const ltephy_cand_t* full_or_null,
                                uint32_t n, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis);
/* 1 if a walk over these survivor forms may ask for the full tables: a subframe overflows, or some RNTI has ever been
 * RAR-activated on this search object.  Unlike the walk's own (exact) test this does not depend on how far the walk has
 * progressed, so the ranks of a sharded run can decide on a collective fetch of the full tables before walking. */
int ltephy_search_needs_full_table(const ltephy_search_t* s, const ltephy_compact_t* comp, uint32_t n);
int ltephy_grants_from_dcis(const ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_dci_t* dcis, uint32_t nd, uint32_t mod, uint32_t rem,
                            ltephy_grant_t* grants, uint32_t* grant_dci, uint32_t max_grants, uint32_t* n_grants);

#ifdef __cplusplus
}
#endif
#endif
