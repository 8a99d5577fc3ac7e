/*
 * lte_sim.h -- synthetic eNB transmitter + channel: produces the seeded cf32 IQ captures that
 * BASELINE.json's configs call for (SURVEY.md section 8d) together with ground truth.
 * TEST / BENCH INPUT GENERATOR: not part of the product and not part of the oracle receiver.
 * The reference ships no IQ recording (SURVEY.md section 4); file layout matches what
 * srsran_filesource_read_multi feeds SubframeWorker buffers (src/src/SubframeWorker.cc:89):
 * one cf32 stream of lte_sf_len() samples per rx antenna per subframe.
 */
#ifndef LTE_SIM_H
#define LTE_SIM_H
#include "lte_common.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  lte_cell_t cell;
  uint64_t   seed;
  uint32_t   cfi;          /* 1..3 (fixed for the capture) */
  uint32_t   nof_ues;      /* C-RNTIs drawn uniformly from [0x0100, 0xFFF3) */
  uint32_t   dl_min, dl_max; /* DL DCIs per subframe */
  uint32_t   ul_min, ul_max; /* DCI format 0 grants per subframe (PDCCH only) */
  uint32_t   tm;           /* 1: format 1 (port0 / tx-div), 3: format 2A (CDD 2CW), 13: mix 1/1A/2A */
  uint32_t   mcs_min, mcs_max;
  uint32_t   si_period;    /* every n-th subframe carries an SI-RNTI 1A in common space (0 = never) */
  float      snr_db;
  uint32_t   chan_delay;   /* max per-path delay in samples (0 = flat) */
  uint32_t   fixed_L;      /* 0xFF = random aggregation level, else 0..3 */
  uint32_t   full_band;    /* 1: partition all PRBs between the scheduled UEs */
  uint32_t   alt_table;    /* 1: C-RNTI grants use the 256QAM MCS table */
  uint32_t   ul_pusch;     /* 1: DCI-0 grants are decodable PUSCH allocations (L_prb in the DFT set, >= 3, back to back from PRB 0, MCS <= 20) */
  uint32_t   tb_swap;      /* 1: two-TB DCIs (2 / 2A) set the TB-to-codeword swap flag at random */
  uint32_t   harq_retx;    /* 1: subframes with (tti / 8) odd repeat the DCIs and transport blocks of tti - 8 with rv = 2 (same NDI, same HARQ process) */
  uint32_t   pbch;         /* 1: subframe 0 of every frame carries the PBCH (MIB: bandwidth, PHICH, SFN = tti / 10) */
  float      cfo_hz;       /* carrier frequency offset applied to the generated samples (phase restarts every subframe, as srsran_cfo_correct sees it) */
  uint32_t   sync;         /* 1: subframes 0 and 5 carry the PSS (symbol 6) and SSS (symbol 5) on port 0 (36.211 6.11, FDD); 0 leaves those REs empty */
  uint32_t   reserved[1];
} lte_sim_cfg_t;

#define LTE_SIM_MAX_DCI 32
typedef struct {
  uint16_t rnti;
  uint8_t  format, L;
  uint16_t ncce;
  uint16_t nbits;
  uint8_t  bits[LTE_DCI_MAX_BITS];
  uint8_t  nof_tb, tx_scheme;
  uint8_t  qm[2], rv[2], mcs[2];
  int32_t  tbs[2];
  uint32_t payload_off[2]; /* byte offset into truth payload buffer */
  uint32_t nof_prb, nof_re;
} lte_sim_dci_truth_t;

typedef struct {
  uint32_t            tti;
  uint32_t            cfi;
  uint32_t            nof_dci;
  lte_sim_dci_truth_t dci[LTE_SIM_MAX_DCI];
  uint32_t            payload_len;
} lte_sim_truth_t;

typedef struct lte_sim lte_sim_t;

lte_sim_t* lte_sim_create(const lte_sim_cfg_t* cfg);
void       lte_sim_destroy(lte_sim_t* s);
/* iq: [nof_rx][sf_len] cf32; payload: caller buffer (>= 64 KiB) receiving the TB bytes back to back */
int lte_sim_subframe(lte_sim_t* s, uint32_t tti, cf_t* iq, lte_sim_truth_t* truth, uint8_t* payload, uint32_t payload_cap);
/* list of RNTIs of the simulated UEs */
uint32_t lte_sim_rntis(lte_sim_t* s, uint16_t* out, uint32_t max);

/* low level, used by unit tests: encode one DCI into E = 72<<L PDCCH bits */
void lte_sim_pdcch_encode(const uint8_t* dci_bits, uint32_t nbits, uint16_t rnti, uint32_t L, uint8_t* e);
/* encode one transport block into G bits (CRC, segmentation, turbo, rate matching) */
int lte_sim_dlsch_encode(const uint8_t* payload, uint32_t tbs, uint32_t rv, uint32_t G, uint32_t Qm, uint32_t NL, uint8_t* e);

#ifdef __cplusplus
}
#endif
#endif

/* ---- uplink: one subframe of PUSCH from several UEs on one rx antenna (the reference decodes PUSCH from
 * antenna buffer 1, src/src/UL_Sniffer_PUSCH.cc:391-392).  grants: already valid (lte_ul_dci_to_grant). */
#ifdef __cplusplus
extern "C" {
#endif
int lte_sim_ul_subframe(lte_sim_t* s, uint32_t tti, const lte_ul_cfg_t* ucfg, const lte_ul_grant_t* grants, uint32_t n, cf_t* iq /* [sf_len] */,
                        uint8_t* payload, uint32_t* payload_off, uint32_t payload_cap);
/* the same subframe received on nof_rx (1..LTE_MAX_ANT) antennas, iq [nof_rx][sf_len]: antenna a sees port 0's channel towards it (gain
 * h[a][0], delay[a][0]) and its own noise, drawn after antenna a - 1's, so antenna 0 equals lte_sim_ul_subframe's output */
int lte_sim_ul_subframe_rx(lte_sim_t* s, uint32_t tti, const lte_ul_cfg_t* ucfg, const lte_ul_grant_t* grants, uint32_t n, uint32_t nof_rx,
                           cf_t* iq /* [nof_rx][sf_len] */, uint8_t* payload, uint32_t* payload_off, uint32_t payload_cap);
#ifdef __cplusplus
}
#endif
