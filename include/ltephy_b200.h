/*
 * ltephy_b200.h -- C-ABI of the H100-native (sm_90a) LTE PHY decode path (libltephy_b200.so).
 *
 * Tier 1 (this file): batched, plain-C entry points.  A "batch" is n independent subframes (the
 * reference's unit of parallel work: one SubframeWorker each, src/src/Phy.cc:29-54).
 *   phase A  = what srsran_ue_dl_decode_fft_estimate + the per-candidate srsran_pdcch_dci_decode calls
 *              compute (src/src/DCISearch.cc:562, lib/src/phy/falcon_phch/falcon_pdcch.c:110-170):
 *              OFDM rx, CRS channel estimate, PCFICH, PDCCH LLRs, and the FULL blind-decode table
 *              T[location][payload size] -> {CRC remainder (RNTI), payload bits}
 *   search   = host replay of FALCON's tree walk (src/src/DCISearch.cc:102-528) over that table,
 *              in subframe order, with the RNTI history (lib/src/util/RNTIManager.cc)
 *   phase B  = srsran_ue_dl_decode_pdsch for every accepted DL grant (src/src/DL_Sniffer_PDSCH.cc:997)
 * Tier 2 (ltephy_srsran_compat.h): the srsRAN/FALCON names on top of tier 1.
 *
 * Error convention follows the reference (falcon_pdcch.c:121,131): 0 success, -1 error,
 * -2 invalid inputs.  A failed decode is NOT an error: it is crc == 0 in the result.
 * No CPU fallback exists: every entry point fails with LTEPHY_ERROR if no CUDA device is usable.
 */
#ifndef LTEPHY_B200_H
#define LTEPHY_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LTEPHY_SUCCESS 0
#define LTEPHY_ERROR -1
#define LTEPHY_ERROR_INVALID_INPUTS -2
#define LTEPHY_NEED_FULL_TABLE -3 /* survivor form insufficient for this walk (see ltephy_compact_t); nothing was consumed */

#define LTEPHY_MAX_PRB 110
#define LTEPHY_MAX_CCE 88
#define LTEPHY_MAX_LOC 160       /* MAX_CANDIDATES_BLIND, lib/include/falcon/phy/falcon_ue/falcon_ue_dl.h:39 */
#define LTEPHY_SEARCH_MAX_CCE 84 /* MAX_NUM_OF_CCE, lib/include/falcon/phy/falcon_phch/falcon_pdcch.h:36 */
#define LTEPHY_NOF_FORMATS 9     /* falcon_ue_all_formats, src/src/DCISearch.cc:84-95 */
#define LTEPHY_MAX_SIZES 8       /* distinct DCI payload sizes among the 9 formats */

typedef struct ltephy ltephy_t;

typedef struct {
  uint32_t nof_prb;        /* 15..100 (control region needs > 10) */
  uint32_t nof_ports;      /* CRS ports 1|2 */
  uint32_t cell_id;        /* PCI */
  uint32_t nof_rx;         /* rx antennas 1|2 */
  uint32_t max_subframes;  /* batch capacity */
  uint32_t max_grants;     /* phase-B capacity per batch (0 = 24 * max_subframes) */
  uint32_t turbo_max_iter; /* max-log-MAP iterations, >= 1 (SURVEY.md App. B.7) */
  int32_t  device;         /* CUDA device ordinal */
  uint32_t flags;          /* LTEPHY_FLAG_* */
  uint32_t symbol_sz;      /* FFT size of one OFDM symbol = samples per subframe / 15: 2^k or 3 * 2^k (2^k >= 128), at most
                              2048 and more than the 12 * nof_prb sub-carriers.
                              0: 256 at 15 PRB, 512 at 25, 1024 at 50, 2048 at 75 and 100 PRB (2048 = 30.72 Msps).  At 75 PRB that is not
                              the 3GPP rate: a 15 MHz capture at 23.04 Msps needs 1536.  srsRAN built without FORCE_STANDARD_RATE -- the
                              reference's default, CMakeLists.txt:289-292 -- samples 25 / 50 / 75 / 100 PRB at 384 / 768 / 1024 / 1536
                              (srsran_symbol_sz): pass that value then. */
  uint32_t phich_resources; /* phich-Resource of the MIB as srsran_phich_r_t (srsran_cell_t.phich_resources): 0 = Ng 1/6 (what the reference presets in file
                               mode, src/src/LTESniffer_Core.cc:242-247), 1 = 1/2, 2 = 1, 3 = 2.  Sets the PHICH groups of symbol 0 and with them the
                               CCE grid of the PDCCH. */
  uint32_t phich_length;    /* phich-Duration of the MIB (srsran_cell_t.phich_length): 0 normal, 1 extended (PHICH REGs in symbols 0, 1 and 2) */
  uint32_t reserved[4];
} ltephy_cfg_t;

#define LTEPHY_FLAG_SKIP_LOW_POWER 1u /* do not decode locations covering a CCE with mean|LLR| < 0.7 (they are never consulted) */

/* ---- phase A results --------------------------------------------------------------------- */
typedef struct {
  uint32_t tti;
  uint32_t cfi;
  uint32_t nof_cce;
  uint32_t nof_locations;
  float    pcfich_corr[3];
  float    noise[2][2], rsrp[2][2]; /* [port][ant] -> chest_res.snr_ant_port_db */
  float    noise_avg, rsrp_avg;
  float    cfo_re, cfo_im;
  float    snr_db; /* host: 10 log10f(rsrp_avg / noise_avg)   -> q->chest_res.snr_db (DCISearch.cc:568) */
  float    cfo;    /*                                          -> q->chest_res.cfo   (SubframeWorker.cc:203) */
  float    rb_power[LTEPHY_MAX_PRB];  /* linear mean RE power, antenna 0 (SubframePower.cc:18-58) */
  float    cce_power[LTEPHY_MAX_CCE]; /* mean |LLR| per CCE (falcon_pdcch.c:595-620) */
} ltephy_sf_info_t;

typedef struct {
  uint64_t bits;  /* payload, bit i of the DCI at position (63 - i) */
  uint16_t rnti;  /* CRC remainder = parity XOR crc16 (falcon_pdcch.c:142-143) */
  uint8_t  valid; /* 1 decoded; 0 skipped (no such location / all-zero LLRs / low power with the flag set) */
  uint8_t  pad[5];
} ltephy_cand_t;

/* Survivor form of one subframe's candidate table: the entries the FALCON walk can possibly act on.
 * An entry (location li, size column si) is listed iff the location has sufficient power (no CCE below 0.7,
 * src/src/DCISearch.cc:473-489) and at least one of
 *   - its RNTI lies in a search space that contains the location (srsran_pdcch_validate_location, falcon_pdcch.c:223-250),
 *   - its RNTI is 0 (includes undecoded all-zero entries),
 *   - it is the first child of a location whose entry in the same column decoded the same RNTI (shortcut test,
 *     DCISearch.cc:163-178).
 * Every other entry makes inspect_dci_location_recursively take the "rnti = 0; continue" branch whatever the RNTI
 * history holds, so the walk over the survivor form equals the walk over the full table (as long as no RNTI is
 * active with reason RAR: that path looks at every format-0 candidate and needs the full table).
 * list[loc[li].off + popcount(loc[li].mask & ((1 << si) - 1))] is the entry of (li, si) when bit si of mask is set.
 * In a listed entry pad[0] = search-space match (0 none, 1 ambiguous, 2 unique) | zero-RNTI << 2 | parent-match << 3,
 * pad[1] = li, pad[2] = si. */
#define LTEPHY_COMPACT_CAP 248
typedef struct {
  uint16_t off;   /* index of the location's first listed entry */
  uint8_t  mask;  /* bit si: column si of this location is listed */
  uint8_t  pad;   /* union of mask over the location and all locations nested in it (aggregation-level tree) */
} ltephy_cloc_t;
typedef struct {
  uint32_t      count;    /* survivors of this subframe; > LTEPHY_COMPACT_CAP: list is truncated, use the full table */
  uint32_t      reserved;
  ltephy_cloc_t loc[LTEPHY_MAX_LOC];
  uint8_t       pad[8];
  ltephy_cand_t list[LTEPHY_COMPACT_CAP];
} ltephy_compact_t;       /* 4624 bytes instead of 20480 */

/* ---- phase B ------------------------------------------------------------------------------ */
enum { LTEPHY_TX_PORT0 = 0, LTEPHY_TX_DIVERSITY = 1, LTEPHY_TX_CDD = 2, LTEPHY_TX_SPATIALMUX = 3 };

typedef struct {
  uint32_t sf;              /* index of the subframe inside the current batch */
  uint16_t rnti;
  uint8_t  tx_scheme;       /* LTEPHY_TX_* -- srsran_pdsch_grant_t.tx_scheme */
  uint8_t  nof_tb;
  uint32_t prb_mask[2][4];  /* per slot, bit (prb & 31) of word (prb >> 5) */
  uint32_t nof_re;          /* srsran_pdsch_grant_t.nof_re */
  uint32_t pmi;             /* srsran_pdsch_grant_t.pmi (spatial multiplexing codebook index) */
  struct {
    int32_t tbs;            /* bits, <= 0 disables the TB */
    uint8_t qm;             /* 2,4,6,8 */
    uint8_t rv;
    uint8_t enabled;
    uint8_t cw_idx;         /* srsran_ra_tb_t.cw_idx (dl_sniffer_pdsch.c:24): codeword this TB travels on -- 1 for TB 1 and 0 for TB 2 when both are
                               enabled and the DCI 2/2A swap flag is set, otherwise the TB's rank among the enabled ones */
    uint8_t  harq_op;       /* LTEPHY_HARQ_*: what pdsch_cfg->softbuffers.rx[t] is at DL_Sniffer_PDSCH.cc:955-985 */
    uint8_t  pad[3];
    uint32_t harq_slot;     /* slot of the HARQ store (ltephy_harq_reserve) for LTEPHY_HARQ_NEW / _RETX */
  } tb[2];
} ltephy_grant_t;
/* HARQ soft-combining store (reference src/src/HARQ.cc:71-151, the -h mode): per-slot int16 accumulators of the rate-dematcher in HBM */
#define LTEPHY_HARQ_NONE 0  /* scratch buffer, reset (srsran_softbuffer_rx_reset_tbs on buffer[i]) */
#define LTEPHY_HARQ_NEW  1  /* the slot is overwritten with this transmission (getHARQBuffer + reset_tbs) */
#define LTEPHY_HARQ_RETX 2  /* this transmission is added to the slot (getHARQBuffer, no reset) */
#define LTEPHY_HARQ_SLOT_BYTES (16u * 18448u * 2u) /* one transport block: up to 16 code blocks of 3 x 6148 values (+ padding) */

typedef struct {
  uint8_t  crc;             /* srsran_pdsch_res_t.crc */
  uint8_t  avg_iters;       /* mean turbo iterations over the code blocks (rounded up) */
  uint16_t nof_cb;
  uint32_t payload_off;     /* byte offset of srsran_pdsch_res_t.payload in the payload buffer */
  uint32_t payload_len;     /* tbs / 8 */
} ltephy_tb_result_t;

/* ---- accepted DCI (output of the host search) --------------------------------------------- */
typedef struct {
  uint32_t sf;
  uint16_t rnti;
  uint8_t  format;          /* index into the 9-format list */
  uint8_t  L;               /* after disambiguation */
  uint16_t ncce;
  uint16_t nof_bits;
  uint64_t bits;
  uint32_t histogram_value; /* hist_max_format_value handed to DCICollection::addCandidate */
} ltephy_dci_t;

/* ---- lifecycle ---------------------------------------------------------------------------- */
int  ltephy_create(const ltephy_cfg_t* cfg, ltephy_t** out);
void ltephy_destroy(ltephy_t* h);
const char* ltephy_last_error(void);

/* static geometry queries (host only) */
uint32_t ltephy_sf_len(const ltephy_t* h);                          /* cf32 samples per antenna-subframe */
uint32_t ltephy_nof_cce(const ltephy_t* h, uint32_t cfi);
uint32_t ltephy_nof_sizes(const ltephy_t* h);                       /* distinct DCI payload sizes */
uint32_t ltephy_dci_size(const ltephy_t* h, uint32_t format);       /* srsran_dci_format_sizeof */
uint32_t ltephy_size_index(const ltephy_t* h, uint32_t format);     /* format -> column of the candidate table */
uint32_t ltephy_locations(const ltephy_t* h, uint32_t cfi, uint16_t* ncce, uint8_t* L, uint32_t max); /* falcon_pdcch.c:321-356 */

/* ---- phase A ------------------------------------------------------------------------------ */
/* iq: n * nof_rx * sf_len cf32 (interleaved re,im), subframe-major then antenna; host memory
 * (pinned memory makes the copy asynchronous).  tti[i] = 10*sfn + sf_idx.  Asynchronous. */
int ltephy_submit_iq(ltephy_t* h, const float* iq, const uint32_t* tti, uint32_t n);
/* same, but iq already lives in device memory (used to time the kernels alone) */
int ltephy_submit_iq_device(ltephy_t* h, const void* iq_dev, const uint32_t* tti, uint32_t n);
/* blocks until phase A of the current batch is done and copies its results to the host:
 * info[n], cands[n][LTEPHY_MAX_LOC][LTEPHY_MAX_SIZES] */
int ltephy_get_phase_a(ltephy_t* h, ltephy_sf_info_t* info, ltephy_cand_t* cands);
/* same, fetching the survivor form (4.5 KB instead of 20 KB per subframe); comp[n].  ltephy_get_phase_a may still be
 * called afterwards for the full table (needed only for subframes whose count exceeds LTEPHY_COMPACT_CAP). */
int ltephy_get_phase_a_compact(ltephy_t* h, ltephy_sf_info_t* info, ltephy_compact_t* comp);
/* comp may be NULL above: the survivor forms then stay in the handle's pinned buffer, valid until the next submit_iq */
const ltephy_compact_t* ltephy_phase_a_compact_buffer(const ltephy_t* h);
/* sharded operation: device-to-device copies of the raw per-subframe records (ltephy_sf_info_t before the host-side
 * snr_db / cfo step) and of the survivor forms of the current batch into caller-owned device buffers, for an all-gather
 * without a host round trip; either pointer may be NULL.  Blocks until the copies are done. */
int ltephy_copy_phase_a_device(ltephy_t* h, void* dst_info_dev, void* dst_compact_dev);
/* host: fills noise_avg / rsrp_avg / snr_db / cfo of raw records from their per-path sums (what ltephy_get_phase_a does
 * before it returns; idempotent) */
void ltephy_finalize_info(ltephy_sf_info_t* info, uint32_t n, uint32_t nof_ports, uint32_t nof_rx);

/* ---- phase B ------------------------------------------------------------------------------ */
int ltephy_submit_grants(ltephy_t* h, const ltephy_grant_t* grants, uint32_t n);
/* results[n][2]; payload receives the TB bytes back to back */
int ltephy_get_phase_b(ltephy_t* h, ltephy_tb_result_t* results, uint8_t* payload, size_t payload_cap);
/* device-to-device copy of the raw payload buffer of the current phase B (transport block i at the running offset
 * sum_{j<i} ((tbs_j/8 + 6) & ~3), followed by its 3 CRC bytes) into dst_dev, for a collective without a host round trip
 * (the "single NCCL gather of decoded transport blocks").  Blocks until the copy is done. */
int ltephy_copy_phase_b_device(ltephy_t* h, void* dst_dev, size_t cap, size_t* nbytes);

/* ---- file-mode front matter (SURVEY 8f-1): what runs before the hot path when LTESniffer reads a recording --------------------------- */
/* constant carrier-frequency-offset correction of every subframe of samples, fused into the OFDM kernel: srsran_cfo_correct in srsran_ue_sync's
 * file mode (args.file_offset_freq -> srsran_ue_sync_init_file_multi, src/src/LTESniffer_Core.cc:252-257); phase restarts at each subframe;
 * 0 switches it off.  Applies to ltephy_submit_iq / _device of this handle (downlink). */
int ltephy_set_cfo(ltephy_t* h, float cfo_hz);
typedef struct {
  uint8_t  found;           /* SRSRAN_UE_MIB_FOUND */
  uint8_t  nof_ports;       /* 1, 2 or 4: from the CRC mask */
  uint8_t  sfn_offset;      /* position of this frame in the 40 ms PBCH period = SFN mod 4 */
  uint8_t  phich_length;    /* 0 normal, 1 extended    (srsran_cell_t.phich_length) */
  uint8_t  phich_resources; /* 0: 1/6, 1: 1/2, 2: 1, 3: 2 (srsran_cell_t.phich_resources); the value to create the decoding handle with
                               (ltephy_cfg_t.phich_resources), as the reference's live mode does through srsran_pbch_mib_unpack + srsran_ue_dl_set_cell */
  uint8_t  bch_payload[3];  /* the 24 MIB bits, first bit in bit 7 of byte 0 (bch_payload of srsran_ue_mib_decode, packed) */
  uint32_t nof_prb;         /* 6, 15, 25, 50, 75, 100 */
  uint32_t sfn;             /* (8 MSBs << 2) + sfn_offset, as LTESniffer_Core.cc:390-392 computes it */
} ltephy_mib_t;
/* PBCH decode of every subframe of the last ltephy_submit_iq whose tti % 10 == 0 (found = 0 elsewhere): srsran_ue_mib_decode +
 * srsran_pbch_mib_unpack (src/src/LTESniffer_Core.cc:382-396).  out[n].  The equaliser uses the handle's port count; one frame is decoded on its
 * own (no soft combining across the 40 ms period). */
int ltephy_mib_decode(ltephy_t* h, ltephy_mib_t* out);

/* nslots HARQ slots of LTEPHY_HARQ_SLOT_BYTES each (150 RNTIs x 8 processes x 2 TBs = 2400 slots = 1.4 GB); contents survive across batches */
int ltephy_harq_reserve(ltephy_t* h, uint32_t nslots);

/* ---- uplink: PUSCH (PUSCH_Decoder::decode / decode_run, src/src/UL_Sniffer_PUSCH.cc:250-263,389-392) ------------ */
typedef struct {
  uint32_t n_dmrs1;       /* cyclicShift of SIB2, 0..7, as ULSchedule::set_config hands it to srsRAN (dmrs_cfg.cyclic_shift, src/src/ULSchedule.cc:143);
                             n_DMRS^(1) = {0, 2, 3, 4, 6, 8, 9, 10}[cyclicShift] (36.211 Table 5.5.2.1.1-2) is looked up inside */
  uint32_t delta_ss;      /* groupAssignmentPUSCH */
  uint32_t group_hopping; /* groupHoppingEnabled    (dmrs_cfg.group_hopping_en, ULSchedule.cc:145): u = (f_gh(ns) + f_ss) mod 30 */
  uint32_t seq_hopping;   /* sequenceHoppingEnabled (dmrs_cfg.sequence_hopping_en, :146): v = c(ns) from 6 PRB on when group hopping is off */
} ltephy_ul_cfg_t;
typedef struct {
  uint32_t sf;            /* index of the UL subframe inside the submitted UL batch */
  uint16_t rnti;
  uint8_t  qm, rv;        /* srsran_pusch_grant_t.tb.mod (2, 4, 6 or 8) / .rv */
  uint32_t L_prb, n_prb;  /* contiguous allocation of slot 0; L_prb in the 2^a 3^b 5^c set (srsran_pusch_grant_t.L_prb / .n_prb[0]) */
  uint32_t n_dmrs2;       /* 36.211 Table 5.5.2.1.1-1 value of the DCI-0 cyclic shift field */
  int32_t  tbs;
  uint32_t n_prb_slot1;   /* with LTEPHY_UL_FLAG_SLOT1: first PRB of slot 1 (srsran_pusch_grant_t.n_prb[1]), which differs from n_prb under
                             type-1 PUSCH hopping (36.213 8.4.1); without the flag slot 1 uses n_prb */
  /* UCI multiplexed with the data (36.212 5.2.2.6 - 5.2.4), as the reference configures it (src/src/UL_Sniffer_PUSCH.cc:429-450) */
  uint8_t  nof_ack;       /* HARQ-ACK bits (0, 1, 2)            -> uci_cfg.ack[0].nof_acks */
  uint8_t  ri_len;        /* rank-indicator bits (0, 1)         -> uci_cfg.cqi.ri_len */
  uint16_t cqi_len;       /* CQI/PMI bits (0 = none)            -> srsran_cqi_size(&uci_cfg.cqi) */
  uint8_t  I_offset_ack, I_offset_cqi, I_offset_ri; /* beta-offset indices (36.213 Tables 8.6.3-1..3) -> uci_offset */
  uint8_t  flags;         /* LTEPHY_UL_FLAG_* */
} ltephy_ul_grant_t;
#define LTEPHY_UL_FLAG_SLOT1 1u
typedef struct {
  float noise, rsrp;      /* srsran_chest_ul_res_t.noise_estimate, RSRP (linear) */
  float snr_db;           /* .snr_db   (UL_Sniffer_PUSCH.cc:268) */
  float ta_us;            /* .ta_us    timing offset from the phase slope of the DMRS estimates (meas_ta_en, UL_Sniffer_PUSCH.cc:424,574) */
} ltephy_ul_chest_t;
int ltephy_set_ul_cfg(ltephy_t* h, const ltephy_ul_cfg_t* cfg);
/* iq_ul: n * sf_len cf32 of the UL carrier (one antenna: the reference uses antenna buffer 1); host memory.  iq_ul may be NULL when the previous
 * call demodulated the same n subframes: their symbols are decoded again with the new grants (srsran_enb_ul_fft once, decode_run per grant).
 * L_prb >= 3: the 1- and 2-PRB DMRS base sequences (36.211 Tables 5.5.1.2-1 / -2) are not carried. */
int ltephy_submit_ul(ltephy_t* h, const float* iq_ul, const uint32_t* tti, uint32_t n, const ltephy_ul_grant_t* grants, uint32_t ngrants);
/* results[ngrants], chest[ngrants]; payload receives the TB bytes back to back */
int ltephy_get_ul(ltephy_t* h, ltephy_tb_result_t* results, ltephy_ul_chest_t* chest, uint8_t* payload, size_t payload_cap);

/* ---- stand-alone batched kernels (BASELINE.json configs 3 and 4) --------------------------- */
/* llr: n subframes x 72*LTEPHY_MAX_CCE float LLRs (host); cfi[n]; fills cands[n][MAX_LOC][MAX_SIZES] */
int ltephy_dci_sweep(ltephy_t* h, const float* llr, const uint32_t* cfi, uint32_t n, ltephy_cand_t* cands);
/* ncb code blocks of size K, d: ncb x 3*(K+4) conditioned int16 streams (host);
 * bits: ncb x K decoded bits (one per byte); iters/crc_ok per code block; crc_type 0 none,1 CRC24A,2 CRC24B */
int ltephy_turbo_batch(ltephy_t* h, const int16_t* d, uint32_t K, uint32_t ncb, uint32_t max_iter, int crc_type, uint8_t* bits,
                       uint8_t* iters, uint8_t* crc_ok);

/* ---- debug / parity taps: copy an internal device buffer of the current batch to the host -- */
enum {
  LTEPHY_TAP_SYM = 0, /* cf32 [n][rx][14][12*nof_prb]          q->sf_symbols */
  LTEPHY_TAP_CE  = 1, /* cf32 [n][port][rx][14][12*nof_prb]    q->chest_res.ce */
  LTEPHY_TAP_LLR = 2, /* f32  [n][72*LTEPHY_MAX_CCE]           q->pdcch.llr */
  LTEPHY_TAP_PDSCH_LLR = 3, /* int16, all codewords of the submitted grants back to back */
  LTEPHY_TAP_TURBO_IN = 4,  /* int16 conditioned streams (debug) */
  LTEPHY_TAP_UL_SYM = 5     /* cf32 [n][14][12*nof_prb]  UL grid after srsran_enb_ul_fft */
};
int ltephy_tap(ltephy_t* h, int what, void* dst, size_t bytes);

/* timing of the last batch, from CUDA events on the library's stream (ms): [0] H2D+phase A, [1] phase B */
int ltephy_last_timing(ltephy_t* h, float ms[4]);
/* user markers on the library's stream: ltephy_mark(h, 0) ... ltephy_mark(h, 1); ltephy_mark_elapsed_ms
 * synchronises the stream and returns the device time between the two markers */
int   ltephy_mark(ltephy_t* h, int slot);
float ltephy_mark_elapsed_ms(ltephy_t* h);
/* algorithmic bytes of the turbo stage of the last phase B: sum over code blocks of 3(K+4)*2 + K/8 (SURVEY.md 8d),
 * number of code blocks and information bits */
int ltephy_last_turbo_work(ltephy_t* h, uint64_t* bytes, uint64_t* code_blocks, uint64_t* info_bits);
/* number of kernel launches issued by the library since creation */
uint64_t ltephy_launch_count(const ltephy_t* h);

#ifdef __cplusplus
}
#endif
#endif
