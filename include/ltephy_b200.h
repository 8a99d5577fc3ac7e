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

#define LTEPHY_MAX_BATCH_SUBFRAMES 65535 /* largest max_subframes ltephy_create accepts (65 s of air time per batch) */

typedef struct ltephy ltephy_t;

/* Sample formats of a narrowband or wideband input: interleaved I/Q, converted to float exactly where the kernels load them, so a run on integer
 * samples equals the cf32 run on value * 2^-15 (sc16) or value * 2^-7 (sc8) bit for bit (DESIGN.md §2 "integer samples").  Outputs -- the
 * tracker's cut, the channeliser's carrier streams -- are always cf32: a decode or search handle fed from them keeps iq_format = 0. */
#define LTEPHY_IQ_CF32 0u /* float32 */
#define LTEPHY_IQ_SC16 1u /* int16, value * 2^-15 */
#define LTEPHY_IQ_SC8 2u  /* int8, value * 2^-7 */

typedef struct {
  uint32_t nof_prb;        /* 15..100 (control region needs > 10) */
  uint32_t nof_ports;      /* CRS ports 1|2 */
  uint32_t cell_id;        /* PCI */
  uint32_t nof_rx;         /* rx antennas 1|2 */
  uint32_t max_subframes;  /* batch capacity, 1..LTEPHY_MAX_BATCH_SUBFRAMES */
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
  uint32_t ul_nof_rx;       /* receive antennas of the uplink carrier: 0 or 1 one antenna, 2 two (PUSCH combined over both, DESIGN.md §2 "uplink
                               receive diversity"); any other value is INVALID_INPUTS.  Sets the shape of ltephy_submit_ul / _device and
                               LTEPHY_TAP_UL_SYM. */
  uint32_t iq_format;       /* LTEPHY_IQ_CF32 (0), LTEPHY_IQ_SC16 or LTEPHY_IQ_SC8: the sample type of ltephy_submit_iq / _device and ltephy_submit_ul /
                               _device (and so of ltephy_decode_subframes*); any other value is INVALID_INPUTS */
  uint32_t reserved[2];
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
uint32_t ltephy_sf_len(const ltephy_t* h);                          /* complex samples per antenna-subframe (of the handle's iq_format) */
uint32_t ltephy_nof_cce(const ltephy_t* h, uint32_t cfi);
uint32_t ltephy_nof_sizes(const ltephy_t* h);                       /* distinct DCI payload sizes */
uint32_t ltephy_dci_size(const ltephy_t* h, uint32_t format);       /* srsran_dci_format_sizeof */
uint32_t ltephy_size_index(const ltephy_t* h, uint32_t format);     /* format -> column of the candidate table */
uint32_t ltephy_locations(const ltephy_t* h, uint32_t cfi, uint16_t* ncce, uint8_t* L, uint32_t max); /* falcon_pdcch.c:321-356 */

/* ---- phase A ------------------------------------------------------------------------------ */
/* iq: n * nof_rx * sf_len samples in the handle's iq_format (interleaved re,im), subframe-major then antenna; host memory
 * (pinned memory makes the copy asynchronous).  tti[i] = 10*sfn + sf_idx.  Asynchronous. */
int ltephy_submit_iq(ltephy_t* h, const void* iq, const uint32_t* tti, uint32_t n);
/* same, but iq already lives in device memory (used to time the kernels alone); INVALID_INPUTS for integer samples whose pointer is not aligned
 * to the sample (4 bytes sc16, 2 bytes sc8) */
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
 * own, any of the three CRC masks is accepted and the lowest position in the 40 ms period wins.  ltephy_mib_decode_combined is the
 * combining decoder; this call neither reads nor changes its state. */
int ltephy_mib_decode(ltephy_t* h, ltephy_mib_t* out);

/* MIB decode with soft combining across the 40 ms PBCH period: srsran_ue_mib_decode as the reference calls it in its DECODE_MIB state
 * (src/src/LTESniffer_Core.cc:382-396), whose PBCH decoder keeps the soft bits of up to four consecutive frames between calls and tries every
 * way to combine them.  The rules are DESIGN.md §2 ("PBCH combining"): the subframes 0 of the last submit are consumed in batch order; a frame
 * that does not follow the last one consumed (SFN 1023 -> 0 does) empties the buffer first; the first hypothesis that passes, in srsRAN's
 * order, wins and empties the buffer; with four frames held and no pass the oldest is dropped.  The state persists across submits and calls.
 * A hypothesis tried with k ports passes only if the CRC remainder is the mask of k ports; 4-port cells are not decoded.
 * flags: LTEPHY_MIB_SEARCH_PORTS tries 1 and then (on a 2-port handle) 2 ports for every frame, as srsRAN's cell search does; without it only
 * the handle's port count is tried (the reference's file mode).  out[n], one entry per subframe of the last submit; found = 0 on subframes
 * other than 0 and on frames where nothing passed (a pass whose bandwidth code is reserved also reports found = 0, after emptying the buffer).
 * Returns LTEPHY_ERROR_INVALID_INPUTS without a submit, with a NULL out or with unknown flags. */
#define LTEPHY_MIB_SEARCH_PORTS 1u
typedef struct {
  ltephy_mib_t mib;        /* as ltephy_mib_decode, except: nof_ports is the port count of the passing hypothesis, and sfn_offset is srsRAN's
                              dst - src + window - 1 (0..6), so that mib.sfn = ((8 MSBs << 2) + sfn_offset) mod 1024 is the SFN of this frame */
  uint8_t      nof_frames; /* n: frames combined (1..4) */
  uint8_t      src;        /* the first of them, as an index into the frames held (0 = oldest) */
  uint8_t      dst;        /* its position in the 40 ms period (0..3) */
  uint8_t      window;     /* frames held when the hypothesis passed, this one included (srsRAN's frame_idx) */
} ltephy_mib_comb_t;
int ltephy_mib_decode_combined(ltephy_t* h, uint32_t flags, ltephy_mib_comb_t* out);
/* empties the combining buffer of ltephy_mib_decode_combined: srsran_ue_mib_reset */
int ltephy_mib_reset(ltephy_t* h);

/* Cell search: the PSS / SSS half of rf_search_and_decode_mib (reference src/src/LTESniffer_Core.cc:193-204) on a continuous FDD recording with
 * normal CP.  For each N_ID_2 it finds the PSS timing, the carrier offset and N_ID_1 with the subframe-0 / subframe-5 decision, and from them the
 * first sample of a subframe 0 -- what ltephy_create (PCI), ltephy_submit_iq (subframe alignment) and ltephy_set_cfo need.  The algorithm and
 * its summation orders are DESIGN.md §2 ("cell search"); the CPU oracle lteo_cell_search defines the results bit for bit. */
typedef struct ltephy_sync ltephy_sync_t;
typedef struct {
  uint32_t symbol_sz;   /* N: 128, 256, 384, 512, 768, 1024, 1536 or 2048 samples per symbol (sample rate 15 kHz * N) */
  uint32_t nof_rx;      /* 1 or 2 antennas */
  uint64_t max_samples; /* longest recording per antenna this handle accepts (device memory is sized for it) */
  int32_t  device;      /* CUDA device ordinal */
  uint32_t iq_format;   /* LTEPHY_IQ_*: the sample type of ltephy_cell_search / _device; any other value is INVALID_INPUTS */
  uint32_t reserved[3];
} ltephy_sync_cfg_t;
typedef struct {
  uint8_t  detected;        /* psr >= 2.5 and sss_ratio >= 1.75 */
  uint8_t  n_id_2, pad[2];
  uint16_t n_id_1, pci;     /* n_id_1 = pci = 0xFFFF when no half-frame had both PSS and SSS inside the capture */
  uint64_t frame_offset;    /* first sample of a subframe 0, in [0, 150 * symbol_sz) */
  uint32_t nof_half_frames; /* half-frames whose PSS and SSS both lie inside the capture */
  float    pss_peak;        /* PSS metric at the refined timing (0..1) */
  float    psr;             /* folded coarse peak / the largest folded value more than 2 bins away */
  float    sss_peak, sss_ratio; /* best SSS hypothesis, and its ratio to the second best */
  float    cfo_hz;          /* carrier offset: the value to pass to ltephy_set_cfo */
  float    cfo_re, cfo_im;  /* the device sum it comes from (cfo_hz = atan2f(im, re) * 15000 / pi) */
} ltephy_cell_t;
int  ltephy_sync_create(const ltephy_sync_cfg_t* cfg, ltephy_sync_t** h);
void ltephy_sync_destroy(ltephy_sync_t* h);
/* iq: [nof_rx][nof_samples] samples in the handle's iq_format, antenna-major, host memory; HF + N <= nof_samples <= max_samples (HF = 75 N, 5 ms).
 * out[3]: one result per N_ID_2, by pss_peak descending, ties to the lower N_ID_2.  Blocks until done. */
int  ltephy_cell_search(ltephy_sync_t* h, const void* iq, uint64_t nof_samples, ltephy_cell_t out[3]);
/* same, with the samples already in device memory (integer samples aligned to the sample) */
int  ltephy_cell_search_device(ltephy_sync_t* h, const void* iq_dev, uint64_t nof_samples, ltephy_cell_t out[3]);
enum {
  LTEPHY_SYNC_TAP_COARSE  = 0, /* f32 [3][9600]       folded coarse metric per N_ID_2 */
  LTEPHY_SYNC_TAP_REFINED = 1, /* f32 [3][2 D - 1]    folded stride-1 metric around the coarse peak, D = N / 128 */
  LTEPHY_SYNC_TAP_CFO     = 2, /* f32 [3][2]          the CFO sum S (re, im) */
  LTEPHY_SYNC_TAP_SSS     = 3  /* f32 [3][168][2]     the SSS table A(N_ID_1, q) */
};
/* copies an intermediate of the last search; bytes must be at least its size */
int  ltephy_sync_tap(ltephy_sync_t* h, int what, void* dst, size_t bytes);

/* Tracking after acquisition: the track state of srsran_ue_sync_zerocopy (reference src/src/LTESniffer_Core.cc:365) on a recording.  From the
 * cell search's frame_offset and cfo_hz, the tracker follows the PSS of every half-frame, corrects the subframe start in whole samples and the
 * carrier offset with a first-order loop, and cuts every subframe into device memory, rotated by the carrier offset that held before it -- the
 * input ltephy_submit_iq_device / ltephy_decode_subframes_device take, with ltephy_set_cfo left at 0.  The rule and its summation orders are
 * DESIGN.md §2 ("tracking"); the CPU oracle lteo_track_* (oracle_track/) defines every record and cut sample bit for bit. */
typedef struct ltephy_track ltephy_track_t;
#define LTEPHY_TRACK_NO_CFO    1u /* keep cfo_hz at its initial value (the reference's disable_cfo) */
/* After 4 half-frames in a row without lock, search the cell again instead of cutting on: the find state of srsran_ue_sync_zerocopy.  The
 * tracker steps through the recording one frame at a time (windows of 150 N + N samples, each searched once it has been fed) with the cell
 * search of pci mod 3, cuts nothing meanwhile, and resumes at the first subframe boundary of the window where the cell is detected with this
 * pci.  Subframe numbers come from the SSS; the SFN continues by sample count, so after dropped samples only the MIB gives it (DESIGN.md §2). */
#define LTEPHY_TRACK_REACQUIRE 2u
typedef struct {
  uint32_t symbol_sz;     /* N, as for ltephy_sync_cfg_t */
  uint32_t nof_rx;        /* 1 or 2 antennas */
  uint32_t pci;           /* 0..503: the PSS tracked is N_ID_2 = pci mod 3 */
  uint32_t first_tti;     /* tti (10 sfn + subframe, 0..10239) of the subframe that starts at frame_offset */
  uint64_t frame_offset;  /* absolute first sample of that subframe */
  float    cfo_hz;        /* initial carrier offset (ltephy_cell_t.cfo_hz), |cfo_hz| <= 7500 */
  float    max_ppm;       /* largest sampling-clock offset the measurement windows are sized for (0 = 50) */
  uint32_t max_subframes; /* most subframes one push cuts (device memory is sized for it) */
  uint32_t flags;         /* LTEPHY_TRACK_* */
  int32_t  device;        /* CUDA device ordinal */
  uint32_t iq_format;     /* LTEPHY_IQ_*: the sample type of every push, the DL and the UL input alike (the cut is cf32); else INVALID_INPUTS */
  uint32_t reserved[4];
} ltephy_track_cfg_t;
#define LTEPHY_TRACK_LOCKED 1u /* subframe: the last half-frame measured before it was locked (or none was measured yet); half-frame: locked */
#define LTEPHY_TRACK_LOST   2u /* 4 or more half-frames in a row were not locked */
#define LTEPHY_TRACK_REACQUIRED 4u /* subframe: the first cut after the find state found the cell again (with LTEPHY_TRACK_LOCKED) */
typedef struct {
  int64_t  start;  /* absolute first sample of the subframe as cut */
  uint32_t tti;
  float    cfo_hz; /* carrier offset it was corrected with */
  uint32_t flags;  /* LTEPHY_TRACK_LOCKED / _LOST / _REACQUIRED */
  uint32_t index;  /* subframe number since frame_offset */
} ltephy_track_sf_t;
typedef struct {
  int64_t  tau;      /* expected first sample of the PSS useful part: start + 13 N / 2 */
  uint32_t index;    /* subframe number (tti mod 5 = 0) */
  int32_t  delta;    /* offset of the metric's argmax from tau, |delta| <= 9 N / 128 */
  float    peak;     /* metric at tau + delta */
  float    s_re, s_im; /* S = sum_a c2 conj(c1) at tau + delta */
  float    f_meas;   /* atan2f(s_im, s_re) * 15000 / pi */
  uint32_t flags;    /* LTEPHY_TRACK_LOCKED / _LOST, after this half-frame */
  uint32_t pad;
} ltephy_track_hf_t;
typedef struct {
  uint32_t                 nof_subframes, nof_half_frames;
  const ltephy_track_sf_t* sf;          /* [nof_subframes], host memory owned by the tracker, valid until the next push */
  const ltephy_track_hf_t* hf;          /* [nof_half_frames], likewise */
  const void*              iq_dev;      /* cf32 [nof_subframes][nof_rx][15 N] in device memory, valid until the next push */
  uint64_t                 next_sample; /* the first absolute sample the next push must still include */
  uint32_t                 remeasured;  /* half-frames whose metric window had to be computed again (diagnostic) */
  uint32_t                 finds;       /* find windows searched during this push (LTEPHY_TRACK_REACQUIRE) */
} ltephy_track_out_t;
int  ltephy_track_create(const ltephy_track_cfg_t* cfg, ltephy_track_t** h);
void ltephy_track_destroy(ltephy_track_t* h);
/* iq: [nof_rx][nof_samples] samples in the handle's iq_format, antenna-major, host memory, absolute samples first_sample .. first_sample + nof_samples - 1, with
 * first_sample <= the previous push's next_sample.  Cuts every subframe (up to max_subframes) that lies wholly inside what has been fed.  The
 * results do not depend on how the recording is split into pushes.  Blocks until the cut is complete. */
int  ltephy_track_push(ltephy_track_t* h, const void* iq, uint64_t first_sample, uint64_t nof_samples, ltephy_track_out_t* out);
/* same, with the samples already in device memory (integer samples aligned to the sample) */
int  ltephy_track_push_device(ltephy_track_t* h, const void* iq_dev, uint64_t first_sample, uint64_t nof_samples, ltephy_track_out_t* out);
/* The uplink carrier of the same radio (the reference's -m 1: channel 1 of srsran_ue_sync_zerocopy, src/src/LTESniffer_Core.cc:174-181,365), cut
 * at the downlink's tracked timing.  UL subframe k starts at start_k + ul_offset and is rotated, with the DL cut's rule, by
 * f_ul = (float)(cfo_hz_k * cfo_ratio).  cfo_ratio = 1 applies the downlink's offset unchanged, as srsRAN's ue_sync does to every channel; with one
 * reference oscillator f_UL / f_DL is the physical value (1747.5 / 1842.5 in band 3).  Call before the first push; afterwards only
 * ltephy_track_push_ul / _device are accepted (ltephy_track_push / _device are refused).  INVALID_INPUTS for 0 >= cfo_ratio, cfo_ratio > 2, NaN,
 * |ul_offset| >= 15 N or frame_offset + ul_offset < 0. */
typedef struct {
  double   cfo_ratio; /* f_UL / f_DL, in (0, 2] */
  int32_t  ul_offset; /* whole samples the UL subframe starts after the DL one, |ul_offset| < 15 N */
  uint32_t nof_rx;    /* UL receive antennas: 0 or 1 one antenna, 2 two (every antenna cut at the same start with the same rotation); else INVALID_INPUTS */
  uint32_t reserved[4];
} ltephy_track_ul_cfg_t;
int  ltephy_track_set_ul(ltephy_track_t* h, const ltephy_track_ul_cfg_t* cfg);
/* iq as ltephy_track_push; iq_ul: [ul nof_rx][nof_samples] in the same iq_format, antenna-major like iq, the same absolute samples.  A subframe is cut only when its
 * DL window and its UL window both lie inside what has been fed; out->next_sample is the lowest sample either pending window still needs.  The DL
 * records and cut equal those of a tracker without the uplink.  *ul_iq_dev: cf32 [nof_subframes][ul nof_rx][15 N] in device memory, valid until the
 * next push: the input ltephy_submit_ul_device takes with ltephy_cfg_t.ul_nof_rx = the same antenna count. */
int  ltephy_track_push_ul(ltephy_track_t* h, const void* iq, const void* iq_ul, uint64_t first_sample, uint64_t nof_samples, ltephy_track_out_t* out,
                          const void** ul_iq_dev);
/* same, with both carriers already in device memory (integer samples aligned to the sample) */
int  ltephy_track_push_ul_device(ltephy_track_t* h, const void* iq_dev, const void* iq_ul_dev, uint64_t first_sample, uint64_t nof_samples,
                                 ltephy_track_out_t* out, const void** ul_iq_dev);

/* Channeliser: several carriers from one wideband capture.  Each carrier is shifted to 0 Hz, low-pass filtered and decimated by an integer
 * D = fs_in / (15 kHz * symbol_sz) to the rate the cell search and the tracker take.  The filter, its arithmetic and the output range of a call are
 * DESIGN.md §2 ("channeliser"); the CPU oracles lteo_chan_run (oracle/lte_chan_oracle.h) and lteo_chan_run_poly (oracle/lte_chan_poly_oracle.h,
 * rational carriers and integer samples) define every output sample bit for bit.  Output m of a
 * carrier belongs to input time m D (zero group delay), so a cell's timing in a carrier stream is its timing in the capture divided by D.
 * The handle keeps no state between calls: the outputs do not depend on how the capture is split. */
#define LTEPHY_CHAN_MAX_CARRIERS 8
#define LTEPHY_CHAN_MAX_FS 245760000u
/* Rational carriers (opt-in).  With LTEPHY_CHAN_RATIONAL, a carrier whose 15 kHz * N / fs_in = L / M in lowest terms is not an integer decimation
 * 2..128 is resampled by L / M through a polyphase filter (DESIGN.md §2): accepted when L <= 1024, M <= 128 L (output at least fs_in / 128),
 * L <= 2 M (upsampling at most 2x) and its phase table L * Kp has at most 2^15 taps.  Output m belongs to capture time m M / L and needs capture
 * samples floor(m M / L) - Ka .. floor(m M / L) + Kb (ltephy_chan_design).  A carrier of integer ratio keeps the integer rule, flag or not. */
#define LTEPHY_CHAN_RATIONAL 1u
/* The input is in one of the LTEPHY_IQ_* formats (ltephy_chan_cfg_t.iq_format): complex sample i of antenna a at index a * nof_samples + i */
typedef struct ltephy_chan ltephy_chan_t;
typedef struct {
  int32_t  offset_hz; /* carrier centre minus capture centre, a multiple of 1000 */
  uint32_t symbol_sz; /* N of the carrier: 128, 256, 384, 512, 768, 1024, 1536 or 2048; its rate is 15 kHz * N */
} ltephy_chan_carrier_t;
typedef struct {
  uint32_t              fs_in;        /* capture rate in Hz, at most LTEPHY_CHAN_MAX_FS; fs_in / (15 kHz * N) an integer 2..128, or any ratio the
                                         rational rule accepts when flags has LTEPHY_CHAN_RATIONAL */
  uint32_t              nof_rx;       /* 1 or 2 antennas */
  uint32_t              nof_carriers; /* 1..LTEPHY_CHAN_MAX_CARRIERS */
  uint32_t              pad;
  ltephy_chan_carrier_t carrier[LTEPHY_CHAN_MAX_CARRIERS];
  uint64_t              max_samples;  /* longest call per antenna, 1..2^31 (device memory is sized for it) */
  int32_t               device;       /* CUDA device ordinal */
  uint32_t              flags;        /* 0 or LTEPHY_CHAN_RATIONAL */
  uint32_t              iq_format;    /* LTEPHY_IQ_CF32 (0), LTEPHY_IQ_SC16 or LTEPHY_IQ_SC8: the sample type of the input */
  uint32_t              reserved[3];
} ltephy_chan_cfg_t;
typedef struct {
  uint64_t    first;  /* carrier sample index of the first output of this call */
  uint64_t    count;  /* outputs per antenna */
  const void* iq_dev; /* cf32 [nof_rx][count] in device memory (what ltephy_cell_search_device / ltephy_track_push_device take), valid until the next call */
} ltephy_chan_out_t;
/* INVALID_INPUTS, before any device is looked for, for: a carrier whose D is not an integer in 2..128 (without LTEPHY_CHAN_RATIONAL) or that
 * breaks the rational limits (with it), an offset off the 1 kHz grid, a carrier whose widest occupied band (|offset_hz| + 90 kHz * the largest PRB
 * count of its N) reaches past fs_in / 2, an unknown N, 0 or more than 8 carriers, nof_rx other than 1 or 2, fs_in above LTEPHY_CHAN_MAX_FS,
 * max_samples 0 or above 2^31, unknown flag bits or an unknown iq_format. */
int  ltephy_chan_create(const ltephy_chan_cfg_t* cfg, ltephy_chan_t** h);
void ltephy_chan_destroy(ltephy_chan_t* h);
/* iq: [nof_rx][nof_samples] complex samples in the plan's iq_format, antenna-major, host memory: capture samples first_sample .. first_sample +
 * nof_samples - 1 (1 <= nof_samples <= max_samples).  out[nof_carriers]: every output m >= 0 of each carrier whose filter window [m D - H, m D + H]
 * ([n - Ka, n + Kb], n = floor(m M / L), for a rational carrier) has all its non-negative samples inside the call (samples before 0 count as zero).
 * *next_sample: the lowest capture sample the next call must still include for every carrier to continue without a gap; a carrier's first output
 * in that call may repeat outputs of this one.  Blocks until the outputs are complete. */
int  ltephy_chan_run(ltephy_chan_t* h, const void* iq, uint64_t first_sample, uint64_t nof_samples, ltephy_chan_out_t* out, uint64_t* next_sample);
/* same, with the samples already in device memory on the handle's device */
int  ltephy_chan_run_device(ltephy_chan_t* h, const void* iq_dev, uint64_t first_sample, uint64_t nof_samples, ltephy_chan_out_t* out,
                            uint64_t* next_sample);
/* host only, needs no device: the tables of carrier c (< nof_carriers) as the kernel uses them.  h: f32 [T] prototype, g: cf32 [T] band-pass taps g[k] at index
 * k + H, rot: cf32 [P] output rotation r[m mod P]; any of the three may be NULL.  *T (odd, H = (T - 1) / 2), *D and *P are always written.
 * A rational carrier is refused: its tables come from ltephy_chan_design. */
int  ltephy_chan_taps(const ltephy_chan_cfg_t* cfg, uint32_t c, float* h, float* g, float* rot, uint32_t* T, uint32_t* D, uint32_t* P);
typedef struct {
  uint32_t L, M; /* output rate / capture rate in lowest terms (L = 1, M = D for an integer carrier) */
  uint32_t Tp;   /* odd prototype length at rate L fs_in (T for an integer carrier), Hp = (Tp - 1) / 2 */
  uint32_t Kp;   /* taps per phase, Ka + Kb + 1 */
  uint32_t Ka, Kb; /* floor(Hp / L), ceil(Hp / L): output m reads capture samples floor(m M / L) - Ka .. floor(m M / L) + Kb */
  uint32_t P;    /* period of the output rotation */
} ltephy_chan_poly_t;
/* host only, needs no device: the geometry and tables of carrier c under the plan's flags, integer or rational.  hp: f32 [Tp] prototype (DC gain
 * L), g: cf32 [L][Kp] phase taps, g_phi[k] at [phi][k + Kb], rot: cf32 [P]; any of the three may be NULL.  For an integer carrier they equal
 * ltephy_chan_taps's h, g and rot. */
int  ltephy_chan_design(const ltephy_chan_cfg_t* cfg, uint32_t c, ltephy_chan_poly_t* out, float* hp, float* g, float* rot);

/* Raster scan: find the cells of a wideband capture without knowing where they are.  Every point of the 100 kHz E-UTRA channel raster (36.101
 * §5.7.2) inside the capture gets the channeliser's N = 128 stream (the central 62 sub-carriers hold the PSS and SSS of every bandwidth) and the
 * cell search of that stream.  Point p has offset o_p = 100 000 k - center_hz, for every integer k whose N = 128 carrier passes the channeliser's
 * band check (|o| + 540 kHz <= fs_in / 2) and lies in [lo_hz, hi_hz] (both 0: every offset), in ascending offset.  A point's three results are
 * exactly what ltephy_cell_search_device returns on what ltephy_chan_run (LTEPHY_CHAN_RATIONAL, the one carrier (o_p, 128)) makes of capture
 * samples [0, n): DESIGN.md §2 ("raster scan"), with lteo_chan_run_poly and lteo_cell_search as its oracle. */
typedef struct ltephy_scan ltephy_scan_t;
typedef struct {
  uint32_t fs_in;               /* capture rate in Hz, as for the channeliser; fs_in -> 1.92 MHz must pass its rational rule */
  uint32_t nof_rx;              /* 1 or 2 antennas */
  uint32_t iq_format;           /* LTEPHY_IQ_CF32 (0), LTEPHY_IQ_SC16 or LTEPHY_IQ_SC8: the sample type of the capture */
  uint32_t max_points_per_pass; /* raster points one batched pass holds; 0 = as many as a fixed device budget (2 GiB) holds.  No result depends on it */
  uint64_t center_hz;           /* absolute centre frequency of the capture, a multiple of 1 kHz */
  int32_t  lo_hz, hi_hz;        /* offset range of the points, lo_hz <= hi_hz; both 0 = every offset */
  uint64_t max_samples;         /* longest capture per antenna, up to 2^31; its N = 128 stream must hold a half-frame plus a symbol (9 728 samples) */
  int32_t  device;              /* CUDA device ordinal */
  uint32_t reserved[5];
} ltephy_scan_cfg_t;
typedef struct {
  int32_t       offset_hz; /* the raster point's offset from center_hz */
  uint32_t      pad;
  ltephy_cell_t cell;      /* its result, with frame_offset in N = 128 stream samples: at N' it is frame_offset * N' / 128, within one N = 128 sample */
} ltephy_scan_cell_t;
/* INVALID_INPUTS, before any device is looked for, for: center_hz off the 1 kHz grid, fs_in outside 1..LTEPHY_CHAN_MAX_FS or a ratio fs_in ->
 * 1.92 MHz the rational rule refuses, nof_rx other than 1 or 2, an unknown iq_format, lo_hz > hi_hz, a configuration without raster points,
 * and max_samples above 2^31 or too short for a half-frame plus a symbol at N = 128. */
int  ltephy_scan_create(const ltephy_scan_cfg_t* cfg, ltephy_scan_t** h);
void ltephy_scan_destroy(ltephy_scan_t* h);
/* iq: [nof_rx][nof_samples] samples in the handle's iq_format, antenna-major, host memory: capture samples 0 .. nof_samples - 1 (nof_samples <=
 * max_samples, its N = 128 stream at least a half-frame plus a symbol).  out[cap]: every result with detected = 1, by offset ascending, then by
 * pss_peak descending; *nof_cells: how many there are (only the first cap are written).  Blocks until done. */
int  ltephy_scan_run(ltephy_scan_t* h, const void* iq, uint64_t nof_samples, ltephy_scan_cell_t* out, uint32_t cap, uint32_t* nof_cells);
/* same, with the samples already in device memory on the handle's device (integer samples aligned to the sample) */
int  ltephy_scan_run_device(ltephy_scan_t* h, const void* iq_dev, uint64_t nof_samples, ltephy_scan_cell_t* out, uint32_t cap, uint32_t* nof_cells);
/* the three results of every point of the last run, point-major, each point's by pss_peak descending as ltephy_cell_search gives them:
 * out[3 * cap]; writes min(cap, points) points */
int  ltephy_scan_points(ltephy_scan_t* h, ltephy_cell_t* out, uint32_t cap);
/* host only, needs no device: the raster offsets of a configuration, ascending; *n: how many (only the first cap are written).  Fails as
 * ltephy_scan_create does, except that a configuration without points gives *n = 0. */
int  ltephy_scan_plan(const ltephy_scan_cfg_t* cfg, int32_t* offsets, uint32_t cap, uint32_t* n);

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
/* iq_ul: [n][A][sf_len] samples of the UL carrier in the handle's iq_format, A = ltephy_cfg_t.ul_nof_rx antennas (one antenna, A = 1, is what the reference decodes: antenna
 * buffer 1); host memory.  With A = 2 the PUSCH is estimated per antenna and equalised over both (DESIGN.md §2 "uplink receive diversity").
 * iq_ul may be NULL when the previous call demodulated the same n subframes: their symbols are decoded again with the new grants
 * (srsran_enb_ul_fft once, decode_run per grant).  L_prb >= 3: the 1- and 2-PRB DMRS base sequences (36.211 Tables 5.5.1.2-1 / -2) are not carried. */
int ltephy_submit_ul(ltephy_t* h, const void* iq_ul, const uint32_t* tti, uint32_t n, const ltephy_ul_grant_t* grants, uint32_t ngrants);
/* same, with iq_ul_dev [n][A][sf_len] already in device memory on the handle's device (integer samples aligned to the sample) (e.g. ltephy_track_push_ul's cut), read in place: the
 * caller keeps it alive until ltephy_get_ul returns.  NULL re-decodes the previous call's symbols, as above. */
int ltephy_submit_ul_device(ltephy_t* h, const void* iq_ul_dev, const uint32_t* tti, uint32_t n, const ltephy_ul_grant_t* grants, uint32_t ngrants);
/* the uplink twin of ltephy_set_cfo: a constant carrier-offset correction of every UL subframe (phase restarting at each subframe, the table of
 * ltephy_set_cfo), applied before the 7.5 kHz half-subcarrier rotation -- lteo_cfo_correct then lteo_ul_ofdm.  0 switches it off.  Kept apart
 * from ltephy_set_cfo's value; applies to every UL antenna.  For pre-aligned captures; the tracked cut of ltephy_track_push_ul is already rotated. */
int ltephy_set_ul_cfo(ltephy_t* h, float cfo_hz);
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
  LTEPHY_TAP_UL_SYM = 5,    /* cf32 [n][ul_nof_rx][14][12*nof_prb]  UL grid after srsran_enb_ul_fft */
  LTEPHY_TAP_PBCH_LLR = 6   /* f32  [frames][2][480]     PBCH soft bits (not descrambled) of the subframes 0 of the last ltephy_mib_decode or
                               ltephy_mib_decode_combined, in batch order, row [port count - 1]; ltephy_mib_decode writes only its handle's port count */
};
int ltephy_tap(ltephy_t* h, int what, void* dst, size_t bytes);
/* turbo rate-dematch tables of a code block of size K with F filler bits, as phase B uses them; no device needed.  LTEPHY_TAP_TURBO_IN
 * holds one buffer of 96*NW + 16 words (NW = ceil(K/32)) per code-block pair: the sys / p1 / p2 streams, stream index i at word
 * (i % 32) * NW + i / 32 of the stream, then 12 tail words and 4 pad words; code block 0 of the pair in the low 16 bits.  The tap pairs
 * code blocks of equal K in submission order, buffers in the order of their first code block (the decoder's own pairs are ltephy_turbo_pairing's).
 * order[k], k < *nn: word that soft bit k (and k + nn, k + 2 nn, ...) of redundancy version rv lands on (3*(K+4) entries of room).
 * inv[w] (96*NW + 16 entries): the word's position j in the order of rv 0, or LTEPHY_RM_FILLER / LTEPHY_RM_NONE; soft bit k of
 * redundancy version v lands on the word with j = (k + rot[v]) mod nn.  Returns -2 for a K that is not a turbo block size. */
#define LTEPHY_RM_FILLER 0xFFFEu /* filler bit of the systematic or first parity stream: a known 0 */
#define LTEPHY_RM_NONE   0xFFFFu /* ragged window slot or pad word: no soft bit lands here */
int ltephy_rm_turbo_tables(uint32_t K, uint32_t F, uint32_t rv, uint32_t* order, uint32_t* nn, uint16_t* inv, uint32_t* rot);

/* Turbo pairs of phase B (host only, needs no device): code block i of a batch -- block size K[i], TBS tbs[i] and rate-matched bits G[i]
 * of its transport block -- is decoded in half half[i] (0 or 1) of pair pair[i], *npairs pairs in all.  Both halves of a pair have the
 * same K.  Blocks of one K are paired in the order of their code rate TBS / G (in steps of 2^-16, saturating at 1), highest first, then
 * by index: a pair decodes until both halves are done, and blocks of similar rate tend to need similar iteration counts.  Pairs are
 * numbered by K (largest first), then in that order.  Returns -2 for bad arguments or a K that is not a turbo block size. */
int ltephy_turbo_pairing(uint32_t ncb, const uint32_t* K, const uint32_t* tbs, const uint32_t* G, uint32_t* pair, uint32_t* half, uint32_t* npairs);

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
