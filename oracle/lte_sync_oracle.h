/*
 * lte_sync_oracle.h -- CPU ORACLE of the cell search (TEST INFRASTRUCTURE): PSS / SSS acquisition of a continuous FDD capture, DESIGN.md §2
 * ("cell search").  srsRAN's ue_cellsearch, which the reference calls from rf_search_and_decode_mib (src/src/LTESniffer_Core.cc:193-204), is not
 * available, so this restatement defines the contract that ltephy_cell_search meets bit for bit.  Built into oracle/liblteosync.so on top of
 * liblteoracle.so (lteo_det_sum) and the shared sequences of sim/lte_common.c (lte_pss, lte_sss).  Every float expression has a fixed evaluation
 * order (build with -ffp-contract=off).
 */
#ifndef LTE_SYNC_ORACLE_H
#define LTE_SYNC_ORACLE_H
#include "lte_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

#define LTEO_SYNC_BINS 9600       /* coarse bins per half-frame: 75 N / D with D = N / 128 */
#define LTEO_SYNC_PSR_MIN 2.5f    /* detection thresholds: noise-only captures stay below 1.7 on both (DESIGN.md §2) */
#define LTEO_SYNC_SSS_MIN 1.75f   /* a clean cell gives about 2: an SSS shares half its elements with the SSS of another N_ID_1 */
typedef struct {
  uint8_t  detected, n_id_2, pad[2];
  uint16_t n_id_1, pci;
  uint64_t frame_offset;
  uint32_t nof_half_frames;
  float    pss_peak, psr, sss_peak, sss_ratio, cfo_hz, cfo_re, cfo_im;
} lteo_cell_t;
/* intermediates, each may be NULL: coarse [3][9600] folded metrics, refined [3][2D-1], cfo [3][2] (re, im of S), sss [3][168][2] */
typedef struct {
  float *coarse, *refined, *cfo, *sss;
} lteo_sync_taps_t;
/* x: cf32 [nof_rx][L], antenna-major; N = symbol size (128 * D, 2^k or 3 * 2^k, <= 2048); out[3] sorted by pss_peak (descending, ties to the lower
 * N_ID_2).  Returns 0, or -2 for unsupported N / nof_rx or L < 75 N + N. */
int lteo_cell_search(uint32_t N, uint32_t nof_rx, const cf_t* x, uint64_t L, lteo_cell_t* out, const lteo_sync_taps_t* taps);


#ifdef __cplusplus
}
#endif
#endif
