/*
 * lte_pusch_rx_oracle.h -- CPU ORACLE of the PUSCH receive path with one or two receive antennas (TEST INFRASTRUCTURE).
 *
 * DESIGN.md §2 ("uplink receive diversity") defines the rule: lteo_pusch_decode (oracle/lte_oracle.h) run per antenna up to the smoothed
 * DMRS estimates and the per-slot sums, then the chest figures from the sums over (antenna, slot) and the equaliser of the downlink's port 0,
 * sum_a conj(h_a) y_a / sum_a |h_a|^2.  It is written apart from lteo_pusch_decode, which stays the one-antenna reference: at nof_rx = 1 the
 * two agree bit for bit, and the tests check that they do.  Every float expression has a fixed evaluation order (-ffp-contract=off) so that
 * the CUDA path can be compared bit for bit.
 */
#ifndef LTE_PUSCH_RX_ORACLE_H
#define LTE_PUSCH_RX_ORACLE_H
#include "../oracle/lte_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif
/* one PUSCH grant received on nof_rx (1 or 2) antennas: sym[a] is antenna a's grid [14][12 nof_prb] (lteo_ul_ofdm).  llr_out (optional) receives
 * the nof_bits descrambled, de-interleaved int16 soft bits, eq_out (optional) the equalised data symbols [12][M] before the IDFT.  0 ok, -1 bad
 * grant or antenna count, -2 DMRS failure. */
int lteo_pusch_decode_rx(const lte_cell_t* cell, const lte_ul_cfg_t* ucfg, uint32_t sf_idx, const lte_ul_grant_t* g, const cf_t* const* sym,
                         uint32_t nof_rx, uint32_t max_iter, uint8_t* payload, int* crc_ok, lteo_ul_chest_t* chest, int16_t* llr_out, cf_t* eq_out);
#ifdef __cplusplus
}
#endif
#endif
