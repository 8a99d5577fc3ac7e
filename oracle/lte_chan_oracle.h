/* lte_chan_oracle.h -- CPU oracle of the channeliser (DESIGN.md §2 "channeliser"): one output at a time, in the order the rule states, in plain C
 * built with -ffp-contract=off.  ltephy_chan_run / _device must equal lteo_chan_run bit for bit, and ltephy_chan_taps must equal lteo_chan_design. */
#ifndef LTE_CHAN_ORACLE_H
#define LTE_CHAN_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* tables of one carrier (offset_hz, N) of a capture at fs_in: h f32 [T], g cf32 [T] (g[k] at index k + H), rot cf32 [P]; any array may be NULL.
 * Returns 0, or -2 for a carrier the rule refuses (D not an integer in 2..128, offset off the 1 kHz grid, band outside the capture, unknown N,
 * fs_in above 245.76 MHz). */
int lteo_chan_design(uint32_t fs_in, int32_t offset_hz, uint32_t N, float* h, float* g, float* rot, uint32_t* T, uint32_t* D, uint32_t* P);

/* x: cf32 [nof_rx][n], antenna-major: capture samples first .. first + n - 1.  For carrier c: out[c] receives cf32 [nof_rx][count[c]] (rows count[c]
 * apart; room for cap outputs per antenna), m_first[c] its first output index.  *next: the lowest capture sample the next call must include.
 * Returns 0, -2 for a refused configuration, -1 when an output range exceeds cap. */
int lteo_chan_run(uint32_t fs_in, uint32_t nof_rx, uint32_t nof_carriers, const int32_t* offset_hz, const uint32_t* N, const float* x, uint64_t first,
                  uint64_t n, float* const* out, uint64_t cap, uint64_t* m_first, uint64_t* count, uint64_t* next);

#ifdef __cplusplus
}
#endif
#endif
