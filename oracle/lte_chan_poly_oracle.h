/* lte_chan_poly_oracle.h -- CPU oracle of the channeliser's rational carriers and integer sample formats (DESIGN.md §2 "channeliser"): one output
 * at a time, in the order the rule states, in plain C built with -ffp-contract=off.  ltephy_chan_run / _device with the plan's flags and iq_format
 * must equal lteo_chan_run_poly bit for bit, and ltephy_chan_design must equal lteo_chan_design_poly. */
#ifndef LTE_CHAN_POLY_ORACLE_H
#define LTE_CHAN_POLY_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Rational carriers and integer samples.  LTEO_CHAN_RATIONAL admits a carrier whose ratio 15 kHz * N / fs_in = L / M (in lowest terms) is not an
 * integer decimation 2..128 when L <= 1024, M <= 128 L, L <= 2 M and L * Kp <= 2^15; a carrier of integer ratio keeps the rule above (L = 1,
 * M = D, Ka = Kb = H).  Formats: cf32, sc16 (int16 I/Q, value * 2^-15) and sc8 (int8 I/Q, value * 2^-7). */
#define LTEO_CHAN_RATIONAL 1u
#define LTEO_IQ_CF32 0u
#define LTEO_IQ_SC16 1u
#define LTEO_IQ_SC8 2u
typedef struct {
  uint32_t L, M, Tp, Kp, Ka, Kb, P;
} lteo_chan_poly_t;

/* geometry and tables of one carrier: hp f32 [Tp] prototype (sum L), g cf32 [L][Kp] (g_phi[k] at [phi][k + Kb]), rot cf32 [P]; any may be NULL.
 * For an integer carrier hp, g and rot are lteo_chan_design's h, g and rot.  Returns 0, -2 for a refused carrier or unknown flag bits. */
int lteo_chan_design_poly(uint32_t fs_in, int32_t offset_hz, uint32_t N, uint32_t flags, lteo_chan_poly_t* out, float* hp, float* g, float* rot);

/* lteo_chan_run for integer and rational carriers alike, x in iq_format ([nof_rx][n] complex samples, antenna-major).  Output m of a rational
 * carrier needs capture samples floor(m M / L) - Ka .. floor(m M / L) + Kb; *next is the least max(0, floor(m' M / L) - Ka) over the carriers'
 * next outputs m'. */
int lteo_chan_run_poly(uint32_t fs_in, uint32_t flags, uint32_t iq_format, uint32_t nof_rx, uint32_t nof_carriers, const int32_t* offset_hz,
                       const uint32_t* N, const void* x, uint64_t first, uint64_t n, float* const* out, uint64_t cap, uint64_t* m_first, uint64_t* count,
                       uint64_t* next);

#ifdef __cplusplus
}
#endif
#endif
