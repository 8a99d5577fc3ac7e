/*
 * lte_track_oracle.h -- CPU oracle of the tracker (DESIGN.md §2, "tracking"): PSS tracking of every half-frame after the cell search, whole-
 * sample timing corrections with a drift estimate, a first-order carrier-offset loop, and the cut of every subframe rotated by the carrier
 * offset that held before it; with LTEO_TRACK_REACQUIRE, after a loss, the cell search (lteo_cell_search) of the known PCI frame by frame
 * until it is found again.  Plain C, one subframe at a time, every float sum in the order DESIGN.md states; the product (ltephy_track_*,
 * include/ltephy_b200.h) must equal its records and cut samples bit for bit.  The records have the layout of ltephy_track_sf_t / _hf_t.
 */
#pragma once
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  float re, im;
} lteo_tcf_t;

#define LTEO_TRACK_NO_CFO     1u
#define LTEO_TRACK_REACQUIRE  2u     /* after a loss, search the cell again frame by frame and resume at the new timing (DESIGN.md §2) */
#define LTEO_TRACK_LOCKED     1u
#define LTEO_TRACK_LOST       2u
#define LTEO_TRACK_REACQUIRED 4u     /* subframe record: the first one cut after a successful find */
#define LTEO_TRACK_P      4u     /* locked half-frames per timing correction */
#define LTEO_TRACK_ALPHA  0.05f  /* gain of the carrier-offset loop */
#define LTEO_TRACK_MISS   4u     /* half-frames in a row without lock after which records are flagged lost */
#define LTEO_TRACK_LOCK_K 20.0f  /* a half-frame is locked when its peak metric reaches LTEO_TRACK_LOCK_K / N */

typedef struct {
  int64_t  start;
  uint32_t tti;
  float    cfo_hz;
  uint32_t flags;
  uint32_t index;
} lteo_track_sf_t;

typedef struct {
  int64_t  tau;
  uint32_t index;
  int32_t  delta;
  float    peak;
  float    s_re, s_im;
  float    f_meas;
  uint32_t flags;
  uint32_t pad;
} lteo_track_hf_t;

typedef struct lteo_track lteo_track_t;

/* N, A (1 or 2), pci, first_tti, frame_offset, cfo_hz and flags as in ltephy_track_cfg_t; NULL on invalid arguments */
lteo_track_t* lteo_track_create(uint32_t N, uint32_t A, uint32_t pci, uint32_t first_tti, uint64_t frame_offset, float cfo_hz, uint32_t flags);
void          lteo_track_destroy(lteo_track_t* t);
/* x: [A][n] absolute samples first .. first + n - 1 (first <= *next of the previous call).  Processes up to max_sf subframes that lie wholly
 * inside; writes their records to sf (and the half-frame records to hf, at most max_sf / 5 + 1), their cut samples to cut [k][A][15 N] (may be
 * NULL), the counts to *nsf / *nhf and the next sample the caller must still include to *next.  0, or -2 on invalid arguments.  With
 * LTEO_TRACK_REACQUIRE, a find window [f0, f0 + 150 N + N) is searched with lteo_cell_search once all of it has been fed. */
int lteo_track_push(lteo_track_t* t, const lteo_tcf_t* x, uint64_t first, uint64_t n, uint32_t max_sf, lteo_track_sf_t* sf, uint32_t* nsf,
                    lteo_track_hf_t* hf, uint32_t* nhf, lteo_tcf_t* cut, uint64_t* next);
/* the number of find windows searched since the tracker was created (LTEO_TRACK_REACQUIRE) */
uint32_t lteo_track_finds(const lteo_track_t* t);
/* the uplink carrier (ltephy_track_set_ul): before the first push, 0 < cfo_ratio <= 2, |ul_offset| < 15 N, frame_offset + ul_offset >= 0; 0 or -2.
 * After it lteo_track_push is refused and lteo_track_push_ul takes both carriers. */
int lteo_track_set_ul(lteo_track_t* t, double cfo_ratio, int32_t ul_offset);
/* the same with nof_rx UL antennas (0 or 1: one, 2: two; else -2): lteo_track_push_ul then takes x_ul [nof_rx][n] and writes cut_ul
 * [k][nof_rx][15 N], every antenna cut and rotated as the one antenna is */
int lteo_track_set_ul_rx(lteo_track_t* t, double cfo_ratio, int32_t ul_offset, uint32_t nof_rx);
/* lteo_track_push with x_ul [n] (one antenna, the same absolute samples): a subframe is processed only when its DL window start .. start + 15 N - 1
 * and its UL window start + ul_offset .. start + ul_offset + 15 N - 1 both lie inside what was fed.  UL subframe k is x_ul from start_k + ul_offset,
 * rotated as the DL cut with f_ul = (float)(cfo_hz_k * cfo_ratio), into cut_ul [k][15 N] (may be NULL).  After lteo_track_set_ul_rx with nof_rx = 2,
 * x_ul is [nof_rx][n], antenna-major, and cut_ul [k][nof_rx][15 N], every antenna cut and rotated as above.  *next is the lower of start and
 * start + ul_offset of the next subframe. */
int lteo_track_push_ul(lteo_track_t* t, const lteo_tcf_t* x, const lteo_tcf_t* x_ul, uint64_t first, uint64_t n, uint32_t max_sf, lteo_track_sf_t* sf,
                       uint32_t* nsf, lteo_track_hf_t* hf, uint32_t* nhf, lteo_tcf_t* cut, lteo_tcf_t* cut_ul, uint64_t* next);

#ifdef __cplusplus
}
#endif
