/* ltephy_compat_ext.h -- extensions of libltephy_srsran_compat beyond the srsRAN names.
 *
 * ltephy_compat_inject: hands the NEXT srsran_ue_dl_decode_fft_estimate call on q a ready-made phase-A result (per-subframe record,
 * blind-decode table T[location][size], PDCCH LLRs) instead of running the GPU.  It exists so that the reference's unmodified
 * blind search (src/src/DCISearch.cc, lib/src/phy/falcon_phch/falcon_pdcch.c) can be run on host-supplied tables -- the parity
 * tests use it to compare the reference's own walk with ltephy_search_batch on identical input, with or without a GPU. */
#ifndef LTEPHY_COMPAT_EXT_H
#define LTEPHY_COMPAT_EXT_H
#include "srsran/phy/ue/ue_dl.h"
#include "../include/ltephy_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
/* info: finalised record of the subframe; table: [LTEPHY_MAX_LOC][LTEPHY_MAX_SIZES]; llr: 72 * info->nof_cce floats (may be NULL: zeros) */
int ltephy_compat_inject(srsran_ue_dl_t* q, const ltephy_sf_info_t* info, const ltephy_cand_t* table, const float* llr);
/* the tier-1 PHY handle behind q (NULL before the first GPU subframe) */
ltephy_t* ltephy_compat_phy(srsran_ue_dl_t* q);

/* HARQ soft combining of srsran_ue_dl_decode_pdsch / srsran_pdsch_decode.  Each srsran_softbuffer_rx_t handed in through
 * pdsch_cfg->softbuffers.rx[t] for an enabled TB owns one slot of the handle's HARQ store (ltephy_harq_reserve):
 *   - softbuffers.rx[t] == NULL: the TB decodes on its own (LTEPHY_HARQ_NONE);
 *   - the buffer's b200_id differs from the one its slot was last decoded with, or the buffer has no slot: the slot is overwritten
 *     with this transmission (LTEPHY_HARQ_NEW).  srsran_softbuffer_rx_init / _reset / _reset_tbs / _reset_cb all renew b200_id, so a
 *     reset buffer, or a buffer freed and initialised again at the same address, starts empty;
 *   - the same b200_id: this transmission is added to the slot's soft values (LTEPHY_HARQ_RETX) -- the reference's retransmission,
 *     getHARQBuffer without a reset (DL_Sniffer_PDSCH.cc:955-990).
 * The store is reserved with its full capacity at the first decode that carries a soft buffer (one LTEPHY_HARQ_SLOT_BYTES slot each:
 * the default LTEPHY_COMPAT_HARQ_SLOTS = 150 RNTIs x 8 processes x 2 TBs + 2 scratch buffers, the reference's HARQ.cc, is 1.42 GB of
 * device memory).  When every slot is taken, the buffer decoded least recently gives up its slot: its next decode is a new transmission
 * even without a reset.  srsran_ue_dl_set_cell and srsran_ue_dl_free drop every slot.  If both TBs of a grant name the same buffer,
 * the second decodes on its own.
 * The store belongs to one srsran_ue_dl_t; it is not shared between objects.  Two consequences for a caller with several objects, such as
 * the reference's SubframeWorkers (DEFAULT_NOF_THREAD = 4, one ue_dl each, one HARQ object shared by all, workers taken from an
 * availability queue):
 *   - a retransmission combines only when it is decoded on the same object as the transmissions before it; on another object the buffer
 *     has no slot there, so it decodes on its own (correct, but without the combining gain, and which of the two happens depends on timing);
 *   - every object reserves its own store at its first decode with a soft buffer, which includes the reference's mode without HARQ (scratch
 *     buffer[i] with reset_tbs on every decode): 4 x 1.42 GB at the defaults.  A caller that only ever hands in those two scratch buffers
 *     needs ltephy_compat_harq_slots(q, 2) (1.2 MB): with two slots they never lose theirs, and a scratch buffer is reset before every
 *     decode anyway. */
#define LTEPHY_COMPAT_HARQ_SLOTS (150u * 8u * 2u + 2u)
/* capacity of q's HARQ store in slots (> 0).  Drops every slot; the store is reserved again at the next decode with a soft buffer. */
int ltephy_compat_harq_slots(srsran_ue_dl_t* q, uint32_t nslots);
#ifdef __cplusplus
}
#endif
#endif
