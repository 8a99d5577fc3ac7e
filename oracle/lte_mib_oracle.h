/*
 * lte_mib_oracle.h -- CPU ORACLE for the MIB decode across the 40 ms PBCH period (TEST INFRASTRUCTURE).
 *
 * Restates srsRAN 21.10's PBCH soft combiner as the reference reaches it through srsran_ue_mib_decode in its DECODE_MIB state
 * (src/src/LTESniffer_Core.cc:382-396) and srsran_ue_mib_reset, with the rules of DESIGN.md §2 ("PBCH combining").  Written sequentially,
 * the way srsRAN is: a real buffer of up to four frames of soft bits per port count, frame_idx, and the nested hypothesis loops calling
 * lteo_dci_decode on the 1920-value rate-matching input.  The GPU evaluates the same hypotheses as a table, so the two formulations check
 * each other's state logic.  Builds into oracle/liblteomib.so, which links liblteoracle.so for lteo_dci_decode and the shared primitives.
 */
#ifndef LTE_MIB_ORACLE_H
#define LTE_MIB_ORACLE_H
#include "lte_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* the 480 QPSK soft bits of the PBCH of one subframe 0, equalised for nant = 1 (port 0, zero forcing) or 2 (SFBC) transmit ports: the first
 * half of lteo_pbch_decode for a given port count.  sym[nof_rx][14 nsc], ce[port * nof_rx + ant][14 nsc] as lteo_chest writes them; 0 ok */
int lteo_pbch_llr(const lte_cell_t* cell, const cf_t* const* sym, const cf_t* const* ce, uint32_t nant, float* llr /* [480] */);

typedef struct {
  uint8_t  found;      /* a hypothesis passed its CRC with the mask of the port count it was tried with */
  uint8_t  nof_ports;  /* that port count */
  uint8_t  sfn_offset; /* dst - src + window - 1 (0..6): 4 * (8 MSBs) + sfn_offset is the SFN of the newest frame */
  uint8_t  nof_frames; /* n: frames combined */
  uint8_t  src, dst;   /* first combined frame in the buffer, its position in the 40 ms period */
  uint8_t  window;     /* frame_idx: frames held when it passed */
  uint8_t  mib[24];    /* the 24 MIB bits */
  uint32_t sfn;        /* ((8 MSBs << 2) + sfn_offset) mod 1024 */
} lteo_mib_res_t;

typedef struct lteo_mib lteo_mib_t;
/* cell: nof_ports is the handle's port count (1 or 2; the buffers kept), nof_rx and nof_prb the grid of sym / ce, cell_id the scrambling */
lteo_mib_t* lteo_mib_create(const lte_cell_t* cell);
void        lteo_mib_destroy(lteo_mib_t* q);
void        lteo_mib_reset(lteo_mib_t* q); /* srsran_ue_mib_reset */
/* one subframe 0 (tti % 10 == 0) in stream order; search_ports: try 1 then 2 (if the cell has 2) ports, else only cell.nof_ports.
 * Returns res->found. */
int lteo_mib_decode(lteo_mib_t* q, uint32_t tti, const cf_t* const* sym, const cf_t* const* ce, int search_ports, lteo_mib_res_t* res);

#ifdef __cplusplus
}
#endif
#endif
