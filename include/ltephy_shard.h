/*
 * ltephy_shard.h -- sharded (multi-GPU, one process per GPU) operation of the decode path, C-ABI.
 *
 * Replaces, for this path, the reference's hand-off of subframes to a pool of workers and the in-order collection of
 * their results (src/src/Phy.cc:29-109: getAvail / putAvailImmediate / putPending / joinPending;
 * src/src/SubframeWorker.cc:142-207 is the per-worker body): global subframe g of a batch belongs to rank g % world
 * ("independent subframes shard round-robin across the GPUs", BASELINE.json north_star).
 *
 *   phase A      local, on the rank's own subframes
 *   exchange     the survivor forms of the candidate tables, packed to their used length on the GPU (ltephy_packed_hdr_t +
 *                location records + survivor list: about 1.8 KB per busy 20 MHz subframe instead of 5.4 KB), are all-gathered
 *                device to device over NCCL and copied to the host once
 *   walk         every rank replays FALCON's walk (src/src/DCISearch.cc:102-528) over ALL subframes in global order -- the RNTI
 *                history (lib/src/util/RNTIManager.cc) is sequential by nature and is never partitioned -- and keeps the grants
 *                of the subframes it owns
 *   phase B      local
 *   gather       ONE NCCL gather of the decoded transport blocks (payload, CRC flags, placement) to rank 0
 *
 * Several host threads may drive different PHY handles of one rank concurrently (batch k on handle k % T): the exchange,
 * the walk and the gather are each entered strictly in batch order (`seq`), on every rank, so all ranks issue the same
 * sequence of collectives; everything else overlaps.
 *
 * NCCL is loaded at run time (dlopen libnccl.so.2): the library itself links without it.
 */
#ifndef LTEPHY_SHARD_H
#define LTEPHY_SHARD_H
#include "ltephy_b200.h"
#include "ltephy_search.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct ltephy_shard ltephy_shard_t;

#define LTEPHY_SHARD_ID_BYTES 384 /* three ncclUniqueId (exchange, gather and full-table communicators) */

/* ---- packed survivor form: what crosses the wire per subframe ------------------------------------------------------- */
typedef struct {
  uint32_t count;          /* survivors; > LTEPHY_COMPACT_CAP: list truncated, the walk needs the full table */
  uint32_t tti, cfi;
  uint32_t nloc;           /* location records that follow (0 when the CFI is invalid) */
  float    noise[2][2], rsrp[2][2]; /* per (port, antenna) sums of the channel estimator -> snr_db on the host (DCISearch.cc:568-569) */
  uint64_t low[2];         /* bit c: CCE c < min(nof_cce, 84) has mean |LLR| < 0.7 (DCISearch.cc:473-489) */
} ltephy_packed_hdr_t;     /* 64 bytes; then ltephy_cloc_t[(nloc + 3) & ~3]; then ltephy_cand_t[min(count, LTEPHY_COMPACT_CAP)] */

/* bytes of one packed record */
size_t ltephy_packed_size(uint32_t nloc, uint32_t count);
/* Host restatement of the GPU's pack kernel (tests; callers that obtained the survivor forms elsewhere): info[n] (raw or
 * finalised), comp[n] -> out (records back to back), offs[n + 1] (byte offset of record i; offs[n] = total).
 * Returns LTEPHY_ERROR_INVALID_INPUTS if cap is too small. */
int ltephy_pack_subframes(const ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_compact_t* comp, uint32_t n, uint8_t* out, size_t cap,
                          uint32_t* offs);
/* The walk turn of a sharded batch (host only, no GPU needed): bufs[r] / offs[r] are rank r's packed records and offsets
 * (n + 1 entries); global subframe g = i * world + r is record i of rank r.  full[r] (optional, may be NULL as a whole) is
 * rank r's full candidate table [n][LTEPHY_MAX_LOC][LTEPHY_MAX_SIZES], consulted where the survivor form cannot serve.
 * dcis[].sf is the global index g.  tti_cfi (optional) receives {tti, cfi} of every global subframe (2 * n * world words).
 * Returns LTEPHY_NEED_FULL_TABLE (nothing consumed) when full == NULL and the survivor forms cannot serve. */
int ltephy_search_batch_packed(ltephy_search_t* s, const uint8_t* const* bufs, const uint32_t* const* offs, const ltephy_cand_t* const* full,
                               uint32_t world, uint32_t n, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis, uint32_t* tti_cfi);
/* 1 if the walk over these records may need the full tables (an overfull subframe, or an RNTI ever RAR-activated on this
 * search object): identical on every rank, so the ranks can agree on a collective fetch before walking */
int ltephy_packed_needs_full_table(const ltephy_search_t* s, const uint8_t* const* bufs, const uint32_t* const* offs, uint32_t world, uint32_t n);
/* ltephy_grants_from_dcis with {tti, cfi} pairs (as written by ltephy_search_batch_packed) instead of full records */
int ltephy_grants_from_dcis_tc(const ltephy_search_t* s, const uint32_t* tti_cfi, const ltephy_dci_t* dcis, uint32_t nd, uint32_t mod, uint32_t rem,
                               ltephy_grant_t* grants, uint32_t* grant_dci, uint32_t max_grants, uint32_t* n_grants);

/* ---- communicator ----------------------------------------------------------------------------------------------------- */
/* rank 0 fills id (LTEPHY_SHARD_ID_BYTES) and hands it to the other ranks out of band (MPI, torch.distributed, a file) */
int ltephy_shard_unique_id(uint8_t* id);
/* collective: every rank calls it with the same id.  device = the CUDA device of this rank's PHY handles. */
int  ltephy_shard_create(const uint8_t* id, uint32_t rank, uint32_t world, int device, ltephy_shard_t** out);
void ltephy_shard_destroy(ltephy_shard_t* sh);
/* Every rank sends its transport blocks to rank 0 in a message of fixed size (no size negotiation inside the ordered section): capacity in bytes
 * per subframe of the batch, default 24576 (a 20 MHz 2x2 cell with both MCS-table readings decoded needs about 18 KB).  Same value on every rank. */
int ltephy_shard_set_gather_capacity(ltephy_shard_t* sh, uint32_t bytes_per_subframe);

typedef struct {
  double   host_ms[8];      /* submit A, wait A, exchange turn (incl. waiting for it), walk turn wait, walk, grants, phase B (submit + wait), gather turn */
  uint64_t exchanged_bytes; /* packed records received from all ranks in this batch */
  uint32_t n_grants;        /* this rank's grants */
  uint32_t used_full_table;
} ltephy_shard_stats_t;

/* One batch: this rank's n subframes (global subframe g = i * world + rank; every rank passes the same n and seq).
 *   iq: host memory (pinned makes the copy asynchronous), or device memory when iq_on_device != 0
 *   seq: 0, 1, 2, ... -- batch number, the same on every rank; calls for different seq may run concurrently on different
 *        handles h of the same rank (h must not be shared between concurrent calls).  A seq whose turn is over (reused, or a restart
 *        from 0 on a shard that has decoded), a seq another call of this rank is decoding, and LTEPHY_SEQ_NONE return
 *        LTEPHY_ERROR_INVALID_INPUTS at once: no section is taken and the rank does not count as failed
 *   info[n]: this rank's subframes
 *   dcis[max_dcis], *n_dcis: accepted DCIs of ALL n * world subframes in the order the walk produced them (sf = g)
 *   tbs[2 * max_dcis]: tbs[2 * i + t] belongs to dcis[i].  Rank 0 receives the transport blocks of every rank; other
 *        ranks see only those of their own subframes (the rest stay zeroed)
 *   payload: transport-block bytes; tbs[].payload_off points into it.  Pinned memory keeps the device->host copy asynchronous.
 * Returns 0 or a negative LTEPHY_* code.  A rank that fails stops taking part in the collectives of later batches: treat
 * an error as fatal for the job, as with any collective program.  A failing call, a refused argument list included, still passes
 * every ordered section on, and later batches of the rank return LTEPHY_ERROR at once. */
int ltephy_decode_subframes_sharded(ltephy_shard_t* sh, ltephy_t* h, ltephy_search_t* s, const void* iq, int iq_on_device, const uint32_t* tti,
                                    uint32_t n, uint64_t seq, ltephy_sf_info_t* info, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis,
                                    ltephy_tb_result_t* tbs, uint8_t* payload, size_t payload_cap, ltephy_shard_stats_t* stats);

/* parity tap: packed records + offsets of the CURRENT batch of h as the GPU pack kernel wrote them (blocks).
 * out_cap bytes at out, offs[n + 1]. */
int ltephy_pack_phase_a(ltephy_t* h, uint8_t* out, size_t out_cap, uint32_t* offs);

#ifdef __cplusplus
}
#endif
#endif
