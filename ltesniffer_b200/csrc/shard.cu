// shard.cu -- sharded (one process per GPU) operation of the decode path behind include/ltephy_shard.h.
// Replaces the reference's worker hand-off and in-order result collection (src/src/Phy.cc:29-109) for N GPUs:
// global subframe g -> rank g % world; packed survivor forms all-gathered over NCCL (device to device), the FALCON walk
// replayed on every rank, phase B local, one NCCL gather of the decoded transport blocks to rank 0.
// NCCL is bound at run time (dlopen), so the library links and loads on hosts without it.
#include "../../include/ltephy_shard.h"
#include "ltephy_internal.cuh"
#include "tb_merge.hpp"
#include "turn.hpp"
#include <atomic>
#include <chrono>
#include <dlfcn.h>
#include <mutex>
#include <nccl.h>

// ====================================================================================================
// pack kernel: ltephy_compact_t + DevSfInfo of every subframe of the batch -> variable-length records, back to back.
// One CTA per subframe; the CTA finds its own byte offset by summing the sizes of the subframes before it (n is a few
// thousand at most: a handful of loads per thread), so there is no second pass and no atomics.
__device__ __forceinline__ uint32_t packed_size_dev(uint32_t nloc, uint32_t count)
{
  return (uint32_t)sizeof(ltephy_packed_hdr_t) + 4u * ((nloc + 3u) & ~3u) + 16u * min(count, (uint32_t)LTEPHY_COMPACT_CAP);
}
__global__ void __launch_bounds__(256) pack_kernel(const __grid_constant__ DevCell c, const DevSfInfo* __restrict__ info,
                                                   const ltephy_compact_t* __restrict__ comp, uint32_t n, uint8_t* __restrict__ out,
                                                   uint32_t* __restrict__ offs)
{
  __shared__ uint32_t red[8];
  __shared__ uint32_t low_s[4];
  const uint32_t i = blockIdx.x, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  uint32_t       acc = 0;
  for (uint32_t j = tid; j < i; j += blockDim.x) {
    const uint32_t cfi = info[j].cfi;
    const bool     ok  = cfi >= 1 && cfi <= 3;
    acc += packed_size_dev(ok ? c.nloc[cfi - 1] : 0u, ok ? comp[j].count : 0u);
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) red[warp] = acc;
  // low-power CCE mask (DCISearch.cc:473-489), bit c of word c >> 5
  const uint32_t cfi = info[i].cfi;
  const bool     ok  = cfi >= 1 && cfi <= 3;
  const uint32_t lim = ok ? min(c.nof_cce[cfi - 1], (uint32_t)LTEPHY_SEARCH_MAX_CCE) : 0u;
  if (tid < 128) {
    const uint32_t b = __ballot_sync(0xffffffffu, tid < lim && info[i].cce_power[tid] < 0.7f);
    if (lane == 0) low_s[warp] = b;
  }
  __syncthreads();
  uint32_t off = 0;
  for (uint32_t w = 0; w < blockDim.x / 32; w++) off += red[w];
  const uint32_t nloc = ok ? c.nloc[cfi - 1] : 0u, cnt = ok ? comp[i].count : 0u, nl4 = (nloc + 3u) & ~3u, nlist = min(cnt, (uint32_t)LTEPHY_COMPACT_CAP);
  if (tid == 0) {
    offs[i] = off;
    if (i + 1 == n) offs[n] = off + packed_size_dev(nloc, cnt);
    ltephy_packed_hdr_t hd;
    hd.count = cnt, hd.tti = info[i].tti, hd.cfi = cfi, hd.nloc = nloc;
    for (int p = 0; p < 2; p++)
      for (int a = 0; a < 2; a++) hd.noise[p][a] = info[i].noise[p][a], hd.rsrp[p][a] = info[i].rsrp[p][a];
    hd.low[0] = (uint64_t)low_s[0] | ((uint64_t)low_s[1] << 32);
    hd.low[1] = (uint64_t)low_s[2] | ((uint64_t)low_s[3] << 32);
    *reinterpret_cast<ltephy_packed_hdr_t*>(out + off) = hd; // records are 16-byte aligned (every size is a multiple of 16)
  }
  uint32_t*       dl = reinterpret_cast<uint32_t*>(out + off + sizeof(ltephy_packed_hdr_t));
  const uint32_t* sl = reinterpret_cast<const uint32_t*>(comp[i].loc);
  for (uint32_t j = tid; j < nl4; j += blockDim.x) dl[j] = j < nloc ? sl[j] : 0u;
  uint4*       dq = reinterpret_cast<uint4*>(out + off + sizeof(ltephy_packed_hdr_t) + 4u * nl4);
  const uint4* sq = reinterpret_cast<const uint4*>(comp[i].list);
  for (uint32_t j = tid; j < nlist; j += blockDim.x) dq[j] = sq[j];
}
static_assert(sizeof(ltephy_packed_hdr_t) == 64 && sizeof(ltephy_cloc_t) == 4 && sizeof(ltephy_cand_t) == 16, "packed layout");
#define PACK_MAX_BYTES (sizeof(ltephy_packed_hdr_t) + 4 * LTEPHY_MAX_LOC + 16 * LTEPHY_COMPACT_CAP) /* 4672 */

// ====================================================================================================
// NCCL, bound at run time
namespace {
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*)                                                                          = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int)                                                   = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t)                                                                             = nullptr;
  const char* (*GetErrorString)(ncclResult_t)                                                                        = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t)                     = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t)                = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t)                            = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t)                                  = nullptr;
  ncclResult_t (*GroupStart)()                                                                                        = nullptr;
  ncclResult_t (*GroupEnd)()                                                                                          = nullptr;
};
NcclApi    g_nccl;
std::mutex g_nccl_mtx;
int        nccl_load()
{
  std::lock_guard<std::mutex> lk(g_nccl_mtx);
  if (g_nccl.lib) return 0;
  // LTEPHY_NCCL_LIB names the library explicitly.  Otherwise the copy the process already holds is used (a process that imported torch gets
  // torch's bundled NCCL; loading an older system copy first would make a later "import torch" fail on the symbols it lacks), then the
  // loader's default libnccl.so.2.
  void*       lib = nullptr;
  const char* env = getenv("LTEPHY_NCCL_LIB");
  if (env && *env) lib = dlopen(env, RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) return fail(LTEPHY_ERROR, "libnccl.so.2 cannot be loaded: %s", dlerror());
#define BIND(field, name)                                                                          \
  *reinterpret_cast<void**>(&g_nccl.field) = dlsym(lib, name);                                     \
  if (!g_nccl.field) return fail(LTEPHY_ERROR, "libnccl: symbol %s not found", name);
  BIND(GetUniqueId, "ncclGetUniqueId")
  BIND(CommInitRank, "ncclCommInitRank")
  BIND(CommDestroy, "ncclCommDestroy")
  BIND(GetErrorString, "ncclGetErrorString")
  BIND(AllGather, "ncclAllGather")
  BIND(Broadcast, "ncclBroadcast")
  BIND(Send, "ncclSend")
  BIND(Recv, "ncclRecv")
  BIND(GroupStart, "ncclGroupStart")
  BIND(GroupEnd, "ncclGroupEnd")
#undef BIND
  g_nccl.lib = lib;
  return 0;
}
#define NC(x)                                                                                      \
  do {                                                                                             \
    ncclResult_t r_ = (x);                                                                         \
    if (r_ != ncclSuccess) return fail(LTEPHY_ERROR, "%s: %s", #x, g_nccl.GetErrorString(r_));     \
  } while (0)

struct TbMeta { // one per result slot (2 per grant) of the sending rank
  uint32_t grant_dci; // global DCI index | LTEPHY_GRANT_ALT_TABLE
  uint32_t tb_index;  // index into the sender's result array, ~0u: no transport block in this slot
  uint32_t byte_off, nbytes;
};
struct GatherHdr {
  uint32_t ng, ntb;
  uint64_t payload_bytes;
};

// per-handle buffers of the sharded path (T batches are in flight, each on its own handle)
struct Slot {
  uint32_t           cap_n = 0;
  DevBuf<uint8_t>    d_pack, d_pack_all, d_full_all, d_g_payload;
  DevBuf<uint32_t>   d_offs, d_offs_all;
  PinBuf<uint8_t>    h_pack_all, h_full_all;
  PinBuf<uint32_t>   h_offs_all;
  DevBuf<uint8_t>    d_msg, d_g_msg;   // gather message of this rank / of every other rank (rank 0): GatherHdr, TbMeta[2 ng], ltephy_tb_result_t[ntb]
  PinBuf<uint8_t>    h_msg, h_g_msg;
  Event              ev_pack, ev_g, ev_x, ev_msg; // created on first use
  std::vector<uint32_t>           tti_cfi, grant_dci;
  std::vector<ltephy_grant_t>     grants;
  std::vector<ltephy_tb_result_t> res;
};
inline double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
} // namespace

struct ltephy_shard {
  uint32_t     rank = 0, world = 1;
  int          device = 0;
  ncclComm_t   comm_x = nullptr, comm_g = nullptr, comm_f = nullptr; // exchange / gather / full-table fetch: one communicator per ordered section
  Stream       st_x, st_g, st_f;
  Turn         turn_x, turn_f, turn_w, turn_g;
  uint32_t     gather_bytes_per_sf = 24576; // fixed payload capacity of one rank's gather message, per subframe of the batch
  std::mutex   slots_mtx;
  std::map<ltephy_t*, std::unique_ptr<Slot>> slots;
  std::atomic<bool> failed{false}; // set and read by the pipelines' threads
  Slot*        slot_of(ltephy_t* h)
  {
    std::lock_guard<std::mutex> lk(slots_mtx);
    std::unique_ptr<Slot>&      s = slots[h];
    if (!s) s = std::make_unique<Slot>();
    return s.get();
  }
};

extern "C" int ltephy_shard_unique_id(uint8_t* id)
{
  if (!id) return fail(LTEPHY_ERROR_INVALID_INPUTS, "shard_unique_id: null argument");
  if (nccl_load()) return LTEPHY_ERROR;
  static_assert(LTEPHY_SHARD_ID_BYTES == 3 * NCCL_UNIQUE_ID_BYTES, "id size");
  for (int i = 0; i < 3; i++) {
    ncclUniqueId u;
    NC(g_nccl.GetUniqueId(&u));
    memcpy(id + i * NCCL_UNIQUE_ID_BYTES, &u, NCCL_UNIQUE_ID_BYTES);
  }
  return LTEPHY_SUCCESS;
}
extern "C" int ltephy_shard_create(const uint8_t* id, uint32_t rank, uint32_t world, int device, ltephy_shard_t** out)
{
  if (!id || !out || world == 0 || rank >= world) return fail(LTEPHY_ERROR_INVALID_INPUTS, "shard_create: bad arguments");
  if (nccl_load()) return LTEPHY_ERROR;
  CU(cudaSetDevice(device));
  ltephy_shard* sh = new ltephy_shard();
  sh->rank = rank, sh->world = world, sh->device = device;
  ncclUniqueId u[3];
  for (int i = 0; i < 3; i++) memcpy(&u[i], id + i * NCCL_UNIQUE_ID_BYTES, NCCL_UNIQUE_ID_BYTES);
  ncclResult_t r = g_nccl.CommInitRank(&sh->comm_x, (int)world, u[0], (int)rank);
  if (r == ncclSuccess) r = g_nccl.CommInitRank(&sh->comm_g, (int)world, u[1], (int)rank);
  if (r == ncclSuccess) r = g_nccl.CommInitRank(&sh->comm_f, (int)world, u[2], (int)rank);
  // highest priority: the collectives are short but sit on the critical path of every batch, and the GPU is kept full by the decode kernels of
  // the other pipelines -- without it an NCCL kernel waits behind whole grids of them
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  if (r != ncclSuccess || cudaStreamCreateWithPriority(&sh->st_x.raw, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
      cudaStreamCreateWithPriority(&sh->st_g.raw, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
      cudaStreamCreateWithPriority(&sh->st_f.raw, cudaStreamNonBlocking, prio_hi) != cudaSuccess) {
    ltephy_shard_destroy(sh);
    return fail(LTEPHY_ERROR, "shard_create: %s", r != ncclSuccess ? g_nccl.GetErrorString(r) : "stream creation failed");
  }
  *out = sh;
  return LTEPHY_SUCCESS;
}
extern "C" int ltephy_shard_set_gather_capacity(ltephy_shard_t* sh, uint32_t bytes_per_subframe)
{
  if (!sh || bytes_per_subframe < 1024) return fail(LTEPHY_ERROR_INVALID_INPUTS, "shard_set_gather_capacity: bad arguments");
  sh->gather_bytes_per_sf = (bytes_per_subframe + 15u) & ~15u;
  return LTEPHY_SUCCESS;
}
extern "C" void ltephy_shard_destroy(ltephy_shard_t* sh)
{
  if (!sh) return;
  cudaSetDevice(sh->device);
  cudaDeviceSynchronize();
  if (sh->comm_x) g_nccl.CommDestroy(sh->comm_x);
  if (sh->comm_g) g_nccl.CommDestroy(sh->comm_g);
  if (sh->comm_f) g_nccl.CommDestroy(sh->comm_f);
  delete sh;
}

// pack the current batch of h on its stream (after phase A) into slot buffers
static int pack_current(ltephy* h, Slot* sl)
{
  const uint32_t n = h->n_cur;
  if (sl->d_pack.reserve((size_t)h->cfg.max_subframes * PACK_MAX_BYTES) || sl->d_offs.reserve(h->cfg.max_subframes + 1))
    return fail(LTEPHY_ERROR, "device allocation failed");
  if (!sl->ev_pack) CU(cudaEventCreateWithFlags(&sl->ev_pack.raw, cudaEventDisableTiming));
  pack_kernel<<<n, 256, 0, h->stream>>>(h->dc, h->d_info.p, h->d_compact.p, n, sl->d_pack.p, sl->d_offs.p);
  h->launches++;
  CU(cudaEventRecord(sl->ev_pack, h->stream));
  CU(cudaGetLastError());
  return LTEPHY_SUCCESS;
}

extern "C" int ltephy_pack_phase_a(ltephy_t* h, uint8_t* out, size_t out_cap, uint32_t* offs)
{
  if (!h || !out || !offs || !h->n_cur) return fail(LTEPHY_ERROR_INVALID_INPUTS, "pack_phase_a: bad arguments");
  CU(cudaSetDevice(h->cfg.device));
  Slot sl;
  int  r = pack_current(h, &sl);
  if (r == LTEPHY_SUCCESS) {
    const uint32_t n = h->n_cur;
    if (cudaMemcpyAsync(offs, sl.d_offs.p, (n + 1) * 4, cudaMemcpyDeviceToHost, h->stream) != cudaSuccess || cudaStreamSynchronize(h->stream) != cudaSuccess)
      r = fail(LTEPHY_ERROR, "pack_phase_a: copy failed");
    else if (offs[n] > out_cap)
      r = fail(LTEPHY_ERROR_INVALID_INPUTS, "pack_phase_a: %u bytes needed, %zu available", offs[n], out_cap);
    else if (cudaMemcpy(out, sl.d_pack.p, offs[n], cudaMemcpyDeviceToHost) != cudaSuccess)
      r = fail(LTEPHY_ERROR, "pack_phase_a: copy failed");
  }
  cudaStreamSynchronize(h->stream);
  return r;
}

// ====================================================================================================
extern "C" int ltephy_decode_subframes_sharded(ltephy_shard_t* sh, ltephy_t* h, ltephy_search_t* s, const void* iq, int iq_on_device, const uint32_t* tti,
                                               uint32_t n, uint64_t seq, ltephy_sf_info_t* info, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis,
                                               ltephy_tb_result_t* tbs, uint8_t* payload, size_t payload_cap, ltephy_shard_stats_t* stats)
{
  if (!sh) return fail(LTEPHY_ERROR_INVALID_INPUTS, "decode_subframes_sharded: bad arguments");
  // every batch takes the exchange turn first, so owning seq there makes it the one call of its batch in every section
  if (seq == LTEPHY_SEQ_NONE || !sh->turn_x.claim(seq))
    return fail(LTEPHY_ERROR_INVALID_INPUTS, "decode_subframes_sharded: seq %llu is not the number of a batch still to come", (unsigned long long)seq);
  const uint32_t W = sh->world, R = sh->rank;
  // the ordered sections of this batch; the guards keep the order intact on every exit path, a refused argument list included
  TurnGuard gx(sh->turn_x, seq), gf(sh->turn_f, seq), gw(sh->turn_w, seq), gg(sh->turn_g, seq);
  if (sh->failed) return fail(LTEPHY_ERROR, "decode_subframes_sharded: an earlier batch failed on this rank");
  struct FailMark {
    ltephy_shard* sh;
    bool          ok = false;
    ~FailMark()
    {
      if (!ok) sh->failed = true;
    }
  } mark{sh};
  if (!h || !s || !iq || !tti || !info || !dcis || !n_dcis || !tbs || n == 0) return fail(LTEPHY_ERROR_INVALID_INPUTS, "decode_subframes_sharded: bad arguments");
  CU(cudaSetDevice(sh->device));
  Slot*  sl = sh->slot_of(h);
  double t[10];
  t[0]  = now_ms();
  // ---- phase A + pack (asynchronous) ----------------------------------------------------------------
  int r = iq_on_device ? ltephy_submit_iq_device(h, iq, tti, n) : ltephy_submit_iq(h, iq, tti, n);
  if (r) return r;
  if ((r = pack_current(h, sl))) return r;
  t[1] = now_ms();
  // this rank's full records (CFI and tti are also what phase B needs on the host)
  if ((r = ltephy_get_phase_a(h, info, nullptr))) return r;
  t[2] = now_ms();
  const size_t cap_rank = (size_t)n * PACK_MAX_BYTES;
  if (sl->d_offs_all.reserve((size_t)W * (n + 1)) || sl->h_offs_all.reserve((size_t)W * (n + 1)) || sl->d_pack_all.reserve(W * cap_rank) ||
      sl->h_pack_all.reserve(W * cap_rank))
    return fail(LTEPHY_ERROR, "allocation of the exchange buffers failed");
  // ---- exchange turn: the turn orders the two collectives of this batch among the batches in flight, nothing else.  Waiting for them
  // (= for the slowest rank) and the copies to the host happen outside it, so a straggler delays its own batch only.
  for (Event* e : {&sl->ev_x, &sl->ev_g, &sl->ev_msg})
    if (!*e) CU(cudaEventCreateWithFlags(&e->raw, cudaEventDisableTiming));
  gx.take();
  CU(cudaStreamWaitEvent(sh->st_x, sl->ev_pack, 0));
  // offsets, then the records at their fixed per-rank capacity (4.6 MB per 1000 subframes, a third of it used: NVLink does not notice, and
  // no host round trip sits between the two collectives); only the used part of every rank's records goes to the host
  NC(g_nccl.AllGather(sl->d_offs.p, sl->d_offs_all.p, n + 1, ncclUint32, sh->comm_x, sh->st_x));
  NC(g_nccl.AllGather(sl->d_pack.p, sl->d_pack_all.p, cap_rank, ncclUint8, sh->comm_x, sh->st_x));
  CU(cudaEventRecord(sl->ev_x, sh->st_x));
  gx.pass();
  CU(cudaStreamWaitEvent(h->stream, sl->ev_x, 0)); // the handle's stream is idle between phase A and phase B
  CU(cudaMemcpyAsync(sl->h_offs_all.p, sl->d_offs_all.p, (size_t)W * (n + 1) * 4, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  uint64_t exch = 0;
  for (uint32_t q = 0; q < W; q++) {
    const uint32_t bytes = sl->h_offs_all.p[(size_t)q * (n + 1) + n];
    if (bytes > cap_rank) return fail(LTEPHY_ERROR, "rank %u announced %u packed bytes for %u subframes", q, bytes, n);
    exch += bytes;
    CU(cudaMemcpyAsync(sl->h_pack_all.p + q * cap_rank, sl->d_pack_all.p + q * cap_rank, bytes, cudaMemcpyDeviceToHost, h->stream));
  }
  CU(cudaStreamSynchronize(h->stream));
  std::vector<const uint8_t*>       bufs(W);
  std::vector<const uint32_t*>      offs(W);
  std::vector<const ltephy_cand_t*> full;
  for (uint32_t q = 0; q < W; q++) bufs[q] = sl->h_pack_all.p + q * cap_rank, offs[q] = sl->h_offs_all.p + (size_t)q * (n + 1);
  // The full tables are needed only for an overfull subframe or RAR-activated RNTIs; every rank sees the same records and the same
  // history, so every rank fetches them (a collective on its own communicator, ordered by its own turn) or none does.
  const int need_full = ltephy_packed_needs_full_table(s, bufs.data(), offs.data(), W, n);
  if (need_full < 0) return need_full;
  gf.take();
  if (need_full) {
    const size_t fb = (size_t)n * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES * sizeof(ltephy_cand_t);
    if (sl->d_full_all.reserve(W * fb) || sl->h_full_all.reserve(W * fb)) return fail(LTEPHY_ERROR, "allocation of the full-table exchange buffers failed");
    NC(g_nccl.AllGather(h->d_cands.p, sl->d_full_all.p, fb, ncclUint8, sh->comm_f, sh->st_f));
    CU(cudaMemcpyAsync(sl->h_full_all.p, sl->d_full_all.p, W * fb, cudaMemcpyDeviceToHost, sh->st_f));
    CU(cudaStreamSynchronize(sh->st_f));
    full.resize(W);
    for (uint32_t q = 0; q < W; q++) full[q] = reinterpret_cast<const ltephy_cand_t*>(sl->h_full_all.p + q * fb);
  }
  gf.pass();
  t[3] = now_ms();
  // ---- walk turn -----------------------------------------------------------------------------------------
  gw.take();
  t[4] = now_ms();
  sl->tti_cfi.resize((size_t)2 * n * W);
  uint32_t nd = 0;
  r = ltephy_search_batch_packed(s, bufs.data(), offs.data(), need_full ? full.data() : nullptr, W, n, dcis, max_dcis, &nd, sl->tti_cfi.data());
  gw.pass();
  if (r) return fail(r, "walk over the exchanged tables failed (%d)", r);
  *n_dcis = nd;
  t[5]    = now_ms();
  sl->grants.resize(2 * (size_t)nd + 1), sl->grant_dci.resize(2 * (size_t)nd + 1);
  uint32_t ng = 0;
  if ((r = ltephy_grants_from_dcis_tc(s, sl->tti_cfi.data(), dcis, nd, W, R, sl->grants.data(), sl->grant_dci.data(), 2 * nd + 1, &ng))) return r;
  t[6] = now_ms();
  // ---- phase B (local) ----------------------------------------------------------------------------------------
  for (uint32_t i = 0; i < 2 * nd; i++) tbs[i] = ltephy_tb_result_t{};
  const size_t cap_p = (size_t)n * sh->gather_bytes_per_sf; // fixed size of one rank's payload message
  if (W > 1 && h->d_payload.reserve(cap_p + 16)) return fail(LTEPHY_ERROR, "device allocation failed");
  if ((r = ltephy_submit_grants(h, sl->grants.data(), ng))) return r;
  sl->res.assign(2 * (size_t)ng + 2, ltephy_tb_result_t{});
  if ((r = ltephy_get_phase_b(h, sl->res.data(), payload, payload_cap))) return r;
  size_t own_bytes = 0;
  for (uint32_t gi = 0; gi < ng; gi++) {
    ltephy_place_grant_result(tbs, sl->grant_dci[gi], sl->res[2 * gi], sl->res[2 * gi + 1]);
    own_bytes += sl->res[2 * gi].payload_len + sl->res[2 * gi + 1].payload_len;
  }
  t[7] = now_ms();
  // ---- gather: the decoded transport blocks of every rank -> rank 0.  Every rank sends two messages of FIXED size (header + per-slot
  // records + result structs; the payload bytes), so no size has to be agreed on first and the turn holds nothing but the NCCL calls.
  const size_t cap_m = 64 + (size_t)n * 64 * (sizeof(TbMeta) + sizeof(ltephy_tb_result_t)); // up to 32 grants (64 result slots) per subframe
  if (W > 1) {
    const size_t ntb = h->pb.tbs.size();
    if (h->pb.payload_bytes > cap_p)
      return fail(LTEPHY_ERROR_INVALID_INPUTS, "%zu transport-block bytes in %u subframes exceed the gather capacity (ltephy_shard_set_gather_capacity)", h->pb.payload_bytes, n);
    if (64 + 2 * (size_t)ng * sizeof(TbMeta) + ntb * sizeof(ltephy_tb_result_t) > cap_m)
      return fail(LTEPHY_ERROR_INVALID_INPUTS, "%u grants in %u subframes exceed the gather message", ng, n);
    if (R != 0) {
      if (sl->h_msg.reserve(cap_m) || sl->d_msg.reserve(cap_m)) return fail(LTEPHY_ERROR, "allocation of the gather buffers failed");
      GatherHdr gh{ng, (uint32_t)ntb, (uint64_t)h->pb.payload_bytes};
      memcpy(sl->h_msg.p, &gh, sizeof(gh));
      TbMeta* hm = reinterpret_cast<TbMeta*>(sl->h_msg.p + 64);
      for (uint32_t j = 0; j < 2 * ng; j++) {
        const uint32_t ti = h->pb.tb_slot[j];
        hm[j].grant_dci = sl->grant_dci[j / 2], hm[j].tb_index = ti;
        hm[j].byte_off = ti != 0xFFFFFFFFu ? h->pb.tbs[ti].byte_off : 0, hm[j].nbytes = ti != 0xFFFFFFFFu ? h->pb.tbs[ti].nbytes : 0;
      }
      const size_t mb = 64 + 2 * (size_t)ng * sizeof(TbMeta);
      ltephy_pull(h, sl->d_msg.p, sl->h_msg.p, (mb + 15) & ~(size_t)15, h->stream);
      if (ntb) CU(cudaMemcpyAsync(sl->d_msg.p + mb, h->d_res.p, ntb * sizeof(ltephy_tb_result_t), cudaMemcpyDeviceToDevice, h->stream));
      CU(cudaEventRecord(sl->ev_msg, h->stream));
      gg.take();
      CU(cudaStreamWaitEvent(sh->st_g, sl->ev_msg, 0));
      NC(g_nccl.GroupStart());
      NC(g_nccl.Send(sl->d_msg.p, cap_m, ncclUint8, 0, sh->comm_g, sh->st_g));
      NC(g_nccl.Send(h->d_payload.p, cap_p, ncclUint8, 0, sh->comm_g, sh->st_g));
      NC(g_nccl.GroupEnd());
      CU(cudaEventRecord(sl->ev_g, sh->st_g));
      gg.pass();
      CU(cudaEventSynchronize(sl->ev_g)); // the handle's buffers are free for its next batch when this call returns
    } else {
      if (sl->d_g_msg.reserve((W - 1) * cap_m) || sl->h_g_msg.reserve((W - 1) * cap_m) || sl->d_g_payload.reserve((W - 1) * cap_p + 16))
        return fail(LTEPHY_ERROR, "allocation of the gather buffers failed");
      gg.take();
      NC(g_nccl.GroupStart());
      for (uint32_t q = 1; q < W; q++) {
        NC(g_nccl.Recv(sl->d_g_msg.p + (q - 1) * cap_m, cap_m, ncclUint8, (int)q, sh->comm_g, sh->st_g));
        NC(g_nccl.Recv(sl->d_g_payload.p + (q - 1) * cap_p, cap_p, ncclUint8, (int)q, sh->comm_g, sh->st_g));
      }
      NC(g_nccl.GroupEnd());
      CU(cudaEventRecord(sl->ev_g, sh->st_g));
      gg.pass();
      // host side, outside the turn: headers first, then exactly the used part of every rank's records and bytes
      CU(cudaStreamWaitEvent(h->stream, sl->ev_g, 0));
      CU(cudaMemcpy2DAsync(sl->h_g_msg.p, cap_m, sl->d_g_msg.p, cap_m, 64, W - 1, cudaMemcpyDeviceToHost, h->stream));
      CU(cudaStreamSynchronize(h->stream));
      const size_t base0 = (own_bytes + 15) & ~(size_t)15;
      size_t       tp    = 0;
      for (uint32_t q = 1; q < W; q++) {
        GatherHdr gh;
        memcpy(&gh, sl->h_g_msg.p + (q - 1) * cap_m, sizeof(gh));
        const size_t mb = 2 * (size_t)gh.ng * sizeof(TbMeta) + (size_t)gh.ntb * sizeof(ltephy_tb_result_t);
        if (64 + mb > cap_m || gh.payload_bytes > cap_p) return fail(LTEPHY_ERROR, "rank %u sent an inconsistent gather header", q);
        if (base0 + tp + gh.payload_bytes > payload_cap)
          return fail(LTEPHY_ERROR_INVALID_INPUTS, "payload buffer too small for the gathered transport blocks (%zu needed)", base0 + tp + (size_t)gh.payload_bytes);
        if (mb) CU(cudaMemcpyAsync(sl->h_g_msg.p + (q - 1) * cap_m + 64, sl->d_g_msg.p + (q - 1) * cap_m + 64, mb, cudaMemcpyDeviceToHost, h->stream));
        if (gh.payload_bytes) CU(cudaMemcpyAsync(payload + base0 + tp, sl->d_g_payload.p + (q - 1) * cap_p, gh.payload_bytes, cudaMemcpyDeviceToHost, h->stream));
        tp += (gh.payload_bytes + 15) & ~(size_t)15;
      }
      CU(cudaStreamSynchronize(h->stream));
      size_t op = 0;
      for (uint32_t q = 1; q < W; q++) {
        GatherHdr gh;
        memcpy(&gh, sl->h_g_msg.p + (q - 1) * cap_m, sizeof(gh));
        const TbMeta*             gm = reinterpret_cast<const TbMeta*>(sl->h_g_msg.p + (q - 1) * cap_m + 64);
        const ltephy_tb_result_t* gr = reinterpret_cast<const ltephy_tb_result_t*>(sl->h_g_msg.p + (q - 1) * cap_m + 64 + 2 * (size_t)gh.ng * sizeof(TbMeta));
        for (uint32_t gi = 0; gi < gh.ng; gi++) {
          ltephy_tb_result_t rr[2] = {ltephy_tb_result_t{}, ltephy_tb_result_t{}};
          for (int tbi = 0; tbi < 2; tbi++) {
            const TbMeta& m = gm[2 * gi + tbi];
            if (m.tb_index == 0xFFFFFFFFu || m.tb_index >= gh.ntb) continue;
            rr[tbi]             = gr[m.tb_index];
            rr[tbi].payload_off = (uint32_t)(base0 + op + m.byte_off);
            rr[tbi].payload_len = m.nbytes;
          }
          const uint32_t gd = gm[2 * gi].grant_dci;
          if ((gd & ~LTEPHY_GRANT_ALT_TABLE) < nd) ltephy_place_grant_result(tbs, gd, rr[0], rr[1]);
        }
        op += (gh.payload_bytes + 15) & ~(size_t)15;
      }
    }
  }
  gg.pass();
  t[8] = now_ms();
  if (stats) {
    stats->host_ms[0] = t[1] - t[0], stats->host_ms[1] = t[2] - t[1], stats->host_ms[2] = t[3] - t[2], stats->host_ms[3] = t[4] - t[3];
    stats->host_ms[4] = t[5] - t[4], stats->host_ms[5] = t[6] - t[5], stats->host_ms[6] = t[7] - t[6], stats->host_ms[7] = t[8] - t[7];
    stats->exchanged_bytes = exch, stats->n_grants = ng, stats->used_full_table = (uint32_t)need_full;
  }
  mark.ok = true;
  return LTEPHY_SUCCESS;
}
