// ltephy_internal.cuh -- the PHY handle and its helpers, shared by ltephy_capi.cu (single-GPU entry points) and shard.cu
// (sharded operation).  Private to libltephy_b200: nothing here is part of the C-ABI.
#pragma once
#include "../../include/ltephy_b200.h"
#include "../../include/ltephy_search.h"
#include "dev_common.cuh"
#include "dev_ul.cuh"
#include "lte_host.hpp"
#include <cstdarg>
#include <cstdio>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

extern thread_local std::string ltephy_g_err;
static inline int fail(int code, const char* fmt, ...)
{
  char    buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  ltephy_g_err = buf;
  return code;
}
// bytes of one complex sample of iq_format fmt (LTEPHY_IQ_*): sizes every sample buffer and host-to-device copy of an input
static inline size_t iq_sample_bytes(uint32_t fmt) { return fmt == LTEPHY_IQ_SC16 ? 4 : fmt == LTEPHY_IQ_SC8 ? 2 : 8; }
// integer samples in device memory are loaded as short2 / char2, so their pointer must be aligned to the sample; cf32 pointers are taken as given
static inline bool iq_misaligned(const void* p, uint32_t fmt) { return fmt != LTEPHY_IQ_CF32 && (uintptr_t)p % iq_sample_bytes(fmt); }
#define CU(x)                                                                                      \
  do {                                                                                             \
    cudaError_t e_ = (x);                                                                          \
    if (e_ != cudaSuccess) return fail(LTEPHY_ERROR, "%s: %s", #x, cudaGetErrorString(e_));        \
  } while (0)

// The owners below free what they hold when they die.  A handle declares its stream before its buffers, so the buffers go first.
template <typename T>
struct DevBuf { // growable device buffer
  T*     p   = nullptr;
  size_t cap = 0;
  DevBuf()   = default;
  DevBuf(const DevBuf&)            = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
  DevBuf& operator=(DevBuf&& o) noexcept // the buffer held before dies with o
  {
    std::swap(p, o.p), std::swap(cap, o.cap);
    return *this;
  }
  ~DevBuf() { release(); }
  int reserve(size_t n)
  {
    if (n <= cap) return 0;
    size_t want = n + n / 4 + 1024;
    if (p) {
      cudaDeviceSynchronize();
      cudaFree(p);
      p = nullptr;
    }
    if (cudaMalloc(&p, want * sizeof(T)) != cudaSuccess) {
      cap = 0;
      return -1;
    }
    cap = want;
    return 0;
  }
  void release()
  {
    if (p) cudaFree(p);
    p = nullptr, cap = 0;
  }
};
template <typename T>
struct PinBuf { // growable pinned host buffer
  T*     p   = nullptr;
  size_t cap = 0;
  PinBuf()   = default;
  PinBuf(const PinBuf&)            = delete;
  PinBuf& operator=(const PinBuf&) = delete;
  PinBuf(PinBuf&& o) noexcept { *this = std::move(o); }
  PinBuf& operator=(PinBuf&& o) noexcept
  {
    std::swap(p, o.p), std::swap(cap, o.cap);
    return *this;
  }
  ~PinBuf() { release(); }
  int reserve(size_t n)
  {
    if (n <= cap) return 0;
    size_t want = n + n / 4 + 1024;
    if (p) cudaFreeHost(p);
    p = nullptr;
    if (cudaMallocHost(&p, want * sizeof(T)) != cudaSuccess) {
      cap = 0;
      return -1;
    }
    cap = want;
    return 0;
  }
  void release()
  {
    if (p) cudaFreeHost(p);
    p = nullptr, cap = 0;
  }
};
// a stream or an event: created into &raw while it is null, used wherever the CUDA type is
template <typename H, cudaError_t (*destroy)(H)>
struct CudaOwned {
  H raw = nullptr;
  CudaOwned() = default;
  CudaOwned(const CudaOwned&)            = delete;
  CudaOwned& operator=(const CudaOwned&) = delete;
  ~CudaOwned()
  {
    if (raw) destroy(raw);
  }
  operator H() const { return raw; }
};
using Stream = CudaOwned<cudaStream_t, cudaStreamDestroy>;
using Event  = CudaOwned<cudaEvent_t, cudaEventDestroy>;

struct ltephy {
  ltephy_cfg_t       cfg{};
  ltehost::Cell      cell;
  ltehost::CtrlMap   cm;
  ltehost::SizeTable st;
  DevCell            dc{};
  Stream             stream;
  Event              ev[6], mark[2], ev_h2d;
  DevBuf<float2>     d_cfo;                  // per-sample rotation of ltephy_set_cfo
  DevBuf<float2>     d_ulcfo;                // per-sample rotation of ltephy_set_ul_cfo
  DevBuf<uint32_t>   d_vwork;                // work list of the Viterbi kernel: count + two-word (subframe, locations, size) items
  DevBuf<uint32_t>   d_mib;                  // PBCH work of one call: subframe of each frame, hypothesis jobs, 2 result words per job (k_pbch.cu)
  DevBuf<float>      d_pbch;                 // PBCH frame store [3 + max_subframes][2][480]: rows 0..2 the frames the combiner carries over
  uint32_t           mib_held     = 0;       // combiner: frames held (srsRAN's frame_idx between calls), in rows 3 - mib_held .. 2
  int32_t            mib_last_sfn = -1;      // combiner: SFN of the last frame consumed, -1 after a reset
  uint32_t           pbch_frames  = 0;       // frames the last PBCH call wrote to rows 3.. of d_pbch (LTEPHY_TAP_PBCH_LLR)
  DevBuf<short>      d_harq;                 // HARQ store: harq_slots x LTEPHY_HARQ_SLOT_BYTES
  uint32_t           harq_slots = 0;
  std::vector<DevBuf<uint8_t>> tables;                 // the cell's constant tables (upload): dc, d_gold_* and d_xpow* point into them
  cudaError_t                  table_err = cudaSuccess; // the first table upload that failed
  uint64_t                     launches  = 0;

  // phase A
  DevBuf<uint8_t>       d_iq;                     // samples of the batch in cfg.iq_format
  DevBuf<float2>        d_sym, d_pil, d_ce; // d_pil: smoothed CRS estimates [n][port][rx][4][2 nof_prb]; d_ce: interpolated grid, filled on demand (tap)
  DevBuf<float>         d_llr;
  DevBuf<DevSfInfo>     d_info;
  DevBuf<ltephy_cand_t> d_cands;
  PinBuf<DevSfInfo>     h_info;
  DevBuf<ltephy_compact_t> d_compact;
  PinBuf<ltephy_compact_t> h_compact;
  uint32_t              n_cur = 0;
  std::vector<uint8_t>  re_cnt; // [3 sf class][3 cfi][14][nof_prb]

  // phase B
  struct PhaseB { // the batch of the last ltephy_submit_grants, ltephy_submit_ul or ltephy_turbo_batch: every submit starts with reset()
    std::vector<DevGrant>   grants;
    std::vector<DevUlGrant> ulgrants;
    std::vector<DevCb>      cbs;
    struct CbHalf {           // what a code block's half of its turbo pair needs, and its pairing key TBS / G (pair_code_blocks)
      uint32_t tbs, G, crc_type, out_bits, out_byte;
    };
    std::vector<CbHalf>     cb_half; // [code block]
    std::vector<DevPair>    pairs;
    std::vector<DevTb>      tbs;
    std::vector<DevScr>     scr;     // [codeword] scrambling sequence to write (alloc_codeword)
    std::vector<uint32_t>   pair_pi_off;
    std::vector<uint32_t>   tb_slot; // result slot (DL: grant*2 + tb, UL: grant) -> tb index or ~0
    std::map<uint32_t, uint32_t> harq_uses; // slot -> uses in this batch
    uint32_t                harq_max_gen = 0;
    size_t                  payload_bytes = 0, pllr_elems = 0;
    size_t                  seq_words = 0, turbo_words = 0; // scrambling-sequence and turbo-pool words
    uint32_t                max_scr_words = 0;              // longest codeword's scrambling words
    void reset(size_t nslots)
    {
      grants.clear(), ulgrants.clear(), cbs.clear(), cb_half.clear(), pairs.clear(), tbs.clear(), scr.clear(), pair_pi_off.clear(), harq_uses.clear();
      tb_slot.assign(nslots, 0xFFFFFFFFu);
      harq_max_gen = 0, payload_bytes = 0, pllr_elems = 0, seq_words = 0, turbo_words = 0, max_scr_words = 0;
    }
  } pb;
  DevBuf<DevGrant>      d_grants;
  DevBuf<DevCb>         d_cbs;
  DevBuf<DevPair>       d_pairs;
  DevBuf<DevTb>         d_tbs;       // pb.tbs, then pb.scr (stage_tbs_and_scramble)
  DevBuf<uint32_t>      d_pair_pi_off;
  DevBuf<uint32_t>      d_seq, d_turbo;
  DevBuf<uint16_t>      d_rm;        // pool of rate-matching inverse tables (pool_append), rm_used entries filled
  size_t                rm_used = 0;
  DevBuf<uint32_t>      d_tscratch, d_tqueue; // persistent turbo kernel: per-CTA state slots, pair counters of the launches
  DevBuf<short>         d_pllr;
  DevBuf<uint16_t>      d_pi;        // pool of QPP interleaver tables (pool_append), pi_used entries filled
  size_t                pi_used = 0;
  DevBuf<uint8_t>       d_payload, d_cb_iters, d_cb_crc;
  DevBuf<ltephy_tb_result_t> d_res;
  PinBuf<ltephy_tb_result_t> h_res;
  PinBuf<uint8_t>            h_payload;
  PinBuf<uint8_t>            h_stage;      // pinned arena for the job descriptors of one phase B (see pull())
  size_t                     stage_used = 0;
  bool                       stage_busy = false; // descriptors staged and possibly still being pulled
  uint32_t *                 d_gold_x1 = nullptr, *d_gold_basis = nullptr, gold_words = 0;
  uint32_t *                 d_xpowA = nullptr, *d_xpowB = nullptr;
  struct RmEntry {
    int64_t  off = -1; // offset of the inverse table in d_rm, -1: not built yet
    uint32_t nn = 0, rot[4]{};
  };
  std::map<std::pair<uint32_t, uint32_t>, RmEntry> rm_cache; // (K, F) -> inverse table
  RmEntry                                          rm_fast[188]; // F == 0 fast path, by qpp index
  int64_t  pi_fast[188];                // offset of K's interleaver table in d_pi by qpp index, -1: not built yet
  std::vector<ltehost::Segm> segm_fast; // index tbs/8, C == 0 means "not computed"
  // uplink
  ltephy_ul_cfg_t            ulcfg{};
  bool                       ulcfg_set = false;
  uint32_t                   n_prs[20]{}, ul_u[20]{}, ul_v[20]{}; // per slot: n_PRS, base-sequence group u and sequence v
  DevBuf<uint8_t>            d_uliq;                    // UL samples in cfg.iq_format
  DevBuf<float2>             d_ulsym, d_ulpool; // d_ulpool: pool of DMRS sequences and IDFT twiddles (pool_append)
  DevBuf<DevUlGrant>         d_ulgrants;
  DevBuf<DevUlChest>         d_ulchest;
  PinBuf<DevUlChest>         h_ulchest;
  std::map<uint64_t, uint32_t> ul_tab_cache; // (kind, M, ncs, u, v) -> offset in d_ulpool
  size_t                     ulpool_used = 0;
  uint32_t                   n_ul = 0;
  float                      t_ms[4]{};
};


// kernel-driven copy of a few bytes from pinned host memory (see ltephy_capi.cu: small transfers avoid the copy engine)
void ltephy_pull(ltephy* h, void* dst_dev, const void* src_pinned, size_t bytes, cudaStream_t st);
