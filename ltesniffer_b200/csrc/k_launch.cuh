// k_launch.cuh -- host entry points of the PHY kernels (k_frontend/k_viterbi/k_pdsch/k_turbo/k_pusch/k_pbch.cu), called by ltephy_capi.cu.
// Each kernel file includes this header, so a definition that differs from its declaration here fails to compile instead of being linked
// by its unmangled name.  Private to libltephy_b200.
#pragma once
#include "dev_common.cuh"
#include "dev_ul.cuh"

extern "C" {
void launch_frontend(const DevCell& c, const void* iq, uint32_t fmt, float2* sym, float2* ce, float* llr, DevSfInfo* info, uint32_t n, cudaStream_t st,
                     uint64_t* launches);
void launch_chest_interp(const DevCell& c, const float2* pil, float2* ce, uint32_t n, cudaStream_t st, uint64_t* launches);
void launch_ul_ofdm(const DevCell& c, const void* iq, uint32_t fmt, float2* sym, uint32_t n, cudaStream_t st, uint64_t* launches);
void launch_viterbi(const DevCell& c, const float* llr, const DevSfInfo* info, ltephy_cand_t* cands, uint32_t* work, uint32_t n, cudaStream_t st,
                    uint64_t* launches);
void launch_compact(const DevCell& c, const DevSfInfo* info, const ltephy_cand_t* cands, ltephy_compact_t* out, uint32_t n, cudaStream_t st,
                    uint64_t* launches);
void launch_scr_seq(const DevScr* cws, uint32_t ncw, uint32_t max_words, const uint32_t* gold_x1, const uint32_t* gold_basis, uint32_t basis_words,
                    uint32_t* seq_pool, cudaStream_t st, uint64_t* launches);
void launch_pdsch_front(const DevCell& c, const DevGrant* grants, uint32_t ngrants, const float2* sym, const float2* ce, const uint32_t* seq_pool,
                        short* llr_pool, cudaStream_t st, uint64_t* launches);
void launch_rm_turbo_rx(const DevCb* cbs, const DevPair* pairs, uint32_t npairs, const short* llr_pool, const uint16_t* rm_pool, uint32_t* turbo_pool,
                        short* harq_pool, uint32_t gen, cudaStream_t st, uint64_t* launches);
void launch_turbo(const DevPair* pairs, uint32_t npairs, uint32_t max_threads, int full, uint32_t* queue, const uint32_t* pool, uint32_t* scratch,
                  size_t scratch_words, const uint16_t* pi_pool, const uint32_t* pi_off, const uint32_t* xpowA, const uint32_t* xpowB, uint8_t* payload,
                  uint8_t* cb_iters, uint8_t* cb_crc, uint32_t max_iter, cudaStream_t st, uint64_t* launches);
void launch_tb_crc(const DevTb* tbs, uint32_t ntb, const uint8_t* payload, const uint8_t* cb_crc, const uint8_t* cb_iters, const uint32_t* xpowA,
                   ltephy_tb_result_t* res, cudaStream_t st, uint64_t* launches);
void launch_pusch(const DevCell& c, const DevUlGrant* grants, uint32_t ngrants, uint32_t max_M, const float2* ulsym, const float2* dmrs_pool,
                  const float2* idft_pool, const uint32_t* seq_pool, short* llr_pool, DevUlChest* chest, cudaStream_t st, uint64_t* launches);
void launch_pbch(const DevCell& c, const float2* sym, const float2* pil, const uint32_t* frame_sf, uint32_t nframes, uint32_t p_first, uint32_t np,
                 float* store, const uint32_t* jobs, uint32_t njobs, void* out, cudaStream_t st, uint64_t* launches);
}
