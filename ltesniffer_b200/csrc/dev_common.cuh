// dev_common.cuh -- device-side structures shared by the sm_90a kernels of libltephy_b200.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/ltephy_b200.h"

#define LLR_STRIDE (72 * LTEPHY_MAX_CCE) /* floats per subframe in the PDCCH LLR buffer */
#define NPILSYM 4

struct DevCell {
  uint32_t nof_prb, nof_ports, cell_id, nof_rx, fft, log2n, nsc, sf_len;
  uint32_t ul_nof_rx;             // antennas of the uplink carrier, 1 or 2 (ltephy_cfg_t.ul_nof_rx)
  uint32_t sub;                   // power-of-two transform length: fft, or fft / 3 for a 3 * 2^k symbol size (log2n = log2(sub))
  uint32_t sym_off[14];
  uint32_t nof_cce[3], nloc[3];
  uint32_t crs_off[2][2]; // [port][0: symbol 0 of slot, 1: symbol 4 of slot]
  float    filt[5], noise_corr, interp_c[17];
  float    t_frac[14];    // time-interpolation weight per symbol
  uint8_t  t_ia[14], t_ib[14];
  uint32_t nsizes, sizes[LTEPHY_MAX_SIZES];
  uint32_t flags;
  uint32_t pcfich_scr[10]; // 32 scrambling bits per subframe index
  uint16_t pcfich_idx[16];
  uint32_t pdcch_scr_words;       // words per subframe index
  const float2*   tw;             // [sub/2]
  const float2*   tw_st;          // [sub] per-stage tables: tw_st[H + pos] = tw[pos * sub / (2 H)], H = 1, 2, .. sub/2, pos < H
  const float2*   w3;             // [2][fft] radix-3 twiddles W_N^k, W_N^(2k) of a 3 * 2^k symbol size, nullptr otherwise
  const float2*   ul_rot;         // [fft] exp(-j pi i / N)
  const float2*   crs;            // [10][2][4][2*nof_prb]
  const uint16_t* pdcch_idx[3];   // [nof_cce*9][4]
  const uint32_t* pdcch_scr;      // [10][pdcch_scr_words]
  const uint16_t* conv_tab[LTEPHY_MAX_SIZES]; // [3K] circular position -> stream-major index
  const uint16_t* loc_tab[3];     // [nloc] ncce | (L << 8)
  const uint16_t* re_mask;        // [3 sf class][3 cfi][14][nof_prb]: 12-bit mask of PDSCH data REs of the PRB in the symbol
  const uint32_t* pbch_re;        // [240] (symbol << 16) | sub-carrier of the PBCH resource elements of subframe 0
  const uint32_t* pbch_scr;       // [60] c(cell_id), 1920 bits
  const uint16_t* pbch_tab;       // [120] conv rate-matching table of K = 40
  const float2*   cfo_rot;        // [sf_len] e^{-j 2 pi f n / (15000 fft)} or nullptr (ltephy_set_cfo)
  const float2*   ul_cfo_rot;     // the same for the uplink, or nullptr (ltephy_set_ul_cfo)
};

// per-subframe device record (layout mirrors the leading part of ltephy_sf_info_t)
struct DevSfInfo {
  uint32_t tti, cfi, nof_cce, nof_locations;
  float    pcfich_corr[3];
  float    noise[2][2], rsrp[2][2];
  float    noise_avg, rsrp_avg, cfo_re, cfo_im, snr_db, cfo;
  float    rb_power[LTEPHY_MAX_PRB];
  float    cce_power[LTEPHY_MAX_CCE];
};
static_assert(sizeof(DevSfInfo) == sizeof(ltephy_sf_info_t), "DevSfInfo must mirror ltephy_sf_info_t");

// One complex input sample as cf32, converted where a kernel loads it: sc16 is value * 2^-15, sc8 value * 2^-7, both exact in fp32, so a run on
// integer samples equals the cf32 run on the converted samples bit for bit (DESIGN.md §2 "integer samples").
__device__ __forceinline__ float2 chan_cf32(float2 v) { return v; }
__device__ __forceinline__ float2 chan_cf32(short2 v) { return make_float2((float)v.x * 0x1p-15f, (float)v.y * 0x1p-15f); }
__device__ __forceinline__ float2 chan_cf32(char2 v) { return make_float2((float)v.x * 0x1p-7f, (float)v.y * 0x1p-7f); }

// host: f(X{}) with X the sample type of iq_format fmt (LTEPHY_IQ_CF32 float2, _SC16 short2, _SC8 char2); callers validate fmt beforehand
template <typename F>
inline auto with_iq_type(uint32_t fmt, F&& f)
{
  return fmt == LTEPHY_IQ_SC16 ? f(short2{}) : fmt == LTEPHY_IQ_SC8 ? f(char2{}) : f(float2{});
}

// deterministic warp sum: lane-strided partials already in v, then the fixed halving tree.
__device__ __forceinline__ float warp_tree_sum(float v)
{
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) v = v + __shfl_down_sync(0xffffffffu, v, off);
  return v;
}

// ---- phase B job descriptors ------------------------------------------------------------------
struct DevGrant {          // one PDSCH grant
  uint32_t sf;             // subframe index in batch
  uint32_t sf_idx;         // tti % 10
  uint32_t cfi;
  uint32_t rnti;
  uint32_t tx_scheme, ncw, pmi;
  uint32_t prb_mask[2][4];
  uint32_t nof_re;
  uint32_t re_off[15];     // prefix sum of data REs per OFDM symbol
  uint32_t cls;            // subframe class for the RE masks: 0 = sf 0, 1 = sf 5, 2 = other
  uint32_t np[2];          // allocated PRBs per slot
  uint8_t  plist[2][112];  // allocated PRB indices per slot, ascending
  uint32_t qm[2];
  uint64_t llr_off[2];     // offset (int16 elements) of codeword LLRs in the LLR pool
  uint32_t scr_off[2];     // offset (words) of the scrambling sequence in the sequence pool
};

struct DevScr {            // one PDSCH or PUSCH codeword's scrambling sequence (scr_seq_kernel)
  uint32_t c_init;         // Gold-sequence initialisation, 36.211 6.3.1 (PDSCH) / 5.3.1 (PUSCH)
  uint32_t words;          // sequence words
  uint32_t scr_off;        // offset (words) of the sequence in the sequence pool
};

// The soft-bit, turbo-stream and HARQ pools of one batch pass 2^32 elements (8.6 GB of soft bits after ~24 000 subframes of a loaded
// 20 MHz cell), so offsets into them are 64-bit.  Scrambling-word and payload-byte offsets (scr_off, DevPair.out_byte, DevTb.byte_off) stay
// 32-bit: they would need ~2^37 soft bits or ~200 GB of turbo pool before they wrap, which no 80 GB card holds.
struct DevCb {             // one code block
  uint64_t llr_off;        // first soft bit of this code block in the LLR pool
  uint64_t harq_off;       // int16 offset of this code block's accumulators in the HARQ store
  uint32_t E;              // soft bits received
  uint32_t K, F;
  uint32_t rm_tab;         // offset into the rate-matching table pool: inverse table of (K, F), one uint16 per pair-buffer word
  uint32_t rm_nn;          // repeat period of the received soft bits
  uint32_t rm_rot;         // redundancy version: soft bit k lands on the word whose table entry is (k + rm_rot) mod rm_nn
  uint32_t shift;          // conditioning shift from Qm
  uint32_t pair, half;     // turbo job and 16-bit lane it occupies
  uint32_t harq_op;        // LTEPHY_HARQ_*: 0 none, 1 overwrite the store, 2 add to it
  uint32_t harq_gen;       // 0: first use of the slot in this batch, 1: second, ... (one rate-dematch launch per generation)
};

struct DevPair {           // turbo job: up to two code blocks of equal K decoded by one CTA
  uint64_t buf_off;        // offset (uint32) of this pair's stream buffers in the turbo pool
  uint32_t K, NW, f1, f2;
  uint32_t ncb;            // 1 or 2
  uint32_t crc_type[2];    // 0 none, 1 CRC24A, 2 CRC24B
  uint32_t out_byte[2];    // byte offset in the payload buffer where the CB's data bits go
  uint32_t out_skip[2];    // filler bits to skip at the start
  uint32_t out_bits[2];    // number of data bits to write (K - F - 24*(C>1))
  uint32_t cb_index[2];    // global code-block index (for iters / crc flags)
};

struct DevTb {             // transport block for the final CRC24A
  uint32_t byte_off, nbytes; // payload bytes (tbs/8) followed by 3 CRC bytes written by the turbo kernel
  uint32_t cb_first, ncb;
};
