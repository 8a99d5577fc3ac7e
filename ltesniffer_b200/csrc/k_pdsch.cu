// k_pdsch.cu -- K6: PDSCH RE gather + equalise + layer demap + max-log soft demodulation + Gold
// descrambling -> int16 LLRs; K7: turbo rate de-matching into the decoder's stream layout.
// Restates the front half of srsran_pdsch_decode reached through srsran_ue_dl_decode_pdsch
// (reference src/src/DL_Sniffer_PDSCH.cc:997): srsran_predecoding_type, srsran_demod_soft_demodulate_s
// (int16, scales 100*sqrt2/400/700/1000), srsran_scrambling, srsran_rm_turbo_rx_lut.
#include "dev_common.cuh"
#include "k_launch.cuh"
#include "dev_eq.cuh"

// ---- scrambling sequences of every codeword of a PDSCH or PUSCH batch: c = x1 ^ XOR_{b in c_init} basis[b]  (36.211 7.2 without the
// 1600-step warm-up).  Grid: x = codeword, y = block of 256 words.  The codeword count goes on x because gridDim.y stops at 65 535 and a
// batch may carry more codewords than that; a codeword needs a few dozen word blocks at most.
__global__ void __launch_bounds__(256) scr_seq_kernel(const DevScr* __restrict__ cws, const uint32_t* __restrict__ x1,
                                                      const uint32_t* __restrict__ basis, uint32_t basis_words, uint32_t* __restrict__ seq_pool)
{
  const DevScr&  cw = cws[blockIdx.x];
  const uint32_t wi = blockIdx.y * blockDim.x + threadIdx.x;
  if (wi >= cw.words || wi >= basis_words) return;
  uint32_t v = x1[wi];
#pragma unroll
  for (uint32_t b = 0; b < 31; b++)
    if ((cw.c_init >> b) & 1u) v ^= basis[(size_t)b * basis_words + wi];
  seq_pool[cw.scr_off + wi] = v;
}

// soft bits of one equalised symbol of codeword cw at its data-RE index gi
__device__ __forceinline__ void emit(const DevGrant& g, uint32_t cw, uint32_t gi, float2 x, const uint32_t* __restrict__ seq_pool,
                                     short* __restrict__ llr_pool)
{
  const uint32_t qm = g.qm[cw];
  soft_bits(x, 1.0f, qm, seq_pool + g.scr_off[cw], gi * qm, llr_pool + g.llr_off[cw] + (size_t)gi * qm);
}

// One CTA per grant.  Work items are (OFDM symbol, allocated PRB, subcarrier) slots; the 12-bit data-RE
// mask of the PRB gives the rank of the RE inside the grant (36.211 6.3.5 mapping order: k first, then l).
__global__ void __launch_bounds__(256) pdsch_demod_kernel(const __grid_constant__ DevCell c, const DevGrant* __restrict__ grants,
                                                          const float2* __restrict__ sym, const float2* __restrict__ ce,
                                                          const uint32_t* __restrict__ seq_pool, short* __restrict__ llr_pool)
{
  __shared__ uint16_t pref[14][LTEPHY_MAX_PRB + 2];
  __shared__ DevGrant gs;
  const uint32_t tid = threadIdx.x, nt = blockDim.x, N = c.nof_prb;
  for (uint32_t i = tid; i < sizeof(DevGrant) / 4; i += nt) reinterpret_cast<uint32_t*>(&gs)[i] = reinterpret_cast<const uint32_t*>(&grants[blockIdx.x])[i];
  __syncthreads();
  const DevGrant& g    = gs;
  const uint16_t* mask = c.re_mask + ((size_t)(g.cls * 3 + g.cfi - 1) * 14) * N;
  if (tid < 14) {
    const uint32_t l = tid, sl = l / 7, np = g.np[sl];
    uint32_t       acc = 0;
    for (uint32_t j = 0; j < np; j++) {
      pref[l][j] = (uint16_t)acc;
      acc += __popc(mask[l * N + g.plist[sl][j]]);
    }
    pref[l][np] = (uint16_t)acc;
  }
  __syncthreads();
  const SfView   v  = make_view(c, sym, ce, g.sf);
  const uint32_t n0 = 7 * 12 * g.np[0], n1 = 7 * 12 * g.np[1];
  for (uint32_t it = tid; it < n0 + n1; it += nt) {
    uint32_t sl, rem;
    if (it < n0)
      sl = 0, rem = it;
    else
      sl = 1, rem = it - n0;
    const uint32_t per = 12 * g.np[sl], l = 7 * sl + rem / per, q = rem % per, j = q / 12, kk = q % 12;
    const uint32_t prb = g.plist[sl][j], m = mask[l * N + prb];
    if (!((m >> kk) & 1u)) continue;
    const uint32_t r = pref[l][j] + __popc(m & ((1u << kk) - 1u)), gi = g.re_off[l] + r, idx = l * c.nsc + 12 * prb + kk;
    if (g.tx_scheme == LTEPHY_TX_PORT0) {
      emit(g, 0, gi, eq_port0(c, v, idx), seq_pool, llr_pool);
    } else if (g.tx_scheme == LTEPHY_TX_DIVERSITY) {
      if (gi & 1u) continue; // handled together with its even partner
      const uint32_t rest = m >> (kk + 1);
      uint32_t       idx2;
      if (rest)
        idx2 = idx + 1 + (uint32_t)(__ffs(rest) - 1);
      else { // partner is the first data RE of the next allocated PRB (never happens for even per-PRB counts)
        const uint32_t prb2 = g.plist[sl][j + 1], m2 = mask[l * N + prb2];
        idx2 = l * c.nsc + 12 * prb2 + (uint32_t)(__ffs(m2) - 1);
      }
      float2 x0, x1;
      eq_sfbc(c, v, idx, idx2, x0, x1);
      emit(g, 0, gi, x0, seq_pool, llr_pool);
      emit(g, 0, gi + 1, x1, seq_pool, llr_pool);
    } else if (g.tx_scheme == LTEPHY_TX_CDD) {
      float2 x0, x1;
      eq_cdd(c, v, idx, (gi & 1u) != 0, x0, x1);
      emit(g, 0, gi, x0, seq_pool, llr_pool);
      emit(g, 1, gi, x1, seq_pool, llr_pool);
    } else if (g.tx_scheme == LTEPHY_TX_SPATIALMUX) {
      if (g.ncw == 1) {
        emit(g, 0, gi, eq_spmux1(c, v, idx, spmux_w(1, g.pmi)), seq_pool, llr_pool);
      } else {
        float2 x0, x1;
        eq_spmux2(c, v, idx, spmux_w(2, g.pmi), x0, x1);
        emit(g, 0, gi, x0, seq_pool, llr_pool);
        emit(g, 1, gi, x1, seq_pool, llr_pool);
      }
    }
  }
}

// ---- K7: one CTA per code-block pair, iterating over the words of the pair buffer.  Word w of a code block sits at
// position j = inv[w] of the rv-0 circular order (the table is shared by every redundancy version); it receives soft bits
// k, k+nn, k+2nn, ... < E with k = (j - rot) mod nn, summed in that (received) order.  Consecutive words are consecutive
// rows of one interleaver column, so the table reads and the stores are coalesced and the gathers of e nearly so.  Every
// word is written, so the stream buffers need no memset.
__device__ __forceinline__ int sat16(int v) { return v > 32767 ? 32767 : (v < -32768 ? -32768 : v); }

#define RM_UNROLL 4 // words per thread whose table reads and first gathers are in flight together

struct RmHalf {
  const short*    e;
  const uint16_t* inv;
  short*          hq; // HARQ accumulators, or nullptr
  uint32_t        E, nn, rot, shift, retx;
};
__device__ __forceinline__ RmHalf rm_half(const DevCb& cb, const short* llr_pool, const uint16_t* rm_pool, short* harq_pool)
{
  // HARQ store (reference src/src/HARQ.cc, DL_Sniffer_PDSCH.cc:955-985): the accumulators of this code block live at the pair-buffer word index,
  // which does not depend on the redundancy version; a retransmission starts from what earlier transmissions left there
  return RmHalf{llr_pool + cb.llr_off, rm_pool + cb.rm_tab, cb.harq_op ? harq_pool + cb.harq_off : nullptr, cb.E, cb.rm_nn, cb.rm_rot, cb.shift,
                cb.harq_op == LTEPHY_HARQ_RETX ? 1u : 0u};
}
// conditioned value of word w with table entry j of one code block: sat16 sum of its soft bits (first one, x0, already loaded)
__device__ __forceinline__ int rm_word_value(const RmHalf& h, uint32_t w, uint32_t j, uint32_t k, int x0, int acc)
{
  if (j == LTEPHY_RM_NONE) return 0;
  if (j == LTEPHY_RM_FILLER) return -255; // filler bits are known zeros: strong "0" in the systematic and first parity streams
  if (k < h.E) {
    acc = sat16(acc + x0);
    for (uint32_t kk = k + h.nn; kk < h.E; kk += h.nn) acc = sat16(acc + (int)h.e[kk]);
  }
  if (h.hq) h.hq[w] = (short)acc;
  const int v = acc >> h.shift;
  return v > 255 ? 255 : (v < -255 ? -255 : v);
}

__global__ void __launch_bounds__(256) rm_turbo_rx_kernel(const DevCb* __restrict__ cbs, const DevPair* __restrict__ pairs,
                                                          const short* __restrict__ llr_pool, const uint16_t* __restrict__ rm_pool,
                                                          uint32_t* __restrict__ turbo_pool, short* __restrict__ harq_pool, uint32_t gen)
{
  const DevPair& pr  = pairs[blockIdx.x];
  const uint32_t ncb = pr.ncb, nwords = 96 * pr.NW + 16;
  const DevCb&   c0 = cbs[pr.cb_index[0]];
  const DevCb&   c1 = cbs[pr.cb_index[ncb - 1]];
  // a HARQ slot used twice in one batch puts its later use in a later launch: only the halves of this generation are written
  const bool do0 = c0.harq_gen == gen, do1 = ncb == 2 && c1.harq_gen == gen;
  if (!do0 && !do1) return;
  const bool     full = do0 && (do1 || ncb == 1); // whole 32-bit words (a single code block keeps its high half at 0)
  const RmHalf   h0 = rm_half(c0, llr_pool, rm_pool, harq_pool), h1 = rm_half(c1, llr_pool, rm_pool, harq_pool);
  uint32_t*      bw = turbo_pool + pr.buf_off;
  short*         bh = reinterpret_cast<short*>(bw);
  for (uint32_t base = threadIdx.x; base < nwords; base += RM_UNROLL * blockDim.x) {
    uint32_t j0[RM_UNROLL], j1[RM_UNROLL], k0[RM_UNROLL], k1[RM_UNROLL];
    int      x0[RM_UNROLL], x1[RM_UNROLL], a0[RM_UNROLL], a1[RM_UNROLL];
#pragma unroll
    for (int u = 0; u < RM_UNROLL; u++) {
      const uint32_t w = base + u * blockDim.x;
      j0[u] = do0 && w < nwords ? h0.inv[w] : LTEPHY_RM_NONE;
      j1[u] = do1 && w < nwords ? h1.inv[w] : LTEPHY_RM_NONE;
    }
#pragma unroll
    for (int u = 0; u < RM_UNROLL; u++) {
      const uint32_t w = base + u * blockDim.x;
      const bool     r0 = j0[u] < h0.nn, r1 = j1[u] < h1.nn;
      k0[u] = j0[u] >= h0.rot ? j0[u] - h0.rot : j0[u] + h0.nn - h0.rot;
      k1[u] = j1[u] >= h1.rot ? j1[u] - h1.rot : j1[u] + h1.nn - h1.rot;
      x0[u] = r0 && k0[u] < h0.E ? (int)h0.e[k0[u]] : 0;
      x1[u] = r1 && k1[u] < h1.E ? (int)h1.e[k1[u]] : 0;
      a0[u] = r0 && h0.retx ? (int)h0.hq[w] : 0;
      a1[u] = r1 && h1.retx ? (int)h1.hq[w] : 0;
    }
#pragma unroll
    for (int u = 0; u < RM_UNROLL; u++) {
      const uint32_t w = base + u * blockDim.x;
      if (w >= nwords) break;
      const int v0 = rm_word_value(h0, w, j0[u], k0[u], x0[u], a0[u]), v1 = rm_word_value(h1, w, j1[u], k1[u], x1[u], a1[u]);
      if (full)
        bw[w] = ((uint32_t)v0 & 0xFFFFu) | ((uint32_t)v1 << 16);
      else if (do0)
        bh[2 * w] = (short)v0;
      else
        bh[2 * w + 1] = (short)v1;
    }
  }
}

extern "C" void launch_scr_seq(const DevScr* cws, uint32_t ncw, uint32_t max_words, const uint32_t* gold_x1, const uint32_t* gold_basis,
                               uint32_t basis_words, uint32_t* seq_pool, cudaStream_t st, uint64_t* launches)
{
  if (!ncw) return;
  scr_seq_kernel<<<dim3(ncw, (max_words + 255) / 256), 256, 0, st>>>(cws, gold_x1, gold_basis, basis_words, seq_pool);
  *launches += 1;
}
extern "C" void launch_pdsch_front(const DevCell& c, const DevGrant* grants, uint32_t ngrants, const float2* sym, const float2* ce,
                                   const uint32_t* seq_pool, short* llr_pool, cudaStream_t st, uint64_t* launches)
{
  if (!ngrants) return;
  pdsch_demod_kernel<<<ngrants, 256, 0, st>>>(c, grants, sym, ce, seq_pool, llr_pool);
  *launches += 1;
}
extern "C" void launch_rm_turbo_rx(const DevCb* cbs, const DevPair* pairs, uint32_t npairs, const short* llr_pool, const uint16_t* rm_pool,
                                   uint32_t* turbo_pool, short* harq_pool, uint32_t gen, cudaStream_t st, uint64_t* launches)
{
  if (!npairs) return;
  rm_turbo_rx_kernel<<<npairs, 256, 0, st>>>(cbs, pairs, llr_pool, rm_pool, turbo_pool, harq_pool, gen);
  *launches += 1;
}
