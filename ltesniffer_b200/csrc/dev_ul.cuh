// dev_ul.cuh -- device descriptors of the PUSCH path
#pragma once
#include "dev_common.cuh"

struct DevUlGrant {
  uint64_t llr_off;       // int16 offset of the codeword in the LLR pool (64-bit: dev_common.cuh, DevCb)
  uint32_t sf, sf_idx, rnti;
  uint32_t M, k0[2], qm;  // M_sc = 12 L_prb, first subcarrier of slot 0 / slot 1 (they differ under type-1 hopping)
  uint32_t dmrs_off[2];   // offsets (float2) of the two slots' DMRS sequences in the DMRS pool
  uint32_t idft_off;      // offset of exp(+j 2 pi m / M), m < M
  uint32_t scr_off;       // word offset of the scrambling sequence (12 M Qm bits)
  uint32_t qp_ack, qp_ri, qp_cqi; // Q' of the multiplexed control information (36.212 5.2.2.6)
  uint32_t nrad, rad;     // IDFT radices, 4 bits each, first stage in the low nibble
};
struct DevUlChest {
  float noise, rsrp;
  float cr[2], ci[2];     // per slot: sum ls[n+1] conj(ls[n]) (timing offset from its argument)
};
