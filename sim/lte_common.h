/*
 * lte_common.h -- LTE (36.211/212/213) primitives shared by the synthetic eNB (sim/) and the
 * CPU oracle (oracle/).  TEST INFRASTRUCTURE: nothing under ltesniffer_b200/ links this.
 *
 * The reference delegates all of this to srsRAN (absent from /root/reference, see SURVEY.md
 * section 8c); each function names the reference call site whose behaviour it restates.
 */
#ifndef LTE_COMMON_H
#define LTE_COMMON_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  float re, im;
} cf_t;

#define LTE_MAX_PRB 110
#define LTE_NRE 12
#define LTE_NSYMB_SF 14 /* normal CP only (file mode assumes normal CP: src/src/LTESniffer_Core.cc:242-247) */
#define LTE_MAX_PORTS 2
#define LTE_MAX_ANT 2
#define LTE_MAX_CCE 88
#define LTE_DCI_MAX_BITS 64

typedef struct {
  uint32_t nof_prb;   /* 6,15,25,50,75,100 */
  uint32_t nof_ports; /* 1 or 2 CRS ports */
  uint32_t cell_id;   /* PCI 0..503 */
  uint32_t nof_rx;    /* rx antennas 1 or 2 */
  uint32_t symbol_sz; /* FFT size; 0 = the standard LTE rate (2048 at 100 PRB).  srsRAN's default build samples at 3/4 of it
                         (srsran_symbol_sz: 1536 at 100 PRB, 768 at 50, 384 at 25), which is what LTESniffer records with */
  uint32_t phich_ng;  /* phich-Resource of the MIB as srsran_phich_r_t: 0 = Ng 1/6, 1 = 1/2, 2 = 1, 3 = 2 */
  uint32_t phich_ext; /* phich-Duration of the MIB: 0 normal, 1 extended */
} lte_cell_t;

/* numerology */
uint32_t lte_fft_size(uint32_t nof_prb);
uint32_t lte_cell_fft(const lte_cell_t* c); /* symbol_sz, or the standard size when it is 0 */
uint32_t lte_cp_len(uint32_t fft, uint32_t symbol_in_slot);
uint32_t lte_sf_len(uint32_t nof_prb);

/* ---- sequences / CRC ---- */
void     lte_gold_bits(uint32_t c_init, uint8_t* c, uint32_t len);               /* 36.211 7.2 */
uint32_t lte_crc(uint32_t poly, uint32_t order, const uint8_t* bits, uint32_t n); /* bitwise, zero init */
#define LTE_CRC24A 0x1864CFBu
#define LTE_CRC24B 0x1800063u
#define LTE_CRC16 0x11021u
#define LTE_CRC8 0x19Bu
void lte_bits_pack(const uint8_t* bits, uint32_t nbits, uint8_t* bytes); /* MSB first */
void lte_bits_unpack(const uint8_t* bytes, uint32_t nbits, uint8_t* bits);

/* ---- CRS (36.211 6.10.1) ---- */
/* fills pilot value r_{l,ns}(m') for m = 0..2*nof_prb-1; returns subcarrier offset (v+v_shift)%6 */
uint32_t lte_crs(const lte_cell_t* c, uint32_t port, uint32_t ns, uint32_t l, cf_t* pilots);
uint32_t lte_crs_offset(const lte_cell_t* c, uint32_t port, uint32_t l_in_slot);

/* ---- control region REG geometry (36.211 6.2.4, 6.7.4, 6.9.3, 6.8.5) ---- */
typedef struct {
  uint16_t k0; /* lowest subcarrier of the REG */
  uint8_t  l;  /* OFDM symbol */
  uint8_t  kind; /* 0 = free for PDCCH, 1 = PCFICH, 2 = PHICH */
  uint16_t k[4]; /* the 4 data REs of the REG (CRS slots skipped) */
} lte_reg_t;

typedef struct {
  lte_cell_t cell;
  uint32_t   nof_regs_sym[3]; /* REGs in symbol 0,1,2 */
  lte_reg_t  regs[3 * 3 * LTE_MAX_PRB];
  uint32_t   nof_regs_total;
  uint32_t   pcfich_reg[4]; /* indices into regs[] */
  uint32_t   nof_phich_groups;
  uint32_t   phich_reg[3 * 28]; /* up to ceil(2 * 110 / 8) groups */
  /* per CFI: */
  uint32_t nof_pdcch_regs[3]; /* (N_reg/9)*9 */
  uint32_t nof_cce[3];
  /* pdcch_map[cfi-1][q] = index into regs[] of the REG carrying quadruplet q of the CCE stream
   * (interleaver + cyclic shift applied; restates srsRAN regs_pdcch_init behaviour used by
   *  srsran_pdcch_extract_llr at src/src/DCISearch.cc:562) */
  uint16_t pdcch_map[3][3 * 3 * LTE_MAX_PRB];
} lte_regs_t;

int lte_regs_init(lte_regs_t* r, const lte_cell_t* cell);

/* ---- convolutional code (36.212 5.1.3.1 / 5.1.4.2) ---- */
void lte_conv_encode(const uint8_t* in, uint32_t K, uint8_t* out /* 3K, stream-major d0|d1|d2 */);
/* w-index table: for circular-buffer position j (NULLs removed, 0..3K-1) gives index into the
 * stream-major coded array (s*K + k). */
void lte_rm_conv_table(uint32_t K, uint16_t* tab /* 3K */);
void lte_rm_conv_tx(const uint8_t* d, uint32_t K, uint8_t* e, uint32_t E);

/* ---- turbo code (36.212 5.1.3.2 / 5.1.4.1) ---- */
typedef struct {
  uint32_t tbs, C, Kp, Km, Cp, Cm, F;
} lte_cbsegm_t;
int      lte_cbsegm(lte_cbsegm_t* s, uint32_t tbs);
uint32_t lte_cb_K(const lte_cbsegm_t* s, uint32_t r); /* first Cm blocks use Km */
void     lte_qpp(uint32_t K, uint16_t* pi);           /* pi[i] = (f1 i + f2 i^2) mod K */
/* encode one code block: in[K] -> d0,d1,d2 each K+4 */
void lte_turbo_encode(const uint8_t* in, uint32_t K, uint8_t* d0, uint8_t* d1, uint8_t* d2);
/* circular-buffer map: for w position j in [0,3*Kpi) returns index into stream-major (s*(K+4)+k)
 * or 0xFFFFFFFF for a <NULL> dummy.  Kpi = 32*ceil((K+4)/32). */
uint32_t lte_rm_turbo_table(uint32_t K, uint32_t* tab /* 3*Kpi */);
uint32_t lte_rm_turbo_k0(uint32_t K, uint32_t rv);
/* rate-match one code block: d (stream-major, 3*(K+4)), F filler bits at the start of d0/d1 are
 * treated as <NULL>; writes E bits */
void lte_rm_turbo_tx(const uint8_t* d, uint32_t K, uint32_t F, uint32_t rv, uint8_t* e, uint32_t E);
/* E_r for code block r (36.212 5.1.4.1.2) */
uint32_t lte_rm_turbo_E(uint32_t G, uint32_t C, uint32_t r, uint32_t Qm, uint32_t NL);

/* ---- modulation (36.211 7.1) ---- */
void lte_modulate(const uint8_t* bits, uint32_t nsym, uint32_t Qm, cf_t* out);

/* ---- DCI (36.212 5.3.3) ---- */
typedef enum {
  LTE_DCI_FORMAT0 = 0,
  LTE_DCI_FORMAT1,
  LTE_DCI_FORMAT1A,
  LTE_DCI_FORMAT1B,
  LTE_DCI_FORMAT1C,
  LTE_DCI_FORMAT1D,
  LTE_DCI_FORMAT2,
  LTE_DCI_FORMAT2A,
  LTE_DCI_FORMAT2B,
  LTE_DCI_NOF_FORMATS
} lte_dci_format_t; /* same order as the reference's list, src/src/DCISearch.cc:84-95 */

uint32_t lte_dci_sizeof(const lte_cell_t* c, lte_dci_format_t f); /* restates srsran_dci_format_sizeof (falcon_pdcch.c:133) */

typedef struct {
  uint16_t rnti;
  uint8_t  format;
  /* resource allocation */
  uint8_t  alloc_type;  /* 0,1,2 */
  uint32_t rbg_bitmask; /* type0 */
  uint32_t t1_vrb_bitmask, t1_subset, t1_shift;
  uint32_t riv;         /* type2 */
  uint8_t  t2_dist;     /* 1 = distributed VRB */
  uint8_t  t2_ngap2;    /* gap selection */
  uint8_t  n_prb1a;     /* 2 or 3 (SI/P/RA-RNTI 1A TBS column) */
  /* TBs */
  uint8_t  mcs[2], rv[2], ndi[2];
  uint8_t  tb_en[2];
  uint8_t  tb_cw_swap;
  uint8_t  pinfo;
  uint8_t  pid, tpc;
  /* format 0 */
  uint8_t  hop, n_dmrs, cqi_req;
} lte_dci_t;

int lte_dci_pack(const lte_cell_t* c, const lte_dci_t* d, uint8_t* bits, uint32_t* nbits);
int lte_dci_unpack(const lte_cell_t* c, lte_dci_format_t f, uint16_t rnti, const uint8_t* bits, uint32_t nbits, lte_dci_t* d);

/* ---- DL grant (36.213 7.1.6 / 7.1.7) ---- */
typedef enum { LTE_TX_PORT0 = 0, LTE_TX_DIVERSITY, LTE_TX_CDD, LTE_TX_SPATIALMUX } lte_txscheme_t;
typedef struct {
  uint8_t  prb_mask[2][LTE_MAX_PRB]; /* per slot */
  uint32_t nof_prb;
  uint32_t nof_tb;
  struct {
    uint8_t  enabled;
    uint8_t  qm;     /* 2,4,6,8 */
    uint8_t  rv;
    uint8_t  mcs;
    int32_t  tbs;
    uint32_t nof_bits; /* G */
  } tb[2];
  uint32_t nof_re;
  uint8_t  tx_scheme;
  uint8_t  nof_layers;
  uint8_t  pmi;
  uint8_t  cw_swap; /* 2 TBs and the "transport block to codeword swap flag" of DCI 2/2A set (36.212 Table 5.3.3.1.5-1): TB1 -> codeword 1, TB2 -> codeword 0 */
} lte_dl_grant_t;

#define LTE_SIRNTI 0xFFFF
#define LTE_PRNTI 0xFFFE
#define LTE_RARNTI_START 0x0001
#define LTE_RARNTI_END 0x000A
#define LTE_CRNTI_START 0x000B
#define LTE_CRNTI_END 0xFFF3
#define LTE_RNTI_ISUSER(r) ((r) >= LTE_CRNTI_START && (r) <= LTE_CRNTI_END)

/* restates dl_sniffer_ra_dl_dci_to_grant (lib/src/phy/falcon_phch/dl_sniffer_pdsch.c:95-132) +
 * dl_sniffer_config_mimo (:255-276); returns 0 ok, <0 error */
int lte_dl_dci_to_grant(const lte_cell_t* c, uint32_t sf_idx, uint32_t cfi, int use_alt_table, const lte_dci_t* d, lte_dl_grant_t* g);
int lte_tbs_from_idx(int itbs, uint32_t nprb);
/* which REs of symbol l in PRB prb are PDSCH data for this cell/subframe; returns count, fills k[] (abs subcarrier) */
uint32_t lte_pdsch_re_in_prb(const lte_cell_t* c, uint32_t sf_idx, uint32_t cfi, uint32_t l, uint32_t prb, uint16_t* k);

/* ---- PDCCH search spaces (36.213 9.1.1) ---- */
uint32_t lte_pdcch_ue_locations(uint32_t nof_cce, uint32_t sf_idx, uint16_t rnti, uint16_t* ncce, uint8_t* L, uint32_t max);
uint32_t lte_pdcch_common_locations(uint32_t nof_cce, uint16_t* ncce, uint8_t* L, uint32_t max);
/* restates srsran_pdcch_validate_location (lib/src/phy/falcon_phch/falcon_pdcch.c:223-250) */
uint32_t lte_pdcch_validate_location(uint32_t nof_cce, uint32_t ncce, uint32_t L, uint32_t sf_idx, uint16_t rnti);

/* ---- PCFICH (36.212 5.3.4) ---- */
extern const uint8_t lte_cfi_codeword[3][32];

/* ---- deterministic RNG (splitmix/xoshiro) so sim + tests are reproducible ---- */
typedef struct {
  uint64_t s[4];
} lte_rng_t;
void     lte_rng_seed(lte_rng_t* r, uint64_t seed);
uint64_t lte_rng_u64(lte_rng_t* r);
double   lte_rng_uniform(lte_rng_t* r);
double   lte_rng_gauss(lte_rng_t* r);

#ifdef __cplusplus
}
#endif
#endif

/* ---- PBCH / MIB (36.211 6.6, 36.212 5.3.1, 36.331 MasterInformationBlock): what srsran_ue_mib_decode + srsran_pbch_mib_unpack deliver
 * at src/src/LTESniffer_Core.cc:382-396 ---- */
#ifndef LTE_COMMON_PBCH_H
#define LTE_COMMON_PBCH_H
#ifdef __cplusplus
extern "C" {
#endif
/* the 240 resource elements of one radio frame's PBCH part: slot 1 of subframe 0, symbols 0..3, the central 72 sub-carriers without the CRS
 * positions of four ports; symbol-major, ascending sub-carrier */
uint32_t lte_pbch_re(const lte_cell_t* c, uint16_t* k /* [240] */, uint8_t* l /* [240], 7..10 */);
/* 24 MIB bits: dl-Bandwidth (3), phich-Duration (1), phich-Resource (2), systemFrameNumber (8 MSBs), 10 spare */
void lte_mib_pack(uint32_t nof_prb, uint32_t phich_ext, uint32_t phich_res, uint32_t sfn, uint8_t* bits);
int  lte_mib_unpack(const uint8_t* bits, uint32_t* nof_prb, uint32_t* phich_ext, uint32_t* phich_res, uint32_t* sfn);
/* CRC mask of the antenna-port count (36.212 Table 5.3.1.1-1): 1 -> 0x0000, 2 -> 0xFFFF, 4 -> 0x5555; 0 for anything else */
uint32_t lte_pbch_crc_mask(uint32_t nof_ports);
/* synchronisation signals (36.211 6.11, FDD): d[n], n = 0..61, goes to the sub-carrier n - 31 (n < 31) or n - 30 (n >= 31) around DC.
 * PSS: Zadoff-Chu root 25 / 29 / 34 of N_ID_2 = 0 / 1 / 2, each value computed in double and rounded to float.
 * SSS: the +-1 sequence of subframe 0 (sf5 = 0) or subframe 5 (sf5 = 1) of N_ID_1 (0..167) and N_ID_2 (6.11.2.1). */
void lte_pss(uint32_t n_id_2, cf_t* d /* [62] */);
void lte_sss(uint32_t n_id_1, uint32_t n_id_2, uint32_t sf5, float* d /* [62] */);
#ifdef __cplusplus
}
#endif
#endif

/* ================================================================== uplink (PUSCH), 36.211 5.x / 36.213 8 */
#ifndef LTE_COMMON_UL_H
#define LTE_COMMON_UL_H
#ifdef __cplusplus
extern "C" {
#endif
typedef struct {
  uint32_t n_dmrs1;       /* cyclicShift of SIB2, 0..7 (ULSchedule::set_config, src/src/ULSchedule.cc:140-158); n_DMRS^(1) by Table 5.5.2.1.1-2 */
  uint32_t delta_ss;      /* groupAssignmentPUSCH */
  uint32_t group_hopping; /* groupHoppingEnabled: u = (f_gh(ns) + f_ss) mod 30, 36.211 5.5.1.3 */
  uint32_t seq_hopping;   /* sequenceHoppingEnabled: v = c(ns) for M_sc >= 72 when group hopping is off, 36.211 5.5.1.4 */
  uint32_t n_rb_ho;       /* pusch-HoppingOffset (SubframeWorker.cc:271, DCICollection.cc:168) */
} lte_ul_cfg_t;

typedef struct {
  uint16_t rnti;
  uint32_t L_prb, n_prb; /* contiguous allocation; n_prb = first PRB of slot 0 */
  uint32_t mcs, qm, rv;
  int32_t  tbs;
  uint32_t n_dmrs2;      /* mapped from the 3-bit cyclic shift field of DCI format 0 */
  uint32_t nof_re, nof_bits; /* nof_bits = G: the bits of the UL-SCH codeword after the CQI / RI symbols are taken out */
  uint32_t hop;          /* 0: both slots at n_prb; 1: type-1 hopping, slot 1 at n_prb_slot1 (ul_sniffer_pusch.c:48-80) */
  uint32_t n_prb_slot1;
  /* control information multiplexed with the data (36.212 5.2.2.6-8); what PUSCH_Decoder::decode sets at UL_Sniffer_PUSCH.cc:429-450 */
  uint32_t nof_ack, ri_len, cqi_len;                  /* O_ACK (0..2), O_RI (0..2), O_CQI (bits, without CRC) */
  uint32_t I_offset_ack, I_offset_ri, I_offset_cqi;   /* betaOffset indices (36.213 Tables 8.6.3-1..3) */
  float    ta_us;        /* simulator only: timing offset of this UE's transmission (decoder ignores it) */
} lte_ul_grant_t;

/* where the control information sits in the R' x 12 channel-interleaver matrix */
typedef struct {
  uint32_t Qp_ack, Qp_ri, Qp_cqi; /* Q' (modulation symbols) */
  uint32_t G;                     /* UL-SCH bits left: (12 M_sc - Q'_cqi - Q'_ri) Qm */
} lte_uci_layout_t;

/* L_prb must be 2^a 3^b 5^c (valid_prb_ul, src/src/UL_Sniffer_PUSCH.cc:3-10) */
int lte_ul_valid_prb(uint32_t L_prb);
/* restates srsran_ra_ul_dci_to_grant as used at falcon_dci.c:222; table: 0 = 16QAM cap (enable_64qam false), 1 = 64QAM.
 * ucfg may be NULL (n_rb_ho = 0).  returns 0 ok */
int lte_ul_dci_to_grant(const lte_cell_t* c, const lte_dci_t* d, int table, lte_ul_grant_t* g);
int lte_ul_dci_to_grant_hop(const lte_cell_t* c, const lte_ul_cfg_t* ucfg, const lte_dci_t* d, int table, lte_ul_grant_t* g);
/* DMRS for PUSCH (36.211 5.5.2.1) for slot ns: M_sc complex values; returns 0, or -1 if M_sc < 36 (the
 * computer-generated 1- and 2-PRB base sequences are not implemented) */
int lte_pusch_dmrs(const lte_cell_t* c, const lte_ul_cfg_t* u, uint32_t ns, uint32_t n_dmrs2, uint32_t M_sc, cf_t* r);
/* base-sequence group u and sequence v of slot ns (36.211 5.5.1.3 / 5.5.1.4) */
void lte_pusch_uv(const lte_cell_t* c, const lte_ul_cfg_t* u, uint32_t ns, uint32_t M_sc, uint32_t* u_out, uint32_t* v_out);
/* Q' of ACK, RI, CQI and the remaining G (36.212 5.2.2.6; srsRAN Q_prime_ri_ack / Q_prime_cqi in phy/phch/uci.c, sch.c) */
void lte_uci_layout(const lte_ul_grant_t* g, lte_uci_layout_t* L);
/* kind[r * 12 + c] for the R' = 12 L_prb rows x 12 columns: 0 data, 1 CQI, 2 RI, 3 ACK (punctures data / CQI); dpos[] = index of the symbol in the
 * UL-SCH (kind 0 / 3) or CQI (kind 1) stream.  36.212 5.2.2.7 / 5.2.2.8 */
void lte_uci_map(uint32_t M_sc, const lte_uci_layout_t* L, uint8_t* kind, uint32_t* dpos);
uint32_t lte_largest_prime_below(uint32_t n);
#ifdef __cplusplus
}
#endif
#endif
