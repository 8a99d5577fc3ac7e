// lte_host.hpp -- host-side (C++17) LTE table builders for the CUDA PHY library.
// Product code: independent of sim/ and oracle/.  Everything here is integer/table work that the
// reference obtains from srsRAN at *_init / *_set_cell time (srsran_ue_dl_set_cell,
// src/src/SubframeWorker.cc:100-107) or per grant (srsran_ra_*, lib/src/phy/falcon_phch/dl_sniffer_pdsch.c).
#pragma once
#include <array>
#include <cstdint>
#include <map>
#include <vector>

namespace ltehost {

struct Cell {
  uint32_t nof_prb = 0, nof_ports = 1, cell_id = 0, nof_rx = 1;
  uint32_t phich_ng = 0;  // phich-Resource of the MIB as srsran_phich_r_t: 0 = 1/6, 1 = 1/2, 2 = 1, 3 = 2
  uint32_t phich_ext = 0; // phich-Duration of the MIB: 0 normal (symbol 0), 1 extended (one REG of every group in each of symbols 0, 1, 2)
};

// ---- numerology
uint32_t fft_size(uint32_t nof_prb);
uint32_t cp_len(uint32_t fft, uint32_t sym_in_slot);
inline uint32_t sf_len(uint32_t nof_prb) { return 15u * fft_size(nof_prb); }

// ---- pseudo-random sequence (36.211 7.2), bit i of the sequence at bit (i & 31) of word i >> 5
std::vector<uint32_t> gold_words(uint32_t c_init, uint32_t nbits);
// basis for the jump-free generator used on the device: seq(c_init) = x1 ^ XOR_{b in c_init} basis[b]
struct GoldBasis {
  uint32_t              nwords = 0;
  std::vector<uint32_t> x1;    // [nwords]
  std::vector<uint32_t> basis; // [31][nwords]
};
GoldBasis gold_basis(uint32_t nbits);

// ---- CRC helpers (host side of the parallel CRC24 used by the turbo kernel)
uint32_t crc_bits(uint32_t poly, uint32_t order, const uint8_t* bits, uint32_t n);
// x^(8*i) mod poly for i = 0..n-1 (24-bit polynomials)
std::vector<uint32_t> crc24_xpow8(uint32_t poly, uint32_t n);
constexpr uint32_t    CRC24A = 0x1864CFBu, CRC24B = 0x1800063u, CRC16 = 0x11021u;

// ---- CRS (36.211 6.10.1): value table [sf 10][port 2][pilot symbol 4][2*nof_prb] as (re,im) floats
std::vector<float> crs_table(const Cell& c);
uint32_t           crs_offset(const Cell& c, uint32_t port, uint32_t sym_in_slot);

// ---- control region geometry
struct CtrlMap {
  uint32_t              nof_cce[3]{};
  std::vector<uint16_t> pdcch_idx[3]; // per CFI: [nof_cce*9][4] grid indices l*nsc + k of the REs of each quadruplet
  uint16_t              pcfich_idx[16]{};
};
bool build_ctrl_map(const Cell& c, CtrlMap& out);

// ---- DCI payload sizes (srsran_dci_format_sizeof, lib/src/phy/falcon_phch/falcon_pdcch.c:133)
enum Format { F0 = 0, F1, F1A, F1B, F1C, F1D, F2, F2A, F2B, NOF_FORMATS };
uint32_t dci_sizeof(const Cell& c, Format f);
struct SizeTable {
  std::vector<uint32_t> sizes;                  // distinct sizes, ascending order of first appearance in the format list
  uint32_t              index_of[NOF_FORMATS]{}; // format -> index into sizes
};
SizeTable dci_size_table(const Cell& c);
// convolutional rate-matching table (36.212 5.1.4.2): circular position j -> stream-major index s*K+k
std::vector<uint16_t> conv_rm_table(uint32_t K);

// ---- blind-search locations (srsran_pdcch_ue_locations_all_map, falcon_pdcch.c:321-356)
struct Location {
  uint16_t ncce;
  uint8_t  L;
};
std::vector<Location> all_locations(uint32_t nof_cce);

// ---- turbo code structure
struct Segm {
  uint32_t tbs = 0, C = 0, Kp = 0, Km = 0, Cp = 0, Cm = 0, F = 0;
  uint32_t K(uint32_t r) const { return r < Cm ? Km : Kp; }
};
bool     cb_segmentation(uint32_t tbs, Segm& s);
// control information multiplexed on PUSCH (36.212 5.2.2.6): Q' modulation symbols of HARQ-ACK, RI, CQI and the UL-SCH bits G that remain.
// false: invalid TBS or a reserved beta-offset index (36.213 Tables 8.6.3-1..3)
struct UciLayout {
  uint32_t Qp_ack, Qp_ri, Qp_cqi, G;
};
bool uci_layout(uint32_t L_prb, uint32_t qm, uint32_t tbs, uint32_t nof_ack, uint32_t ri_len, uint32_t cqi_len, uint32_t I_ack, uint32_t I_ri, uint32_t I_cqi,
                UciLayout& out);
bool     qpp_params(uint32_t K, uint32_t& f1, uint32_t& f2);
uint32_t rm_turbo_E(uint32_t G, uint32_t C, uint32_t r, uint32_t Qm, uint32_t NL);
// order[k], k in [0, nn): the stream position (s*(K+4)+i) that receives soft bit k, k+nn, k+2nn, ...
// nn = number of transmittable circular-buffer positions (the repeat period).
struct RmTurboTable {
  uint32_t              nn = 0;
  std::vector<uint32_t> order; // [nn]
};
RmTurboTable rm_turbo_table(uint32_t K, uint32_t F, uint32_t rv);
// word of the turbo pair buffer that holds stream position s = st*(K+4)+i: the window-transposed sys / p1 / p2 streams ([32][NW]
// each, i < K), then the 12 tail words; 4 pad words end the buffer (96*NW + 16 words)
uint32_t rm_turbo_word(uint32_t K, uint32_t s);
// rm_turbo_table inverted per pair-buffer word, for every redundancy version at once: inv[w] = position j in [0, nn) of word w in the
// rv-0 order, LTEPHY_RM_FILLER for a filler bit of sys / p1, LTEPHY_RM_NONE for a word no soft bit reaches.  nn does not depend on
// rv (N_cb = K_w), so the order of rv is the rv-0 order rotated by rot[rv]: soft bit k of rv lands on the word with j = (k + rot[rv]) mod nn.
struct RmTurboInverse {
  uint32_t              nn = 0, rot[4]{};
  std::vector<uint16_t> inv; // [96*NW + 16]
};
RmTurboInverse rm_turbo_inverse(uint32_t K, uint32_t F);

// ---- PDSCH resource elements: count of data REs of symbol l in PRB prb (and which k) ---------
uint32_t pdsch_re_in_prb(const Cell& c, uint32_t sf_idx, uint32_t cfi, uint32_t l, uint32_t prb, uint16_t* k /*12*/);

// ---- DCI fields as unpacked from the payload (stage 1 of the DCI -> grant chain; srsran_dci_dl_t without the grant) -------------
struct DlDciFields {
  uint8_t  format;
  uint16_t rnti;
  uint32_t alloc;                                    // resource allocation type 0 / 1 / 2
  uint32_t rbg_mask, t1_subset, t1_shift, t1_mask;   // type 0 / type 1
  uint32_t riv;                                      // type 2
  bool     dist, ngap2;                              // distributed VRBs, N_gap2
  uint32_t n_prb1a;                                  // 2 or 3 (format 1A to a non-user RNTI: TBS column)
  uint8_t  mcs[2], rv[2], ndi[2];
  bool     tb_en[2];
  uint8_t  harq_pid, tpc, tb_cw_swap, pinfo;
};

} // namespace ltehost
// host_search.cpp: the stages of ltephy_dci_to_grant, shared with the srsRAN-compatible shim (compat/src)
int ltehost_unpack_dl_dci(const ltehost::Cell& c, uint32_t format, uint16_t rnti, uint64_t bits, ltehost::DlDciFields& f);
int ltehost_dl_prb_allocation(uint32_t N, const ltehost::DlDciFields& f, uint32_t mask[2][4], uint32_t* nof_prb);
