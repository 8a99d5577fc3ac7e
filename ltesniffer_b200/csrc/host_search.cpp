// host_search.cpp -- host (C++17) half of the drop-in path: replays FALCON's recursive blind DCI search
// over the candidate table produced by the Viterbi kernel, in subframe order, with a restatement of the
// reference's RNTI history, and converts accepted DL DCIs into PDSCH grants.
//   reference: src/src/DCISearch.cc:102-578 (inspect_dci_location_recursively, recursive_blind_dci_search,
//   search), lib/src/util/RNTIManager.cc + Histogram.cc, src/src/MetaFormats.cc:41-89,
//   lib/src/phy/falcon_phch/falcon_pdcch.c:183-250 (search-space validation), falcon_dci.c:148-352 and
//   dl_sniffer_pdsch.c:14-276 (DCI -> grant).  Integer control flow only: the GPU never sees this state.
#include "../../include/ltephy_b200.h"
#include "../../include/ltephy_sinks.h"
#include "../../include/ltephy_shard.h"
#include "../../include/lte_tables.h"
#include "lte_host.hpp"
#include "tb_merge.hpp"
#include "turn.hpp"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <vector>

namespace {

constexpr int      NF            = LTEPHY_NOF_FORMATS;
constexpr uint32_t HIST_DEPTH    = 200 * (304 / 5); // RNTI_HISTORY_DEPTH, RNTIManager.h:47-49
constexpr uint32_t PER_SF        = 304 / 5;         // RNTI_PER_SUBFRAME
constexpr uint32_t LIFETIME      = 10000;           // RRC_INACTIVITY_TIMER_MS
constexpr uint16_t RARNTI_START = 0x0001, RARNTI_END = 0x000A, CRNTI_START = 0x000B, CRNTI_END = 0xFFF3, MRNTI = 0xFFFD, PRNTI = 0xFFFE;
enum { ACT_UNSET = 0, ACT_EVERGREEN, ACT_RAR, ACT_SHORTCUT, ACT_HISTOGRAM, ACT_OTHER };

// ---------------------------------------------------------------------------------------------------
// RNTI history: same observable behaviour as RNTIManager (per-format 200 ms sliding histogram padded to
// 60 entries per subframe, active set with 10 s expiry, evergreen / forbidden intervals).
struct RntiManager {
  // Sliding histogram over the last HIST_DEPTH added entries (Histogram.cc).  Only non-zero RNTIs are stored,
  // with the add-position they were written at, so the zero padding of stepTime costs O(1) plus the entries it
  // expires; observable behaviour (getFrequency of any value, including 0) is unchanged.
  // Everything the walk needs to know about one RNTI sits in one 32-byte record (histogram counts of all formats,
  // active-set state), so that validating a candidate touches one cache line instead of a dozen arrays.
  struct alignas(32) Rec {
    uint16_t cnt[NF];
    uint8_t  active, reason, assoc, pad;
    uint32_t last_seen;
    uint16_t ever, forb; // bit f: this RNTI lies in an evergreen / forbidden interval of format f
  };
  struct Hist {
    struct Ent {
      uint64_t pos;
      uint16_t rnti;
    };
    std::vector<Ent> q = std::vector<Ent>(HIST_DEPTH); // circular FIFO of the non-zero entries in the window
    Rec*             rec = nullptr;                       // shared per-RNTI records; this histogram owns cnt[f]
    uint32_t         f   = 0;
    uint32_t         head = 0, size = 0;
    uint64_t              pos  = 0; // number of adds so far
    inline void           expire()
    {
      while (size && q[head].pos + HIST_DEPTH <= pos - 1) {
        rec[q[head].rnti].cnt[f]--;
        head = head + 1 == HIST_DEPTH ? 0 : head + 1;
        size--;
      }
    }
    inline void add(uint16_t v)
    {
      pos++;
      expire();
      if (v) {
        uint32_t tail = head + size;
        if (tail >= HIST_DEPTH) tail -= HIST_DEPTH;
        q[tail] = {pos - 1, v};
        size++;
        rec[v].cnt[f]++;
      }
    }
    inline void add_zeros(uint32_t n)
    {
      pos += n;
      expire();
    }
    inline uint32_t freq(uint16_t v) const { return v ? rec[v].cnt[f] : (uint32_t)(std::min<uint64_t>(pos, HIST_DEPTH) - size); }
  };
  struct Interval {
    uint16_t a, b;
  };
  Hist                  hist[NF];
  std::vector<Interval> evergreen[NF], forbidden[NF];
  std::vector<Rec>      rec = std::vector<Rec>(65536, Rec{});
  uint32_t              timestamp = 0, threshold = 5;
  int32_t               remaining[NF];
  RntiManager()
  {
    std::fill(remaining, remaining + NF, (int32_t)PER_SF);
    for (int i = 0; i < NF; i++) hist[i].rec = rec.data(), hist[i].f = (uint32_t)i;
  }
  RntiManager(const RntiManager&)            = delete;
  RntiManager& operator=(const RntiManager&) = delete;

  bool is_evergreen(uint16_t r, uint32_t f) const { return (rec[r].ever >> f) & 1u; }
  bool is_forbidden(uint16_t r, uint32_t f) const { return (rec[r].forb >> f) & 1u; }
  void add_evergreen(uint16_t a, uint16_t b, uint32_t f)
  {
    evergreen[f].push_back({a, b});
    for (uint32_t r = a; r <= b; r++) rec[r].ever |= (uint16_t)(1u << f);
  }
  void add_forbidden(uint16_t a, uint16_t b, uint32_t f)
  {
    forbidden[f].push_back({a, b});
    for (uint32_t r = a; r <= b; r++) rec[r].forb |= (uint16_t)(1u << f);
  }
  uint32_t freq(uint16_t r, uint32_t f) const { return hist[f].freq(r); }
  void     add_candidate(uint16_t r, uint32_t f)
  {
    hist[f].add(r);
    remaining[f]--;
  }
  uint32_t n_rar = 0;        // RNTIs currently active with reason RAR (they make the walk look at every format-0 candidate)
  bool     rar_seen = false; // sticky: some RNTI has been RAR-activated since creation (ltephy_search::may_need_full_table)
  void     activate(uint16_t r, uint8_t why)
  {
    if (!rec[r].active) rec[r].active = 1, rec[r].reason = why, n_rar += why == ACT_RAR, rar_seen |= why == ACT_RAR;
  }
  void deactivate(uint16_t r)
  {
    if (rec[r].active) n_rar -= rec[r].reason == ACT_RAR, rec[r].active = 0, rec[r].assoc = 0, rec[r].reason = ACT_UNSET;
  }
  bool expired(uint16_t r) const { return !(rec[r].active && timestamp - rec[r].last_seen < LIFETIME); }
  bool validate(uint16_t r, uint32_t f)
  {
    Rec& R = rec[r];
    if ((R.ever >> f) & 1u) return true;
    if ((R.forb >> f) & 1u) return false;
    if (R.active) {
      if (timestamp - R.last_seen < LIFETIME) return true;
      deactivate(r);
    }
    // validateByHistogram (RNTIManager.cc:335-365).  Most candidates that reach this point carry a chance RNTI that is in
    // no histogram at all: likely = 0 and ul + dl = 0 <= threshold, whatever f is.
    uint32_t likely = 0, maxf = 0;
    if (r) {
      uint64_t a, b;
      memcpy(&a, &R.cnt[0], 8), memcpy(&b, &R.cnt[4], 8);
      if (!(a | b | R.cnt[8])) return false;
      for (uint32_t i = 1; i < NF; i++)
        if (R.cnt[i] > maxf) maxf = R.cnt[i], likely = i;
    } else {
      for (uint32_t i = 1; i < NF; i++)
        if (hist[i].freq(r) > maxf) maxf = hist[i].freq(r), likely = i;
    }
    if (f != 0 && f != likely) return false;
    const uint32_t ul = hist[0].freq(r), dl = likely ? maxf : 0;
    if (ul + dl > threshold) {
      activate(r, ACT_HISTOGRAM);
      R.assoc = (uint8_t)(dl > threshold ? likely : 0);
      return true;
    }
    return false;
  }
  bool validate_and_refresh(uint16_t r, uint32_t f)
  {
    const bool ok = validate(r, f);
    if (ok) rec[r].last_seen = timestamp;
    return ok;
  }
  void activate_and_refresh(uint16_t r, uint32_t f, uint8_t why)
  {
    activate(r, why);
    rec[r].last_seen = timestamp;
    rec[r].assoc     = (uint8_t)f;
  }
  void step_time()
  {
    for (int i = 0; i < NF; i++) {
      if (remaining[i] > 0) hist[i].add_zeros((uint32_t)remaining[i]);
      remaining[i] = (int32_t)PER_SF;
    }
    timestamp++;
  }
};

// 36.213 9.1.1 search-space membership in O(1); equals srsran_pdcch_validate_location (falcon_pdcch.c:223-250)
inline bool in_ue_space(uint32_t nof_cce, uint32_t ncce, uint32_t l, uint32_t Yk)
{
  static const uint32_t M[4] = {6, 6, 2, 2};
  const uint32_t        L = 1u << l;
  if (nof_cce < L || (ncce & (L - 1))) return false;
  const uint32_t n = nof_cce / L, q = ncce / L;
  if (q >= n) return false;
  return (q + n - Yk % n) % n < M[l];
}
inline bool in_common_space(uint32_t nof_cce, uint32_t ncce, uint32_t l)
{
  if (l < 2) return false;
  const uint32_t L = 1u << l;
  if (nof_cce < L || (ncce & (L - 1))) return false;
  const uint32_t lim = std::min<uint32_t>(nof_cce, 16) / L, q = ncce / L;
  return q < lim && q < nof_cce / L;
}
uint32_t validate_location(uint32_t nof_cce, uint32_t ncce, uint32_t l, uint32_t sf_idx, uint16_t rnti)
{
  bool ue = false, common = false;
  if (rnti >= RARNTI_START && rnti <= RARNTI_END)
    common = true;
  else if (rnti >= CRNTI_START && rnti <= CRNTI_END)
    ue = common = true;
  else if (rnti >= MRNTI)
    common = true;
  else
    return 0;
  uint32_t Yk = rnti;
  if (ue)
    for (uint32_t m = 0; m < sf_idx + 1; m++) Yk = (39827u * Yk) % 65537u;
  const bool valid = (ue && in_ue_space(nof_cce, ncce, l, Yk)) || (common && in_common_space(nof_cce, ncce, l));
  if (!valid) return 0;
  const bool amb = l > 0 && ((ue && in_ue_space(nof_cce, ncce, l - 1, Yk)) || (common && in_common_space(nof_cce, ncce, l - 1)));
  return amb ? 1 : 2;
}

struct Cand { // no default initialisers: inspect() creates nine of them per visited location and clears only what it reads
  uint64_t bits;
  uint16_t rnti;
  uint8_t  format; // decoded format
  uint8_t  ssm;
  uint16_t nof_bits;
};
typedef unsigned __int128 u128;
struct Loc {
  uint8_t L;
  uint8_t ncce;
  bool    used, occupied, checked, sufficient_power;
};
struct Meta {
  uint8_t  format;
  uint32_t hits;
};
struct TempDci0 {
  uint16_t rnti;
  uint8_t  L, format;
  uint16_t ncce;
  Cand     cand;
};

} // namespace

struct ltephy_search {
  ltehost::Cell      cell;
  ltehost::SizeTable st;
  uint32_t           nof_cce[3]{};
  std::vector<uint16_t> re_slot; // [3 sf class][3 cfi][2 slots][nof_prb]: data REs of a PRB in a slot
  RntiManager        rm;
  Meta               all[NF];
  uint8_t            primary[NF], secondary[NF];
  uint32_t           n_primary = 0, n_secondary = 0;
  double             split_ratio     = 0.99;
  bool               skip_secondary  = false, shortcut = true;
  bool               ul_mode = false;           // ltephy_grants_from_dcis selects as PDSCH_Decoder::decode_ul_mode does instead of decode_dl_mode
  uint16_t           ul_target_rnti = 0;
  bool               keep_reserved_mcs = false; // HARQ mode: a C-RNTI grant whose first block has a reserved MCS is kept, ltephy_harq_prepare_grant sizes it
  bool               speculate_256qam = false; // grants_from_dcis emits both MCS-table readings of a C-RNTI DCI (DL_Sniffer_PDSCH.cc:1089-1210)
  uint32_t           update_interval = 500, sf_cnt = 0;
  uint32_t           ul_n_rb_ho = 0; // pusch-HoppingOffset of SIB2 (hopping_cfg.n_rb_ho, src/src/DCICollection.cc:168)
  ltephy_search_stats_t stats{};
  // per-subframe scratch
  const ltephy_cand_t*    T  = nullptr;
  const ltephy_cloc_t*    CL = nullptr; // survivor form (then T is null): per-location records ...
  const ltephy_cand_t*    CLIST = nullptr; // ... and the survivor list (ltephy_compact_t, or a packed record of ltephy_shard.h)
  uint32_t                sf_idx = 0, ncce_sf = 0, sf_batch = 0, pass_mask = 0;
  // Location state of the subframe being walked, as bit masks in CCE space: location (L, ncce) is bit ncce of the level-L
  // masks (only multiples of 2^L are meaningful there).
  //   low    - CCEs whose mean |LLR| is below 0.7 (a location covering one has insufficient power, DCISearch.cc:473-489)
  //   occ    - CCEs of the accepted locations (= the reference's `used` of the location itself, and `occupied` of every
  //            location overlapping it, DCISearch.cc:381-392)
  //   blk[L] - locations of level L that cover a CCE of low | occ (fold of the CCE mask, refreshed on acceptance)
  //   chk[L] - locations of level L already inspected in the current pass
  //   val[L] - locations of level L that exist in this subframe (srsran_pdcch_ue_locations_all_map, falcon_pdcch.c:321-356)
  u128     low = 0, occ = 0, blk[4]{}, chk[4]{}, val[4]{};
  uint32_t nq[4]{};
  inline void refold()
  {
    blk[0] = low | occ;
    blk[1] = blk[0] | (blk[0] >> 1);
    blk[2] = blk[1] | (blk[1] >> 2);
    blk[3] = blk[2] | (blk[2] >> 4);
  }
  struct LocTemplate {
    uint32_t n = 0;
    Loc      loc[LTEPHY_MAX_LOC];
    int16_t  loc_of[4][LTEPHY_MAX_CCE];
    u128     val[4]{};
    uint32_t nq[4]{};
  } tmpl[3];
  std::vector<TempDci0> temp_dci0;
  ltephy_dci_t*        out = nullptr;
  uint32_t             out_cap = 0, out_n = 0;
  Turn turn; // the walks of concurrent ltephy_decode_subframes calls, in seq order; its lock also keeps RNTI updates out of a walk

  void update_formats()
  {
    uint8_t sorted[NF];
    double  total = 0;
    for (int i = 0; i < NF; i++) sorted[i] = (uint8_t)i, total += all[i].hits;
    for (int i = 0; i < NF - 1; i++) {
      int mx = i;
      for (int j = mx; j < NF; j++)
        if (all[sorted[j]].hits > all[sorted[mx]].hits) mx = j;
      std::swap(sorted[i], sorted[mx]);
    }
    const double thr = total * split_ratio;
    double       cum = 0;
    n_primary = n_secondary = 0;
    for (int i = 0; i < NF; i++) {
      if (cum <= thr)
        primary[n_primary++] = sorted[i];
      else
        secondary[n_secondary++] = sorted[i];
      cum += all[sorted[i]].hits;
      all[sorted[i]].hits = 0;
    }
  }
  inline void fetch(uint32_t li, uint32_t format, Cand& c) const
  {
    const uint32_t       si = st.index_of[format];
    const ltephy_cand_t& t  = CL ? CLIST[CL[li].off + (uint32_t)__builtin_popcount(CL[li].mask & ((1u << si) - 1u))]
                                 : T[(size_t)li * LTEPHY_MAX_SIZES + si];
    c.bits = 0, c.rnti = 0, c.format = 0, c.ssm = 0;
    c.nof_bits             = (uint16_t)st.sizes[st.index_of[format]];
    if (!t.valid) return; // all-zero LLRs: the reference leaves the calloc'ed candidate untouched
    c.bits = t.bits, c.rnti = t.rnti;
    if (CL) c.ssm = t.pad[0] & 3u;
    if (format == ltehost::F0 || format == ltehost::F1A)
      c.format = (t.bits >> 63) ? ltehost::F1A : ltehost::F0;
    else
      c.format = (uint8_t)format;
  }
  void emit(const Cand& c, uint32_t L, uint32_t ncce, uint32_t histval)
  {
    if (out_n < out_cap) {
      ltephy_dci_t& o = out[out_n];
      o.sf = sf_batch, o.rnti = c.rnti, o.format = c.format, o.L = (uint8_t)L, o.ncce = (uint16_t)ncce, o.nof_bits = c.nof_bits, o.bits = c.bits;
      o.histogram_value = histval;
    }
    out_n++;
  }
  static inline u128 cce_range(uint32_t ncce, uint32_t L) { return ((((u128)1) << (1u << L)) - 1) << ncce; }
  inline bool        skip(uint32_t ncce, uint32_t L) const { return (uint64_t)((blk[L] | chk[L]) >> ncce) & 1u; }
  // location index in the candidate table: levels are laid out 3,2,1,0
  inline uint32_t loc_index(uint32_t ncce, uint32_t L) const
  {
    uint32_t b = 0;
    for (uint32_t l = 3; l > L; l--) b += nq[l];
    return b + (ncce >> L);
  }
  // A location whose whole subtree holds no survivor for the formats of this pass: the reference's recursion decodes
  // every reachable location, finds nothing, and marks them inspected.  Returns the number of locations it would visit.
  uint32_t sweep_empty(uint32_t ncce, uint32_t L, uint32_t max_depth)
  {
    chk[L] |= (u128)1 << ncce;
    uint32_t n = 1;
    if (L > 0 && max_depth > 0) {
      if (!skip(ncce, L - 1)) n += sweep_empty(ncce, L - 1, max_depth - 1);
      if (!skip(ncce + (1u << (L - 1)), L - 1)) n += sweep_empty(ncce + (1u << (L - 1)), L - 1, max_depth - 1);
    }
    return n;
  }
  int inspect(uint32_t ncce, uint32_t L, uint32_t max_depth, const uint8_t* mf, uint32_t nf, bool discovery, const Cand* parent)
  {
    if (!((uint64_t)(val[L] >> ncce) & 1u) || skip(ncce, L)) return 0;
    const uint32_t li = loc_index(ncce, L);
    if (CL && !(CL[li].pad & pass_mask)) { // pad = union of the survivor masks over the subtree
      stats.nof_decoded_locations += nf * sweep_empty(ncce, L, max_depth);
      return 0;
    }
    Cand     cand[NF];
    for (uint32_t f = 0; f < nf; f++) cand[f].rnti = 0, cand[f].ssm = 0;
    int      best = -1;
    uint32_t best_val = 0, n_above = 0;
    if (CL && !(CL[li].mask & pass_mask)) // no survivor in any column this pass looks at: every candidate ends as rnti = 0
      stats.nof_decoded_locations += nf;
    else
    for (uint32_t f = 0; f < nf; f++) {
      const uint32_t fmt = mf[f];
      stats.nof_decoded_locations++;
      if (CL && !((CL[li].mask >> st.index_of[fmt]) & 1u)) continue; // not a survivor: every path below ends in rnti = 0
      fetch((uint32_t)li, fmt, cand[f]);
      if (rm.rec[cand[f].rnti].reason == ACT_RAR && cand[f].format == 0) {
        bool add = true;
        for (auto& m : temp_dci0)
          if (m.format == cand[f].format && m.rnti == cand[f].rnti && m.ncce == ncce) add = false;
        if (add) temp_dci0.push_back({cand[f].rnti, (uint8_t)L, cand[f].format, (uint16_t)ncce, cand[f]});
      }
      if (fmt != cand[f].format) {
        cand[f].rnti = 0;
        continue;
      }
      const uint16_t r = cand[f].rnti;
      if (fmt == ltehost::F1C && r > RARNTI_END && r < PRNTI) {
        cand[f].rnti = 0;
        continue;
      }
      if (r > RARNTI_START && r < RARNTI_END && fmt != ltehost::F1A && fmt != ltehost::F1C) {
        cand[f].rnti = 0;
        continue;
      }
      if (shortcut && discovery && parent && parent[f].rnti == r && !rm.is_forbidden(r, fmt)) return -((int)f + 1);
      cand[f].ssm = CL ? cand[f].ssm : (uint8_t)validate_location(ncce_sf, ncce, L, sf_idx, r); // the survivor form carries it
      if (cand[f].ssm == 0) {
        cand[f].rnti = 0;
        continue;
      }
      if (rm.validate_and_refresh(r, fmt)) {
        n_above++;
        best     = (int)f;
        best_val = rm.freq(r, fmt);
      }
    }
    if (n_above > 1) {
      best = -1;
      uint32_t hmax = 0;
      for (uint32_t f = 0; f < nf; f++)
        if (cand[f].rnti != 0) {
          const uint32_t h = rm.freq(cand[f].rnti, mf[f]);
          if (h > hmax) hmax = h, best = (int)f, best_val = h;
        }
      if (best < 0) n_above = 0;
    }
    chk[L] |= (u128)1 << ncce;
    int disamb = 0;
    if (n_above > 0 && cand[best].ssm == 1) {
      if (L > 0 && max_depth > 0) disamb = inspect(ncce + (1u << (L - 1)), L - 1, max_depth - 1, mf, nf, false, nullptr);
    } else if (n_above == 0) {
      int rr = 0;
      if (L > 0 && max_depth > 0) {
        rr += inspect(ncce, L - 1, max_depth - 1, mf, nf, discovery, cand);
        if (rr < 0) {
          best     = -rr - 1;
          best_val = rm.freq(cand[best].rnti, mf[best]);
          n_above  = 1;
          if (cand[best].ssm == 1) disamb = inspect(ncce + (1u << (L - 1)), L - 1, std::min<uint32_t>(max_depth, 99) - 1, mf, nf, false, nullptr);
          rm.activate_and_refresh(cand[best].rnti, mf[best], ACT_SHORTCUT);
        } else
          rr += inspect(ncce + (1u << (L - 1)), L - 1, max_depth - 1, mf, nf, discovery, nullptr);
      }
      if (rr == 0) {
        if (discovery)
          for (uint32_t f = 0; f < nf; f++)
            if (cand[f].rnti != 0) rm.add_candidate(cand[f].rnti, mf[f]);
        return 0;
      }
      if (rr > 0) return rr;
    }
    if (n_above > 0) {
      occ |= cce_range(ncce, L);
      refold();
      rm.add_candidate(cand[best].rnti, mf[best]);
      all[mf[best]].hits++;
      const uint32_t L_dis = disamb > 0 ? L - 1 : L;
      const Cand&    b     = cand[best];
      if (b.rnti != 0) {
        bool add = true;
        if (b.format == 0)
          for (auto& m : temp_dci0)
            if (m.format == b.format && m.rnti == b.rnti && m.ncce == ncce) add = false;
        if (add) emit(b, L_dis, ncce, best_val);
        for (auto& m : temp_dci0) emit(m.cand, m.L, m.ncce, rm.freq(m.rnti, m.format));
        temp_dci0.clear();
      }
      return 1 + disamb;
    }
    return 0;
  }
  // What the walk needs to know about one subframe: either the full table, or the survivor form (loc + list).
  struct WalkIn {
    uint32_t             tti, cfi;
    float                snr_db;
    uint64_t             low[2]; // bit c: CCE c has mean |LLR| < 0.7 (DCISearch.cc:473-489), c < min(nof_cce, 84)
    uint32_t             count;  // survivors (survivor form only)
    const ltephy_cand_t* table;
    const ltephy_cloc_t* loc;
    const ltephy_cand_t* list;
  };
  WalkIn walk_in(const ltephy_sf_info_t& info, const ltephy_cand_t* table, const ltephy_compact_t* comp) const
  {
    WalkIn w{info.tti, info.cfi, info.snr_db, {0, 0}, comp ? comp->count : 0, table, comp ? comp->loc : nullptr, comp ? comp->list : nullptr};
    if (info.cfi >= 1 && info.cfi <= 3) {
      const uint32_t lim = std::min<uint32_t>(nof_cce[info.cfi - 1], LTEPHY_SEARCH_MAX_CCE);
      for (uint32_t c = 0; c < lim; c++) w.low[c >> 6] |= (uint64_t)(info.cce_power[c] < 0.7f) << (c & 63u);
    }
    return w;
  }
  // exactly one of table / comp is given.  The survivor form cannot serve a walk that has RAR-activated RNTIs (the
  // temp_dci0 rule looks at every format-0 candidate) nor a truncated list: LTEPHY_NEED_FULL_TABLE, nothing consumed.
  int search_subframe(const ltephy_sf_info_t& info, const ltephy_cand_t* table, const ltephy_compact_t* comp, uint32_t sf_in_batch, ltephy_dci_t* o,
                      uint32_t cap, uint32_t* n)
  {
    return search_subframe(walk_in(info, table, comp), sf_in_batch, o, cap, n);
  }
  int search_subframe(const WalkIn& info, uint32_t sf_in_batch, ltephy_dci_t* o, uint32_t cap, uint32_t* n)
  {
    if (info.loc && (rm.n_rar || info.count > LTEPHY_COMPACT_CAP)) return LTEPHY_NEED_FULL_TABLE;
    if (update_interval && (sf_cnt % update_interval) == 0) update_formats();
    sf_cnt++;
    out = o, out_cap = cap, out_n = 0, sf_batch = sf_in_batch, T = info.table, CL = info.loc, CLIST = info.list;
    int ret = LTEPHY_ERROR;
    if (info.snr_db > 6.0f && info.cfi >= 1 && info.cfi <= 3) {
      temp_dci0.clear();
      sf_idx  = info.tti % 10;
      ncce_sf = nof_cce[info.cfi - 1];
      stats.nof_cce += ncce_sf;
      const uint32_t lim = std::min<uint32_t>(ncce_sf, LTEPHY_SEARCH_MAX_CCE);
      const uint32_t k   = tmpl[info.cfi - 1].n;
      stats.nof_locations += k;
      low = ((u128)info.low[1] << 64) | info.low[0], occ = 0;
      refold();
      for (uint32_t l = 0; l < 4; l++) nq[l] = tmpl[info.cfi - 1].nq[l], val[l] = tmpl[info.cfi - 1].val[l];
      ret = 0;
      for (int pass = 0; pass < (skip_secondary ? 1 : 2); pass++) {
        const uint8_t* mf = pass ? secondary : primary;
        const uint32_t nf = pass ? n_secondary : n_primary;
        pass_mask = 0;
        for (uint32_t f = 0; f < nf; f++) pass_mask |= 1u << st.index_of[mf[f]];
        chk[0] = chk[1] = chk[2] = chk[3] = 0;
        for (int l = 3; l >= 0; l--) // table order: level 3 first, ascending CCE; inspecting only ever removes locations from `todo`
          for (;;) {
            const u128     todo = val[l] & ~(blk[l] | chk[l]);
            const uint64_t lo = (uint64_t)todo, hi = (uint64_t)(todo >> 64);
            if (!(lo | hi)) break;
            const uint32_t ncce = lo ? (uint32_t)__builtin_ctzll(lo) : 64u + (uint32_t)__builtin_ctzll(hi);
            ret += inspect(ncce, (uint32_t)l, 99, mf, nf, true, nullptr);
          }
      }
      const u128     all = lim >= 128 ? ~(u128)0 : (((u128)1 << lim) - 1), rest = all & ~low & ~occ;
      const uint32_t missed = (uint32_t)(__builtin_popcountll((uint64_t)rest) + __builtin_popcountll((uint64_t)(rest >> 64)));
      stats.nof_missed_cce += missed;
      rm.step_time();
    }
    stats.nof_subframes++;
    if (n) *n = out_n;
    return out_n > cap ? LTEPHY_ERROR_INVALID_INPUTS : (ret < 0 ? 0 : ret);
  }
  // One subframe of a batch: what the walk reads, and the subframe's full table when the caller gave full tables (else nullptr)
  struct WalkSf {
    WalkIn               in;
    const ltephy_cand_t* full;
  };
  // The walk over a batch: at(i) -> WalkSf of subframe i, for i = 0 .. n - 1 in order; dci.sf = i.  A subframe whose survivor form
  // cannot serve is walked over its full table instead.
  template <class At>
  int search_batch(uint32_t n, At at, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis)
  {
    uint32_t nd = 0;
    for (uint32_t i = 0; i < n; i++) {
      WalkSf   sf = at(i);
      uint32_t k  = 0;
      int      r  = search_subframe(sf.in, i, dcis + nd, max_dcis - nd, &k);
      if (r == LTEPHY_NEED_FULL_TABLE && sf.full) {
        sf.in.table = sf.full, sf.in.loc = nullptr, sf.in.list = nullptr;
        r = search_subframe(sf.in, i, dcis + nd, max_dcis - nd, &k);
      }
      if (r < 0) return r;
      nd += std::min(k, max_dcis - nd);
    }
    *n_dcis = nd;
    return LTEPHY_SUCCESS;
  }
  // Whether a walk over n survivor forms may need the full tables: some subframe overflows its survivor list (count(i) survivors), or
  // RAR-activated RNTIs make the walk look at every format-0 candidate.  The RAR test depends on the use:
  //   FOR_WALK        a walk given no full tables refuses such a batch before it consumes anything.  It asks for RNTIs active with reason
  //                   RAR now (n_rar), which is exact: RAR activations only arrive between batches.
  //   FOR_COLLECTIVE  the ranks of a sharded run decide on a collective fetch of the full tables before they walk.  They ask whether any
  //                   RNTI was ever RAR-activated (rar_seen), a superset of n_rar > 0 that does not depend on how far the walk has progressed,
  //                   so that every rank decides alike.
  enum FullTableUse { FOR_WALK, FOR_COLLECTIVE };
  template <class Count>
  bool may_need_full_table(FullTableUse use, uint32_t n, Count count) const
  {
    if (use == FOR_WALK ? rm.n_rar != 0 : rm.rar_seen) return true;
    for (uint32_t i = 0; i < n; i++)
      if (count(i) > LTEPHY_COMPACT_CAP) return true;
    return false;
  }
};

// ===================================================================================================
// DCI -> grant (a10).  srsran_dci_msg_unpack_pdsch + dl_sniffer_ra_dl_dci_to_grant + dl_sniffer_config_mimo.
namespace {
struct Bits {
  uint64_t v;
  uint32_t pos = 0;
  uint32_t get(uint32_t n)
  {
    uint32_t r = n ? (uint32_t)((v << pos) >> (64 - n)) : 0;
    pos += n;
    return r;
  }
};
uint32_t clog2(uint32_t v)
{
  uint32_t n = 0;
  while ((1u << n) < v) n++;
  return n;
}
uint32_t rbg_size(uint32_t n) { return n <= 10 ? 1 : n <= 26 ? 2 : n <= 63 ? 3 : 4; }
uint32_t gap1(uint32_t n) { return n <= 10 ? (n + 1) / 2 : n == 11 ? 4 : n <= 19 ? 8 : n <= 26 ? 12 : n <= 44 ? 18 : n <= 63 ? 27 : n <= 79 ? 32 : 48; }
uint32_t gap2(uint32_t n) { return n < 50 ? 0 : n <= 63 ? 9 : 16; }
uint32_t nvrb(uint32_t n, bool g2)
{
  if (!g2) {
    uint32_t g = gap1(n);
    return 2 * std::min(g, n - g);
  }
  uint32_t g = gap2(n);
  return g ? (n / (2 * g)) * 2 * g : 0;
}
void riv_decode(uint32_t riv, uint32_t N, uint32_t& L, uint32_t& S)
{
  L = riv / N + 1, S = riv % N;
  if (L + S > N) L = N - L + 2, S = N - 1 - S;
}
void dvrb(uint32_t N, bool g2, uint32_t v, uint32_t& p0, uint32_t& p1)
{
  const uint32_t P = rbg_size(N), Ng = g2 ? gap2(N) : gap1(N), Nt = g2 ? 2 * Ng : nvrb(N, false);
  const uint32_t Nrow = ((Nt + 4 * P - 1) / (4 * P)) * P, Nnull = 4 * Nrow - Nt, nt = v % Nt, blk = v / Nt;
  const int      a = (int)(2 * Nrow * (nt % 2) + nt / 2 + Nt * blk), b = (int)(Nrow * (nt % 4) + nt / 4 + Nt * blk);
  int            e;
  if (Nnull && nt >= Nt - Nnull && (nt & 1))
    e = a - (int)Nrow;
  else if (Nnull && nt >= Nt - Nnull)
    e = a - (int)Nrow + (int)Nnull / 2;
  else if (Nnull && (nt % 4) >= 2)
    e = b - (int)Nnull / 2;
  else
    e = b;
  const uint32_t ee = (uint32_t)e, oo = (ee + Nt / 2) % Nt + Nt * blk;
  p0 = (ee % Nt) < Nt / 2 ? ee : ee + Ng - Nt / 2;
  p1 = (oo % Nt) < Nt / 2 ? oo : oo + Ng - Nt / 2;
}
inline void set_prb(ltephy_grant_t& g, int slot, uint32_t prb) { g.prb_mask[slot][prb >> 5] |= 1u << (prb & 31); }
inline bool user_rnti(uint16_t r) { return r >= CRNTI_START && r <= CRNTI_END; }
} // namespace

extern "C" {

} // extern "C"

// ---- stage 1: srsran_dci_msg_unpack_pdsch -- payload bits -> fields (36.212 5.3.3.1.2-5.3.3.1.5A), formats 1, 1A, 1C, 2, 2A
int ltehost_unpack_dl_dci(const ltehost::Cell& c, uint32_t format, uint16_t rnti, uint64_t bits, ltehost::DlDciFields& f)
{
  const uint32_t N = c.nof_prb, P = rbg_size(N), nrbg = (N + P - 1) / P, hdr = N > 10, rivb = clog2(N * (N + 1) / 2);
  f        = ltehost::DlDciFields{};
  f.format = (uint8_t)format, f.rnti = rnti, f.n_prb1a = 2;
  Bits b{bits};
  switch (format) {
    case ltehost::F1A:
      if (b.get(1) != 1) return LTEPHY_ERROR;
      f.alloc = 2;
      f.dist  = b.get(1);
      if (f.dist && N >= 50) {
        f.ngap2 = b.get(1);
        f.riv   = b.get(rivb - 1);
      } else
        f.riv = b.get(rivb);
      f.mcs[0] = (uint8_t)b.get(5), f.harq_pid = (uint8_t)b.get(3), f.ndi[0] = (uint8_t)b.get(1), f.rv[0] = (uint8_t)b.get(2);
      {
        const uint32_t t = b.get(2);
        if (user_rnti(rnti))
          f.tpc = (uint8_t)t;
        else
          f.n_prb1a = (t & 1) ? 3 : 2;
      }
      f.tb_en[0] = true;
      break;
    case ltehost::F1C:
      f.alloc = 2, f.dist = true;
      if (N >= 50) f.ngap2 = b.get(1);
      {
        const uint32_t nv = nvrb(N, false) / (N < 50 ? 2 : 4);
        f.riv             = b.get(clog2(nv * (nv + 1) / 2));
      }
      f.mcs[0]   = (uint8_t)b.get(5);
      f.tb_en[0] = true;
      break;
    case ltehost::F1:
    case ltehost::F2:
    case ltehost::F2A:
      f.alloc = hdr ? b.get(1) : 0;
      if (f.alloc == 0)
        f.rbg_mask = b.get(nrbg);
      else {
        const uint32_t sb = clog2(P);
        f.t1_subset = b.get(sb), f.t1_shift = b.get(1), f.t1_mask = b.get(nrbg - sb - 1);
      }
      if (format == ltehost::F1) {
        f.mcs[0] = (uint8_t)b.get(5), f.harq_pid = (uint8_t)b.get(3), f.ndi[0] = (uint8_t)b.get(1), f.rv[0] = (uint8_t)b.get(2), f.tpc = (uint8_t)b.get(2);
        f.tb_en[0] = true;
      } else {
        f.tpc = (uint8_t)b.get(2), f.harq_pid = (uint8_t)b.get(3), f.tb_cw_swap = (uint8_t)b.get(1);
        for (int i = 0; i < 2; i++) {
          f.mcs[i] = (uint8_t)b.get(5), f.ndi[i] = (uint8_t)b.get(1), f.rv[i] = (uint8_t)b.get(2);
          f.tb_en[i] = !(f.mcs[i] == 0 && f.rv[i] == 1);
        }
        if (format == ltehost::F2) f.pinfo = (uint8_t)b.get(c.nof_ports == 2 ? 3 : c.nof_ports == 4 ? 6 : 0);
        if (format == ltehost::F2A && c.nof_ports == 4) f.pinfo = (uint8_t)b.get(2);
      }
      break;
    default: return LTEPHY_ERROR; // format 0 is an uplink grant; 1B/1D/2B are rejected by dl_sniffer_config_mimo_type
  }
  return LTEPHY_SUCCESS;
}
// ---- stage 2: srsran_ra_dl_grant_to_grant_prb_allocation -- allocation fields -> PRBs of both slots (36.213 7.1.6)
int ltehost_dl_prb_allocation(uint32_t N, const ltehost::DlDciFields& f, uint32_t mask[2][4], uint32_t* nof_prb_out)
{
  const uint32_t P = rbg_size(N), nrbg = (N + P - 1) / P;
  auto           set = [&](uint32_t sl, uint32_t prb) { mask[sl][prb >> 5] |= 1u << (prb & 31u); };
  memset(mask, 0, sizeof(uint32_t) * 8);
  uint32_t nof_prb = 0;
  if (f.alloc == 0) {
    for (uint32_t i = 0; i < nrbg; i++)
      if (f.rbg_mask & (1u << (nrbg - 1 - i)))
        for (uint32_t j = i * P; j < (i + 1) * P && j < N; j++) set(0, j), set(1, j), nof_prb++;
  } else if (f.alloc == 1) {
    const uint32_t sb = clog2(P), nb = nrbg - sb - 1, q = (N - 1) / (P * P), pm = ((N - 1) / P) % P;
    const uint32_t nsub  = f.t1_subset < pm ? q * P + P : f.t1_subset == pm ? q * P + (N - 1) % P + 1 : q * P;
    const uint32_t shift = f.t1_shift ? nsub - nb : 0;
    for (uint32_t i = 0; i < nb; i++)
      if (f.t1_mask & (1u << (nb - 1 - i))) {
        const uint32_t v = ((i + shift) / P) * P * P + f.t1_subset * P + (i + shift) % P;
        if (v >= N) return LTEPHY_ERROR;
        set(0, v), set(1, v), nof_prb++;
      }
  } else {
    uint32_t L, S;
    if (f.format == ltehost::F1C) {
      const uint32_t step = N < 50 ? 2 : 4;
      riv_decode(f.riv, nvrb(N, f.ngap2) / step, L, S);
      L *= step, S *= step;
    } else if (f.dist)
      riv_decode(f.riv, nvrb(N, f.ngap2), L, S);
    else
      riv_decode(f.riv, N, L, S);
    {
      const uint32_t lim = f.dist ? nvrb(N, f.ngap2) : N; // an out-of-range RIV decodes to nonsense: reject it
      if (L < 1 || L > lim || S >= lim || S + L > lim) return LTEPHY_ERROR;
    }
    if (!f.dist) {
      for (uint32_t j = S; j < S + L; j++) set(0, j), set(1, j);
    } else {
      for (uint32_t v = S; v < S + L; v++) {
        uint32_t p0, p1;
        dvrb(N, f.ngap2, v, p0, p1);
        if (p0 >= N || p1 >= N) return LTEPHY_ERROR;
        set(0, p0), set(1, p1);
      }
    }
    nof_prb = L;
  }
  if (!nof_prb) return LTEPHY_ERROR;
  *nof_prb_out = nof_prb;
  return LTEPHY_SUCCESS;
}

extern "C" {
int ltephy_dci_to_grant(const ltephy_search_t* s, const ltephy_dci_t* d, uint32_t sf_idx, uint32_t cfi, int use_256qam_table, ltephy_grant_t* g,
                        ltephy_dci_fields_t* fields)
{
  if (!s || !d || !g || cfi < 1 || cfi > 3 || sf_idx > 9) return LTEPHY_ERROR_INVALID_INPUTS;
  const ltehost::Cell& c = s->cell;
  const uint32_t       N = c.nof_prb;
  memset(g, 0, sizeof(*g));
  ltehost::DlDciFields u;
  if (ltehost_unpack_dl_dci(c, d->format, d->rnti, d->bits, u)) return LTEPHY_ERROR;
  ltephy_dci_fields_t f{};
  f.format = d->format, f.rnti = d->rnti, f.alloc_type = (uint8_t)u.alloc, f.harq_pid = u.harq_pid, f.tpc = u.tpc, f.tb_cw_swap = u.tb_cw_swap,
  f.pinfo = u.pinfo;
  for (int i = 0; i < 2; i++) f.mcs[i] = u.mcs[i], f.rv[i] = u.rv[i], f.ndi[i] = u.ndi[i];
  const bool     tb_en[2] = {u.tb_en[0], u.tb_en[1]};
  const uint32_t n_prb1a  = u.n_prb1a;
  uint32_t       nof_prb  = 0;
  if (ltehost_dl_prb_allocation(N, u, g->prb_mask, &nof_prb)) return LTEPHY_ERROR;
  if (!nof_prb) return LTEPHY_ERROR;
  f.nof_prb = nof_prb;
  // ---- transport blocks (dl_sniffer_compute_tb, dl_sniffer_pdsch.c:14-92) ----
  bool alt = use_256qam_table != 0;
  if (d->format == ltehost::F1A || !user_rnti(d->rnti)) alt = false;
  for (int i = 0; i < 2; i++) {
    g->tb[i].rv = f.rv[i];
    if ((tb_en[i] && d->format >= ltehost::F2) || (d->format < ltehost::F2 && i == 0)) g->tb[i].enabled = 1, g->tb[i].cw_idx = g->nof_tb, g->nof_tb++;
  }
  // transport block to codeword swap flag (36.212 Table 5.3.3.1.5-1): with both TBs enabled, TB1 -> codeword 1 and TB2 -> codeword 0;
  // with one TB disabled the other one always maps to codeword 0 (Table 5.3.3.1.5-2).  srsRAN carries this as tb[i].cw_idx
  // (dl_sniffer_pdsch.c:24) into scrambling (q << 13) and layer mapping.
  if (g->nof_tb == 2 && f.tb_cw_swap) g->tb[0].cw_idx = 1, g->tb[1].cw_idx = 0;
  if (!user_rnti(d->rnti)) {
    int tbs;
    if (d->format == ltehost::F1A)
      tbs = f.mcs[0] < LTE_TBS_NOF_ITBS ? lte_tbs_table[f.mcs[0]][n_prb1a - 1] : -1;
    else if (d->format == ltehost::F1C)
      tbs = lte_tbs_format1c[f.mcs[0] & 31];
    else
      return LTEPHY_ERROR;
    if (tbs < 0) return LTEPHY_ERROR;
    g->tb[0].qm = 2, g->tb[0].tbs = tbs;
  } else {
    for (int i = 0; i < 2; i++) {
      if (!g->tb[i].enabled) continue;
      const int itbs = alt ? lte_dl_mcs_itbs_alt[f.mcs[i]] : lte_dl_mcs_itbs[f.mcs[i]];
      g->tb[i].qm    = (uint8_t)(alt ? lte_dl_mcs_qm_alt[f.mcs[i]] : lte_dl_mcs_qm[f.mcs[i]]);
      g->tb[i].tbs   = itbs >= 0 ? lte_tbs_table[itbs][nof_prb - 1] : 0;
    }
  }
  // ---- nof_re (srsran_ra_dl_compute_nof_re) ----
  {
    const uint32_t  cls = sf_idx == 0 ? 0 : sf_idx == 5 ? 1 : 2;
    const uint16_t* cnt = &s->re_slot[((size_t)cls * 3 + cfi - 1) * 2 * N];
    for (uint32_t sl = 0; sl < 2; sl++)
      for (uint32_t w = 0; w < 4; w++) {
        uint32_t m = g->prb_mask[sl][w];
        while (m) {
          const uint32_t b = (uint32_t)__builtin_ctz(m);
          m &= m - 1;
          g->nof_re += cnt[sl * N + 32 * w + b];
        }
      }
  }
  if (d->format == ltehost::F1C && (d->rnti <= RARNTI_END || d->rnti == PRNTI))
    for (int i = 0; i < 2; i++) g->tb[i].rv = 0;
  // ---- MIMO (dl_sniffer_config_mimo, dl_sniffer_pdsch.c:134-276) ----
  switch (d->format) {
    case ltehost::F2: g->tx_scheme = (g->nof_tb == 1 && f.pinfo == 0) ? LTEPHY_TX_DIVERSITY : LTEPHY_TX_SPATIALMUX; break;
    case ltehost::F2A: g->tx_scheme = (g->nof_tb == 1 && f.pinfo == 0) ? LTEPHY_TX_DIVERSITY : LTEPHY_TX_CDD; break;
    default: g->tx_scheme = c.nof_ports == 1 ? LTEPHY_TX_PORT0 : LTEPHY_TX_DIVERSITY; break;
  }
  if (g->tx_scheme == LTEPHY_TX_SPATIALMUX) { // dl_sniffer_config_mimo_pmi, dl_sniffer_pdsch.c:181-209
    if (g->nof_tb == 1) {
      if (!(f.pinfo > 0 && f.pinfo < 5)) return LTEPHY_MIMO_PMI_WRONG;
      g->pmi = f.pinfo - 1u;
    } else {
      if (f.pinfo >= 2) return LTEPHY_MIMO_PMI_WRONG;
      g->pmi = f.pinfo % 2u;
    }
  }
  if ((g->tx_scheme == LTEPHY_TX_PORT0 || g->tx_scheme == LTEPHY_TX_DIVERSITY) && g->nof_tb != 1) return LTEPHY_MIMO_LAYER_WRONG;
  if (g->tx_scheme == LTEPHY_TX_CDD && g->nof_tb != 2) return LTEPHY_MIMO_LAYER_WRONG;
  if (g->tx_scheme == LTEPHY_TX_SPATIALMUX && g->nof_tb != 1 && g->nof_tb != 2) return LTEPHY_MIMO_LAYER_WRONG; // both TBs disabled, dl_sniffer_pdsch.c:229-237
  g->rnti = d->rnti, g->sf = d->sf;
  if (fields) *fields = f;
  return LTEPHY_SUCCESS;
}

// fields of a format-0 DCI or of a RAR grant -> PUSCH grant.  hop_kind: 0xFF none, 0 +1/4, 1 -1/4, 2 +1/2 (type 1), 3 type 2
static int ul_fields_to_grant(const ltephy_search_t* s, uint32_t sf, uint16_t rnti, uint32_t hop_kind, uint32_t riv, uint32_t mcs, uint32_t cs, int enable_64qam,
                              ltephy_ul_grant_t* g)
{
  static const uint8_t dmrs2_map[8] = {0, 6, 3, 4, 2, 8, 10, 9}; // 36.211 Table 5.5.2.1.1-1
  const uint32_t       N = s->cell.nof_prb;
  uint32_t             L, S;
  riv_decode(riv, N, L, S);
  if (L < 3 || L > N || S >= N || S + L > N) return LTEPHY_ERROR;
  uint32_t t = L;
  while (t % 2 == 0) t /= 2;
  while (t % 3 == 0) t /= 3;
  while (t % 5 == 0) t /= 5;
  if (t != 1) return LTEPHY_ERROR;                   // valid_prb_ul, src/src/UL_Sniffer_PUSCH.cc:3-10
  uint32_t S1 = S;
  if (hop_kind < 3) { // type 1: ul_sniffer_ra_ul_grant_to_grant_prb_allocation, lib/src/phy/falcon_phch/ul_sniffer_pusch.c:48-80
    uint32_t ho = s->ul_n_rb_ho;
    if (ho % 2) ho++;
    const uint32_t nrb = N - ho - (N % 2);
    if (S < ho / 2) return LTEPHY_ERROR;
    S1 = hop_kind == 0 ? (nrb / 4 + S) % nrb : hop_kind == 1 ? (S < nrb / 4 ? nrb + S - nrb / 4 : S - nrb / 4) : (nrb / 2 + S) % nrb;
    if (S1 + L > N) return LTEPHY_ERROR;
  } // type 2 (hop_kind 3): the reference keeps n_prb_tilde = n_prb for both slots (ul_sniffer_pusch.c:32-44,224-226)
  memset(g, 0, sizeof(*g));
  int itbs;
  if (mcs > 28) return LTEPHY_ERROR;
  if (enable_64qam == 2) { // 36.213 Table 8.6.1-3 as restated by ul_fill_ra_mcs_256 (lib/src/phy/falcon_phch/ul_sniffer_pusch.c:91-135)
    if (mcs < 6)
      g->qm = 2, itbs = 2 * (int)mcs;
    else if (mcs < 14)
      g->qm = 4, itbs = (int)mcs + (mcs < 10 ? 5 : 6);
    else if (mcs < 23)
      g->qm = 6, itbs = (int)mcs + (mcs < 19 ? 6 : 7);
    else
      g->qm = 8, itbs = (int)mcs + (mcs < 26 ? 7 : 6);
    if (mcs == 26)
      g->tbs = lte_tbs_32a(L); // row 32A
    else if (itbs > 33)
      return LTEPHY_ERROR;     // MCS 28 -> I_TBS 34: srsran_ra_tbs_from_idx has no such row
    else
      g->tbs = lte_tbs_table[itbs][L - 1];
  } else {
    if (mcs <= 10)
      g->qm = 2, itbs = (int)mcs;
    else if (mcs <= 20)
      g->qm = 4, itbs = (int)mcs - 1;
    else
      g->qm = enable_64qam ? 6 : 4, itbs = (int)mcs - 2;
    g->tbs = lte_tbs_table[itbs][L - 1];
  }
  if (g->tbs <= 0) return LTEPHY_ERROR;
  g->sf = sf, g->rnti = rnti, g->rv = 0, g->L_prb = L, g->n_prb = S, g->n_dmrs2 = dmrs2_map[cs & 7];
  g->n_prb_slot1 = S1, g->flags = LTEPHY_UL_FLAG_SLOT1;
  return LTEPHY_SUCCESS;
}
int ltephy_ul_dci_to_grant(const ltephy_search_t* s, const ltephy_dci_t* d, int enable_64qam, ltephy_ul_grant_t* g)
{
  if (!s || !d || !g || d->format != ltehost::F0) return LTEPHY_ERROR_INVALID_INPUTS;
  const uint32_t N = s->cell.nof_prb, rivb = clog2(N * (N + 1) / 2);
  Bits           b{d->bits};
  if (b.get(1) != 0) return LTEPHY_ERROR;            // format 0/1A flag
  const uint32_t hop = b.get(1);                     // frequency hopping flag
  uint32_t       riv = b.get(rivb), hop_kind = 0xFF;
  const uint32_t mcs = b.get(5);
  b.get(1);                                          // ndi
  b.get(2);                                          // tpc
  const uint32_t cs = b.get(3);
  if (hop) { // the N_UL_hop most significant bits of the allocation select the hop (36.213 Tables 8.4-1 / 8.4-2): 0 +1/4, 1 -1/4, 2 +1/2, 3 type 2
    const uint32_t nh = N < 50 ? 1 : 2, hb = riv >> (rivb - nh);
    riv &= (1u << (rivb - nh)) - 1;
    hop_kind = nh == 1 ? (hb == 0 ? 2 : 3) : hb;
  }
  return ul_fields_to_grant(s, d->sf, d->rnti, hop_kind, riv, mcs, cs, enable_64qam, g);
}

// MAC Random Access Response PDU (36.321 6.1.5 / 6.2.2 / 6.2.3; srsran::rar_pdu in the reference) -> one entry per MAC RAR with its msg-3 PUSCH grant, as
// PDSCH_Decoder::unpack_rar_response_ul_mode builds it (reference src/src/DL_Sniffer_PDSCH.cc:632-665): the 20-bit grant is split by ul_sniffer_dci_rar_unpack,
// turned into an uplink DCI by ul_sniffer_dci_rar_to_ul_dci (lib/src/phy/falcon_phch/falcon_dci.c:648-684: RIV = the 10 allocation bits as they are, MCS = the
// truncated MCS, a set hopping flag read as hop value 1) and into a grant by ul_sniffer_ra_ul_dci_to_grant (Table 8.6.1-1).
int ltephy_rar_unpack(const ltephy_search_t* s, const uint8_t* pdu, uint32_t len, ltephy_rar_t* out, uint32_t max_out, uint32_t* n_out, int* backoff)
{
  if (!s || !pdu || !out || !n_out) return LTEPHY_ERROR_INVALID_INPUTS;
  *n_out = 0;
  if (backoff) *backoff = -1;
  uint8_t  rapid[64];
  uint32_t nr = 0, pos = 0;
  for (bool more = true; more;) { // subheaders: E | T | RAPID(6), or E | T=0 | R R | BI(4)
    if (pos >= len) return LTEPHY_ERROR;
    const uint8_t h = pdu[pos++];
    more            = (h & 0x80) != 0;
    if (h & 0x40) {
      if (nr >= 64) return LTEPHY_ERROR;
      rapid[nr++] = h & 0x3F;
    } else if (backoff)
      *backoff = h & 0x0F;
  }
  if (pos + 6 * (size_t)nr > len) return LTEPHY_ERROR;
  for (uint32_t k = 0; k < nr; k++, pos += 6) {
    if (*n_out >= max_out) return LTEPHY_ERROR_INVALID_INPUTS;
    const uint8_t* r = pdu + pos; // R(1) TA(11) UL grant(20) T-CRNTI(16)
    ltephy_rar_t&  o = out[(*n_out)++];
    memset(&o, 0, sizeof(o));
    o.rapid = rapid[k], o.ta = (uint16_t)(((r[0] & 0x7Fu) << 4) | (r[1] >> 4)), o.t_crnti = (uint16_t)((r[4] << 8) | r[5]);
    const uint32_t gr = ((r[1] & 0x0Fu) << 16) | ((uint32_t)r[2] << 8) | r[3];
    o.hopping_flag = (gr >> 19) & 1, o.tpc = (gr >> 2) & 7, o.ul_delay = (gr >> 1) & 1, o.cqi_request = gr & 1;
    const uint32_t rba = (gr >> 9) & 0x3FF, mcs = (gr >> 5) & 0xF;
    o.valid = ul_fields_to_grant(s, 0, o.t_crnti, o.hopping_flag ? 1u : 0xFFu, rba, mcs, 0, 1, &o.grant) == LTEPHY_SUCCESS;
  }
  return LTEPHY_SUCCESS;
}

// The readings of one accepted format-0 DCI that PUSCH_Decoder::decode tries, in its order (reference src/src/UL_Sniffer_PUSCH.cc:417-570), given what
// MCSTracking knows of the UE (mcs_mod = ul_sniffer_mod_tracking_t).  The reference runs them one after the other and stops at the first CRC pass; a
// batch caller submits them all in one ltephy_submit_ul and keeps the first in this order whose CRC passed -- same outcome, one launch.
int ltephy_ul_decode_plan(const ltephy_search_t* s, const ltephy_dci_t* d, int mcs_mod, ltephy_ul_grant_t* grants, uint8_t* reading)
{
  if (!s || !d || !grants || !reading || mcs_mod < LTEPHY_UL_MOD_16QAM_MAX || mcs_mod > LTEPHY_UL_MOD_UNKNOWN) return LTEPHY_ERROR_INVALID_INPUTS;
  // investigate_valid_ul_grant (:894-918): RNTI 0, no transport block size in either table (retransmission MCS, failed allocation) or an L_prb that is no DFT
  // size -> not decoded.  All of it is what makes the Table 8.6.1-1 conversion fail here.
  ltephy_ul_grant_t g1;
  if (d->rnti == 0 || ltephy_ul_dci_to_grant(s, d, 1, &g1) != LTEPHY_SUCCESS) return 0;
  const uint32_t N = s->cell.nof_prb, rivb = clog2(N * (N + 1) / 2);
  Bits           b{d->bits};
  b.get(2), b.get(rivb);
  const uint32_t mcs = b.get(5);
  int            order[3], n = 0;
  if (mcs > 20) { // :456-529
    if (mcs_mod == LTEPHY_UL_MOD_UNKNOWN)
      order[n++] = 0, order[n++] = 1, order[n++] = 2;
    else
      order[n++] = mcs_mod;
  } else { // :531-569: up to MCS 20 the 16QAM and 64QAM readings are the same grant
    if (mcs_mod == LTEPHY_UL_MOD_16QAM_MAX || mcs_mod == LTEPHY_UL_MOD_64QAM_MAX)
      order[n++] = 0;
    else if (mcs_mod == LTEPHY_UL_MOD_256QAM_MAX)
      order[n++] = 2;
    else
      order[n++] = 0, order[n++] = 2;
  }
  int m = 0;
  for (int k = 0; k < n; k++) { // a reading without a transport block size (MCS 28 has no row in Table 8.6.1-3) cannot pass a CRC in the reference either
    if (ltephy_ul_dci_to_grant(s, d, order[k], &grants[m]) != LTEPHY_SUCCESS) continue;
    reading[m++] = (uint8_t)order[k];
  }
  return m;
}

// One line of the DCI trace file, DCIToFile::printDCICollection (reference src/src/SubframeInfoConsumer.cc:66-138); the hex column is
// sprint_hex of the payload bits (lib/src/phy/falcon_phch/falcon_dci.c:37-58).  Declared in include/ltephy_sinks.h.
extern "C" int ltephy_dci_trace_line(const ltephy_search_t* s, const ltephy_dci_t* d, uint32_t tti, uint32_t cfi, int use_256qam_table, uint32_t ts_sec,
                                     uint32_t ts_usec, char* out, size_t cap)
{
  if (!s || !d || !out || cap < 2 || d->nof_bits == 0 || d->nof_bits > 64) return LTEPHY_ERROR_INVALID_INPUTS;
  char           hex[2 * 8 + 1];
  const uint32_t nbytes = (d->nof_bits + 7) / 8;
  for (uint32_t i = 0; i < nbytes; i++) snprintf(hex + 2 * i, 3, "%02x", (unsigned)((d->bits >> (56 - 8 * i)) & 0xFFu));
  const uint32_t sfn = tti / 10, sf = tti % 10;
  int            n;
  if (d->format == ltehost::F0) {
    const uint32_t N = s->cell.nof_prb, rivb = clog2(N * (N + 1) / 2);
    Bits           b{d->bits};
    b.get(1), b.get(1);
    const uint32_t riv = b.get(rivb), mcs = b.get(5), ndi = b.get(1);
    uint32_t       L, S;
    riv_decode(riv, N, L, S);
    if (L < 1 || L > N || S >= N || S + L > N) return LTEPHY_ERROR;
    const int itbs = mcs <= 10 ? (int)mcs : mcs <= 20 ? (int)mcs - 1 : (int)mcs - 2;
    const int tbs  = mcs < 29 ? lte_tbs_table[itbs][L - 1] : 0;
    n = snprintf(out, cap, "%ld.%06ld\t%04d\t%d\t%d\t0\t%d\t%d\t%d\t%d\t%d\t0\t%d\t-1\t%d\t%d\t%d\t%d\t%d\t%d\t%s\n", (long)ts_sec, (long)ts_usec, (int)sfn,
                 (int)sf, (int)d->rnti, (int)mcs, (int)L, tbs, -1, -1, (int)ndi, (int)((10 * sfn + sf) % 8), (int)d->ncce, (int)d->L, (int)cfi,
                 (int)d->histogram_value, (int)d->nof_bits, hex);
  } else {
    ltephy_grant_t      g;
    ltephy_dci_fields_t f;
    if (ltephy_dci_to_grant(s, d, sf, cfi, use_256qam_table, &g, &f) != LTEPHY_SUCCESS) return LTEPHY_ERROR;
    const bool two  = d->format >= ltehost::F2;
    // The reference's convert_dl_grant fills BOTH legacy mcs[] entries from the first transport block (ran_dl_grant->tb->tbs,
    // lib/src/phy/falcon_phch/falcon_dci.c:608-612), so a two-TB line reads "2 x tbs0, tbs0, tbs0" whatever the second block carries: reproduced,
    // because the trace file is an output format (checked line by line against DCIToFile::printDCICollection in tests/test_reference_code.py)
    const int  tbs0 = g.tb[0].tbs > 0 ? g.tb[0].tbs : 0, tbs1 = tbs0;
    n = snprintf(out, cap, "%ld.%06ld\t%04d\t%d\t%d\t1\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%s\n", (long)ts_sec, (long)ts_usec, (int)sfn,
                 (int)sf, (int)d->rnti, (int)f.mcs[0], (int)f.nof_prb, two ? tbs0 + tbs1 : tbs0, two ? tbs0 : -1, two ? tbs1 : -1, (int)d->format + 1,
                 (int)f.ndi[0], two ? (int)f.ndi[1] : -1, (int)f.harq_pid, (int)d->ncce, (int)d->L, (int)cfi, (int)d->histogram_value, (int)d->nof_bits, hex);
  }
  return (n < 0 || (size_t)n >= cap) ? LTEPHY_ERROR_INVALID_INPUTS : n;
}

// ===================================================================================================
// Control-region geometry of a cell as the PHY uses it (tables uploaded by ltephy_create): for one CFI the grid indices l * 12 nof_prb + k of the four REs of
// every PDCCH quadruplet in CCE order (36.211 6.8.5: interleaver and cell-specific shift applied; PCFICH and PHICH REGs left out), and the 16 PCFICH REs.
int ltephy_ctrl_region_map(uint32_t nof_prb, uint32_t nof_ports, uint32_t cell_id, uint32_t phich_resources, uint32_t cfi, uint16_t* pdcch_idx, uint32_t cap,
                           uint32_t* nof_cce, uint16_t* pcfich_idx)
{
  if (cfi < 1 || cfi > 3 || !nof_cce) return LTEPHY_ERROR_INVALID_INPUTS;
  ltehost::CtrlMap cm;
  if (!ltehost::build_ctrl_map(ltehost::Cell{nof_prb, nof_ports, cell_id, 1, phich_resources & 0xFFu, phich_resources >> 8}, cm)) return LTEPHY_ERROR_INVALID_INPUTS;
  *nof_cce = cm.nof_cce[cfi - 1];
  if (pdcch_idx) {
    if (cap < cm.pdcch_idx[cfi - 1].size()) return LTEPHY_ERROR_INVALID_INPUTS;
    memcpy(pdcch_idx, cm.pdcch_idx[cfi - 1].data(), cm.pdcch_idx[cfi - 1].size() * sizeof(uint16_t));
  }
  if (pcfich_idx) memcpy(pcfich_idx, cm.pcfich_idx, sizeof(cm.pcfich_idx));
  return LTEPHY_SUCCESS;
}
ltephy_search_t* ltephy_search_create_cell(uint32_t nof_prb, uint32_t nof_ports, uint32_t cell_id, uint32_t nof_rx, uint32_t histogram_threshold)
{
  return ltephy_search_create_cell_ng(nof_prb, nof_ports, cell_id, nof_rx, 0, histogram_threshold);
}
ltephy_search_t* ltephy_search_create_cell_ng(uint32_t nof_prb, uint32_t nof_ports, uint32_t cell_id, uint32_t nof_rx, uint32_t phich_resources,
                                              uint32_t histogram_threshold)
{
  ltehost::CtrlMap cm;
  ltehost::Cell    cell{nof_prb, nof_ports, cell_id, nof_rx, phich_resources & 0xFFu, phich_resources >> 8};
  if (!ltehost::build_ctrl_map(cell, cm)) return nullptr;
  ltephy_search* s = new ltephy_search();
  s->cell          = cell;
  s->st = ltehost::dci_size_table(s->cell);
  for (uint32_t cfi = 1; cfi <= 3; cfi++) s->nof_cce[cfi - 1] = cm.nof_cce[cfi - 1];
  for (uint32_t cfi = 0; cfi < 3; cfi++) { // srsran_pdcch_ue_locations_all_map, falcon_pdcch.c:321-356
    auto& tp = s->tmpl[cfi];
    memset(tp.loc_of, 0xFF, sizeof(tp.loc_of));
    const uint32_t lim = std::min<uint32_t>(s->nof_cce[cfi], LTEPHY_SEARCH_MAX_CCE);
    uint32_t       k   = 0;
    for (int l = 3; l >= 0; l--) {
      const uint32_t Lc = 1u << l;
      tp.nq[l] = lim / Lc;
      for (uint32_t i = 0; i < lim / Lc && k < LTEPHY_MAX_LOC; i++) {
        tp.loc[k]            = {(uint8_t)l, (uint8_t)(Lc * i), false, false, false, true};
        tp.loc_of[l][Lc * i] = (int16_t)k;
        tp.val[l] |= (u128)1 << (Lc * i);
        k++;
      }
    }
    tp.n = k;
  }
  {
    const uint32_t cls_sf[3] = {0, 5, 1};
    uint16_t       kk[12];
    s->re_slot.assign((size_t)3 * 3 * 2 * nof_prb, 0);
    for (uint32_t cls = 0; cls < 3; cls++)
      for (uint32_t cfi = 1; cfi <= 3; cfi++)
        for (uint32_t l = 0; l < 14; l++)
          for (uint32_t prb = 0; prb < nof_prb; prb++)
            s->re_slot[(((size_t)cls * 3 + cfi - 1) * 2 + l / 7) * nof_prb + prb] += (uint16_t)ltehost::pdsch_re_in_prb(cell, cls_sf[cls], cfi, l, prb, kk);
  }
  s->rm.threshold = histogram_threshold;
  for (int i = 0; i < NF; i++) s->all[i] = {(uint8_t)i, 0};
  s->update_formats();
  // evergreen / forbidden ranges exactly as LTESniffer_Core.cc:398-417 seeds them after the MIB
  for (int f : {(int)ltehost::F1A, (int)ltehost::F1C}) {
    s->rm.add_evergreen(RARNTI_START, RARNTI_END, (uint32_t)f);
    s->rm.add_evergreen(PRNTI, 0xFFFF, (uint32_t)f);
  }
  for (int f = 0; f < NF; f++) s->rm.add_forbidden(0, 0, (uint32_t)f);
  return s;
}
ltephy_search_t* ltephy_search_create(const ltephy_t* h, uint32_t histogram_threshold)
{
  if (!h) return nullptr;
  uint32_t a, b, c, d;
  ltephy_cell_of(h, &a, &b, &c, &d);
  return ltephy_search_create_cell_ng(a, b, c, d, ltephy_phich_resources(h), histogram_threshold);
}
void ltephy_search_destroy(ltephy_search_t* s) { delete s; }
void ltephy_search_set_ul_hopping(ltephy_search_t* s, uint32_t n_rb_ho)
{
  if (s) s->ul_n_rb_ho = n_rb_ho;
}
// Redundancy version of a format-1C SI-RNTI transmission, which carries no rv field (srsRAN leaves tb.rv = -1): PDSCH_Decoder::decode_SIB (the SIB
// acquisition of the UL mode, DL_Sniffer_PDSCH.cc:505-511) uses k = (SFN / 2) % 4, rv = ceil(1.5 k) % 4 (36.321 5.3.1), while decode_dl_mode uses 0
// (:891-898), which is what ltephy_dci_to_grant writes.
uint32_t ltephy_si_format1c_rv(uint32_t tti)
{
  static const uint8_t rv_of_k[4] = {0, 2, 3, 1};
  return rv_of_k[((tti / 10) / 2) % 4];
}
void ltephy_search_set_ul_mode(ltephy_search_t* s, int on, uint16_t target_rnti)
{
  if (s) s->ul_mode = on != 0, s->ul_target_rnti = target_rnti;
}
void ltephy_search_keep_reserved_mcs(ltephy_search_t* s, int on)
{
  if (s) s->keep_reserved_mcs = on != 0;
}
void ltephy_search_speculate_256qam(ltephy_search_t* s, int on)
{
  if (s) s->speculate_256qam = on != 0;
}
void ltephy_search_config(ltephy_search_t* s, int shortcut, int skip_secondary, uint32_t update_interval)
{
  s->shortcut = shortcut != 0, s->skip_secondary = skip_secondary != 0, s->update_interval = update_interval;
}
void ltephy_search_add_evergreen(ltephy_search_t* s, uint16_t a, uint16_t b, uint32_t f)
{
  std::lock_guard<std::mutex> lk(s->turn.m);
  if (f < NF && a <= b) s->rm.add_evergreen(a, b, f);
}
void ltephy_search_add_forbidden(ltephy_search_t* s, uint16_t a, uint16_t b, uint32_t f)
{
  std::lock_guard<std::mutex> lk(s->turn.m);
  if (f < NF && a <= b) s->rm.add_forbidden(a, b, f);
}
void ltephy_search_activate(ltephy_search_t* s, uint16_t rnti, uint32_t format_idx, int reason)
{
  std::lock_guard<std::mutex> lk(s->turn.m); // another pipeline thread may be inside the walk
  s->rm.activate_and_refresh(rnti, format_idx, (uint8_t)reason);
}
int  ltephy_search_subframe(ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_cand_t* cands, uint32_t sf_in_batch, ltephy_dci_t* out,
                            uint32_t max_out, uint32_t* n_out)
{
  if (!s || !info || !cands) return LTEPHY_ERROR_INVALID_INPUTS;
  return s->search_subframe(*info, cands, nullptr, sf_in_batch, out, max_out, n_out);
}
int ltephy_search_subframe_compact(ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_compact_t* comp, uint32_t sf_in_batch, ltephy_dci_t* out,
                                   uint32_t max_out, uint32_t* n_out)
{
  if (!s || !info || !comp) return LTEPHY_ERROR_INVALID_INPUTS;
  return s->search_subframe(*info, nullptr, comp, sf_in_batch, out, max_out, n_out);
}
// Host restatement of the survivor selection the GPU does in cand_compact_kernel (k_viterbi.cu); same bytes out.
int ltephy_compact_from_table(const ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_cand_t* cands, ltephy_compact_t* out)
{
  if (!s || !info || !cands || !out) return LTEPHY_ERROR_INVALID_INPUTS;
  memset(out, 0, sizeof(*out));
  if (info->cfi < 1 || info->cfi > 3) return LTEPHY_SUCCESS;
  const auto&    tp      = s->tmpl[info->cfi - 1];
  const uint32_t ncce_sf = s->nof_cce[info->cfi - 1], lim = std::min<uint32_t>(ncce_sf, LTEPHY_SEARCH_MAX_CCE), sf_idx = info->tti % 10;
  uint32_t       cnt     = 0;
  for (uint32_t li = 0; li < tp.n; li++) {
    const uint32_t L = tp.loc[li].L, ncce = tp.loc[li].ncce;
    bool           suff = true;
    for (uint32_t c = ncce; c < ncce + (1u << L); c++)
      if (c < lim && info->cce_power[c] < 0.7f) suff = false;
    const int par = (L < 3 && (ncce & ((2u << L) - 1u)) == 0) ? tp.loc_of[L + 1][ncce] : -1;
    out->loc[li].off = (uint16_t)std::min<uint32_t>(cnt, 0xFFFF);
    uint32_t mask    = 0;
    for (uint32_t si = 0; suff && si < s->st.sizes.size(); si++) {
      const ltephy_cand_t& e  = cands[(size_t)li * LTEPHY_MAX_SIZES + si];
      const uint16_t       r  = e.valid ? e.rnti : 0;
      const uint32_t       sm = validate_location(ncce_sf, ncce, L, sf_idx, r);
      bool                 eq = false;
      if (par >= 0) {
        const ltephy_cand_t& pe = cands[(size_t)par * LTEPHY_MAX_SIZES + si];
        eq                      = (pe.valid ? pe.rnti : 0) == r;
      }
      if (sm == 0 && r != 0 && !eq) continue;
      mask |= 1u << si;
      if (cnt < LTEPHY_COMPACT_CAP) {
        ltephy_cand_t& o = out->list[cnt];
        o                = e;
        if (!e.valid) o.bits = 0, o.rnti = 0;
        memset(o.pad, 0, sizeof(o.pad));
        o.pad[0] = (uint8_t)(sm | ((r == 0) << 2) | (eq << 3)), o.pad[1] = (uint8_t)li, o.pad[2] = (uint8_t)si;
      }
      cnt++;
    }
    out->loc[li].mask = (uint8_t)mask;
  }
  for (uint32_t li = 0; li < tp.n; li++) { // pad = union of the masks over the location's subtree (itself included)
    const uint32_t L = tp.loc[li].L, ncce = tp.loc[li].ncce;
    uint32_t       u = out->loc[li].mask;
    for (uint32_t l2 = 0; l2 < L; l2++)
      for (uint32_t c = ncce; c < ncce + (1u << L); c += 1u << l2) {
        const int j = tp.loc_of[l2][c];
        if (j >= 0) u |= out->loc[j].mask;
      }
    out->loc[li].pad = (uint8_t)u;
  }
  out->count = cnt;
  return LTEPHY_SUCCESS;
}
void ltephy_search_get_stats(const ltephy_search_t* s, ltephy_search_stats_t* st) { *st = s->stats; }
uint32_t ltephy_search_validate_location(uint32_t nof_cce, uint32_t ncce, uint32_t L, uint32_t sf_idx, uint16_t rnti)
{
  return validate_location(nof_cce, ncce, L, sf_idx, rnti);
}
// thin test hooks onto the RNTI history (parity with the reference's rnti_manager_* C wrappers)
int      ltephy_search_rnti_validate_and_refresh(ltephy_search_t* s, uint16_t r, uint32_t f) { return s->rm.validate_and_refresh(r, f); }
void     ltephy_search_rnti_add_candidate(ltephy_search_t* s, uint16_t r, uint32_t f) { s->rm.add_candidate(r, f); }
void     ltephy_search_rnti_step_time(ltephy_search_t* s) { s->rm.step_time(); }
uint32_t ltephy_search_rnti_frequency(const ltephy_search_t* s, uint16_t r, uint32_t f) { return s->rm.freq(r, f); }
uint32_t ltephy_search_rnti_assoc_format(const ltephy_search_t* s, uint16_t r) { return s->rm.rec[r].assoc; }
int      ltephy_search_rnti_reason(const ltephy_search_t* s, uint16_t r) { return s->rm.rec[r].reason; }
int      ltephy_search_rnti_is_forbidden(const ltephy_search_t* s, uint16_t r, uint32_t f) { return s->rm.is_forbidden(r, f); }
int      ltephy_search_rnti_is_evergreen(const ltephy_search_t* s, uint16_t r, uint32_t f) { return s->rm.is_evergreen(r, f); }

// ===================================================================================================
// Batch helpers: the FALCON walk over n subframes in order (dci.sf = index in the batch), over full tables or survivor forms.
int ltephy_search_batch(ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_cand_t* cands, uint32_t n, ltephy_dci_t* dcis, uint32_t max_dcis,
                        uint32_t* n_dcis)
{
  if (!s || !info || !cands || !dcis || !n_dcis) return LTEPHY_ERROR_INVALID_INPUTS;
  return s->search_batch(
      n, [&](uint32_t i) { return ltephy_search::WalkSf{s->walk_in(info[i], cands + (size_t)i * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES, nullptr), nullptr}; },
      dcis, max_dcis, n_dcis);
}
// Same walk over the survivor form.  full (optional) is the full table of the same batch; it is consulted for the
// subframes the survivor form cannot serve.  Without it such a batch is refused up front, before anything is consumed.
int ltephy_search_batch_compact(ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_compact_t* comp, const ltephy_cand_t* full, uint32_t n,
                                ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis)
{
  if (!s || !info || !comp || !dcis || !n_dcis) return LTEPHY_ERROR_INVALID_INPUTS;
  if (!full && s->may_need_full_table(ltephy_search::FOR_WALK, n, [&](uint32_t i) { return comp[i].count; })) return LTEPHY_NEED_FULL_TABLE;
  return s->search_batch(
      n,
      [&](uint32_t i) {
        if (i + 2 < n) __builtin_prefetch(&comp[i + 2], 0, 3), __builtin_prefetch(&info[i + 2], 0, 3);
        if (i + 1 < n) { // the inputs stream through once: have the next subframe's records in cache when its walk starts
          const char*    c  = reinterpret_cast<const char*>(&comp[i + 1]);
          const uint32_t nb = (uint32_t)offsetof(ltephy_compact_t, list) + 16u * std::min<uint32_t>(comp[i + 1].count, LTEPHY_COMPACT_CAP);
          for (uint32_t o = 64; o < nb; o += 64) __builtin_prefetch(c + o, 0, 3);
          const char* f = reinterpret_cast<const char*>(&info[i + 1]);
          for (uint32_t o = 0; o < sizeof(ltephy_sf_info_t); o += 64) __builtin_prefetch(f + o, 0, 3);
        }
        return ltephy_search::WalkSf{s->walk_in(info[i], nullptr, &comp[i]), full ? full + (size_t)i * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES : nullptr};
      },
      dcis, max_dcis, n_dcis);
}
int ltephy_search_needs_full_table(const ltephy_search_t* s, const ltephy_compact_t* comp, uint32_t n)
{
  if (!s || !comp) return LTEPHY_ERROR_INVALID_INPUTS;
  return s->may_need_full_table(ltephy_search::FOR_COLLECTIVE, n, [&](uint32_t i) { return comp[i].count; });
}
// Accepted DL DCIs -> PDSCH grants, applying decode_dl_mode's skip rule (src/src/DL_Sniffer_PDSCH.cc:887-889).
// Only subframes with sf % mod == rem are taken (multi-GPU sharding); grant.sf = sf / mod (local index).
} // extern "C"
template <class TtiCfi>
static int grants_from_dcis_impl(const ltephy_search_t* s, TtiCfi tc, const ltephy_dci_t* dcis, uint32_t nd, uint32_t mod, uint32_t rem,
                                 ltephy_grant_t* grants, uint32_t* grant_dci, uint32_t max_grants, uint32_t* n_grants)
{
  uint32_t ng = 0;
  auto eligible = [&](const ltephy_grant_t& g) {
    // tbs = 0: reserved MCS.  The reference applies this rule after DCICollection gave such a block the size of its HARQ process' last transmission
    // (DCICollection.cc:236-252), which here is the caller's ltephy_harq_prepare_grant -- so in that mode the grant has to get through
    const bool sized = g.tb[0].tbs > 0 || (s->keep_reserved_mcs && g.tb[0].enabled && user_rnti(g.rnti));
    if (!(sized && !(s->cell.nof_rx == 1 && g.nof_tb == 2))) return false;
    if (g.tx_scheme == LTEPHY_TX_SPATIALMUX && (s->cell.nof_ports != 2 || (g.nof_tb == 2 && s->cell.nof_rx != 2))) return false;
    return true;
  };
  for (uint32_t i = 0; i < nd; i++) {
    const ltephy_dci_t& d = dcis[i];
    if (d.sf % mod != rem || d.format == ltehost::F0 || d.rnti == 0) continue;
    ltephy_grant_t g[2];
    bool           ok[2] = {false, false};
    uint32_t tti_sf, cfi_sf;
    tc(d.sf, tti_sf, cfi_sf);
    ok[0] = ltephy_dci_to_grant(s, &d, tti_sf % 10, cfi_sf, 0, &g[0], nullptr) == LTEPHY_SUCCESS && eligible(g[0]);
    if (s->ul_mode) { // PDSCH_Decoder::decode_ul_mode (DL_Sniffer_PDSCH.cc:362-457): Random Access Responses, and format 1 / 1A of everything but the SI-RNTI,
                      // with the 64QAM table only
      const bool rar = d.rnti >= RARNTI_START && d.rnti <= RARNTI_END;
      const bool sel = d.rnti == s->ul_target_rnti || s->ul_target_rnti == 0 || d.rnti > RARNTI_END;
      if (!rar && !(sel && (d.format == ltehost::F1 || d.format == ltehost::F1A) && d.rnti != 0xFFFF)) ok[0] = false;
    } else if (s->speculate_256qam && user_rnti(d.rnti)) { // MCS table of the UE unknown: 64QAM reading first, then the 256QAM one
      ok[1] = ltephy_dci_to_grant(s, &d, tti_sf % 10, cfi_sf, 1, &g[1], nullptr) == LTEPHY_SUCCESS && eligible(g[1]);
      if (ok[0] && ok[1]) {
        bool same = g[0].nof_tb == g[1].nof_tb;
        for (int t = 0; t < 2 && same; t++) same = g[0].tb[t].enabled == g[1].tb[t].enabled && g[0].tb[t].qm == g[1].tb[t].qm && g[0].tb[t].tbs == g[1].tb[t].tbs;
        if (same) ok[1] = false;
      }
    }
    for (uint32_t a = 0; a < 2; a++) {
      if (!ok[a]) continue;
      if (ng >= max_grants) return LTEPHY_ERROR_INVALID_INPUTS;
      g[a].sf       = d.sf / mod;
      grants[ng]    = g[a];
      grant_dci[ng] = i | (a ? LTEPHY_GRANT_ALT_TABLE : 0u);
      ng++;
    }
  }
  *n_grants = ng;
  return LTEPHY_SUCCESS;
}
extern "C" {
int ltephy_grants_from_dcis(const ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_dci_t* dcis, uint32_t nd, uint32_t mod, uint32_t rem,
                            ltephy_grant_t* grants, uint32_t* grant_dci, uint32_t max_grants, uint32_t* n_grants)
{
  if (!s || !info || !dcis || !grants || !grant_dci || !n_grants || mod == 0) return LTEPHY_ERROR_INVALID_INPUTS;
  return grants_from_dcis_impl(s, [&](uint32_t sf, uint32_t& t, uint32_t& c) { t = info[sf].tti, c = info[sf].cfi; }, dcis, nd, mod, rem, grants,
                               grant_dci, max_grants, n_grants);
}
int ltephy_grants_from_dcis_tc(const ltephy_search_t* s, const uint32_t* tti_cfi, const ltephy_dci_t* dcis, uint32_t nd, uint32_t mod, uint32_t rem,
                               ltephy_grant_t* grants, uint32_t* grant_dci, uint32_t max_grants, uint32_t* n_grants)
{
  if (!s || !tti_cfi || !dcis || !grants || !grant_dci || !n_grants || mod == 0) return LTEPHY_ERROR_INVALID_INPUTS;
  return grants_from_dcis_impl(s, [&](uint32_t sf, uint32_t& t, uint32_t& c) { t = tti_cfi[2 * sf], c = tti_cfi[2 * sf + 1]; }, dcis, nd, mod, rem,
                               grants, grant_dci, max_grants, n_grants);
}

// What ltephy_submit_ul reserves for the control information of a grant (36.212 5.2.2.6; srsRAN Q_prime_ri_ack / Q_prime_cqi): the numbers of modulation
// symbols Q' of HARQ-ACK, rank indication and CQI, and the UL-SCH bits G that are left -- for a caller that sizes buffers or wants to know the code rate.
int ltephy_ul_uci_layout(const ltephy_ul_grant_t* g, uint32_t* qp_ack, uint32_t* qp_ri, uint32_t* qp_cqi, uint32_t* G)
{
  if (!g || g->tbs <= 0 || g->L_prb == 0) return LTEPHY_ERROR_INVALID_INPUTS;
  ltehost::UciLayout L;
  if (!ltehost::uci_layout(g->L_prb, g->qm, (uint32_t)g->tbs, g->nof_ack, g->ri_len, g->cqi_len, g->I_offset_ack, g->I_offset_ri, g->I_offset_cqi, L))
    return LTEPHY_ERROR_INVALID_INPUTS;
  if (qp_ack) *qp_ack = L.Qp_ack;
  if (qp_ri) *qp_ri = L.Qp_ri;
  if (qp_cqi) *qp_cqi = L.Qp_cqi;
  if (G) *G = L.G;
  return LTEPHY_SUCCESS;
}

// Size of the aperiodic CQI report multiplexed into a PUSCH whose DCI-0 requests one, for the report types the reference configures
// (UL_Sniffer_PUSCH.cc:434-445: uci_cfg.cqi.type from the UE's RRC configuration, default SRSRAN_CQI_TYPE_SUBBAND_HL, MCSTracking.cc:1538; N =
// ul_sniffer_cqi_hl_get_no_subbands, lib/src/phy/falcon_phch/dl_sniffer_pdsch.c:277-302; no PMI, rank 1): 36.212 Tables 5.2.2.6.1-1 (wideband, 4 bits)
// and 5.2.2.6.2-1 (higher-layer configured subbands, 4 + 2 N bits).  cqi_type: srsran_cqi_type_t (0 wideband, 3 subband HL).
int ltephy_ul_cqi_len(uint32_t nof_prb, int cqi_type)
{
  if (cqi_type == 0) return 4;
  if (cqi_type != 3 || nof_prb < 7 || nof_prb > 110) return LTEPHY_ERROR_INVALID_INPUTS;
  const uint32_t k = nof_prb <= 26 ? 4 : nof_prb <= 63 ? 6 : 8;
  return (int)(4 + 2 * ((nof_prb + k - 1) / k));
}

// UL mode, one batch: what SubframeWorker does per subframe between the search and PUSCH_Decoder::decode (reference src/src/SubframeWorker.cc:296-345)
// and the attempts that decoder then makes (ltephy_ul_decode_plan), for all DCI-0s of a batch of downlink subframes at once.
//   * the PUSCH of a DCI-0 seen at tti n is on the air at n + 4 (ULSchedule::pushULSche / get_ul_tti, src/src/ULSchedule.cc:112-124): grant.sf = dci.sf + 4,
//     an index into the uplink batch that starts at the same tti as the downlink batch -- indices >= the batch length belong to the next one;
//   * nof_ack = number of transport blocks of a downlink DCI of the same RNTI in the same subframe, the last such DCI winning (SubframeWorker.cc:318-337);
//   * an aperiodic CSI request (last payload bit, FDD) adds ri_len = 1 and the UE's CQI size (UL_Sniffer_PUSCH.cc:437-450);
//   * beta offsets and the MCS-table knowledge come per RNTI from ue[] (MCSTracking::get_ue_config_rnti / find_tracking_info_RNTI_ul), entry rnti = 0
//     being the default; without any: unknown table, 10 / 8 / 11 (SubframeWorker::setup_default_ul_cfg, SubframeWorker.cc:347-352); cqi_len 0 = the
//     reference's default report (subband CQI configured by higher layers, ltephy_ul_cqi_len).
int ltephy_ul_grants_from_dcis(const ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_dci_t* dcis, uint32_t nd, const ltephy_ul_ue_cfg_t* ue,
                               uint32_t n_ue, ltephy_ul_grant_t* grants, uint32_t* grant_dci, uint8_t* reading, uint32_t max_grants, uint32_t* n_grants)
{
  if (!s || !info || !dcis || !grants || !grant_dci || !reading || !n_grants || (n_ue && !ue)) return LTEPHY_ERROR_INVALID_INPUTS;
  const uint32_t N = s->cell.nof_prb, rivb = clog2(N * (N + 1) / 2);
  uint32_t       ng = 0;
  for (uint32_t i = 0; i < nd; i++) {
    const ltephy_dci_t& d = dcis[i];
    if (d.format != ltehost::F0 || d.rnti == 0) continue;
    ltephy_ul_ue_cfg_t cfg{0, LTEPHY_UL_MOD_UNKNOWN, 10, 8, 11, 0};
    for (uint32_t k = 0; k < n_ue; k++)
      if (ue[k].rnti == 0) cfg = ue[k];
    for (uint32_t k = 0; k < n_ue; k++)
      if (ue[k].rnti == d.rnti) cfg = ue[k];
    ltephy_ul_grant_t g[3];
    uint8_t           rd[3];
    const int         n = ltephy_ul_decode_plan(s, &d, cfg.mcs_mod, g, rd);
    if (n < 0) return n;
    if (n == 0) continue;
    uint8_t nof_ack = 0;
    uint32_t lo = i, hi = i + 1; // the accepted DCIs of one subframe are adjacent (the search emits subframe after subframe)
    while (lo > 0 && dcis[lo - 1].sf == d.sf) lo--;
    while (hi < nd && dcis[hi].sf == d.sf) hi++;
    for (uint32_t j = lo; j < hi; j++) {
      const ltephy_dci_t& dl = dcis[j];
      if (dl.format == ltehost::F0 || dl.rnti != d.rnti) continue;
      ltephy_grant_t gd;
      const int      r = ltephy_dci_to_grant(s, &dl, info[dl.sf].tti % 10, info[dl.sf].cfi, 0, &gd, nullptr);
      // a DCI whose conversion fails has its RNTI zeroed by the reference (falcon_dci.c:286-305); the MIMO checks come later, in the decoder
      if (r != LTEPHY_SUCCESS && r != LTEPHY_MIMO_NOT_SUPPORT && r != LTEPHY_MIMO_PMI_WRONG && r != LTEPHY_MIMO_LAYER_WRONG) continue;
      if (gd.nof_tb == 1 || gd.nof_tb == 2) nof_ack = (uint8_t)gd.nof_tb;
    }
    Bits b{d.bits};
    b.get(2), b.get(rivb), b.get(5 + 1 + 2 + 3);
    const bool cqi_request = b.get(1) != 0;
    const int  dflt        = ltephy_ul_cqi_len(N, 3); // the reference's default report type (MCSTracking::set_default_of_default_config)
    const uint16_t cqi_len = cfg.cqi_len ? cfg.cqi_len : (uint16_t)(dflt > 0 ? dflt : 0);
    for (int k = 0; k < n; k++) {
      if (ng >= max_grants) return LTEPHY_ERROR_INVALID_INPUTS;
      g[k].sf = d.sf + 4, g[k].nof_ack = nof_ack, g[k].ri_len = cqi_request ? 1 : 0, g[k].cqi_len = cqi_request ? cqi_len : 0;
      g[k].I_offset_ack = cfg.I_offset_ack, g[k].I_offset_cqi = cfg.I_offset_cqi, g[k].I_offset_ri = cfg.I_offset_ri;
      grants[ng] = g[k], grant_dci[ng] = i, reading[ng] = rd[k];
      ng++;
    }
  }
  *n_grants = ng;
  return LTEPHY_SUCCESS;
}

// ===================================================================================================
// Packed survivor form (include/ltephy_shard.h): header + location records + survivor list, back to back.
size_t ltephy_packed_size(uint32_t nloc, uint32_t count)
{
  return sizeof(ltephy_packed_hdr_t) + sizeof(ltephy_cloc_t) * ((nloc + 3u) & ~3u) + sizeof(ltephy_cand_t) * std::min<uint32_t>(count, LTEPHY_COMPACT_CAP);
}
int ltephy_pack_subframes(const ltephy_search_t* s, const ltephy_sf_info_t* info, const ltephy_compact_t* comp, uint32_t n, uint8_t* out, size_t cap,
                          uint32_t* offs)
{
  if (!s || !info || !comp || !out || !offs) return LTEPHY_ERROR_INVALID_INPUTS;
  size_t pos = 0;
  for (uint32_t i = 0; i < n; i++) {
    const bool     ok   = info[i].cfi >= 1 && info[i].cfi <= 3;
    const uint32_t nloc = ok ? s->tmpl[info[i].cfi - 1].n : 0, cnt = ok ? comp[i].count : 0;
    const size_t   sz   = ltephy_packed_size(nloc, cnt);
    if (pos + sz > cap) return LTEPHY_ERROR_INVALID_INPUTS;
    offs[i] = (uint32_t)pos;
    ltephy_packed_hdr_t hd{};
    hd.count = cnt, hd.tti = info[i].tti, hd.cfi = info[i].cfi, hd.nloc = nloc;
    memcpy(hd.noise, info[i].noise, sizeof(hd.noise)), memcpy(hd.rsrp, info[i].rsrp, sizeof(hd.rsrp));
    if (ok) {
      const ltephy_search::WalkIn w = s->walk_in(info[i], nullptr, nullptr);
      hd.low[0] = w.low[0], hd.low[1] = w.low[1];
    }
    memcpy(out + pos, &hd, sizeof(hd));
    ltephy_cloc_t* loc = reinterpret_cast<ltephy_cloc_t*>(out + pos + sizeof(hd));
    for (uint32_t j = 0; j < ((nloc + 3u) & ~3u); j++) loc[j] = j < nloc ? comp[i].loc[j] : ltephy_cloc_t{0, 0, 0};
    memcpy(out + pos + sizeof(hd) + sizeof(ltephy_cloc_t) * ((nloc + 3u) & ~3u), comp[i].list, sizeof(ltephy_cand_t) * std::min<uint32_t>(cnt, LTEPHY_COMPACT_CAP));
    pos += sz;
  }
  offs[n] = (uint32_t)pos;
  return LTEPHY_SUCCESS;
}
// record i of rank r = global subframe g = i * world + r
static inline const ltephy_packed_hdr_t* packed_hdr(const uint8_t* const* bufs, const uint32_t* const* offs, uint32_t world, uint32_t g)
{
  return reinterpret_cast<const ltephy_packed_hdr_t*>(bufs[g % world] + offs[g % world][g / world]);
}
static inline ltephy_search::WalkIn walk_in_packed(const ltephy_search_t* s, const ltephy_packed_hdr_t* hd)
{
  // snr_db exactly as ltephy_finalize_info evaluates it (DESIGN.md section 2: log10f on the host from bit-exact device sums)
  const uint32_t P = s->cell.nof_ports, A = s->cell.nof_rx;
  float          ns = 0.0f, ps = 0.0f;
  for (uint32_t p = 0; p < P; p++)
    for (uint32_t a = 0; a < A; a++) ns = ns + hd->noise[p][a], ps = ps + hd->rsrp[p][a];
  const float npa = (float)(P * A), snr = 10.0f * log10f((ps / npa) / (ns / npa));
  const ltephy_cloc_t* loc = reinterpret_cast<const ltephy_cloc_t*>(hd + 1);
  return ltephy_search::WalkIn{hd->tti, hd->cfi, snr, {hd->low[0], hd->low[1]}, hd->count, nullptr, loc, reinterpret_cast<const ltephy_cand_t*>(loc + ((hd->nloc + 3u) & ~3u))};
}
int ltephy_packed_needs_full_table(const ltephy_search_t* s, const uint8_t* const* bufs, const uint32_t* const* offs, uint32_t world, uint32_t n)
{
  if (!s || !bufs || !offs) return LTEPHY_ERROR_INVALID_INPUTS;
  return s->may_need_full_table(ltephy_search::FOR_COLLECTIVE, n * world, [&](uint32_t g) { return packed_hdr(bufs, offs, world, g)->count; });
}
int ltephy_search_batch_packed(ltephy_search_t* s, const uint8_t* const* bufs, const uint32_t* const* offs, const ltephy_cand_t* const* full,
                               uint32_t world, uint32_t n, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis, uint32_t* tti_cfi)
{
  if (!s || !bufs || !offs || !dcis || !n_dcis || world == 0) return LTEPHY_ERROR_INVALID_INPUTS;
  const uint32_t total = n * world;
  if (!full && s->may_need_full_table(ltephy_search::FOR_WALK, total, [&](uint32_t g) { return packed_hdr(bufs, offs, world, g)->count; }))
    return LTEPHY_NEED_FULL_TABLE;
  return s->search_batch(
      total,
      [&](uint32_t g) {
        if (g + 1 < total) { // the records stream through once: pull the next one towards the core while this one is walked
          const uint32_t r2 = (g + 1) % world, i2 = (g + 1) / world;
          const uint8_t* nx = bufs[r2] + offs[r2][i2];
          const uint32_t nb = offs[r2][i2 + 1] - offs[r2][i2];
          for (uint32_t o = 0; o < nb; o += 64) __builtin_prefetch(nx + o, 0, 3);
        }
        const ltephy_packed_hdr_t* hd = packed_hdr(bufs, offs, world, g);
        if (tti_cfi) tti_cfi[2 * g] = hd->tti, tti_cfi[2 * g + 1] = hd->cfi;
        return ltephy_search::WalkSf{walk_in_packed(s, hd), full ? full[g % world] + (size_t)(g / world) * LTEPHY_MAX_LOC * LTEPHY_MAX_SIZES : nullptr};
      },
      dcis, max_dcis, n_dcis);
}

// One call = what SubframeWorker::work does for every subframe of the batch (src/src/SubframeWorker.cc:142-207):
// phase A on the GPU, FALCON search on the host in subframe order, phase B on the GPU for the DL grants.
static double     g_host_ms[8];
static std::mutex g_host_ms_mtx;
static inline double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
void ltephy_last_host_timing(double* ms8)
{
  std::lock_guard<std::mutex> lk(g_host_ms_mtx);
  memcpy(ms8, g_host_ms, sizeof(g_host_ms));
}

static int decode_common(ltephy_t* h, ltephy_search_t* s, const void* iq, bool iq_on_device, const uint32_t* tti, uint32_t n, uint64_t seq,
                         ltephy_sf_info_t* info, ltephy_cand_t* cand_scratch, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis,
                         ltephy_tb_result_t* tbs, uint8_t* payload, size_t payload_cap)
{
  if (!s) return LTEPHY_ERROR_INVALID_INPUTS;
  double t0 = now_ms();
  if (!s->turn.claim(seq)) return LTEPHY_ERROR_INVALID_INPUTS;
  // Whatever happens before this batch's turn in the walk, the argument check included, the turn is passed on: a failing
  // batch must not leave the other pipelines of this search object waiting for a sequence number that never comes.
  TurnGuard turn(s->turn, seq);
  if (!h || !iq || !tti || !info || !cand_scratch || !dcis || !n_dcis || !tbs) return LTEPHY_ERROR_INVALID_INPUTS;
  int r = iq_on_device ? ltephy_submit_iq_device(h, iq, tti, n) : ltephy_submit_iq(h, iq, tti, n);
  if (r) return r;
  double t1 = now_ms();
  r = ltephy_get_phase_a_compact(h, info, nullptr); // survivor form (4.5 KB / subframe) stays in the handle's pinned buffer
  if (r) return r;
  const ltephy_compact_t* comp = ltephy_phase_a_compact_buffer(h);
  double t2 = now_ms();
  uint32_t nd = 0;
  turn.take();
  r = ltephy_search_batch_compact(s, info, comp, nullptr, n, dcis, max_dcis, &nd);
  if (r == LTEPHY_NEED_FULL_TABLE) { // RAR-activated RNTIs or an overfull subframe: fetch the 20 KB / subframe table after all
    r = ltephy_get_phase_a(h, nullptr, cand_scratch);
    if (r == LTEPHY_SUCCESS) r = ltephy_search_batch_compact(s, info, comp, cand_scratch, n, dcis, max_dcis, &nd);
  }
  turn.pass();
  if (r < 0) return r;
  double t3 = now_ms();
  *n_dcis = nd;
  std::vector<ltephy_grant_t> grants(2 * (size_t)nd + 1);
  std::vector<uint32_t>       grant_dci(2 * (size_t)nd + 1);
  uint32_t                    ng = 0;
  r = ltephy_grants_from_dcis(s, info, dcis, nd, 1, 0, grants.data(), grant_dci.data(), 2 * nd + 1, &ng);
  if (r) return r;
  double t4 = now_ms();
  for (uint32_t i = 0; i < 2 * nd; i++) tbs[i] = ltephy_tb_result_t{};
  r = ltephy_submit_grants(h, grants.data(), ng);
  if (r) return r;
  double t5 = now_ms();
  std::vector<ltephy_tb_result_t> res(2 * (size_t)ng + 2);
  r = ltephy_get_phase_b(h, res.data(), payload, payload_cap);
  if (r) return r;
  double t6 = now_ms();
  {
    std::lock_guard<std::mutex> lk(g_host_ms_mtx);
    g_host_ms[0] = t1 - t0, g_host_ms[1] = t2 - t1, g_host_ms[2] = t3 - t2, g_host_ms[3] = t4 - t3, g_host_ms[4] = t5 - t4, g_host_ms[5] = t6 - t5;
  }
  for (uint32_t gi = 0; gi < ng; gi++) ltephy_place_grant_result(tbs, grant_dci[gi], res[2 * gi], res[2 * gi + 1]);
  return LTEPHY_SUCCESS;
}
int ltephy_decode_subframes(ltephy_t* h, ltephy_search_t* s, const void* iq, const uint32_t* tti, uint32_t n, uint64_t seq, ltephy_sf_info_t* info,
                            ltephy_cand_t* cand_scratch, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis, ltephy_tb_result_t* tbs,
                            uint8_t* payload, size_t payload_cap)
{
  return decode_common(h, s, iq, false, tti, n, seq, info, cand_scratch, dcis, max_dcis, n_dcis, tbs, payload, payload_cap);
}
int ltephy_decode_subframes_device(ltephy_t* h, ltephy_search_t* s, const void* iq_dev, const uint32_t* tti, uint32_t n, uint64_t seq,
                                   ltephy_sf_info_t* info, ltephy_cand_t* cand_scratch, ltephy_dci_t* dcis, uint32_t max_dcis, uint32_t* n_dcis,
                                   ltephy_tb_result_t* tbs, uint8_t* payload, size_t payload_cap)
{
  return decode_common(h, s, iq_dev, true, tti, n, seq, info, cand_scratch, dcis, max_dcis, n_dcis, tbs, payload, payload_cap);
}

} // extern "C"
