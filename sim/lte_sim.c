/*
 * lte_sim.c -- synthetic eNB + channel (see lte_sim.h).  Ground truth generator for the parity
 * tests and input generator for bench.py.  Not product code, not oracle-receiver code.
 */
#include "lte_sim.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

struct lte_sim {
  lte_sim_cfg_t cfg;
  lte_regs_t    regs;
  uint16_t*     rntis;
  float         h_re[LTE_MAX_ANT][LTE_MAX_PORTS], h_im[LTE_MAX_ANT][LTE_MAX_PORTS];
  uint32_t      delay[LTE_MAX_ANT][LTE_MAX_PORTS];
  uint32_t      fft, nsc, sf_len;
  /* scratch */
  cf_t*    grid[LTE_MAX_PORTS]; /* [14][nsc] */
  cf_t*    td[LTE_MAX_PORTS];   /* [sf_len] */
  double*  fre;
  double*  fim;
  uint8_t* ebits;  /* up to 2 * 110*12*14*8 */
  uint8_t* tbbits; /* tbs + crc */
  cf_t*    dsym[2];
};

/* ---------------------------------------------------------------- small helpers */
static void fft_pow2(double* re, double* im, uint32_t n, int inverse)
{
  for (uint32_t i = 1, j = 0; i < n; i++) {
    uint32_t bit = n >> 1;
    for (; j & bit; bit >>= 1) j ^= bit;
    j ^= bit;
    if (i < j) {
      double t = re[i];
      re[i]    = re[j];
      re[j]    = t;
      t        = im[i];
      im[i]    = im[j];
      im[j]    = t;
    }
  }
  for (uint32_t len = 2; len <= n; len <<= 1) {
    double ang = (inverse ? 2.0 : -2.0) * M_PI / len;
    for (uint32_t i = 0; i < n; i += len)
      for (uint32_t j = 0; j < len / 2; j++) {
        double wr = cos(ang * j), wi = sin(ang * j);
        double ur = re[i + j], ui = im[i + j];
        double vr = re[i + j + len / 2] * wr - im[i + j + len / 2] * wi;
        double vi = re[i + j + len / 2] * wi + im[i + j + len / 2] * wr;
        re[i + j] = ur + vr, im[i + j] = ui + vi;
        re[i + j + len / 2] = ur - vr, im[i + j + len / 2] = ui - vi;
      }
  }
}

/* n = 2^k or 3 * 2^k (srsRAN's default sampling rates): one radix-3 decimation-in-time step around three power-of-two transforms */
static void fft_inplace(double* re, double* im, uint32_t n, int inverse)
{
  if (n % 3) {
    fft_pow2(re, im, n, inverse);
    return;
  }
  const uint32_t m = n / 3;
  double*        t = (double*)malloc(sizeof(double) * 2 * n);
  for (uint32_t r = 0; r < 3; r++)
    for (uint32_t i = 0; i < m; i++) t[r * m + i] = re[3 * i + r], t[n + r * m + i] = im[3 * i + r];
  for (uint32_t r = 0; r < 3; r++) fft_pow2(t + r * m, t + n + r * m, m, inverse);
  for (uint32_t k = 0; k < n; k++) {
    double ar = 0.0, ai = 0.0;
    for (uint32_t r = 0; r < 3; r++) {
      const double ang = (inverse ? 2.0 : -2.0) * M_PI * (double)((uint64_t)r * k % n) / (double)n, wr = cos(ang), wi = sin(ang);
      const double fr = t[r * m + k % m], fi = t[n + r * m + k % m];
      ar += fr * wr - fi * wi, ai += fr * wi + fi * wr;
    }
    re[k] = ar, im[k] = ai;
  }
  free(t);
}

void lte_sim_pdcch_encode(const uint8_t* dci_bits, uint32_t nbits, uint16_t rnti, uint32_t L, uint8_t* e)
{
  uint8_t  c[LTE_DCI_MAX_BITS + 16], d[3 * (LTE_DCI_MAX_BITS + 16)];
  uint32_t crc = lte_crc(LTE_CRC16, 16, dci_bits, nbits) ^ rnti;
  memcpy(c, dci_bits, nbits);
  for (uint32_t i = 0; i < 16; i++) c[nbits + i] = (crc >> (15 - i)) & 1;
  lte_conv_encode(c, nbits + 16, d);
  lte_rm_conv_tx(d, nbits + 16, e, 72u << L);
}

int lte_sim_dlsch_encode(const uint8_t* payload, uint32_t tbs, uint32_t rv, uint32_t G, uint32_t Qm, uint32_t NL, uint8_t* e)
{
  lte_cbsegm_t s;
  if (lte_cbsegm(&s, tbs)) return -1;
  uint8_t* tb = (uint8_t*)malloc(tbs + 24);
  lte_bits_unpack(payload, tbs, tb);
  uint32_t crc = lte_crc(LTE_CRC24A, 24, tb, tbs);
  for (uint32_t i = 0; i < 24; i++) tb[tbs + i] = (crc >> (23 - i)) & 1;
  static __thread uint8_t cb[6144], d[3 * 6148];
  uint32_t                rp = 0, wp = 0;
  for (uint32_t r = 0; r < s.C; r++) {
    uint32_t K = lte_cb_K(&s, r), F = (r == 0) ? s.F : 0;
    uint32_t nd = K - F - (s.C > 1 ? 24 : 0);
    memset(cb, 0, F);
    memcpy(cb + F, tb + rp, nd);
    rp += nd;
    if (s.C > 1) {
      uint32_t c2 = lte_crc(LTE_CRC24B, 24, cb, K - 24);
      for (uint32_t i = 0; i < 24; i++) cb[K - 24 + i] = (c2 >> (23 - i)) & 1;
    }
    lte_turbo_encode(cb, K, d, d + (K + 4), d + 2 * (K + 4));
    uint32_t E = lte_rm_turbo_E(G, s.C, r, Qm, NL);
    lte_rm_turbo_tx(d, K, F, rv, e + wp, E);
    wp += E;
  }
  free(tb);
  return wp == G ? 0 : -2;
}

/* ---------------------------------------------------------------- create / destroy */
lte_sim_t* lte_sim_create(const lte_sim_cfg_t* cfg)
{
  lte_sim_t* s = (lte_sim_t*)calloc(1, sizeof(*s));
  s->cfg       = *cfg;
  if (lte_regs_init(&s->regs, &cfg->cell)) {
    free(s);
    return NULL;
  }
  s->fft    = lte_cell_fft(&cfg->cell);
  s->nsc    = 12 * cfg->cell.nof_prb;
  s->sf_len = 15u * s->fft;
  lte_rng_t rng;
  lte_rng_seed(&rng, cfg->seed ^ 0xC0FFEEull);
  s->rntis = (uint16_t*)calloc(cfg->nof_ues ? cfg->nof_ues : 1, sizeof(uint16_t));
  for (uint32_t i = 0; i < cfg->nof_ues; i++) {
    for (;;) {
      uint16_t r = (uint16_t)(0x0100 + lte_rng_u64(&rng) % (0xFFF3 - 0x0100));
      int      dup = 0;
      for (uint32_t j = 0; j < i; j++) dup |= (s->rntis[j] == r);
      if (!dup) {
        s->rntis[i] = r;
        break;
      }
    }
  }
  for (uint32_t a = 0; a < LTE_MAX_ANT; a++)
    for (uint32_t p = 0; p < LTE_MAX_PORTS; p++) {
      double mag = (a == p) ? 1.0 : 0.35, ph = 2.0 * M_PI * lte_rng_uniform(&rng);
      s->h_re[a][p]  = (float)(mag * cos(ph));
      s->h_im[a][p]  = (float)(mag * sin(ph));
      s->delay[a][p] = cfg->chan_delay ? (uint32_t)(lte_rng_u64(&rng) % (cfg->chan_delay + 1)) : 0;
    }
  for (uint32_t p = 0; p < LTE_MAX_PORTS; p++) {
    s->grid[p] = (cf_t*)calloc(14 * s->nsc, sizeof(cf_t));
    s->td[p]   = (cf_t*)calloc(s->sf_len, sizeof(cf_t));
  }
  s->fre    = (double*)calloc(s->fft, sizeof(double));
  s->fim    = (double*)calloc(s->fft, sizeof(double));
  s->ebits  = (uint8_t*)calloc(110 * 12 * 14 * 8 + 64, 1);
  s->tbbits = (uint8_t*)calloc(110 * 12 * 14 * 8 + 64, 1);
  for (int q = 0; q < 2; q++) s->dsym[q] = (cf_t*)calloc(110 * 12 * 14, sizeof(cf_t));
  return s;
}
void lte_sim_destroy(lte_sim_t* s)
{
  if (!s) return;
  for (uint32_t p = 0; p < LTE_MAX_PORTS; p++) {
    free(s->grid[p]);
    free(s->td[p]);
  }
  free(s->fre), free(s->fim), free(s->ebits), free(s->tbbits), free(s->dsym[0]), free(s->dsym[1]), free(s->rntis);
  free(s);
}
uint32_t lte_sim_rntis(lte_sim_t* s, uint16_t* out, uint32_t max)
{
  uint32_t n = s->cfg.nof_ues < max ? s->cfg.nof_ues : max;
  memcpy(out, s->rntis, n * sizeof(uint16_t));
  return n;
}

/* place symbol(s) of a 2-port SFBC pair or a single-port symbol into the grids */
static void put_txdiv(lte_sim_t* s, uint32_t l0, uint32_t k0, uint32_t l1, uint32_t k1, cf_t x0, cf_t x1)
{
  const float a = (float)M_SQRT1_2;
  cf_t *      g0 = s->grid[0], *g1 = s->grid[1];
  g0[l0 * s->nsc + k0] = (cf_t){x0.re * a, x0.im * a};
  g1[l0 * s->nsc + k0] = (cf_t){-x1.re * a, x1.im * a}; /* -conj(x1) */
  g0[l1 * s->nsc + k1] = (cf_t){x1.re * a, x1.im * a};
  g1[l1 * s->nsc + k1] = (cf_t){x0.re * a, -x0.im * a}; /* conj(x0) */
}

/* map a block of QPSK/QAM symbols d[0..n) to a list of REs with the cell's control-channel scheme */
static void map_ctrl(lte_sim_t* s, const cf_t* d, const uint16_t* ks, const uint8_t* ls, uint32_t n)
{
  if (s->cfg.cell.nof_ports == 1) {
    for (uint32_t i = 0; i < n; i++) s->grid[0][ls[i] * s->nsc + ks[i]] = d[i];
  } else {
    for (uint32_t i = 0; i + 1 < n; i += 2) put_txdiv(s, ls[i], ks[i], ls[i + 1], ks[i + 1], d[i], d[i + 1]);
  }
}

static int cce_free(const uint8_t* used, uint32_t ncce, uint32_t L)
{
  for (uint32_t i = ncce; i < ncce + (1u << L); i++)
    if (used[i]) return 0;
  return 1;
}

/* ---------------------------------------------------------------- one subframe */
int lte_sim_subframe(lte_sim_t* s, uint32_t tti, cf_t* iq, lte_sim_truth_t* truth, uint8_t* payload, uint32_t payload_cap)
{
  const lte_sim_cfg_t* cfg  = &s->cfg;
  const lte_cell_t*    cell = &cfg->cell;
  uint32_t             sf_idx = tti % 10, cfi = cfg->cfi, nsc = s->nsc, N = cell->nof_prb;
  lte_rng_t            rng;
  const int retx = cfg->harq_retx && ((tti / 8) & 1); /* scheduling and payload of tti - 8, sent again with rv 2 */
  lte_rng_seed(&rng, cfg->seed * 0x9E3779B97F4A7C15ull + (retx ? tti - 8 : tti));
  memset(truth, 0, sizeof(*truth));
  truth->tti = tti;
  truth->cfi = cfi;
  for (uint32_t p = 0; p < LTE_MAX_PORTS; p++) memset(s->grid[p], 0, 14 * nsc * sizeof(cf_t));

  /* ---- CRS ---- */
  cf_t pil[2 * LTE_MAX_PRB];
  for (uint32_t p = 0; p < cell->nof_ports; p++)
    for (uint32_t sl = 0; sl < 2; sl++)
      for (uint32_t li = 0; li < 2; li++) {
        uint32_t l = li ? 4 : 0, off = lte_crs(cell, p, 2 * sf_idx + sl, l, pil);
        for (uint32_t m = 0; m < 2 * N; m++) s->grid[p][(7 * sl + l) * nsc + 6 * m + off] = pil[m];
      }

  /* ---- PCFICH ---- */
  {
    uint8_t  sc[32], b[32];
    cf_t     d[16];
    uint16_t ks[16];
    uint8_t  ls[16];
    lte_gold_bits((sf_idx + 1) * (2 * cell->cell_id + 1) * 512u + cell->cell_id, sc, 32);
    for (int i = 0; i < 32; i++) b[i] = lte_cfi_codeword[cfi - 1][i] ^ sc[i];
    lte_modulate(b, 16, 2, d);
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) {
        ks[4 * i + j] = s->regs.regs[s->regs.pcfich_reg[i]].k[j];
        ls[4 * i + j] = 0;
      }
    map_ctrl(s, d, ks, ls, 16);
  }

  /* ---- PSS / SSS: the 62 sub-carriers around DC, d[n] on grid index n - 31 + nsc / 2 ---- */
  if (cfg->sync && (sf_idx == 0 || sf_idx == 5)) {
    cf_t  pss[62];
    float sss[62];
    lte_pss(cell->cell_id % 3, pss);
    lte_sss(cell->cell_id / 3, cell->cell_id % 3, sf_idx == 5, sss);
    for (uint32_t n = 0; n < 62; n++) {
      s->grid[0][6 * nsc + n - 31 + nsc / 2] = pss[n];
      s->grid[0][5 * nsc + n - 31 + nsc / 2] = (cf_t){sss[n], 0.0f};
    }
  }

  /* ---- PBCH ---- */
  if (cfg->pbch && sf_idx == 0) {
    const uint32_t sfn = (tti / 10) % 1024;
    uint8_t        c40[40], d120[120], *e = (uint8_t*)malloc(1920), *sc = (uint8_t*)malloc(1920);
    cf_t*          dq = (cf_t*)malloc(sizeof(cf_t) * 960);
    lte_mib_pack(N, cell->phich_ext, cell->phich_ng, sfn, c40); /* the PHICH configuration this cell's control region is mapped with */
    const uint32_t crc = lte_crc(LTE_CRC16, 16, c40, 24) ^ lte_pbch_crc_mask(cell->nof_ports);
    for (int i = 0; i < 16; i++) c40[24 + i] = (crc >> (15 - i)) & 1;
    lte_conv_encode(c40, 40, d120);
    lte_rm_conv_tx(d120, 40, e, 1920);
    lte_gold_bits(cell->cell_id, sc, 1920);
    for (uint32_t i = 0; i < 1920; i++) e[i] ^= sc[i];
    lte_modulate(e, 960, 2, dq);
    uint16_t ks[240];
    uint8_t  ls[240];
    const uint32_t nre = lte_pbch_re(cell, ks, ls);
    map_ctrl(s, dq + 240 * (sfn % 4), ks, ls, nre);
    free(e), free(sc), free(dq);
  }

  /* ---- scheduling ---- */
  uint32_t nof_cce = s->regs.nof_cce[cfi - 1];
  uint32_t search_cce = nof_cce; /* place DCIs anywhere legal; FALCON only searches the first 84 (falcon_pdcch.h:36) */
  uint8_t  used[LTE_MAX_CCE + 8];
  memset(used, 0, sizeof(used));
  uint8_t* cce_bits = (uint8_t*)malloc(nof_cce * 72);
  memset(cce_bits, 2, nof_cce * 72); /* 2 = <NIL> */
  uint32_t P = N <= 10 ? 1 : N <= 26 ? 2 : N <= 63 ? 3 : 4, nrbg = (N + P - 1) / P;
  uint32_t rbg_next = 0, pl_off = 0;

  typedef struct {
    lte_dci_t dci;
    int       is_dl;
  } job_t;
  job_t    jobs[LTE_SIM_MAX_DCI];
  uint32_t njobs = 0;

  if (cfg->si_period && (tti % cfg->si_period) == 0) {
    job_t* j       = &jobs[njobs++];
    memset(j, 0, sizeof(*j));
    j->is_dl       = 1;
    j->dci.rnti    = LTE_SIRNTI;
    j->dci.format  = LTE_DCI_FORMAT1A;
    j->dci.alloc_type = 2;
    uint32_t L = P, S = 0; /* first RBG */
    j->dci.riv     = N * (L - 1) + S;
    j->dci.mcs[0]  = 5;
    j->dci.n_prb1a = 3;
    j->dci.tb_en[0] = 1;
    rbg_next       = 1;
  }
  uint32_t n_dl = cfg->dl_min + (cfg->dl_max > cfg->dl_min ? (uint32_t)(lte_rng_u64(&rng) % (cfg->dl_max - cfg->dl_min + 1)) : 0);
  uint32_t n_ul = cfg->ul_min + (cfg->ul_max > cfg->ul_min ? (uint32_t)(lte_rng_u64(&rng) % (cfg->ul_max - cfg->ul_min + 1)) : 0);
  if (cfg->nof_ues == 0) n_dl = n_ul = 0;
  if (n_dl > cfg->nof_ues) n_dl = cfg->nof_ues;
  if (n_dl > nrbg - rbg_next) n_dl = nrbg - rbg_next;
  /* RBG partition */
  uint32_t chunk[LTE_SIM_MAX_DCI];
  {
    uint32_t avail = nrbg - rbg_next;
    for (uint32_t i = 0; i < n_dl; i++) chunk[i] = 1;
    uint32_t rest = avail - n_dl;
    if (cfg->full_band) {
      for (uint32_t i = 0; i < rest; i++) chunk[lte_rng_u64(&rng) % n_dl]++;
    } else {
      for (uint32_t i = 0; i < n_dl && rest; i++) {
        uint32_t e = (uint32_t)(lte_rng_u64(&rng) % 3);
        if (e > rest) e = rest;
        chunk[i] += e;
        rest -= e;
      }
    }
  }
  uint32_t ue0 = (uint32_t)(((uint64_t)tti * (cfg->dl_max ? cfg->dl_max : 1)) % (cfg->nof_ues ? cfg->nof_ues : 1));
  for (uint32_t i = 0; i < n_dl && njobs < LTE_SIM_MAX_DCI; i++) {
    job_t* j = &jobs[njobs++];
    memset(j, 0, sizeof(*j));
    j->is_dl       = 1;
    lte_dci_t* d   = &j->dci;
    d->rnti        = s->rntis[(ue0 + i) % cfg->nof_ues];
    uint32_t kind  = cfg->tm;
    if (cfg->tm == 13) {
      uint32_t r = (uint32_t)(lte_rng_u64(&rng) % 4);
      kind       = r == 0 ? 1 : r == 1 ? 101 : r == 2 ? 3 : 103;
      if (cell->nof_ports == 1 && kind != 101) kind = 1;
    }
    if (cfg->tm == 4) { /* closed-loop spatial multiplexing (DCI format 2): 2 codewords, or 1 codeword on 1 layer */
      uint32_t r = (uint32_t)(lte_rng_u64(&rng) % 3);
      kind       = r == 0 ? 104 : 4;
    }
    if ((kind == 3 || kind == 4 || kind == 104) && cell->nof_ports != 2) kind = 1;
    if (kind == 4 && cell->nof_rx != 2) kind = 104;
    uint32_t rb0 = rbg_next, nr = chunk[i];
    rbg_next += nr;
    if (kind == 101) { /* 1A localized */
      d->format     = LTE_DCI_FORMAT1A;
      d->alloc_type = 2;
      uint32_t S = rb0 * P, L = nr * P;
      if (S + L > N) L = N - S;
      d->riv = (L - 1 <= N / 2) ? N * (L - 1) + S : N * (N - L + 1) + (N - 1 - S);
    } else {
      d->format     = (kind == 1) ? LTE_DCI_FORMAT1 : (kind == 4 || kind == 104) ? LTE_DCI_FORMAT2 : LTE_DCI_FORMAT2A;
      if (kind == 4) d->pinfo = (uint8_t)(lte_rng_u64(&rng) % 2);
      if (kind == 104) d->pinfo = (uint8_t)(1 + lte_rng_u64(&rng) % 4);
      d->alloc_type = 0;
      for (uint32_t r = rb0; r < rb0 + nr; r++) d->rbg_bitmask |= 1u << (nrbg - 1 - r);
    }
    d->pid = (uint8_t)(lte_rng_u64(&rng) % 8);
    if (cfg->harq_retx) d->pid = (uint8_t)(tti % 8); /* one process per subframe of the 8 ms round trip, as an FDD eNB schedules them */
    d->tpc = 1;
    for (int t = 0; t < 2; t++) {
      d->mcs[t] = (uint8_t)(cfg->mcs_min + lte_rng_u64(&rng) % (cfg->mcs_max - cfg->mcs_min + 1));
      d->ndi[t] = (uint8_t)(lte_rng_u64(&rng) & 1);
      d->rv[t]  = retx ? 2 : 0;
    }
    d->tb_en[0] = 1;
    d->tb_en[1] = (kind == 3 || kind == 4);
    if (cfg->tb_swap && d->tb_en[1]) d->tb_cw_swap = (uint8_t)(lte_rng_u64(&rng) & 1);
    if (kind == 101 && d->mcs[0] > 28) d->mcs[0] = 28;
  }
  uint32_t ul_next = 0;
  for (uint32_t i = 0; i < n_ul && njobs < LTE_SIM_MAX_DCI; i++) {
    job_t* j = &jobs[njobs++];
    memset(j, 0, sizeof(*j));
    lte_dci_t* d  = &j->dci;
    d->rnti       = s->rntis[(ue0 + n_dl + i) % cfg->nof_ues];
    d->format     = LTE_DCI_FORMAT0;
    d->alloc_type = 2;
    uint32_t L = 1 + (uint32_t)(lte_rng_u64(&rng) % 8), S = (uint32_t)(lte_rng_u64(&rng) % (N - L));
    if (cfg->ul_pusch) {
      static const uint8_t okL[8] = {3, 4, 5, 6, 8, 9, 10, 12};
      L = okL[lte_rng_u64(&rng) % 8];
      S = ul_next;
      if (S + L > N) {
        njobs--;
        break;
      }
      ul_next += L;
    }
    d->riv        = N * (L - 1) + S;
    d->mcs[0]     = cfg->ul_pusch ? (uint8_t)(2 + lte_rng_u64(&rng) % 19) : (uint8_t)(10 + lte_rng_u64(&rng) % 15);
    d->ndi[0]     = (uint8_t)(lte_rng_u64(&rng) & 1);
    d->tpc        = 1;
    d->n_dmrs     = (uint8_t)(lte_rng_u64(&rng) % 8);
  }

  /* ---- encode every job: PDCCH + PDSCH ---- */
  for (uint32_t ji = 0; ji < njobs; ji++) {
    lte_dci_t* d = &jobs[ji].dci;
    uint8_t    bits[LTE_DCI_MAX_BITS];
    uint32_t   nbits = 0;
    if (lte_dci_pack(cell, d, bits, &nbits)) continue;
    /* choose a PDCCH location */
    uint16_t nc[22];
    uint8_t  Lv[22];
    uint32_t ncand;
    if (LTE_RNTI_ISUSER(d->rnti))
      ncand = lte_pdcch_ue_locations(search_cce, sf_idx, d->rnti, nc, Lv, 22);
    else
      ncand = lte_pdcch_common_locations(search_cce, nc, Lv, 22);
    uint32_t minL = (nbits + 16 <= 48) ? 0 : 1;
    uint32_t wantL;
    if (cfg->fixed_L != 0xFF)
      wantL = cfg->fixed_L;
    else {
      uint32_t r = (uint32_t)(lte_rng_u64(&rng) % 100);
      wantL      = r < 20 ? 0 : r < 55 ? 1 : r < 85 ? 2 : 3;
    }
    if (wantL < minL) wantL = minL;
    if (!LTE_RNTI_ISUSER(d->rnti) && wantL < 2) wantL = 2;
    int      chosen = -1;
    for (uint32_t dl = 0; dl < 4 && chosen < 0; dl++) {
      uint32_t tryL = (wantL + dl) % 4;
      if (tryL < minL) continue;
      for (uint32_t c = 0; c < ncand; c++)
        if (Lv[c] == tryL && nc[c] + (1u << tryL) <= search_cce && cce_free(used, nc[c], tryL)) {
          chosen = (int)c;
          break;
        }
    }
    if (chosen < 0) continue; /* blocked: UE not scheduled this subframe */
    uint32_t ncce = nc[chosen], L = Lv[chosen];
    lte_dl_grant_t g;
    memset(&g, 0, sizeof(g));
    if (jobs[ji].is_dl) {
      if (lte_dl_dci_to_grant(cell, sf_idx, cfi, (int)cfg->alt_table, d, &g)) continue;
      int ok = 1;
      for (int t = 0; t < 2; t++)
        if (g.tb[t].enabled && g.tb[t].tbs <= 0) ok = 0;
      for (int t = 0; t < 2; t++) /* keep the code rate decodable: drop MCS until rate <= 0.93 */
        while (g.tb[t].enabled && g.tb[t].tbs > 0 && (double)(g.tb[t].tbs + 24) > 0.93 * g.tb[t].nof_bits && d->mcs[t] > 0) {
          d->mcs[t]--;
          lte_dl_dci_to_grant(cell, sf_idx, cfi, (int)cfg->alt_table, d, &g);
        }
      if (!ok) continue;
      lte_dci_pack(cell, d, bits, &nbits);
      uint32_t need = 0;
      for (int t = 0; t < 2; t++)
        if (g.tb[t].enabled) need += (uint32_t)g.tb[t].tbs / 8;
      if (pl_off + need > payload_cap) continue;
    }
    for (uint32_t i = ncce; i < ncce + (1u << L); i++) used[i] = 1;
    lte_sim_pdcch_encode(bits, nbits, d->rnti, L, &cce_bits[72 * ncce]);

    lte_sim_dci_truth_t* tr = &truth->dci[truth->nof_dci++];
    tr->rnti                = d->rnti;
    tr->format              = d->format;
    tr->L                   = (uint8_t)L;
    tr->ncce                = (uint16_t)ncce;
    tr->nbits               = (uint16_t)nbits;
    memcpy(tr->bits, bits, nbits);
    if (!jobs[ji].is_dl) continue;
    tr->nof_tb    = (uint8_t)g.nof_tb;
    tr->tx_scheme = g.tx_scheme;
    tr->nof_prb   = g.nof_prb;
    tr->nof_re    = g.nof_re;

    /* ---- PDSCH ---- */
    uint32_t ncw = 0;
    for (int t = 0; t < 2; t++) {
      if (!g.tb[t].enabled) continue;
      uint32_t tbs = (uint32_t)g.tb[t].tbs, G = g.tb[t].nof_bits, Qm = g.tb[t].qm;
      tr->tbs[t]   = (int32_t)tbs;
      tr->qm[t]    = (uint8_t)Qm;
      tr->rv[t]    = g.tb[t].rv;
      tr->mcs[t]   = d->mcs[t];
      tr->payload_off[t] = pl_off;
      uint8_t* pl  = payload + pl_off;
      for (uint32_t i = 0; i < tbs / 8; i++) pl[i] = (uint8_t)lte_rng_u64(&rng);
      pl_off += tbs / 8;
      uint32_t NL = (g.tx_scheme == LTE_TX_DIVERSITY) ? 2 : 1;
      if (lte_sim_dlsch_encode(pl, tbs, g.tb[t].rv, G, Qm, NL, s->ebits)) {
        free(cce_bits);
        return -10;
      }
      uint8_t* sc = s->tbbits;
      uint32_t q  = g.cw_swap ? 1 - ncw : ncw; /* codeword index (36.212 Table 5.3.3.1.5-1) */
      lte_gold_bits(((uint32_t)d->rnti << 14) + (q << 13) + (sf_idx << 9) + cell->cell_id, sc, G);
      for (uint32_t i = 0; i < G; i++) s->ebits[i] ^= sc[i];
      lte_modulate(s->ebits, G / Qm, Qm, s->dsym[q]);
      ncw++;
    }
    /* layer mapping + precoding + RE mapping */
    uint16_t kk[12];
    uint32_t isym = 0, pair_l = 0, pair_k = 0;
    for (uint32_t l = 0; l < 14; l++)
      for (uint32_t prb = 0; prb < N; prb++) {
        if (!g.prb_mask[l / 7][prb]) continue;
        uint32_t n = lte_pdsch_re_in_prb(cell, sf_idx, cfi, l, prb, kk);
        for (uint32_t i = 0; i < n; i++, isym++) {
          uint32_t k = kk[i];
          if (g.tx_scheme == LTE_TX_PORT0) {
            s->grid[0][l * nsc + k] = s->dsym[0][isym];
          } else if (g.tx_scheme == LTE_TX_DIVERSITY) {
            /* nof_re is even; SFBC pairs are consecutive REs of the mapping order */
            if ((isym & 1) == 0) {
              pair_l = l;
              pair_k = k;
            } else
              put_txdiv(s, pair_l, pair_k, l, k, s->dsym[0][isym - 1], s->dsym[0][isym]);
          } else if (g.tx_scheme == LTE_TX_SPATIALMUX) { /* codebook precoding, 36.211 Table 6.3.4.2.3-1, 2 ports */
            static const float W1[4][2] = {{1, 0}, {-1, 0}, {0, 1}, {0, -1}};
            if (g.nof_layers == 1) {
              cf_t        x = s->dsym[0][isym];
              const float a = (float)M_SQRT1_2, wr = W1[g.pmi & 3][0], wi = W1[g.pmi & 3][1];
              s->grid[0][l * nsc + k] = (cf_t){a * x.re, a * x.im};
              s->grid[1][l * nsc + k] = (cf_t){a * (wr * x.re - wi * x.im), a * (wr * x.im + wi * x.re)};
            } else {
              cf_t        x0 = s->dsym[0][isym], x1 = s->dsym[1][isym];
              const float wr = (g.pmi & 1) ? 0.0f : 1.0f, wi = (g.pmi & 1) ? 1.0f : 0.0f;
              cf_t        dd = {x0.re - x1.re, x0.im - x1.im};
              s->grid[0][l * nsc + k] = (cf_t){0.5f * (x0.re + x1.re), 0.5f * (x0.im + x1.im)};
              s->grid[1][l * nsc + k] = (cf_t){0.5f * (wr * dd.re - wi * dd.im), 0.5f * (wr * dd.im + wi * dd.re)};
            }
          } else { /* large-delay CDD, 2 layers, 2 ports: y = W D(i) U x */
            cf_t  x0 = s->dsym[0][isym], x1 = s->dsym[1][isym];
            float sg = (isym & 1) ? -1.0f : 1.0f;
            s->grid[0][l * nsc + k] = (cf_t){0.5f * (x0.re + x1.re), 0.5f * (x0.im + x1.im)};
            s->grid[1][l * nsc + k] = (cf_t){sg * 0.5f * (x0.re - x1.re), sg * 0.5f * (x0.im - x1.im)};
          }
        }
      }
  }
  truth->payload_len = pl_off;

  /* ---- PDCCH: scramble, modulate, interleave, map ---- */
  {
    uint32_t nbits = nof_cce * 72, nq = nof_cce * 9;
    uint8_t* sc    = (uint8_t*)malloc(nbits);
    lte_gold_bits((sf_idx << 9) + cell->cell_id, sc, nbits);
    for (uint32_t q = 0; q < nq; q++) {
      const uint8_t* b = &cce_bits[8 * q];
      if (b[0] == 2) continue; /* NIL quadruplet */
      uint8_t  bb[8];
      cf_t     d[4];
      uint16_t ks[4];
      uint8_t  ls[4];
      for (int i = 0; i < 8; i++) bb[i] = b[i] ^ sc[8 * q + i];
      lte_modulate(bb, 4, 2, d);
      const lte_reg_t* rg = &s->regs.regs[s->regs.pdcch_map[cfi - 1][q]];
      for (int i = 0; i < 4; i++) {
        ks[i] = rg->k[i];
        ls[i] = rg->l;
      }
      map_ctrl(s, d, ks, ls, 4);
    }
    free(sc);
  }
  free(cce_bits);

  /* ---- OFDM modulation per port ---- */
  double sc = 1.0 / sqrt((double)s->fft);
  for (uint32_t p = 0; p < cell->nof_ports; p++) {
    uint32_t pos = 0;
    for (uint32_t l = 0; l < 14; l++) {
      memset(s->fre, 0, s->fft * sizeof(double));
      memset(s->fim, 0, s->fft * sizeof(double));
      for (uint32_t k = 0; k < nsc; k++) {
        uint32_t bin = (k < nsc / 2) ? s->fft - nsc / 2 + k : k - nsc / 2 + 1;
        s->fre[bin]  = s->grid[p][l * nsc + k].re;
        s->fim[bin]  = s->grid[p][l * nsc + k].im;
      }
      fft_inplace(s->fre, s->fim, s->fft, 1);
      uint32_t cp = lte_cp_len(s->fft, l % 7);
      for (uint32_t n = 0; n < cp; n++) s->td[p][pos + n] = (cf_t){(float)(s->fre[s->fft - cp + n] * sc), (float)(s->fim[s->fft - cp + n] * sc)};
      for (uint32_t n = 0; n < s->fft; n++) s->td[p][pos + cp + n] = (cf_t){(float)(s->fre[n] * sc), (float)(s->fim[n] * sc)};
      pos += cp + s->fft;
    }
  }
  /* ---- channel + AWGN ---- */
  const double cfo_w = 2.0 * M_PI * (double)cfg->cfo_hz / (15000.0 * (double)s->fft); /* radians per sample */
  if (cfg->harq_retx) lte_rng_seed(&rng, cfg->seed * 0x2545F4914F6CDD1Dull + 31ull * tti + 7); /* a retransmission meets its own noise */
  double sigma = pow(10.0, -cfg->snr_db / 20.0) * M_SQRT1_2;
  for (uint32_t a = 0; a < cell->nof_rx; a++) {
    cf_t* out = iq + (size_t)a * s->sf_len;
    for (uint32_t n = 0; n < s->sf_len; n++) {
      double re = sigma * lte_rng_gauss(&rng), im = sigma * lte_rng_gauss(&rng), sr = 0.0, si = 0.0;
      for (uint32_t p = 0; p < cell->nof_ports; p++) {
        uint32_t dl = s->delay[a][p];
        if (n < dl) continue;
        cf_t x = s->td[p][n - dl];
        sr += (double)s->h_re[a][p] * x.re - (double)s->h_im[a][p] * x.im;
        si += (double)s->h_re[a][p] * x.im + (double)s->h_im[a][p] * x.re;
      }
      if (cfo_w != 0.0) { /* receiver's oscillator is off by cfo_hz */
        const double cr = cos(cfo_w * (double)n), ci = sin(cfo_w * (double)n), tr = sr * cr - si * ci;
        si = sr * ci + si * cr, sr = tr;
      }
      out[n] = (cf_t){(float)(re + sr), (float)(im + si)};
    }
  }
  return 0;
}

/* ================================================================== uplink: PUSCH transmitter */
int lte_sim_ul_subframe(lte_sim_t* s, uint32_t tti, const lte_ul_cfg_t* ucfg, const lte_ul_grant_t* grants, uint32_t n, cf_t* iq, uint8_t* payload,
                        uint32_t* payload_off, uint32_t payload_cap)
{
  return lte_sim_ul_subframe_rx(s, tti, ucfg, grants, n, 1, iq, payload, payload_off, payload_cap);
}

int lte_sim_ul_subframe_rx(lte_sim_t* s, uint32_t tti, const lte_ul_cfg_t* ucfg, const lte_ul_grant_t* grants, uint32_t n, uint32_t nof_rx, cf_t* iq,
                           uint8_t* payload, uint32_t* payload_off, uint32_t payload_cap)
{
  if (nof_rx < 1 || nof_rx > LTE_MAX_ANT) return -5;
  const lte_cell_t* cell = &s->cfg.cell;
  const uint32_t    sf_idx = tti % 10, nsc = s->nsc, N = s->fft;
  lte_rng_t         rng;
  lte_rng_seed(&rng, s->cfg.seed * 0x51ED27ull + 977ull * tti + 5);
  cf_t* grid = s->grid[0];
  memset(grid, 0, 14 * nsc * sizeof(cf_t));
  uint32_t pl_off = 0;
  static const uint32_t DATA_SYM[12] = {0, 1, 2, 4, 5, 6, 7, 8, 9, 11, 12, 13};
  for (uint32_t gi = 0; gi < n; gi++) {
    const lte_ul_grant_t* g = &grants[gi];
    const uint32_t        M = 12 * g->L_prb, Qm = g->qm, H = 12 * M;
    const uint32_t        k0s[2] = {12 * g->n_prb, 12 * (g->hop ? g->n_prb_slot1 : g->n_prb)};
    lte_uci_layout_t      L;
    lte_uci_layout(g, &L);
    const uint32_t G = L.G;
    if ((uint32_t)g->tbs / 8 + pl_off > payload_cap) return -1;
    uint8_t* pl = payload + pl_off;
    payload_off[gi] = pl_off;
    for (uint32_t i = 0; i < (uint32_t)g->tbs / 8; i++) pl[i] = (uint8_t)lte_rng_u64(&rng);
    pl_off += (uint32_t)g->tbs / 8;
    uint8_t* e = s->ebits;
    if (lte_sim_dlsch_encode(pl, (uint32_t)g->tbs, g->rv, G, Qm, 1, e)) return -2;
    /* data / control multiplexing and channel interleaver, 36.212 5.2.2.7 / 5.2.2.8: R' x 12 matrix of Qm-bit groups, row-wise in,
     * column-wise out.  Values: 0 / 1 bits, 2 = placeholder x, 3 = placeholder y (36.212 Tables 5.2.2.6-1 / -2) */
    uint8_t*  kind = (uint8_t*)malloc(H);
    uint32_t* dpos = (uint32_t*)malloc(sizeof(uint32_t) * H);
    lte_uci_map(M, &L, kind, dpos);
    uint8_t o_ack[3], o_ri[3];
    for (int i = 0; i < 2; i++) o_ack[i] = (uint8_t)(lte_rng_u64(&rng) & 1), o_ri[i] = (uint8_t)(lte_rng_u64(&rng) & 1);
    o_ack[2] = o_ack[0] ^ o_ack[1], o_ri[2] = o_ri[0] ^ o_ri[1];
    uint8_t* h = s->tbbits;
    uint32_t n_ack = 0, n_ri = 0;
    /* the i-th ACK / RI symbol is counted from the bottom row upwards in column-set order, as lte_uci_map lays them out */
    static const uint32_t RI_COL[4] = {1, 4, 7, 10}, ACK_COL[4] = {2, 3, 8, 9};
    for (uint32_t c = 0; c < 12; c++)
      for (uint32_t r = 0; r < M; r++) {
        uint8_t*       dst = &h[(c * M + r) * Qm];
        const uint32_t p = r * 12 + c, kd = kind[p];
        if (kd == 0)
          memcpy(dst, &e[dpos[p] * Qm], Qm);
        else if (kd == 1)
          for (uint32_t b = 0; b < Qm; b++) dst[b] = (uint8_t)(lte_rng_u64(&rng) & 1); /* CQI codeword bits: content is not examined by the receiver */
        else {
          const int       is_ri = kd == 2;
          const uint32_t* cols = is_ri ? RI_COL : ACK_COL;
          uint32_t        j = 0;
          while (cols[j] != c) j++;
          const uint32_t  t = (3 * j) % 4, i = 4 * (M - 1 - r) + t; /* index of this symbol in the coded ACK / RI sequence */
          const uint32_t  O = is_ri ? g->ri_len : g->nof_ack;
          const uint8_t*  o = is_ri ? o_ri : o_ack;
          for (uint32_t b = 0; b < Qm; b++) dst[b] = 2;
          if (O <= 1)
            dst[0] = o[0], dst[1] = 3;
          else
            dst[0] = o[(2 * i) % 3], dst[1] = o[(2 * i + 1) % 3];
          if (is_ri) n_ri++; else n_ack++;
        }
      }
    if (n_ri != L.Qp_ri || n_ack != L.Qp_ack) return -4;
    free(kind), free(dpos);
    uint8_t* sc = (uint8_t*)malloc(H * Qm);
    lte_gold_bits(((uint32_t)g->rnti << 14) + (sf_idx << 9) + cell->cell_id, sc, H * Qm);
    for (uint32_t i = 0; i < H * Qm; i++) { /* 36.211 5.3.1: x -> 1, y -> the previous scrambled bit */
      if (h[i] == 2)
        h[i] = 1;
      else if (h[i] == 3)
        h[i] = i ? h[i - 1] : 0;
      else
        h[i] ^= sc[i];
    }
    free(sc);
    lte_modulate(h, H, Qm, s->dsym[0]);
    /* transform precoding + mapping (slot 1 at its own PRBs under type-1 hopping); the UE's timing offset is a phase ramp over its sub-carriers */
    double* wr = (double*)malloc(sizeof(double) * M * 2);
    for (uint32_t m = 0; m < M; m++) {
      wr[2 * m]     = cos(2.0 * M_PI * m / M);
      wr[2 * m + 1] = -sin(2.0 * M_PI * m / M);
    }
    double sc_dft = 1.0 / sqrt((double)M);
    for (uint32_t c = 0; c < 12; c++) {
      const cf_t*    d  = &s->dsym[0][c * M];
      const uint32_t k0 = k0s[c / 6];
      for (uint32_t k = 0; k < M; k++) {
        double ar = 0, ai = 0;
        for (uint32_t i = 0; i < M; i++) {
          uint32_t t = (uint32_t)(((uint64_t)i * k) % M);
          ar += d[i].re * wr[2 * t] - d[i].im * wr[2 * t + 1];
          ai += d[i].re * wr[2 * t + 1] + d[i].im * wr[2 * t];
        }
        grid[DATA_SYM[c] * nsc + k0 + k] = (cf_t){(float)(ar * sc_dft), (float)(ai * sc_dft)};
      }
    }
    free(wr);
    cf_t* r = (cf_t*)malloc(sizeof(cf_t) * M);
    for (uint32_t sl = 0; sl < 2; sl++) {
      if (lte_pusch_dmrs(cell, ucfg, 2 * sf_idx + sl, g->n_dmrs2, M, r)) {
        free(r);
        return -3;
      }
      for (uint32_t k = 0; k < M; k++) grid[(7 * sl + 3) * nsc + k0s[sl] + k] = r[k];
    }
    free(r);
    if (g->ta_us != 0.0f)
      for (uint32_t l = 0; l < 14; l++) {
        const uint32_t k0 = k0s[l / 7];
        for (uint32_t k = 0; k < M; k++) {
          const double f  = ((double)(k0 + k) - (double)nsc / 2.0 + 0.5) * 15e3; /* Hz */
          const double ph = -2.0 * M_PI * f * (double)g->ta_us * 1e-6;
          cf_t*        x  = &grid[l * nsc + k0 + k];
          const double xr = x->re * cos(ph) - x->im * sin(ph), xi = x->re * sin(ph) + x->im * cos(ph);
          *x              = (cf_t){(float)xr, (float)xi};
        }
      }
  }
  /* SC-FDMA modulation with the half-subcarrier shift (36.211 5.6) */
  double scl = 1.0 / sqrt((double)N);
  uint32_t pos = 0;
  for (uint32_t l = 0; l < 14; l++) {
    memset(s->fre, 0, N * sizeof(double));
    memset(s->fim, 0, N * sizeof(double));
    for (uint32_t kk = 0; kk < nsc; kk++) {
      uint32_t bin = (kk + N - nsc / 2) % N;
      s->fre[bin]  = grid[l * nsc + kk].re;
      s->fim[bin]  = grid[l * nsc + kk].im;
    }
    fft_inplace(s->fre, s->fim, N, 1);
    uint32_t cp = lte_cp_len(N, l % 7);
    for (int nn = -(int)cp; nn < (int)N; nn++) {
      uint32_t m  = (uint32_t)((nn + (int)N) % (int)N);
      double   ph = M_PI * (double)nn / (double)N;
      double   re = s->fre[m] * cos(ph) - s->fim[m] * sin(ph), im = s->fre[m] * sin(ph) + s->fim[m] * cos(ph);
      s->td[0][pos++] = (cf_t){(float)(re * scl), (float)(im * scl)};
    }
  }
  /* antenna a: port 0's gain and delay towards it, and its own noise, drawn after antenna a - 1's */
  double sigma = pow(10.0, -s->cfg.snr_db / 20.0) * M_SQRT1_2;
  for (uint32_t a = 0; a < nof_rx; a++) {
    const float    hr = s->h_re[a][0], hi = s->h_im[a][0];
    const uint32_t dl = s->delay[a][0];
    cf_t*          out = iq + (size_t)a * s->sf_len;
    for (uint32_t i = 0; i < s->sf_len; i++) {
      double re = sigma * lte_rng_gauss(&rng), im = sigma * lte_rng_gauss(&rng);
      if (i >= dl) {
        cf_t x = s->td[0][i - dl];
        re += (double)hr * x.re - (double)hi * x.im;
        im += (double)hr * x.im + (double)hi * x.re;
      }
      out[i] = (cf_t){(float)re, (float)im};
    }
  }
  return 0;
}
