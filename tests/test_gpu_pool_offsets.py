"""Phase B with pools past 2^32 elements, and phase A at LTEPHY_MAX_BATCH_SUBFRAMES (pytest -m gpu).

Every phase-B pool of a batch is addressed by offsets that the host writes into the device descriptors.  The soft-bit pool (int16), the turbo
pool (uint32 words) and the HARQ store (int16) pass 2^32 elements on an 80 GB card, so an offset that was kept in 32 bits would wrap without a
fault: a later codeword, pair or HARQ slot would land on an earlier one, and transport blocks would come back with another block's soft bits.
Each case below builds a batch whose pool crosses 2^32 and puts real transport blocks on both sides of it:

(a) downlink soft bits: real grant T0, ~18 600 two-codeword 256QAM fillers with tbs = 0 (they take soft bits and scrambling words, no turbo pool),
    real grant T1 whose codeword straddles 2^32 (its grant offset fits 32 bits, its later code blocks' offsets do not), then T2 wholly past it,
    at an offset that is congruent, mod 2^32, to a point inside T0's codeword;
(b) the same through ltephy_submit_ul (~37 300 full-band 256QAM fillers, 115 200 soft bits each);
(c) the turbo pool: 29 200 grants, each one 97 896-bit transport block of 16 code blocks of K = 6144 (8 pairs of 18 448 words), 17.2 GB of pool;
    the grants cycle through 7 different transmitted subframes, so a wrapped pair would overlap a pair of a different transport block;
(d) the HARQ store: ltephy_harq_reserve(14 552), first transmissions into slots 0 and 14 551, then retransmissions at another redundancy version,
    against the same sequence on a store of two slots (0 and 1), including the turbo-decoder input;
(e) phase A at 65 535 subframes (grids with the subframe on gridDim.y / z at their limit): one ltephy_decode_subframes of a 15 PRB capture
    against the same samples in batches of 1 000 on a fresh search, and one ltephy_submit_ul of 65 535 uplink subframes against the two loaded
    subframes alone.

Reference for (a)-(d): the same real grants submitted alone on a fresh handle over the same phase A.  crc, avg_iters, nof_cb, payload_len and the
payload bytes must equal it, and the payload must equal what was sent; a prefix of the soft-bit pool (ltephy_tap copies a prefix, never the whole
multi-GB pool) must equal it over the codeword that a wrapped offset lands on.  Each case first checks that the card has the memory it needs
(computed from its shapes) and skips, printing the bytes, when another user holds it.  tests/test_pool_offsets.py shows from the same layouts,
without a GPU, that 32-bit offsets would make these batches overlap real transport blocks."""
import ctypes as C
import functools
import time

import numpy as np
import pytest

import ltelib
import ref64
import ref64_ul
import ref_dec
import rm_ref
from ltelib import Cell
from test_decoder_reference import crafted_codeword
from test_float64_reference import Case, tbs_of
from test_gpu_batch_limits import CHEST_DT, GRANT_DT, RES_DT, UL_GRANT_DT, _p
from test_gpu_concurrent_pipelines import decode, snapshot
from test_pusch_float64_reference import Subframe, encode, tbs as ul_tbs
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu

WRAP = 1 << 32
GROWTH = 1.25                     # DevBuf::reserve allocates n + n / 4
MARGIN = 2 << 30
NOISE = 1e-4
CFI = 1
UCFG = (0, 0, 0, 0)
FULL = list(range(100))


def cw_len(G):
    """soft bits a codeword of G bits takes in the pool"""
    return (int(G) + 7) & ~7


def nof_re(cell, tti, prbs):
    mask = np.zeros((2, 110), np.uint8)
    mask[:, list(prbs)] = 1
    return len(ref64.pdsch_res(cell, tti % 10, CFI, mask)[0])


def cb_E(tbs, G, qm, NL):
    Cn = ref_dec.segmentation(tbs)[0]
    return [rm_ref.rm_E(G, Cn, r, qm, NL) for r in range(Cn)]


def dl_grant(sf, rnti, scheme, prbs, nre, tbs_qm):
    """GRANT_DT [1]: TB t = tbs_qm[t] = (tbs, qm) on codeword t"""
    g = np.zeros(1, GRANT_DT)
    g["sf"], g["rnti"], g["tx_scheme"], g["nof_tb"], g["nof_re"] = sf, rnti, scheme, len(tbs_qm), nre
    for p in prbs:
        g["prb_mask"][0, :, p >> 5] |= np.uint32(1 << (p & 31))
    for t, (tbs, qm) in enumerate(tbs_qm):
        g["tb"]["tbs"][0, t], g["tb"]["qm"][0, t], g["tb"]["enabled"][0, t], g["tb"]["cw_idx"][0, t] = tbs, qm, 1, t
    return g


def ul_grant(sf, rnti, L, qm, tbs):
    """UL_GRANT_DT [1], allocation from PRB 0"""
    g = np.zeros(1, UL_GRANT_DT)
    g["sf"], g["rnti"], g["qm"], g["L_prb"], g["n_prb"], g["tbs"] = sf, rnti, qm, L, 0, tbs
    return g


def fill_to(pos, lo, hi, big, small):
    """numbers of big and small fillers that take a pool position pos to a point in [lo, hi]"""
    nb = (hi - pos) // big
    ns = (hi - pos - nb * big) // small
    end = pos + nb * big + ns * small
    assert lo <= end <= hi, (lo, end, hi)
    return nb, ns


def repeat(rec, n, rnti0):
    out = np.repeat(rec, n)
    out["rnti"] = rnti0 + np.arange(n) % 3000
    return out


# ------------------------------------------------------------------------------------------------------------------------------------ layouts
# The batches as grant lists and pool offsets, computed from the shapes alone (no IQ): shared with the CPU test.
DL_CELL = Cell(100, 2, 7, 2)
A_TTI = (1, 2, 3)
A_QM, A_ITBS = 4, 12


@functools.lru_cache(None)
def a_layout():
    """-> (grants, indices of T0 / T1 / T2, soft-bit offset of every grant's first codeword, G of the real codeword, its E per code block)"""
    cell = DL_CELL
    nre = nof_re(cell, A_TTI[0], tuple(FULL))
    assert all(nof_re(cell, t, tuple(FULL)) == nre for t in A_TTI)
    G, tbs = nre * A_QM, tbs_of(A_ITBS, 100)
    E = cb_E(tbs, G, A_QM, 2)
    big = dl_grant(0, 0, capi.TX_CDD, FULL, nre, [(0, 8), (0, 8)])           # 2 x 256QAM codewords, no transport block
    small_prbs = tuple(range(25))
    small = dl_grant(0, 0, capi.TX_PORT0, small_prbs, nof_re(cell, A_TTI[0], small_prbs), [(0, 2)])
    lb, ls, lt = 2 * cw_len(nre * 8), cw_len(small["nof_re"][0] * 2), cw_len(G)
    # T1 starts below 2^32 with its first code block, and its last code block starts past it
    nb, ns = fill_to(lt, WRAP - sum(E[:-1]), WRAP - E[0], lb, ls)
    real = [dl_grant(i, 0x4001 + i, capi.TX_DIVERSITY, FULL, nre, [(tbs, A_QM)]) for i in range(3)]
    grants = np.concatenate(real[:1] + [repeat(big, nb, 0x100), repeat(small, ns, 0x100)] + real[1:])
    lens = np.array([lt] + [lb] * nb + [ls] * ns + [lt, lt], np.int64)
    off = np.cumsum(lens) - lens
    idx = [0, 1 + nb + ns, 2 + nb + ns]
    return grants, idx, off, G, E


UL_CELL = Cell(100, 1, 7, 1)
B_TTI = (1, 2, 3)
B_QM = 4


@functools.lru_cache(None)
def b_layout():
    L = 100
    tbs = ul_tbs(L, B_QM)
    G = 12 * 12 * L * B_QM
    E = cb_E(tbs, G, B_QM, 1)
    big, small = ul_grant(0, 0, 100, 8, ul_tbs(100, 8, 0)), ul_grant(0, 0, 25, 2, ul_tbs(25, 2, 0))
    lb, ls, lt = cw_len(12 * 1200 * 8), cw_len(12 * 300 * 2), cw_len(G)
    nb, ns = fill_to(lt, WRAP - sum(E[:-1]), WRAP - E[0], lb, ls)
    real = [ul_grant(i, 0x5001 + i, L, B_QM, tbs) for i in range(3)]
    grants = np.concatenate(real[:1] + [repeat(big, nb, 0x100), repeat(small, ns, 0x100)] + real[1:])
    lens = np.array([lt] + [lb] * nb + [ls] * ns + [lt, lt], np.int64)
    off = np.cumsum(lens) - lens
    return grants, [0, 1 + nb + ns, 2 + nb + ns], off, G, E


TB_CELL = Cell(100, 1, 1, 1)
C_TTI = (1, 2, 3, 4, 6, 7, 8)        # no PSS / SSS / PBCH: every subframe has the same G
C_TBS, C_QM, C_GRANTS = 97896, 8, 29200


@functools.lru_cache(None)
def c_layout():
    """-> (grants, G): grant i carries the transport block of subframe i mod 7"""
    nre = nof_re(TB_CELL, C_TTI[0], tuple(FULL))
    assert all(nof_re(TB_CELL, t, tuple(FULL)) == nre for t in C_TTI)
    real = [dl_grant(s, 0x6001 + s, capi.TX_PORT0, FULL, nre, [(C_TBS, C_QM)]) for s in range(len(C_TTI))]
    grants = np.concatenate(real)[np.arange(C_GRANTS) % len(C_TTI)]
    return grants, nre * C_QM


D_TTI = (1, 2, 3, 4)                 # X rv 0, Y rv 0, X rv 2, Y rv 2
D_QM, D_SLOTS = 2, 14552


@functools.lru_cache(None)
def d_tbs():
    """a transport block of about 1.05 G: one transmission alone cannot pass its CRC, two redundancy versions together have rate ~0.53"""
    G = nof_re(TB_CELL, D_TTI[0], tuple(FULL)) * D_QM
    S = ltelib.sim()
    cands = sorted({int(S.lte_tbs_from_idx(i, n)) for i in range(27) for n in range(1, 111)})
    return G, min(cands, key=lambda t: abs(t - 1.05 * G))


def d_grants(sy):
    """(batch 1, batch 2) with X in HARQ slot 0 and Y in slot sy; batch 2 also decodes both retransmissions alone (no HARQ)"""
    G, tbs = d_tbs()
    nre = G // D_QM

    def g(sf, rnti, rv, op, slot):
        r = dl_grant(sf, rnti, capi.TX_PORT0, FULL, nre, [(tbs, D_QM)])
        r["tb"]["rv"][0], r["tb"]["harq_op"][0], r["tb"]["harq_slot"][0] = rv, op, slot
        return r
    b1 = np.concatenate([g(0, 0x7001, 0, capi.HARQ_NEW, 0), g(1, 0x7002, 0, capi.HARQ_NEW, sy)])
    b2 = np.concatenate([g(2, 0x7001, 2, capi.HARQ_RETX, 0), g(3, 0x7002, 2, capi.HARQ_RETX, sy),
                         g(2, 0x7001, 2, capi.HARQ_NONE, 0), g(3, 0x7002, 2, capi.HARQ_NONE, 0)])
    return b1, b2


# ------------------------------------------------------------------------------------------------------------------------------------ helpers
def guard(nbytes, what):
    import torch
    free = torch.cuda.mem_get_info()[0]
    print("%s: %.2f GB of device memory needed, %.2f GB free" % (what, nbytes / 1e9, free / 1e9))
    if free < nbytes + MARGIN:
        pytest.skip("%s needs %d bytes of free device memory (+ %d margin), %d free" % (what, nbytes, MARGIN, free))


def new_phy(cell, n, iq=None, tti=None):
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8)
    if iq is not None:
        phy.submit_iq(iq, tti)
        info, _ = phy.get_phase_a(want_cands=False)
        assert all(info[i].cfi == CFI for i in range(n))
    return phy


def dl_run(phy, grants):
    L = phy.L
    g = np.ascontiguousarray(grants)
    assert L.ltephy_submit_grants(phy.h, _p(g), len(g)) == 0, L.ltephy_last_error().decode()
    res = np.zeros(2 * len(g), RES_DT)
    cap = int(g["tb"]["tbs"].astype(np.int64).sum() // 8 + 8 * len(g) + 4096)
    pl = np.zeros(cap, np.uint8)
    assert L.ltephy_get_phase_b(phy.h, _p(res), _p(pl), cap) == 0, L.ltephy_last_error().decode()
    return res, pl


def tb(res, pl, slot):
    r = res[slot]
    return (int(r["crc"]), int(r["avg_iters"]), int(r["nof_cb"]), int(r["payload_len"]),
            pl[int(r["payload_off"]):int(r["payload_off"]) + int(r["payload_len"])].tobytes())


def dl_case(cell, tti, qm, prbs, tbs, rnti, seed, NL, rv=0, scheme="sfbc"):
    """the IQ of one subframe carrying one crafted transport block -> (iq [rx][sf_len], payload bytes)"""
    S = ltelib.sim()
    S.lte_turbo_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    kw = dict(chan="flat", noise_var=NOISE, seed=seed, rnti=rnti)
    G = nof_re(cell, tti, tuple(prbs)) * qm
    e, pl = crafted_codeword(S, np.random.default_rng(seed), tbs, G, qm, NL, rv)
    c = Case(cell, tti % 10, CFI, scheme, [qm], prbs, cw_bits=[e], **kw)
    assert c.grant.nof_re * qm == G
    return c.iq, pl.tobytes()


# ------------------------------------------------------------------------------------------------------------------------------------ (a)
def test_downlink_soft_bits_past_2_32(infra, phylib):
    grants, idx, off, G, E = a_layout()
    tot = int(off[-1]) + cw_len(G)
    assert off[idx[1]] < WRAP < off[idx[1]] + sum(E[:-1]) and off[idx[2]] >= WRAP and (off[idx[2]] - WRAP) < off[1]
    guard(GROWTH * (2 * tot + tot // 8) + 1 * len(grants) * 512, "(a) %d grants, %d soft bits" % (len(grants), tot))
    cell = DL_CELL
    tbs = int(grants["tb"]["tbs"][0, 0])
    sig = [dl_case(cell, A_TTI[i], A_QM, FULL, tbs, 0x4001 + i, 500 + i, 2) for i in range(3)]
    iq, tti = np.stack([s[0] for s in sig]), np.array(A_TTI, np.uint32)
    real = grants[idx]
    ref = new_phy(cell, 3, iq, tti)
    want = dl_run(ref, real)
    llr_ref = ref.tap(capi.TAP_PDSCH_LLR, (cw_len(G),), np.int16)
    ref.close()
    for k in range(3):
        assert want[0][2 * k]["crc"] == 1 and tb(*want, 2 * k)[4] == sig[k][1], k
    phy = new_phy(cell, 3, iq, tti)
    try:
        t0 = time.time()
        got = dl_run(phy, grants)
        print("(a) %d grants in %.1f s" % (len(grants), time.time() - t0))
        llr = phy.tap(capi.TAP_PDSCH_LLR, (cw_len(G),), np.int16)
    finally:
        phy.close()
    for k, i in enumerate(idx):
        assert tb(*got, 2 * i) == tb(*want, 2 * k), ("T%d" % k, tb(*got, 2 * i)[:4], tb(*want, 2 * k)[:4])
        assert tb(*got, 2 * i)[4] == sig[k][1], "T%d payload" % k
    assert got[0]["payload_len"][2 * np.arange(len(grants))].sum() == 3 * (tbs // 8)
    assert np.array_equal(llr[:G], llr_ref[:G]), ("T0 soft bits", np.flatnonzero(llr[:G] != llr_ref[:G])[:8])


# ------------------------------------------------------------------------------------------------------------------------------------ (b)
def ul_run(phy, iq, tti, grants):
    L = phy.L
    g = np.ascontiguousarray(grants)
    assert L.ltephy_submit_ul(phy.h, _p(iq), _p(tti), len(tti), _p(g), len(g)) == 0, L.ltephy_last_error().decode()
    res = np.zeros(len(g), RES_DT)
    ch = np.zeros(len(g), CHEST_DT)
    cap = int(g["tbs"].astype(np.int64).sum() // 8 + 8 * len(g) + 4096)
    pl = np.zeros(cap, np.uint8)
    assert L.ltephy_get_ul(phy.h, _p(res), _p(ch), _p(pl), cap) == 0, L.ltephy_last_error().decode()
    return res, pl, ch


def new_ul_phy(cell, n):
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8)
    phy.set_ul_cfg(*UCFG)
    return phy


def ul_signal(cell, tti, g, seed):
    """uplink IQ [sf_len] of one ref64_ul grant with an encoded transport block -> (iq, payload bytes)"""
    pl, e = encode(g, np.random.default_rng(seed))
    s = Subframe(cell, tti % 10, UCFG, [g], chan="flat", noise_var=NOISE, seed=seed, bits=[e])
    return s.iq, pl.tobytes()


def test_uplink_soft_bits_past_2_32(infra, phylib):
    grants, idx, off, G, E = b_layout()
    tot = int(off[-1]) + cw_len(G)
    assert off[idx[1]] < WRAP < off[idx[1]] + sum(E[:-1]) and off[idx[2]] >= WRAP and (off[idx[2]] - WRAP) < off[1]
    npairs = (len(grants) + 1) // 2
    guard(GROWTH * (2 * tot + tot // 8 + 4 * npairs * rm_ref.pair_words(6144)), "(b) %d UL grants, %d soft bits" % (len(grants), tot))
    cell = UL_CELL
    sig = [ul_signal(cell, B_TTI[k], ref64_ul.Grant(100, 0, B_QM, int(grants["tbs"][i]), rnti=int(grants["rnti"][i])), 600 + k)
           for k, i in enumerate(idx)]
    iq, tti = np.ascontiguousarray(np.stack([s[0] for s in sig]), np.complex64), np.array(B_TTI, np.uint32)
    real = grants[idx]
    ref = new_ul_phy(cell, 3)
    want = ul_run(ref, iq, tti, real)
    llr_ref = ref.tap(capi.TAP_PDSCH_LLR, (cw_len(G),), np.int16)
    ref.close()
    for k in range(3):
        assert want[0][k]["crc"] == 1 and tb(want[0], want[1], k)[4] == sig[k][1], k
    phy = new_ul_phy(cell, 3)
    try:
        t0 = time.time()
        got = ul_run(phy, iq, tti, grants)
        print("(b) %d UL grants in %.1f s" % (len(grants), time.time() - t0))
        llr = phy.tap(capi.TAP_PDSCH_LLR, (cw_len(G),), np.int16)
    finally:
        phy.close()
    for k, i in enumerate(idx):
        assert tb(got[0], got[1], i) == tb(want[0], want[1], k), ("Tu%d" % k, tb(got[0], got[1], i)[:4], tb(want[0], want[1], k)[:4])
        assert tb(got[0], got[1], i)[4] == sig[k][1], "Tu%d payload" % k
        assert got[2][i].tobytes() == want[2][k].tobytes(), "Tu%d channel estimate" % k
    assert np.array_equal(llr[:G], llr_ref[:G]), ("Tu0 soft bits", np.flatnonzero(llr[:G] != llr_ref[:G])[:8])


# ------------------------------------------------------------------------------------------------------------------------------------ (c)
def test_turbo_pool_past_2_32_words(infra, phylib):
    grants, G = c_layout()
    n = len(grants)
    ncb = 16 * n
    words = (ncb // 2) * rm_ref.pair_words(6144)
    assert words > WRAP
    guard(GROWTH * (4 * words + 2 * n * cw_len(G) + 4 * n * (G // 32 + 2) + 2 * n * 12300) + 64 * ncb, "(c) %d turbo-pool words" % words)
    cell = TB_CELL
    sig = [dl_case(cell, t, C_QM, FULL, C_TBS, 0x6001 + s, 700 + s, 1, scheme="port0") for s, t in enumerate(C_TTI)]
    assert len({s[1] for s in sig}) == len(C_TTI)
    iq, tti = np.stack([s[0] for s in sig]), np.array(C_TTI, np.uint32)
    ref = new_phy(cell, len(C_TTI), iq, tti)
    want = dl_run(ref, grants[:len(C_TTI)])
    ref.close()
    want_tb = [tb(*want, 2 * s) for s in range(len(C_TTI))]
    for s in range(len(C_TTI)):
        assert want_tb[s][0] == 1 and want_tb[s][2] == 16 and want_tb[s][4] == sig[s][1], s
    phy = new_phy(cell, len(C_TTI), iq, tti)
    try:
        t0 = time.time()
        res, pl = dl_run(phy, grants)
        print("(c) %d grants, %d code blocks in %.1f s" % (n, ncb, time.time() - t0))
    finally:
        phy.close()
    bad = [i for i in range(n) if tb(res, pl, 2 * i) != want_tb[i % len(C_TTI)]]
    assert not bad, ("transport blocks differ from the reference", len(bad), bad[:8], [tb(res, pl, 2 * i)[:4] for i in bad[:4]])


# ------------------------------------------------------------------------------------------------------------------------------------ (d)
def turbo_in_words(tbs, ntb):
    """turbo-pool words the TAP_TURBO_IN layout holds for ntb transport blocks of tbs bits (equal K paired in submission order)"""
    Cn, Ks, _ = ref_dec.segmentation(tbs)
    return sum(-(-(ntb * Ks.count(K)) // 2) * rm_ref.pair_words(K) for K in set(Ks))


def d_sequence(phy, sy, tbs):
    out = []
    for batch in d_grants(sy):
        res, pl = dl_run(phy, batch)
        out.append(([tb(res, pl, 2 * i) for i in range(len(batch))], phy.tap(capi.TAP_TURBO_IN, (turbo_in_words(tbs, len(batch)),), np.uint32)))
    return out


def test_harq_slot_past_2_32_elements(infra, phylib):
    G, tbs = d_tbs()
    Cn = ref_dec.segmentation(tbs)[0]
    assert Cn >= 2 and (D_SLOTS - 2) * rm_ref.HARQ_SLOT_ELEMS < WRAP <= (D_SLOTS - 1) * rm_ref.HARQ_SLOT_ELEMS   # only the last slot starts past 2^32
    guard(GROWTH * D_SLOTS * capi.HARQ_SLOT_BYTES, "(d) %d HARQ slots" % D_SLOTS)
    cell = TB_CELL
    sig = [dl_case(cell, t, D_QM, FULL, tbs, (0x7001, 0x7002)[k % 2], 800 + k % 2, 1, rv=(0, 0, 2, 2)[k], scheme="port0")
           for k, t in enumerate(D_TTI)]
    assert sig[0][1] == sig[2][1] and sig[1][1] == sig[3][1] and sig[0][1] != sig[1][1]
    iq, tti = np.stack([s[0] for s in sig]), np.array(D_TTI, np.uint32)
    ref = new_phy(cell, 4, iq, tti)
    ref.harq_reserve(2)
    want = d_sequence(ref, 1, tbs)
    ref.close()
    # first transmissions and retransmissions alone fail; the combined retransmissions pass with what was sent
    assert [r[0] for r in want[0][0]] == [0, 0] and [r[0] for r in want[1][0]] == [1, 1, 0, 0], want
    assert want[1][0][0][4] == sig[0][1] and want[1][0][1][4] == sig[1][1]
    phy = new_phy(cell, 4, iq, tti)
    try:
        phy.harq_reserve(D_SLOTS)
        got = d_sequence(phy, D_SLOTS - 1, tbs)
    finally:
        phy.close()
    for b in range(2):
        assert got[b][0] == want[b][0], ("batch %d" % (b + 1), [r[:4] for r in got[b][0]], [r[:4] for r in want[b][0]])
        assert np.array_equal(got[b][1], want[b][1]), ("batch %d turbo input" % (b + 1), np.flatnonzero(got[b][1] != want[b][1])[:8])


# ------------------------------------------------------------------------------------------------------------------------------------ (e)
E_CELL = Cell(15, 1, 31, 1)
E_N = 65535                          # LTEPHY_MAX_BATCH_SUBFRAMES
E_CYCLE = 10240
E_CHUNK = 1000


class Outputs:
    """caller-owned outputs of decode_subframes, sized for a lightly loaded 15 PRB cell"""

    def __init__(self, n):
        self.max_dcis = 8 * n
        self.info = (capi.SfInfo * n)()
        self.cands = np.zeros((n, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
        self.dcis = np.zeros(self.max_dcis, capi.DCI_DTYPE)
        self.tbs = (capi.TbResult * (2 * self.max_dcis))()
        self.payload = np.zeros(self.max_dcis * 2 * 1024, np.uint8)
        self.nd = C.c_uint32(0)


def test_phase_a_at_the_largest_batch(infra, phylib):
    cell = E_CELL
    sf_len = 3840
    per_sf = 8 * sf_len + 8 * 14 * 12 * cell.nof_prb * 3 + 4 * capi.LLR_STRIDE + 16 * capi.MAX_LOC * capi.MAX_SIZES + capi.COMPACT_DTYPE.itemsize + 1024
    guard(GROWTH * E_N * per_sf, "(e) %d subframes" % E_N)
    from helpers import make_capture
    sim, iq_c, tti_c, truths, payloads = make_capture(cell, E_CYCLE, seed=61, cfi=2, nof_ues=4, dl_min=1, dl_max=2, tm=1, mcs_min=4, mcs_max=12,
                                                      snr_db=25.0)
    assert iq_c.shape[2] == sf_len
    src = np.arange(E_N) % E_CYCLE
    iq, tti = np.ascontiguousarray(iq_c[src]), np.ascontiguousarray(tti_c[src])
    del iq_c
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=E_N, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
    try:
        S = Outputs(E_N)
        t0 = time.time()
        r = decode(phy, srch, iq, tti, 0, E_N, capi.SEQ_NONE, S)
        assert r == 0, (r, phy.L.ltephy_last_error().decode())
        print("(e) one batch of %d subframes in %.1f s, %d DCIs" % (E_N, time.time() - t0, S.nd.value))
        assert S.nd.value < S.max_dcis
        big = snapshot(S, E_N)
    finally:
        phy.close()
        srch.close()
    del S
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=E_CHUNK, turbo_max_iter=8,
                      flags=capi.FLAG_SKIP_LOW_POWER)
    info, dcis, tbs = [], [], []
    try:
        S = Outputs(E_CHUNK)
        for lo in range(0, E_N, E_CHUNK):
            hi = min(lo + E_CHUNK, E_N)
            assert decode(phy, srch, iq, tti, lo, hi, capi.SEQ_NONE, S) == 0, phy.L.ltephy_last_error().decode()
            i, d, t = snapshot(S, hi - lo)
            info += i
            dcis += [(x[0] + lo,) + x[1:] for x in d]
            tbs += t
    finally:
        phy.close()
        srch.close()
    assert big[0] == info, "SfInfo differs from the batches of %d" % E_CHUNK
    assert big[1] == dcis, "DCIs differ from the batches of %d" % E_CHUNK
    assert big[2] == tbs, "transport blocks differ from the batches of %d" % E_CHUNK
    cfi = {capi.SfInfo.from_buffer_copy(b).cfi for b in info}
    assert cfi == {2}, cfi
    # every transmitted transport block after the first SFN cycle (the search learns the RNTIs in the first) is decoded with what was sent
    got = {}
    for k, d in enumerate(dcis):
        for t in range(2):
            crc, _, _, _, pl = tbs[2 * k + t]
            if crc:
                got[(d[0], d[1], t)] = pl
    nsent = 0
    for sf in range(E_CYCLE, E_N):
        tr, pls = truths[sf % E_CYCLE], payloads[sf % E_CYCLE]
        for i in range(tr.nof_dci):
            d = tr.dci[i]
            for t in range(2):
                if d.tbs[t] > 0:
                    nsent += 1
                    assert got.get((sf, d.rnti, t)) == pls[d.payload_off[t]:d.payload_off[t] + d.tbs[t] // 8].tobytes(), (sf, hex(d.rnti), t)
    assert nsent > 50000


def test_uplink_at_the_largest_batch(infra, phylib):
    cell = E_CELL
    sf_len = 3840
    guard(GROWTH * E_N * (8 * sf_len + 8 * 14 * 12 * cell.nof_prb), "(e) %d uplink subframes" % E_N)
    g = [ref64_ul.Grant(12, 1, 4, ul_tbs(12, 4), rnti=0x3001), ref64_ul.Grant(15, 0, 2, ul_tbs(15, 2), rnti=0x3002)]
    tti = (np.arange(E_N) % E_CYCLE).astype(np.uint32)
    ends = (0, E_N - 1)
    sig = [ul_signal(cell, int(tti[s]), g[k], 900 + k) for k, s in enumerate(ends)]
    grants = np.concatenate([ul_grant(s, g[k].rnti, g[k].L, g[k].qm, g[k].tbs) for k, s in enumerate(ends)])
    grants["n_prb"] = [g[0].n_prb, g[1].n_prb]
    want = []
    phy = new_ul_phy(cell, 1)
    try:
        for k, s in enumerate(ends):
            one = grants[k:k + 1].copy()
            one["sf"] = 0
            res, pl, ch = ul_run(phy, np.ascontiguousarray(sig[k][0][None]), tti[s:s + 1].copy(), one)
            assert res[0]["crc"] == 1 and tb(res, pl, 0)[4] == sig[k][1], k
            want.append((tb(res, pl, 0), ch[0].tobytes()))
    finally:
        phy.close()
    iq = np.zeros((E_N, sf_len), np.complex64)
    for k, s in enumerate(ends):
        iq[s] = sig[k][0]
    phy = new_ul_phy(cell, E_N)
    try:
        res, pl, ch = ul_run(phy, iq, tti, grants)
    finally:
        phy.close()
    for k in range(2):
        assert (tb(res, pl, k), ch[k].tobytes()) == want[k], (k, tb(res, pl, k)[:4], want[k][0][:4])
