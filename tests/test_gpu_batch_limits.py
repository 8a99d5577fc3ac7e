"""Phase B at grant counts that reach CUDA's 65 535 limit on gridDim.y / gridDim.z (pytest -m gpu).

One batch of numpy-synthesised subframes (tests/test_float64_reference.Case downlink, tests/ref64_ul uplink), each with its transmitted block and
many decoy grants: other RNTIs, small PRB sets, QPSK / 16QAM, port 0 and SFBC.  Grants are decode hypotheses, so decoys may overlap.  The whole
list goes through one submit at counts on both sides of where a grid that puts the grant on y or z could no longer launch: 32 767 / 32 768 and
~70 000 downlink grants (two codewords per grant), 65 535 / 65 536 uplink grants.  The soft bits (TAP_PDSCH_LLR), crc, avg_iters, nof_cb, the
payload -- and, uplink, the channel estimate -- must equal the same grants decoded in chunks of at most 1 000 on a fresh handle, and the
transmitted blocks must equal what was sent."""
import ctypes as C

import numpy as np
import pytest

import ltelib
import ref64
import ref64_ul
from ltelib import Cell
from test_decoder_reference import crafted_codeword
from test_float64_reference import Case, tbs_of
from test_pusch_float64_reference import Subframe, encode, tbs as ul_tbs
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu

CHUNK = 1000
GRANT_DT = np.dtype(capi.Grant)
UL_GRANT_DT = np.dtype(capi.UlGrant)
RES_DT = np.dtype(capi.TbResult)
CHEST_DT = np.dtype(capi.UlChest)

DL_CELL = Cell(25, 2, 150, 2)
DL_NSF = 20
DL_COUNTS = (32767, 32768, 70000)
UL_CELL = Cell(25, 1, 150, 1)
UL_NSF = 10
UL_COUNTS = (65535, 65536)
UCFG = (0, 0, 0, 0)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def payload_bytes(res, pl):
    """the payload bytes of every result slot, concatenated in slot order"""
    lens = res["payload_len"].astype(np.int64)
    if lens.sum() == 0:
        return np.zeros(0, np.uint8)
    start = np.cumsum(lens) - lens
    idx = np.repeat(res["payload_off"].astype(np.int64) - start, lens) + np.arange(lens.sum())
    return pl[idx]


def fields(res):
    return {k: res[k].copy() for k in ("crc", "avg_iters", "nof_cb", "payload_len")}


def written(G, llr_len):
    """the soft bits a codeword of G bits writes in its (G + 7) & ~7 slot of the LLR pool (the padding is never written)"""
    start = np.cumsum(llr_len) - llr_len
    return (np.arange(llr_len.sum()) - np.repeat(start, llr_len)) < np.repeat(G, llr_len)


def assert_same(got, want, what, valid):
    for k in ("crc", "avg_iters", "nof_cb", "payload_len"):
        assert np.array_equal(got[0][k], want[0][k]), (what, k, np.flatnonzero(got[0][k] != want[0][k])[:8])
    assert np.array_equal(got[1], want[1]), (what, "payload")
    assert np.array_equal(got[2][valid], want[2][valid]), (what, "soft bits", np.flatnonzero((got[2] != want[2]) & valid)[:8])


# ------------------------------------------------------------------------------------------------------------------------------------ downlink
def dl_batch():
    """-> (iq [n][rx][sf_len], tti, grants GRANT_DT [70 000], llr length of each grant, payload sent in the first DL_NSF grants)"""
    cell = DL_CELL
    N = cell.nof_prb
    S = ltelib.sim()
    S.lte_turbo_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(23)
    iq, cfis, sent = [], [], []
    tx = np.zeros(DL_NSF, GRANT_DT)
    for i in range(DL_NSF):                                           # tti = i: every subframe index twice, CFI 1..3
        sf, cfi, qm = i % 10, 1 + i % 3, (2, 4)[i % 2]
        prbs = list(range(2 + i % 6, 17 + i % 6))
        kw = dict(chan="flat", noise_var=1e-4, seed=300 + i, rnti=0x4000 + i)
        G = Case(cell, sf, cfi, "sfbc", [qm], prbs, **kw).grant.nof_re * qm
        tbs = tbs_of(6 if qm == 2 else 12, len(prbs))
        e, pl = crafted_codeword(S, rng, tbs, G, qm, 2, 0)           # SFBC: two layers in the rate matching
        c = Case(cell, sf, cfi, "sfbc", [qm], prbs, cw_bits=[e], **kw)
        iq.append(c.iq)
        cfis.append(cfi)
        sent.append(pl)
        g = tx[i]
        g["sf"], g["rnti"], g["tx_scheme"], g["nof_tb"], g["nof_re"] = i, 0x4000 + i, capi.TX_DIVERSITY, 1, c.grant.nof_re
        for p in prbs:
            g["prb_mask"][:, p >> 5] |= np.uint32(1 << (p & 31))
        g["tb"]["tbs"][0], g["tb"]["qm"][0], g["tb"]["enabled"][0] = tbs, qm, 1
    # resource elements of every PRB of every subframe (both slots), from the 36.211 map of ref64
    re_cnt = np.zeros((DL_NSF, N), np.int64)
    for i in range(DL_NSF):
        for p in range(N):
            mask = np.zeros((2, 110), np.uint8)
            mask[:, p] = 1
            re_cnt[i, p] = len(ref64.pdsch_res(cell, i % 10, cfis[i], mask)[0])
    nd = DL_COUNTS[-1] - DL_NSF
    j = np.arange(nd)
    d = np.zeros(nd, GRANT_DT)
    sfi = j % DL_NSF
    nprb = 1 + j % 3
    start = (j * 7) % (N - 2)
    qm = np.where((j // 2) % 2 == 0, 2, 4)
    d["sf"], d["rnti"], d["tx_scheme"], d["nof_tb"] = sfi, 0x100 + j % 3000, np.where(j % 2 == 0, capi.TX_PORT0, capi.TX_DIVERSITY), 1
    d["nof_re"] = sum(np.where(nprb > q, re_cnt[sfi, np.minimum(start + q, N - 1)], 0) for q in range(3))
    for q in range(3):
        p = start + q
        on = nprb > q
        np.bitwise_or.at(d["prb_mask"], (np.flatnonzero(on), slice(None), p[on] >> 5), (np.uint32(1) << (p[on] & 31).astype(np.uint32))[:, None])
    d["tb"]["tbs"][:, 0] = [tbs_of(int(a), int(b)) for a, b in zip(j % 6, nprb)]
    d["tb"]["qm"][:, 0], d["tb"]["enabled"][:, 0] = qm, 1
    grants = np.concatenate([tx, d])
    llr_len = ((grants["nof_re"].astype(np.int64) * grants["tb"]["qm"][:, 0] + 7) & ~7)
    return np.stack(iq), np.arange(DL_NSF, dtype=np.uint32), grants, llr_len, sent, cfis


def dl_decode(phy, grants, llr_len):
    L = phy.L
    g = np.ascontiguousarray(grants)
    assert L.ltephy_submit_grants(phy.h, _p(g), len(g)) == 0, L.ltephy_last_error().decode()
    res = np.zeros(2 * len(g), RES_DT)
    cap = int(g["tb"]["tbs"][:, 0].sum() // 8 + 16 * len(g) + 4096)
    pl = np.zeros(cap, np.uint8)
    assert L.ltephy_get_phase_b(phy.h, _p(res), _p(pl), cap) == 0, L.ltephy_last_error().decode()
    llr = phy.tap(capi.TAP_PDSCH_LLR, (int(llr_len.sum()),), np.int16)
    return res, payload_bytes(res, pl), llr


def new_dl_phy(iq, tti, cfis):
    cell = DL_CELL
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=len(tti), turbo_max_iter=8)
    phy.submit_iq(iq, tti)
    info, _ = phy.get_phase_a(want_cands=False)
    assert [info[i].cfi for i in range(len(tti))] == cfis
    return phy


def test_downlink_grant_counts_beyond_the_grid_y_limit(infra, phylib):
    iq, tti, grants, llr_len, sent, cfis = dl_batch()
    ref = new_dl_phy(iq, tti, cfis)
    parts = [dl_decode(ref, grants[a:a + CHUNK], llr_len[a:a + CHUNK]) for a in range(0, len(grants), CHUNK)]
    ref.close()
    res_r = np.concatenate([p[0] for p in parts])
    pl_r = np.concatenate([p[1] for p in parts])
    llr_r = np.concatenate([p[2] for p in parts])
    pl_end = np.cumsum(res_r["payload_len"].astype(np.int64))
    llr_end = np.cumsum(llr_len)
    # the transmitted blocks (grants 0 .. DL_NSF - 1, result slot 2 i) against what was sent; the decoys fail their CRC
    for i in range(DL_NSF):
        r = res_r[2 * i]
        assert r["crc"] == 1 and r["payload_len"] == len(sent[i]), (i, r)
        assert np.array_equal(pl_r[pl_end[2 * i] - r["payload_len"]:pl_end[2 * i]], sent[i]), i
    assert res_r["crc"][2 * DL_NSF:].sum() == 0
    valid = written(grants["nof_re"].astype(np.int64) * grants["tb"]["qm"][:, 0], llr_len)
    phy = new_dl_phy(iq, tti, cfis)
    try:
        for n in DL_COUNTS:
            got = dl_decode(phy, grants[:n], llr_len[:n])
            want = (res_r[:2 * n], pl_r[:pl_end[2 * n - 1]], llr_r[:llr_end[n - 1]])
            assert_same(got, want, "%d grants" % n, valid[:llr_end[n - 1]])
    finally:
        phy.close()


# ------------------------------------------------------------------------------------------------------------------------------------ uplink
def ul_batch():
    cell = UL_CELL
    N = cell.nof_prb
    rng = np.random.default_rng(29)
    iq, sent = [], []
    tx = np.zeros(UL_NSF, UL_GRANT_DT)
    for i in range(UL_NSF):
        qm, Lp, n0 = (2, 4)[i % 2], (10, 12, 15)[i % 3], i % 8
        g = ref64_ul.Grant(Lp, n0, qm, ul_tbs(Lp, qm), rnti=0x5000 + i)
        pl, e = encode(g, rng)
        s = Subframe(cell, i % 10, UCFG, [g], chan="flat", noise_var=1e-4, seed=400 + i, bits=[e])
        iq.append(s.iq)
        sent.append(pl)
        t = tx[i]
        t["sf"], t["rnti"], t["qm"], t["L_prb"], t["n_prb"], t["tbs"] = i, g.rnti, qm, Lp, n0, g.tbs
    nd = UL_COUNTS[-1] - UL_NSF
    j = np.arange(nd)
    d = np.zeros(nd, UL_GRANT_DT)
    Lp = np.array([3, 4, 5, 6])[j % 4]
    qm = np.where((j // 4) % 4 == 3, 4, 2)
    d["sf"], d["rnti"], d["qm"], d["L_prb"] = j % UL_NSF, 0x100 + j % 3000, qm, Lp
    d["n_prb"] = (j * 5) % (N - Lp + 1)
    d["n_dmrs2"] = j % 12
    d["tbs"] = [ul_tbs(int(a), int(b), int(c)) for a, b, c in zip(Lp, qm, j % 5)]
    grants = np.concatenate([tx, d])
    llr_len = (12 * 12 * grants["L_prb"].astype(np.int64) * grants["qm"] + 7) & ~7
    return np.stack(iq), np.arange(UL_NSF, dtype=np.uint32), grants, llr_len, sent


def ul_decode(phy, iq, tti, grants, llr_len):
    L = phy.L
    g = np.ascontiguousarray(grants)
    assert L.ltephy_submit_ul(phy.h, _p(iq), _p(tti), len(tti), _p(g), len(g)) == 0, L.ltephy_last_error().decode()
    res = np.zeros(len(g), RES_DT)
    ch = np.zeros(len(g), CHEST_DT)
    cap = int(g["tbs"].sum() // 8 + 16 * len(g) + 4096)
    pl = np.zeros(cap, np.uint8)
    assert L.ltephy_get_ul(phy.h, _p(res), _p(ch), _p(pl), cap) == 0, L.ltephy_last_error().decode()
    llr = phy.tap(capi.TAP_PDSCH_LLR, (int(llr_len.sum()),), np.int16)
    return res, payload_bytes(res, pl), llr, ch


def new_ul_phy():
    cell = UL_CELL
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=UL_NSF, turbo_max_iter=8)
    phy.set_ul_cfg(*UCFG)
    return phy


def test_uplink_grant_counts_beyond_the_grid_y_limit(infra, phylib):
    iq, tti, grants, llr_len, sent = ul_batch()
    iq = np.ascontiguousarray(iq, np.complex64)
    ref = new_ul_phy()
    parts = [ul_decode(ref, iq, tti, grants[a:a + CHUNK], llr_len[a:a + CHUNK]) for a in range(0, len(grants), CHUNK)]
    ref.close()
    res_r = np.concatenate([p[0] for p in parts])
    pl_r = np.concatenate([p[1] for p in parts])
    llr_r = np.concatenate([p[2] for p in parts])
    ch_r = np.concatenate([p[3] for p in parts])
    pl_end = np.cumsum(res_r["payload_len"].astype(np.int64))
    llr_end = np.cumsum(llr_len)
    for i in range(UL_NSF):
        r = res_r[i]
        assert r["crc"] == 1 and r["payload_len"] == len(sent[i]), (i, r)
        assert np.array_equal(pl_r[pl_end[i] - r["payload_len"]:pl_end[i]], sent[i]), i
    assert res_r["crc"][UL_NSF:].sum() == 0
    valid = written(12 * 12 * grants["L_prb"].astype(np.int64) * grants["qm"], llr_len)
    phy = new_ul_phy()
    try:
        for n in UL_COUNTS:
            res, pl, llr, ch = ul_decode(phy, iq, tti, grants[:n], llr_len[:n])
            assert_same((res, pl, llr), (res_r[:n], pl_r[:pl_end[n - 1]], llr_r[:llr_end[n - 1]]), "%d UL grants" % n, valid[:llr_end[n - 1]])
            assert ch.tobytes() == ch_r[:n].tobytes(), n
    finally:
        phy.close()
