"""Which candidates or code blocks share an int16x2 decode must not change any result.

* DCI Viterbi: with FLAG_SKIP_LOW_POWER the work list pairs the decodable locations of a subframe densely.  The full candidate table
  equals the oracle: a decodable location holds lteo_dci_decode's bits and RNTI, every other entry is all zero.  The captures give
  odd and even counts of decodable locations per subframe, subframes with none (low SNR), and a CFI change on one handle.
* Turbo: code blocks of equal K are paired by code rate (ltephy_turbo_pairing).  Per transport block, crc, avg_iters and payload
  equal the oracle's lteo_dlsch_decode on the same soft bits, on a batch with many K and MCS, HARQ retransmissions inside the
  batch, and an uplink batch.
* The pairing itself, on the host (no GPU): every code block once, equal K in a pair, deterministic."""
import ctypes as C

import numpy as np
import pytest

import ltelib
import rm_ref
from helpers import make_capture, oracle_frontend, to_phy_grant, truth_grants
from ltesniffer_b200 import capi

CFG2 = dict(cfi=3, nof_ues=150, dl_min=8, dl_max=12, tm=3, mcs_min=17, mcs_max=28, snr_db=25.0, full_band=1)   # bench.py SIM_KW


def _pairing(lib, K, tbs, G):
    n = len(K)
    arr = [np.ascontiguousarray(a, np.uint32) for a in (K, tbs, G)]
    pair, half, npairs = np.zeros(n, np.uint32), np.zeros(n, np.uint32), C.c_uint32(0)
    lib.ltephy_turbo_pairing.argtypes = [C.c_uint32] + [C.c_void_p] * 5 + [C.POINTER(C.c_uint32)]
    assert lib.ltephy_turbo_pairing(n, *[a.ctypes.data for a in arr], pair.ctypes.data, half.ctypes.data, C.byref(npairs)) == 0
    return pair, half, npairs.value


def test_pairing_covers_every_block_once_with_equal_k(phylib):
    rng = np.random.default_rng(7)
    n = 501
    K = rng.choice([40, 1056, 2048, 6144], n)
    tbs = rng.integers(100, 60000, n) // 8 * 8
    G = (tbs * rng.uniform(0.8, 12.0, n)).astype(np.int64)      # a few rates above 1 (saturated), most below
    G[:3] = 0
    pair, half, npairs = _pairing(phylib, K, tbs, G)
    slots = set(zip(pair.tolist(), half.tolist()))
    assert len(slots) == n and pair.max() == npairs - 1
    for p in range(npairs):
        m = np.flatnonzero(pair == p)
        assert len(m) in (1, 2) and sorted(half[m].tolist()) == list(range(len(m))) and len(set(K[m].tolist())) == 1, p
    # one single-block pair per K of odd count, none otherwise
    for k in set(K.tolist()):
        assert sum(1 for p in range(npairs) if (pair == p).sum() == 1 and K[pair == p][0] == k) == (K == k).sum() % 2
    # the documented order: K descending, then TBS / G in steps of 2^-16 (saturating at 1) descending, then index; neighbours paired
    rq = np.where(G > 0, np.minimum((tbs.astype(np.int64) << 16) // np.maximum(G, 1), 0xFFFF), 0xFFFF)
    want_pair, want_half, np_, open_k = np.zeros(n, np.int64), np.zeros(n, np.int64), 0, None
    for i in sorted(range(n), key=lambda i: (-K[i], -rq[i], i)):
        if open_k == K[i]:
            want_pair[i], want_half[i], open_k = np_ - 1, 1, None
        else:
            want_pair[i], np_, open_k = np_, np_ + 1, K[i]
    assert np.array_equal(pair, want_pair) and np.array_equal(half, want_half) and npairs == np_
    again = _pairing(phylib, K, tbs, G)
    assert np.array_equal(again[0], pair) and np.array_equal(again[1], half) and again[2] == npairs


def test_pairing_rejects_bad_arguments(phylib):
    phylib.ltephy_turbo_pairing.argtypes = [C.c_uint32] + [C.c_void_p] * 5 + [C.POINTER(C.c_uint32)]
    n = C.c_uint32(0)
    assert phylib.ltephy_turbo_pairing(3, None, None, None, None, None, C.byref(n)) == -2
    assert phylib.ltephy_turbo_pairing(0, None, None, None, None, None, C.byref(n)) == 0 and n.value == 0
    bad = [np.array([40, 41], np.uint32), np.array([16, 16], np.uint32), np.array([100, 100], np.uint32), np.zeros(2, np.uint32), np.zeros(2, np.uint32)]
    assert phylib.ltephy_turbo_pairing(2, *[a.ctypes.data for a in bad], C.byref(n)) == -2       # 41 is not a turbo block size


# ------------------------------------------------------------------------------------------------------------------------------
def _check_table(phy, o, ref, cands, info):
    """full table of one batch vs the oracle under the power floor; -> decodable locations per subframe"""
    sizes, sidx = phy.sizes()
    distinct = sorted({sidx[f]: sizes[f] for f in range(capi.NOF_FORMATS)}.items())
    counts = []
    for i, r in enumerate(ref):
        nc, Ls = phy.locations(r["cfi"])
        assert info[i].cfi == r["cfi"] and info[i].nof_locations == len(nc)
        pw = np.array(info[i].cce_power[:], np.float32)
        assert np.array_equal(pw[:len(r["cce_power"])], r["cce_power"])
        want = np.zeros((capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
        nval = 0
        for li in range(len(nc)):
            n0, L = int(nc[li]), 1 << int(Ls[li])
            if not np.all(pw[n0:n0 + L] >= np.float32(0.7)):
                continue
            nval += 1
            e = r["llr"][72 * n0:72 * (n0 + L)]
            for si, nb in distinct:
                ret, bits, crc = o.dci_decode(e, nb)
                if ret != 0:
                    continue
                v = 0
                for b in range(nb):
                    v |= int(bits[b]) << (63 - b)
                want[li, si]["bits"], want[li, si]["rnti"], want[li, si]["valid"] = v, crc, 1
        got = cands[i][:, :len(distinct)]
        bad = np.argwhere(got.view(np.uint8).reshape(capi.MAX_LOC, len(distinct), 16) != want[:, :len(distinct)].view(np.uint8).reshape(capi.MAX_LOC, len(distinct), 16))
        assert bad.size == 0, "sf %d: %d bytes differ, first at location %d size %d" % (i, len(bad), bad[0][0], bad[0][1])
        counts.append(nval)
    return counts


def _phase_a(phy, o, cell, n, **kw):
    sim, iq, tti, truths, payloads = make_capture(cell, n, **kw)
    ref = oracle_frontend(o, iq, tti)
    phy.submit_iq(iq, tti)
    info, cands = phy.get_phase_a()
    return ref, info, cands


@pytest.mark.gpu
def test_dense_viterbi_table_matches_oracle(infra, phylib):
    cell = ltelib.Cell(100, 2, 7, 2)
    o = ltelib.Oracle(cell)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=6, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
    try:
        counts = []
        # cfg-2 traffic (CFI 3)
        ref, info, cands = _phase_a(phy, o, cell, 6, seed=2, **CFG2)
        counts += _check_table(phy, o, ref, cands, info)
        # the same handle, CFI 1 and few DCIs: fewer locations, so entries written at CFI 3 must not survive
        ref, info, cands = _phase_a(phy, o, cell, 4, seed=21, cfi=1, nof_ues=3, dl_min=0, dl_max=1, tm=1, mcs_min=5, mcs_max=9, snr_db=25.0)
        assert all(r["cfi"] == 1 for r in ref)
        counts += _check_table(phy, o, ref, cands, info)
        # no DCI at all: no location above the power floor
        ref, info, cands = _phase_a(phy, o, cell, 2, seed=22, cfi=2, nof_ues=1, dl_min=0, dl_max=0, tm=1, mcs_min=5, mcs_max=5, snr_db=25.0)
        counts += _check_table(phy, o, ref, cands, info)
        assert any(c % 2 == 1 for c in counts) and any(c > 0 and c % 2 == 0 for c in counts), counts
        assert 0 in counts, counts
    finally:
        phy.close()


# ------------------------------------------------------------------------------------------------------------------------------
def _oracle_tb(llr, G, tbs, rv, qm, NL, soft=None, combine=0):
    O = ltelib.oracle()
    e = np.ascontiguousarray(llr[:G], np.int16)
    pl = np.zeros(tbs // 8 + 16, np.uint8)
    it = np.zeros(64, np.uint32)
    if soft is None:
        ok = O.lteo_dlsch_decode(ltelib.ptr(e), G, tbs, rv, qm, NL, 8, 1, ltelib.ptr(pl), ltelib.ptr(it))
    else:
        P = C.c_void_p
        O.lteo_dlsch_decode_harq.argtypes = [P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, P, P, P, C.c_int]
        ok = O.lteo_dlsch_decode_harq(ltelib.ptr(e), G, tbs, rv, qm, NL, 8, 1, ltelib.ptr(pl), ltelib.ptr(it), ltelib.ptr(soft), combine)
    assert ok >= 0
    ncb = rm_ref.check_tables.segm(tbs)[0]
    return ok, pl[:tbs // 8], -(-int(it[:ncb].sum()) // ncb)


def _check_tbs(res, pl, results):
    assert len(results) > 0
    ks = set()
    for slot, (ok, opl, its, K) in results:
        rr = res[slot]
        assert rr.crc == ok and rr.avg_iters == its, (slot, rr.crc, ok, rr.avg_iters, its)
        assert np.array_equal(pl[rr.payload_off:rr.payload_off + len(opl)], opl), slot
        ks |= K
    return ks


@pytest.mark.gpu
def test_turbo_pairs_by_rate_match_oracle_dl_with_harq(infra, phylib):
    cell = ltelib.Cell(100, 2, 7, 2)
    sim, iq, tti, truths, payloads = make_capture(cell, 4, seed=3, **CFG2)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=4, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
    try:
        phy.submit_iq(iq, tti)
        phy.get_phase_a()
        tg = truth_grants(cell, truths, tti)
        grants = [to_phy_grant(sf, d.rnti, g) for sf, d, g in tg]
        # a HARQ first transmission and its retransmission (other rv) inside the same batch: the grant's allocation again
        phy.harq_reserve(4)
        first = grants[0]
        first.tb[0].harq_op, first.tb[0].harq_slot = capi.HARQ_NEW, 1
        retx = to_phy_grant(tg[0][0], tg[0][1].rnti, tg[0][2])
        retx.tb[0].harq_op, retx.tb[0].harq_slot, retx.tb[0].rv = capi.HARQ_RETX, 1, 2
        grants.append(retx)
        phy.submit_grants(grants)
        res, pl = phy.get_phase_b()
        total = sum(((g.nof_re * g.tb[t].qm + 7) & ~7) for g in grants for t in range(2) if g.tb[t].enabled)
        llr = phy.tap(capi.TAP_PDSCH_LLR, (total,), np.int16)
        soft = np.zeros(16 * rm_ref.HARQ_CB_STRIDE, np.int16)
        out, off = [], 0
        for gi, g in enumerate(grants):
            for t in range(2):
                if not g.tb[t].enabled:
                    continue
                G, tb = g.nof_re * g.tb[t].qm, g.tb[t]
                NL = 2 if g.tx_scheme == capi.TX_DIVERSITY else 1
                harq = tb.harq_op != capi.HARQ_NONE
                ok, opl, its = _oracle_tb(llr[off:], G, tb.tbs, tb.rv, tb.qm, NL, soft if harq else None, 1 if tb.harq_op == capi.HARQ_RETX else 0)
                C_, Kp, Km, Cp, Cm, F = rm_ref.check_tables.segm(tb.tbs)
                out.append((2 * gi + t, (ok, opl, its, {Kp, Km} - {0})))
                off += (G + 7) & ~7
        ks = _check_tbs(res, pl, out)
        assert len(ks) >= 8 and len({g.tb[0].tbs for g in grants}) >= 8, ks
        assert any(r.avg_iters > 1 for r in res[:2 * len(grants)]) and sum(1 for r in res[:2 * len(grants)] if r.crc) > 0
    finally:
        phy.close()


@pytest.mark.gpu
def test_turbo_pairs_by_rate_match_oracle_ul(infra, phylib):
    cell = ltelib.Cell(50, 1, 9, 1)
    ucfg = ltelib.UlCfg(n_dmrs1=3, delta_ss=2)
    s = ltelib.Sim(cell=cell, seed=6, snr_db=22.0, nof_ues=1)
    rng = np.random.default_rng(6)
    iq = np.zeros((3, s.sf_len), np.complex64)
    grants, cg = [], []
    for i in range(3):
        gr = ltelib.make_ul_grants(cell, rng, 5, table=1)
        iq[i] = ltelib.sim_ul_subframe(s, i, ucfg, gr)[0]
        grants += gr
        cg += [capi.UlGrant(sf=i, rnti=g.rnti, qm=g.qm, rv=g.rv, L_prb=g.L_prb, n_prb=g.n_prb, n_dmrs2=g.n_dmrs2, tbs=g.tbs, n_prb_slot1=g.n_prb,
                            flags=capi.UL_FLAG_SLOT1, nof_ack=g.nof_ack, ri_len=g.ri_len, cqi_len=g.cqi_len, I_offset_ack=g.I_offset_ack,
                            I_offset_ri=g.I_offset_ri, I_offset_cqi=g.I_offset_cqi) for g in gr]
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=3)
    try:
        phy.set_ul_cfg(3, 2)
        res, ch, payload = phy.decode_ul(iq, np.arange(3, dtype=np.uint32), cg)
        Gs = [ltelib.uci_layout(g).G for g in grants]
        llr = phy.tap(capi.TAP_PDSCH_LLR, (sum((G + 7) & ~7 for G in Gs),), np.int16)
        out, off = [], 0
        for gi, (g, G) in enumerate(zip(grants, Gs)):
            ok, opl, its = _oracle_tb(llr[off:], G, g.tbs, g.rv, g.qm, 1)
            C_, Kp, Km, Cp, Cm, F = rm_ref.check_tables.segm(g.tbs)
            out.append((gi, (ok, opl, its, {Kp, Km} - {0})))
            off += (G + 7) & ~7
        _check_tbs(res, payload, out)
        assert sum(1 for r in res[:len(grants)] if r.crc) > 0
    finally:
        phy.close()
