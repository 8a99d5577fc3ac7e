"""Host search (product, table-driven) against the oracle walk (lazy decodes + the reference's own
RNTIManager) on the same captures; search-space validation and DCI->grant against the oracle's versions."""
import ctypes as C
import os
import numpy as np
import pytest
import ltelib
from ltelib import Cell, Sim, Oracle, OracleWalk, FORMATS
from ltesniffer_b200 import capi


def oracle_table(o, phy_sizes, nc, Ls, llr):
    """the candidate table exactly as the Viterbi kernel defines it, built with the CPU oracle"""
    sizes, sidx = phy_sizes
    T = np.zeros((capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
    distinct = {sidx[f]: sizes[f] for f in range(9)}
    for li in range(len(nc)):
        e = llr[72 * int(nc[li]):72 * int(nc[li]) + (72 << int(Ls[li]))]
        for si, nb in distinct.items():
            r, bits, crc = o.dci_decode(e, nb)
            if r == 0:
                v = 0
                for i, b in enumerate(bits):
                    v |= int(b) << (63 - i)
                T[li, si] = (v, crc, 1, [0] * 5)
    return T


def host_geometry(cell):
    """sizes / size index / locations from the sim's DCI size function (no GPU needed)"""
    S = ltelib.sim()
    sizes = [S.lte_dci_sizeof(C.byref(cell), f) for f in range(9)]
    order = []
    for s in sizes:
        if s not in order:
            order.append(s)
    return sizes, [order.index(s) for s in sizes]


def locations(nof_cce):
    nc, Ls = [], []
    lim = min(nof_cce, 84)
    for l in (3, 2, 1, 0):
        for i in range(lim // (1 << l)):
            nc.append((1 << l) * i)
            Ls.append(l)
    return np.array(nc), np.array(Ls)


def test_validate_location_matches_list_based_version(infra):
    S, L = infra.sim(), capi.load_library()
    capi._bind_search(L)
    rng = np.random.default_rng(0)
    for nof_cce in (20, 25, 54, 87, 41, 8, 3):
        for _ in range(4000):
            rnti = int(rng.choice([rng.integers(0, 65536), rng.integers(0, 12), rng.integers(0xFFF0, 0x10000)]))
            l = int(rng.integers(0, 4))
            ncce = int(rng.integers(0, max(1, nof_cce))) // (1 << l) * (1 << l)
            sf = int(rng.integers(0, 10))
            assert L.ltephy_search_validate_location(nof_cce, ncce, l, sf, rnti) == S.lte_pdcch_validate_location(nof_cce, ncce, l, sf, rnti), (nof_cce, ncce, l, sf, rnti)


@pytest.mark.parametrize("name,cell,n,kw", [
    ("tm1_shortcut", Cell(100, 1, 1, 1), 30, dict(seed=1, cfi=2, nof_ues=2, dl_min=1, dl_max=2, tm=1, mcs_min=5, mcs_max=5, snr_db=30.0, fixed_L=2, si_period=5)),
    ("busy_tm3", Cell(50, 2, 7, 2), 60, dict(seed=2, cfi=3, nof_ues=12, dl_min=3, dl_max=5, ul_min=1, ul_max=2, tm=13, mcs_min=3, mcs_max=12, snr_db=26.0)),
    ("low_snr_gate", Cell(25, 1, 9, 1), 6, dict(seed=3, cfi=2, nof_ues=2, dl_min=1, dl_max=1, tm=1, mcs_min=2, mcs_max=2, snr_db=3.0)),
])
def test_search_matches_oracle_walk(infra, name, cell, n, kw):
    s, o = Sim(cell=cell, **kw), Oracle(cell)
    walk = OracleWalk(cell, golden="oraclewalk_host_" + name)     # tests/golden stands in for oracle/_ref where it cannot be built
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    srch_c = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)   # same walk over the survivor form of the table
    walk.config(1, 0, 10)
    srch.config(1, 0, 10)
    srch_c.config(1, 0, 10)
    counts = []
    geo = host_geometry(cell)
    found = set()
    sent = set()
    total = 0
    for tti in range(n):
        iq, tr, pl = s.subframe(tti)
        sym = o.ofdm(iq)
        ce, res = o.chest(tti % 10, sym)
        cfi, corr = o.pcfich(tti % 10, sym, ce)
        llr = o.pdcch_llr(tti % 10, cfi, sym, ce)
        ncce = len(llr) // 72
        ref = walk.subframe(tti % 10, cfi, ncce, llr, res.snr_db)
        info = capi.SfInfo()
        info.tti, info.cfi, info.nof_cce, info.snr_db = tti, cfi, ncce, res.snr_db
        pw = np.zeros(ncce, np.float32)
        ltelib.oracle().lteo_cce_power(ltelib.ptr(llr), ncce, ltelib.ptr(pw))
        for i in range(ncce):
            info.cce_power[i] = pw[i]
        nc, Ls = locations(ncce)
        T = oracle_table(o, geo, nc, Ls, llr) if res.snr_db > 6.0 else np.zeros((capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
        got = srch.subframe(info, T)
        comp = srch_c.compact_from_table(info, T)
        counts.append(int(comp["count"][0]))
        got_c = srch_c.subframe_compact(info, comp)
        assert got_c is not None and len(got_c) == len(got) and all(np.array_equal(got_c[k], got[k]) for k in got.dtype.names), \
            (name, tti, "survivor-form walk differs")
        assert len(got) == len(ref), (name, tti, len(got), len(ref))
        for a, b in zip(got, ref):
            assert (int(a["rnti"]), int(a["format"]), int(a["L"]), int(a["ncce"]), int(a["nof_bits"]), int(a["histogram_value"])) == \
                   (b.rnti, b.format, b.L, b.ncce, b.nof_bits, b.histval), (name, tti)
            assert np.array_equal(capi.cand_bits(a["bits"], b.nof_bits), np.frombuffer(bytes(b.bits), np.uint8)[:b.nof_bits])
            found.add((tti, int(a["rnti"]), int(a["ncce"])))
        total += len(got)
        for i in range(tr.nof_dci):
            sent.add((tti, tr.dci[i].rnti, tr.dci[i].ncce))
    walk.save_record()
    ws, ps, cs = walk.stats(), srch.stats(), srch_c.stats()
    assert (ws.nof_decoded_locations, ws.nof_cce, ws.nof_missed_cce, ws.nof_subframes, ws.nof_locations) == \
           (ps.nof_decoded_locations, ps.nof_cce, ps.nof_missed_cce, ps.nof_subframes, ps.nof_locations)
    assert (cs.nof_decoded_locations, cs.nof_cce, cs.nof_missed_cce, cs.nof_subframes, cs.nof_locations) == \
           (ps.nof_decoded_locations, ps.nof_cce, ps.nof_missed_cce, ps.nof_subframes, ps.nof_locations)
    print(name, "survivors per subframe: max", max(counts), "mean", sum(counts) / len(counts))
    assert max(counts) <= capi.COMPACT_CAP
    if name == "low_snr_gate":
        assert total == 0
    else:
        late = {x for x in sent if x[0] >= n // 2}
        assert len(late & found) >= 0.9 * len(late), "search finds %d of %d transmitted DCIs in the second half" % (len(late & found), len(late))


def test_dci_to_grant_matches_oracle(infra):
    """random valid DCIs of every decodable DL format: product ltephy_dci_to_grant == oracle lte_dl_dci_to_grant"""
    S = infra.sim()
    rng = np.random.default_rng(5)
    ncheck = nswap = 0
    for cell in (Cell(100, 2, 3, 2), Cell(50, 1, 9, 1), Cell(25, 2, 100, 2), Cell(75, 2, 5, 2), Cell(15, 1, 7, 1), Cell(15, 2, 8, 2)):
        srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
        for _ in range(1500):
            f = int(rng.choice([1, 2, 4, 6, 7]))
            nb = S.lte_dci_sizeof(C.byref(cell), f)
            bits = rng.integers(0, 2, nb).astype(np.uint8)
            if f == 2:
                bits[0] = 1
            rnti = int(rng.choice([rng.integers(11, 0xFFF3), 0xFFFF, 0xFFFE, rng.integers(1, 11)]))
            sf_idx, cfi, alt = int(rng.integers(0, 10)), int(rng.integers(1, 4)), int(rng.integers(0, 2))
            r0, d, g = ltelib.unpack_and_grant(cell, f, rnti, bits, sf_idx, cfi, alt)
            v = 0
            for i, b in enumerate(bits):
                v |= int(b) << (63 - i)
            row = np.zeros(1, capi.DCI_DTYPE)[0]
            row["rnti"], row["format"], row["nof_bits"], row["bits"] = rnti, f, nb, v
            r1, pg, fl = srch.dci_to_grant(row, sf_idx, cfi, alt)
            assert (r0 == 0) == (r1 == 0), (cell.nof_prb, FORMATS[f], r0, r1, hex(rnti))
            if r0 != 0:
                continue
            ncheck += 1
            assert (pg.nof_re, pg.tx_scheme, pg.nof_tb) == (g.nof_re, g.tx_scheme, g.nof_tb)
            for t in range(2):
                assert (pg.tb[t].enabled, pg.tb[t].tbs if g.tb[t].enabled else 0, pg.tb[t].qm if g.tb[t].enabled else 0) == \
                       (g.tb[t].enabled, g.tb[t].tbs if g.tb[t].enabled else 0, g.tb[t].qm if g.tb[t].enabled else 0)
                if g.tb[t].enabled:
                    assert pg.tb[t].rv == g.tb[t].rv
            if g.nof_tb == 2:        # srsran_ra_tb_t.cw_idx: TB -> codeword, swapped by the DCI 2/2A flag
                assert (pg.tb[0].cw_idx, pg.tb[1].cw_idx) == ((1, 0) if g.cw_swap else (0, 1))
                nswap += g.cw_swap
            else:
                assert all(pg.tb[t].cw_idx == 0 for t in range(2) if g.tb[t].enabled)
            for sl in range(2):
                for prb in range(cell.nof_prb):
                    assert ((pg.prb_mask[sl][prb >> 5] >> (prb & 31)) & 1) == g.prb_mask[sl][prb]
    assert ncheck > 2000 and nswap > 50


def test_ul_dci_to_grant_matches_oracle(infra):
    """random format-0 DCIs: product ltephy_ul_dci_to_grant == oracle lte_dci_unpack + lte_ul_dci_to_grant, restricted to what
    PUSCH_Decoder accepts (valid_prb_ul, src/src/UL_Sniffer_PUSCH.cc:3-10: L_prb = 2^a 3^b 5^c; the product also needs L_prb >= 3)"""
    S = infra.sim()
    S.lte_ul_dci_to_grant.argtypes = [C.POINTER(Cell), C.POINTER(ltelib.Dci), C.c_int, C.POINTER(ltelib.UlGrant)]
    S.lte_ul_valid_prb.argtypes = [C.c_uint32]
    rng = np.random.default_rng(8)
    nok = 0
    for cell in (Cell(100, 2, 3, 2), Cell(50, 1, 9, 1), Cell(25, 2, 100, 2), Cell(75, 2, 5, 2), Cell(15, 1, 2, 1)):
        srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
        nb = S.lte_dci_sizeof(C.byref(cell), 0)
        for it in range(2500):
            bits = rng.integers(0, 2, nb).astype(np.uint8)
            bits[0] = 0
            if it % 4:
                bits[1] = 0                                  # mostly non-hopping
            rnti, q64 = int(rng.integers(11, 0xFFF3)), int(rng.integers(0, 3))     # 16QAM cap / 64QAM table / 256QAM table
            d, g0 = ltelib.Dci(), ltelib.UlGrant()
            r0 = S.lte_dci_unpack(C.byref(cell), 0, rnti, ltelib.ptr(bits), nb, C.byref(d))
            if r0 == 0:
                r0 = S.lte_ul_dci_to_grant(C.byref(cell), C.byref(d), q64, C.byref(g0))
            expect = r0 == 0 and g0.L_prb >= 3 and bool(S.lte_ul_valid_prb(g0.L_prb))
            v = 0
            for i, b in enumerate(bits):
                v |= int(b) << (63 - i)
            row = np.zeros(1, capi.DCI_DTYPE)[0]
            row["sf"], row["rnti"], row["format"], row["nof_bits"], row["bits"] = 7, rnti, 0, nb, v
            r1, g1 = capi.ul_dci_to_grant(srch, row, q64)
            assert (r1 == 0) == expect, (cell.nof_prb, it, r0, r1, g0.L_prb, g0.n_prb)
            if r1 == 0:
                assert (g1.sf, g1.rnti, g1.qm, g1.rv, g1.L_prb, g1.n_prb, g1.n_dmrs2, g1.tbs) == \
                       (7, rnti, g0.qm, g0.rv, g0.L_prb, g0.n_prb, g0.n_dmrs2, g0.tbs)
                nok += 1
    assert nok > 500


def test_finalize_info_and_full_table_decision(infra):
    """host-only helpers of the sharded path: ltephy_finalize_info reproduces the averages / dB / CFO step and is idempotent;
    ltephy_search_needs_full_table reacts to an overfull subframe and to a RAR activation, and only to those"""
    L = capi.load_library()
    capi._bind_search(L)
    rng = np.random.default_rng(12)
    n = 5
    info = (capi.SfInfo * n)()
    for i in range(n):
        for p in range(2):
            for a in range(2):
                info[i].noise[p][a] = float(rng.uniform(1e-3, 2e-3))
                info[i].rsrp[p][a] = float(rng.uniform(0.5, 1.5))
        info[i].cfo_re, info[i].cfo_im = float(rng.uniform(0.5, 1.0)), float(rng.uniform(-0.1, 0.1))
    L.ltephy_finalize_info(info, n, 2, 2)
    first = bytes(info)
    for i in range(n):
        ns = np.float32(0)
        ps = np.float32(0)
        for p in range(2):
            for a in range(2):
                ns = np.float32(ns + np.float32(info[i].noise[p][a]))
                ps = np.float32(ps + np.float32(info[i].rsrp[p][a]))
        assert info[i].noise_avg == np.float32(ns / np.float32(4)) and info[i].rsrp_avg == np.float32(ps / np.float32(4))
        assert abs(info[i].snr_db - 10 * np.log10(float(info[i].rsrp_avg) / float(info[i].noise_avg))) < 1e-4
        assert abs(info[i].cfo - np.arctan2(info[i].cfo_im, info[i].cfo_re) / (2 * np.pi * 7.5)) < 1e-7
    L.ltephy_finalize_info(info, n, 2, 2)
    assert bytes(info) == first
    srch = capi.Search(50, 2, 3, 2)
    comp = np.zeros(n, capi.COMPACT_DTYPE)
    assert L.ltephy_search_needs_full_table(srch.h, comp.ctypes.data_as(C.c_void_p), n) == 0
    comp["count"][3] = capi.COMPACT_CAP + 1
    assert L.ltephy_search_needs_full_table(srch.h, comp.ctypes.data_as(C.c_void_p), n) == 1
    comp["count"][3] = capi.COMPACT_CAP
    assert L.ltephy_search_needs_full_table(srch.h, comp.ctypes.data_as(C.c_void_p), n) == 0
    L.ltephy_search_activate(srch.h, 0x1234, 2, 4)          # activation for another reason does not count
    assert L.ltephy_search_needs_full_table(srch.h, comp.ctypes.data_as(C.c_void_p), n) == 0
    L.ltephy_search_activate(srch.h, 0x2345, 0, 2)          # RAR
    assert L.ltephy_search_needs_full_table(srch.h, comp.ctypes.data_as(C.c_void_p), n) == 1


def test_grants_from_dcis_speculation_and_sharding_filters(infra):
    """ltephy_grants_from_dcis (host only): owner filter sf % mod == rem with local sf = sf // mod; with ltephy_search_speculate_256qam
    a C-RNTI DCI whose two MCS-table readings differ yields two adjacent grants, the second flagged LTEPHY_GRANT_ALT_TABLE; SI / RA /
    paging RNTIs and DCI format 0 never do."""
    S = infra.sim()
    L = capi.load_library()
    capi._bind_search(L)
    cell = Cell(50, 2, 3, 2)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    rng = np.random.default_rng(21)
    n_sf = 6
    info = (capi.SfInfo * n_sf)()
    for i in range(n_sf):
        info[i].tti, info[i].cfi = 20 + i, 2
    rows = []
    for sf in range(n_sf):
        for rnti, f in ((0xFFFF, 2), (0x0004, 2), (int(rng.integers(0x100, 0xFFF0)), 1), (int(rng.integers(0x100, 0xFFF0)), 7), (int(rng.integers(0x100, 0xFFF0)), 0)):
            nb = S.lte_dci_sizeof(C.byref(cell), f)
            for _ in range(50):                                  # draw until the 64QAM-table reading is a valid grant (format 0 excepted)
                bits = rng.integers(0, 2, nb).astype(np.uint8)
                bits[0] = 1 if f == 2 else (0 if f == 0 else bits[0])
                r0, d, g = ltelib.unpack_and_grant(cell, f, rnti, bits, info[sf].tti % 10, 2, 0) if f else (0, None, None)
                if f == 0 or (r0 == 0 and g.tb[0].tbs > 0):
                    break
            v = 0
            for k, b in enumerate(bits):
                v |= int(b) << (63 - k)
            rows.append((sf, rnti, f, nb, v))
    dcis = np.zeros(len(rows), capi.DCI_DTYPE)
    for i, (sf, rnti, f, nb, v) in enumerate(rows):
        dcis[i]["sf"], dcis[i]["rnti"], dcis[i]["format"], dcis[i]["nof_bits"], dcis[i]["bits"] = sf, rnti, f, nb, v
    grants = (capi.Grant * (4 * len(rows)))()
    gidx = np.zeros(4 * len(rows), np.uint32)
    ng = C.c_uint32(0)

    def run(mod, rem):
        assert L.ltephy_grants_from_dcis(srch.h, info, dcis.ctypes.data_as(C.c_void_p), len(rows), mod, rem, grants, gidx.ctypes.data_as(C.c_void_p), len(gidx),
                                         C.byref(ng)) == 0
        return [(int(gidx[i]) & 0x7FFFFFFF, int(gidx[i]) >> 31, int(grants[i].sf), int(grants[i].rnti), int(grants[i].tb[0].qm), int(grants[i].tb[0].tbs)) for i in range(ng.value)]
    plain = run(1, 0)
    assert all(a == 0 for _, a, *_ in plain) and all(rows[di][2] != 0 for di, *_ in plain)      # no alternates, no format 0
    assert len(plain) >= 3 * n_sf
    halves = [run(2, r) for r in range(2)]
    assert sorted([(di, a) for h in halves for di, a, *_ in h]) == sorted([(di, a) for di, a, *_ in plain])
    for r, h in enumerate(halves):
        assert all(rows[di][0] % 2 == r and sf == rows[di][0] // 2 for di, a, sf, *_ in h)
    L.ltephy_search_speculate_256qam(srch.h, 1)
    spec = run(1, 0)
    alts = [x for x in spec if x[1] == 1]
    assert alts and [x for x in spec if x[1] == 0] == plain
    for k, x in enumerate(spec):
        if x[1] == 1:
            di = x[0]
            assert 0x000A < rows[di][1] < 0xFFF4                  # user RNTIs only
            assert spec[k - 1][0] == di and spec[k - 1][1] == 0  # adjacent to its primary, after it
            assert (x[4], x[5]) != (spec[k - 1][4], spec[k - 1][5])
    # UL mode (PDSCH_Decoder::decode_ul_mode, DL_Sniffer_PDSCH.cc:362-457): the RA-RNTI DCIs and format 1 / 1A of everything but the SI-RNTI, 64QAM table only
    L.ltephy_search_set_ul_mode(srch.h, 1, 0)
    ulm = run(1, 0)
    assert all(a == 0 for _, a, *_ in ulm)
    assert sorted(di for di, *_ in ulm) == sorted(di for di, *_ in plain if rows[di][1] != 0xFFFF and rows[di][2] in (1, 2))
    assert {rows[di][1] for di, *_ in ulm} >= {0x0004} and 0xFFFF not in {rows[di][1] for di, *_ in ulm}
    L.ltephy_search_set_ul_mode(srch.h, 0, 0)
    assert run(1, 0) == spec
    L.ltephy_si_format1c_rv.argtypes = [C.c_uint32]
    assert [L.ltephy_si_format1c_rv(10 * sfn + 5) for sfn in range(10)] == [int(np.ceil(1.5 * ((sfn // 2) % 4))) % 4 for sfn in range(10)] == [0, 0, 2, 2, 3, 3, 1, 1, 0, 0]


def test_empty_and_degenerate_inputs(infra):
    """host entry points on empty batches, an invalid CFI, a subframe below the 6 dB gate and null pointers: defined results, no crash"""
    L = capi.load_library()
    capi._bind_search(L)
    srch = capi.Search(100, 2, 1, 2)
    dcis = np.zeros(8, capi.DCI_DTYPE)
    nd = C.c_uint32(77)
    info = (capi.SfInfo * 2)()
    cands = np.zeros((2, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
    comp = np.zeros(2, capi.COMPACT_DTYPE)
    assert L.ltephy_search_batch(srch.h, info, cands.ctypes.data_as(C.c_void_p), 0, dcis.ctypes.data_as(C.c_void_p), 8, C.byref(nd)) == 0 and nd.value == 0
    assert L.ltephy_search_batch_compact(srch.h, info, comp.ctypes.data_as(C.c_void_p), None, 0, dcis.ctypes.data_as(C.c_void_p), 8, C.byref(nd)) == 0 and nd.value == 0
    assert L.ltephy_search_batch(None, info, cands.ctypes.data_as(C.c_void_p), 1, dcis.ctypes.data_as(C.c_void_p), 8, C.byref(nd)) == -2
    # cfi 0 / 4 and low SNR: the subframe is counted but nothing is walked (DCISearch.cc:569)
    for cfi, snr in ((0, 20.0), (4, 20.0), (2, 5.9)):
        info[0].cfi, info[0].snr_db, info[0].tti = cfi, snr, 3
        before = srch.stats().nof_subframes
        assert len(srch.subframe(info[0], cands[0])) == 0
        c = srch.compact_from_table(info[0], cands[0])
        assert len(srch.subframe_compact(info[0], c)) == 0
        assert srch.stats().nof_subframes == before + 2
        if cfi in (0, 4):
            assert int(c["count"][0]) == 0 and not c["loc"]["mask"].any()
    # an all-zero table at good SNR: every entry is "undecoded", nothing is accepted, statistics still advance
    info[0].cfi, info[0].snr_db = 3, 20.0
    for i in range(87):
        info[0].cce_power[i] = 1.0
    assert len(srch.subframe(info[0], cands[0])) == 0
    # grants from no DCIs
    grants = (capi.Grant * 4)()
    gidx = np.zeros(4, np.uint32)
    ng = C.c_uint32(9)
    assert L.ltephy_grants_from_dcis(srch.h, info, dcis.ctypes.data_as(C.c_void_p), 0, 1, 0, grants, gidx.ctypes.data_as(C.c_void_p), 4, C.byref(ng)) == 0 and ng.value == 0
    assert L.ltephy_grants_from_dcis(srch.h, info, dcis.ctypes.data_as(C.c_void_p), 0, 0, 0, grants, gidx.ctypes.data_as(C.c_void_p), 4, C.byref(ng)) == -2   # mod 0
    # an all-zero DL DCI (RIV 0, MCS 0): converts or is rejected, but never crashes; format index out of range is rejected
    row = np.zeros(1, capi.DCI_DTYPE)[0]
    row["rnti"], row["format"], row["nof_bits"] = 0x1234, 2, 28
    r, g, f = srch.dci_to_grant(row, 0, 2, 0)
    assert r in (0, -1)
    row["format"] = 9
    r, g, f = srch.dci_to_grant(row, 0, 2, 0)
    assert r != 0


def test_ul_decode_plan_follows_pusch_decoder(infra):
    """ltephy_ul_decode_plan: the attempts of PUSCH_Decoder::decode (reference src/src/UL_Sniffer_PUSCH.cc:417-570) per MCS range and MCSTracking answer,
    behind investigate_valid_ul_grant (:894-918).  Expectations written out from the reference's branches:
      MCS 21..28: 16QAM_MAX -> [16]; 64QAM_MAX -> [64]; 256QAM_MAX -> [256]; unknown -> [16, 64, 256]
      MCS  0..20: 16QAM_MAX / 64QAM_MAX -> [16]; 256QAM_MAX -> [256]; unknown -> [16, 256]
      MCS 29..31 (no size), L_prb that is no DFT size, RNTI 0: nothing
    MCS 28 has no row in Table 8.6.1-3 (I_TBS 34): that reading is dropped (in the reference it runs with tbs = -1 and cannot pass)."""
    S = infra.sim()
    cell = Cell(50, 2, 3, 2)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    nb = S.lte_dci_sizeof(C.byref(cell), 0)
    N = cell.nof_prb
    rivb = int(np.ceil(np.log2(N * (N + 1) / 2)))

    def dci(L, start, mcs, rnti=0x1234):
        riv = N * (L - 1) + start if L - 1 <= N // 2 else N * (N - L + 1) + (N - 1 - start)
        fields = [(0, 1), (0, 1), (riv, rivb), (mcs, 5), (1, 1), (0, 2), (3, 3), (0, 1)]
        v, pos = 0, 0
        for val, w in fields:
            v |= val << (64 - pos - w)
            pos += w
        row = np.zeros(1, capi.DCI_DTYPE)
        row["rnti"], row["format"], row["nof_bits"], row["bits"], row["L"] = rnti, 0, nb, v, 2
        return row[0]
    M16, M64, M256, UNK = 0, 1, 2, 3
    want = {}
    for mcs in range(32):
        if mcs > 28:
            want[mcs] = {m: [] for m in (M16, M64, M256, UNK)}
        elif mcs > 20:
            want[mcs] = {M16: [0], M64: [1], M256: [2], UNK: [0, 1, 2]}
        else:
            want[mcs] = {M16: [0], M64: [0], M256: [2], UNK: [0, 2]}
    for mcs in range(32):
        for mod in (M16, M64, M256, UNK):
            plan = capi.ul_decode_plan(srch, dci(10, 7, mcs), mod)
            exp = [r for r in want[mcs][mod] if not (r == 2 and mcs == 28)]
            assert [r for r, _ in plan] == exp, (mcs, mod, plan)
            for r, g in plan:
                rc, gd = capi.ul_dci_to_grant(srch, dci(10, 7, mcs), r)
                assert rc == 0 and bytes(g) == bytes(gd) and (g.L_prb, g.n_prb, g.rnti) == (10, 7, 0x1234)
            if mcs in range(21, 28) and mod == UNK:           # the three readings differ where they should
                assert [g.qm for _, g in plan][:2] == [4, 6] and plan[2][1].qm in (6, 8)
    assert capi.ul_decode_plan(srch, dci(7, 0, 10), UNK) == []                 # valid_prb_ul[7] is false
    assert capi.ul_decode_plan(srch, dci(10, 7, 10, rnti=0), UNK) == []
    with pytest.raises(ValueError):
        capi.ul_decode_plan(srch, dci(10, 7, 10), 4)


def test_ul_grants_from_dcis_follows_subframe_worker(infra):
    """ltephy_ul_grants_from_dcis: the UL-mode bookkeeping of SubframeWorker (reference src/src/SubframeWorker.cc:296-345) for a batch --
    PUSCH 4 subframes after its DCI-0 (ULSchedule::get_ul_tti), nof_ack = transport blocks of the same RNTI's downlink DCI in the same subframe (last one
    wins), CSI request -> ri_len 1 + the UE's CQI size, per-RNTI beta offsets / MCS-table knowledge with a default entry, attempts in PUSCH_Decoder's order."""
    S = infra.sim()
    cell = Cell(50, 2, 3, 2)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    N = cell.nof_prb
    rivb = int(np.ceil(np.log2(N * (N + 1) / 2)))
    nb0 = S.lte_dci_sizeof(C.byref(cell), 0)
    rng = np.random.default_rng(8)
    A, B, Cc, D = 0x1001, 0x1002, 0x1003, 0x1004

    def dci0(sf, rnti, L, start, mcs, cqi_req):
        riv = N * (L - 1) + start if L - 1 <= N // 2 else N * (N - L + 1) + (N - 1 - start)
        v, pos = 0, 0
        for val, w in [(0, 1), (0, 1), (riv, rivb), (mcs, 5), (1, 1), (0, 2), (3, 3), (cqi_req, 1)]:
            v |= val << (64 - pos - w)
            pos += w
        return (sf, rnti, 0, nb0, v)

    def dl(sf, rnti, f, want_tb):
        nb = S.lte_dci_sizeof(C.byref(cell), f)
        for _ in range(5000):
            bits = rng.integers(0, 2, nb).astype(np.uint8)
            r0, d, g = ltelib.unpack_and_grant(cell, f, rnti, bits, (20 + sf) % 10, 2, 0)
            if r0 == 0 and g.nof_tb == want_tb and g.tb[0].tbs > 0:
                break
        else:
            raise AssertionError("no payload found")
        v = 0
        for k, b in enumerate(bits):
            v |= int(b) << (63 - k)
        return (sf, rnti, f, nb, v)
    rows = [dl(0, A, 1, 1), dl(0, B, 6, 2), dl(0, B, 1, 1), dci0(0, A, 10, 7, 22, 0), dci0(0, B, 12, 20, 5, 0), dci0(0, Cc, 6, 2, 15, 1),
            dl(1, Cc, 6, 2), dci0(1, Cc, 8, 0, 27, 1), dci0(1, D, 7, 0, 3, 0), dci0(1, A, 10, 7, 30, 0),
            dl(2, A, 6, 2), dci0(3, A, 10, 7, 22, 0)]
    dcis = np.zeros(len(rows), capi.DCI_DTYPE)
    for i, (sf, rnti, f, nb, v) in enumerate(rows):
        dcis[i]["sf"], dcis[i]["rnti"], dcis[i]["format"], dcis[i]["nof_bits"], dcis[i]["bits"] = sf, rnti, f, nb, v
    info = (capi.SfInfo * 4)()
    for i in range(4):
        info[i].tti, info[i].cfi = 20 + i, 2
    ue = [capi.UlUeCfg(rnti=A, mcs_mod=1, I_offset_ack=9, I_offset_cqi=6, I_offset_ri=5, cqi_len=0), capi.UlUeCfg(rnti=0, mcs_mod=3, I_offset_ack=10, I_offset_cqi=8, I_offset_ri=11, cqi_len=20)]
    out = capi.ul_grants_from_dcis(srch, info, dcis, ue)
    got = [(di, rd, g.sf, g.rnti, g.nof_ack, g.ri_len, g.cqi_len, (g.I_offset_ack, g.I_offset_cqi, g.I_offset_ri), g.L_prb, g.qm) for di, rd, g in out]
    dflt, ofsA = (10, 8, 11), (9, 6, 5)
    assert got == [
        (3, 1, 4, A, 1, 0, 0, ofsA, 10, 6),                               # A: 64QAM known, MCS 22 -> one attempt; one downlink TB in its subframe
        (4, 0, 4, B, 1, 0, 0, dflt, 12, 2), (4, 2, 4, B, 1, 0, 0, dflt, 12, 2),      # B: unknown, MCS 5 -> 16QAM and 256QAM readings; last downlink DCI (1 TB) wins
        (5, 0, 4, Cc, 0, 1, 20, dflt, 6, 4), (5, 2, 4, Cc, 0, 1, 20, dflt, 6, 6),    # C: no downlink DCI in subframe 0; CSI request -> RI bit + 20 CQI bits
        (7, 0, 5, Cc, 2, 1, 20, dflt, 8, 4), (7, 1, 5, Cc, 2, 1, 20, dflt, 8, 6), (7, 2, 5, Cc, 2, 1, 20, dflt, 8, 8),   # MCS 27 unknown: 16, 64, 256; two TBs
        # D: 7 PRB is no DFT size; A at MCS 30: no size -> neither is decoded (investigate_valid_ul_grant)
        (11, 1, 7, A, 0, 0, 0, ofsA, 10, 6)]                              # the two-TB DCI of A is in subframe 2, not 3; sf 7 belongs to the next uplink batch
    assert capi.ul_grants_from_dcis(srch, info, dcis[:3]) == [] and capi.ul_grants_from_dcis(srch, info, dcis[:0]) == []
    nodef = capi.ul_grants_from_dcis(srch, info, dcis[3:4])               # no UE table at all: unknown table, 10 / 8 / 11
    assert [(rd, g.I_offset_ack, g.I_offset_cqi, g.I_offset_ri) for _, rd, g in nodef] == [(0, 10, 8, 11), (1, 10, 8, 11), (2, 10, 8, 11)]


def test_rar_unpack_known_answers_from_the_references_captures(infra):
    """ltephy_rar_unpack on the two Random Access Responses in the reference's own example captures (pcap_file_example/ltesniffer_dl_mode.pcap, record of
    RA-RNTI 2 at tti 5636; ltesniffer_ul_mode.pcap, tti 8516), quoted here.  In the UL-mode capture the msg 3 the grant schedules is there too: an uplink
    record of RNTI 70 exactly 6 subframes later (ULSchedule::get_rar_ul_tti) with 7 bytes = the 56-bit transport block of MCS 0 on 3 PRB -- what the grant
    decodes to.  The records are read from the sample of that capture in tests/golden."""
    srch = capi.Search(100, 2, 1, 2)
    for hexpdu, rapid in (("620011940c004600000000", 34), ("720011940c004600000000", 50)):
        r, rars, bo = capi.rar_unpack(srch, bytes.fromhex(hexpdu))
        assert r == 0 and bo == -1 and len(rars) == 1
        x = rars[0]
        assert (x.rapid, x.ta, x.t_crnti, x.hopping_flag, x.tpc, x.ul_delay, x.cqi_request, x.valid) == (rapid, 1, 70, 0, 3, 0, 0, 1)
        g = x.grant
        assert (g.rnti, g.L_prb, g.n_prb, g.n_prb_slot1, g.tbs, g.qm, g.rv, g.n_dmrs2, g.sf) == (70, 3, 2, 2, 56, 2, 0, 0, 0)
    import test_sinks
    _, recs = test_sinks.parse(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_ltesniffer_ul_mode_sample.pcap"))
    rar = [x for x in recs if x["rnti_type"] == 2]
    assert len(rar) == 1 and rar[0]["pdu"].hex() == "720011940c004600000000"
    r, rars, _ = capi.rar_unpack(srch, rar[0]["pdu"])
    msg3 = [x for x in recs if x["direction"] == 0 and x["rnti"] == rars[0].t_crnti and x["tti"] == (rar[0]["tti"] + 6) % 10240]
    assert len(msg3) == 1 and len(msg3[0]["pdu"]) * 8 == rars[0].grant.tbs
    # a backoff-indicator subheader, then two RARs; the second grant hops and asks for CSI
    g2 = (1 << 19) | (((100 * 5 + 30) & 0x3FF) << 9) | (7 << 5) | (5 << 2) | (1 << 1) | 1
    pdu = bytes([0x80 | 0x09, 0xC0 | 3, 0x40 | 61]) + bytes([0x12, 0x31, 0x94, 0x0C, 0xAB, 0xCD]) + bytes([0x7F, 0xF0 | (g2 >> 16), (g2 >> 8) & 255, g2 & 255, 0x00, 0x63]) + b"\0\0"
    r, rars, bo = capi.rar_unpack(srch, pdu)
    assert r == 0 and bo == 9 and [(x.rapid, x.t_crnti, x.ta) for x in rars] == [(3, 0xABCD, 0x123), (61, 0x63, 0x7FF)]
    assert (rars[1].hopping_flag, rars[1].tpc, rars[1].ul_delay, rars[1].cqi_request) == (1, 5, 1, 1)
    riv = (100 * 5 + 30) & 0x3FF                                        # the 10 allocation bits as they are (falcon_dci.c:672-680)
    L, S = riv // 100 + 1, riv % 100
    assert rars[1].valid == 1 and (rars[1].grant.L_prb, rars[1].grant.n_prb, rars[1].grant.qm) == (L, S, 2)
    assert rars[1].grant.n_prb_slot1 == (S - 25 if S >= 25 else 100 + S - 25)          # hopping flag read as hop value 1: -1/4 of the band (n_rb_ho = 0)
    # malformed: no subheader end, RAR body cut short; more RARs than the caller has room for
    assert capi.rar_unpack(srch, bytes([0xC1]))[0] == -1 and capi.rar_unpack(srch, bytes([0x41, 0, 0, 0]))[0] == -1 and capi.rar_unpack(srch, b"")[0] == -1
    assert capi.rar_unpack(srch, pdu, max_out=1)[0] == -2


def test_ul_default_cqi_report_size(infra):
    """without a UE entry a CSI request is sized as the reference's default report (subband CQI configured by higher layers, 4 + 2 N bits)"""
    L = capi.load_library()
    capi._bind_search(L)
    assert [L.ltephy_ul_cqi_len(n, 3) for n in (15, 25, 50, 75, 100)] == [12, 18, 22, 24, 30] and L.ltephy_ul_cqi_len(50, 0) == 4
    assert L.ltephy_ul_cqi_len(6, 3) == -2 and L.ltephy_ul_cqi_len(50, 1) == -2
    srch = capi.Search(50, 2, 3, 2)
    N, rivb = 50, 11
    v, pos = 0, 0
    for val, w in [(0, 1), (0, 1), (N * 5 + 2, rivb), (15, 5), (1, 1), (0, 2), (3, 3), (1, 1)]:
        v |= val << (64 - pos - w)
        pos += w
    dcis = np.zeros(1, capi.DCI_DTYPE)
    dcis[0]["rnti"], dcis[0]["format"], dcis[0]["nof_bits"], dcis[0]["bits"] = 0x2222, 0, 27, v
    info = (capi.SfInfo * 1)()
    info[0].tti, info[0].cfi = 20, 2
    out = capi.ul_grants_from_dcis(srch, info, dcis)
    assert [(rd, g.ri_len, g.cqi_len) for _, rd, g in out] == [(0, 1, 22), (2, 1, 22)]


def test_ul_uci_layout_matches_oracle_side_and_formula(infra):
    """ltephy_ul_uci_layout (= what ltephy_submit_ul reserves, ltehost::uci_layout) on 4 000 random grants against the simulator / oracle's lte_uci_layout (an
    independent C restatement) and against 36.212 5.2.2.6 evaluated in Python float32: Q' = min(ceil(O M_sc N_symb beta / sum K_r), 4 M_sc) for HARQ-ACK and
    RI, min(ceil((O + L) M_sc N_symb beta / sum K_r), M_sc N_symb - Q'_RI) with L = 8 from 12 bits on for CQI, G = (M_sc N_symb - Q'_CQI - Q'_RI) Qm"""
    import sys as _sys
    _sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import check_tables
    L = capi.load_library()
    capi._bind_search(L)
    B_ACK = [2.0, 2.5, 3.125, 4.0, 5.0, 6.25, 8.0, 10.0, 12.625, 15.875, 20.0, 31.0, 50.0, 80.0, 126.0]
    B_RI = [1.25, 1.625, 2.0, 2.5, 3.125, 4.0, 5.0, 6.25, 8.0, 10.0, 12.625, 15.875, 20.0]
    B_CQI = [None, None, 1.125, 1.25, 1.375, 1.625, 1.75, 2.0, 2.25, 2.5, 2.875, 3.125, 3.5, 4.0, 5.0, 6.25]
    _, _, tbs_tab, _ = check_tables.load()
    T = np.array(tbs_tab).reshape(34, 110)
    rng = np.random.default_rng(77)
    valid_L = [l for l in range(1, 101) if ltelib.sim().lte_ul_valid_prb(l)]
    f32 = np.float32
    n = 0
    for _ in range(4000):
        Lp = int(rng.choice(valid_L))
        qm = int(rng.choice([2, 4, 6, 8]))
        tbs = int(T[int(rng.integers(0, 27)), Lp - 1])
        nack, ri, cqi = int(rng.integers(0, 3)), int(rng.integers(0, 2)), int(rng.choice([0, 0, 4, 11, 12, 20, 30, 64]))
        ia, ir, ic = int(rng.integers(0, 15)), int(rng.integers(0, 13)), int(rng.integers(2, 16))
        g = capi.UlGrant(rnti=1, qm=qm, L_prb=Lp, n_prb=0, tbs=tbs, nof_ack=nack, ri_len=ri, cqi_len=cqi, I_offset_ack=ia, I_offset_cqi=ic, I_offset_ri=ir)
        out = [C.c_uint32(0) for _ in range(4)]
        assert L.ltephy_ul_uci_layout(C.byref(g), *[C.byref(o) for o in out]) == 0
        got = tuple(o.value for o in out)
        og = ltelib.UlGrant(rnti=1, L_prb=Lp, qm=qm, tbs=tbs, nof_ack=nack, ri_len=ri, cqi_len=cqi, I_offset_ack=ia, I_offset_ri=ir, I_offset_cqi=ic)
        ol = ltelib.uci_layout(og)
        assert got == (ol.Qp_ack, ol.Qp_ri, ol.Qp_cqi, ol.G), (Lp, qm, tbs, nack, ri, cqi)
        Cn, Kp, Km, Cp, Cm, F = check_tables.segm(tbs)
        ksum = f32(Cp * Kp + Cm * Km)
        M = 12 * Lp
        qp = lambda O, b: int(np.ceil(f32(O) * f32(M) * f32(12) * f32(b) / ksum))
        q_ri = min(qp(ri, B_RI[ir]), 4 * M) if ri else 0
        q_ack = min(qp(nack, B_ACK[ia]), 4 * M) if nack else 0
        q_cqi = min(qp(cqi + (8 if cqi > 11 else 0), B_CQI[ic]), 12 * M - q_ri) if cqi else 0
        assert got == (q_ack, q_ri, q_cqi, (12 * M - q_cqi - q_ri) * qm), (Lp, qm, tbs, nack, ri, cqi, got)
        n += bool(nack or ri or cqi)
    assert n > 2500
    g = capi.UlGrant(rnti=1, qm=2, L_prb=10, tbs=1000, cqi_len=20, I_offset_cqi=1)
    assert L.ltephy_ul_uci_layout(C.byref(g), None, None, None, None) == -2           # reserved beta offset index
