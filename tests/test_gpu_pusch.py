"""GPU parity of the PUSCH path (pytest -m gpu): UL OFDM demodulation and every PUSCH grant's channel estimate
figures, transport-block bytes and CRC against the CPU oracle, bit-exact; ground truth from the synthetic UEs."""
import numpy as np
import pytest
import ltelib
from ltelib import Cell, Sim, Oracle, UlCfg
from helpers import feq, describe_mismatch
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cell,snr,nsf,ngr,table", [(Cell(50, 1, 17, 1), 25.0, 3, 4, 1), (Cell(100, 2, 301, 2), 23.0, 3, 6, 1), (Cell(25, 1, 5, 1), 20.0, 2, 2, 1),
                                                      (Cell(50, 1, 9, 1), 34.0, 3, 4, 2),      # table 2: 36.213 Table 8.6.1-3, Qm up to 8
                                                      (Cell(15, 1, 6, 1), 22.0, 3, 2, 1), (Cell(15, 2, 7, 2), 24.0, 2, 3, 2),
                                                      (Cell(75, 1, 18, 1), 23.0, 3, 4, 1), (Cell(75, 2, 19, 2), 30.0, 2, 5, 2)])
def test_pusch_bit_exact(infra, phylib, cell, snr, nsf, ngr, table):
    """at 75 PRB the first subframe carries one grant of the whole band (75 = 3 * 5^2 PRB: the largest three- and five-point DFT steps)"""
    s = Sim(cell=cell, seed=21, snr_db=snr, nof_ues=1, chan_delay=3)
    o = Oracle(cell)
    rng = np.random.default_rng(cell.nof_prb)
    ucfg = UlCfg(n_dmrs1=3, delta_ss=2)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=nsf)
    phy.set_ul_cfg(3, 2)
    iq = np.zeros((nsf, s.sf_len), np.complex64)
    tti = np.arange(4, 4 + nsf, dtype=np.uint32)
    grants_o, pls, offs, grants_p = [], [], [], []
    for i in range(nsf):
        full = i == 0 and cell.nof_prb == 75
        gr = ltelib.make_ul_grants(cell, rng, 1 if full else ngr, table=table, min_prb=cell.nof_prb if full else 3)
        assert not full or (gr[0].L_prb, gr[0].n_prb) == (75, 0)
        x, pl, off = ltelib.sim_ul_subframe(s, int(tti[i]), ucfg, gr)
        iq[i] = x
        grants_o.append(gr), pls.append(pl), offs.append(off)
        for g in gr:
            grants_p.append(capi.UlGrant(sf=i, rnti=g.rnti, qm=g.qm, rv=g.rv, L_prb=g.L_prb, n_prb=g.n_prb, n_dmrs2=g.n_dmrs2, tbs=g.tbs))
    res, ch, payload = phy.decode_ul(iq, tti, grants_p)
    ulsym = phy.tap(capi.TAP_UL_SYM, (nsf, 14 * phy.nsc), np.complex64)
    k = 0
    nok = 0
    for i in range(nsf):
        sym, ref = ltelib.oracle_ul(o, ucfg, int(tti[i]), grants_o[i], iq[i])
        assert feq(ulsym[i], sym), describe_mismatch(ulsym[i], sym, "UL grid sf %d" % i)
        for g, (r, opl, ocrc, och, _), off in zip(grants_o[i], ref, offs[i]):
            assert r == 0
            rr = res[k]
            nby = g.tbs // 8
            assert (ch[k].noise, ch[k].rsrp, ch[k].snr_db) == (och.noise, och.rsrp, och.snr_db), (k, ch[k].noise, och.noise)
            assert rr.crc == ocrc and rr.payload_len == nby
            assert np.array_equal(payload[rr.payload_off:rr.payload_off + nby], opl[:nby])
            if rr.crc:
                assert np.array_equal(payload[rr.payload_off:rr.payload_off + nby], pls[i][off:off + nby])
                nok += 1
            k += 1
    assert nok >= k - 1
    phy.close()


def _to_capi(i, g):
    return capi.UlGrant(sf=i, rnti=g.rnti, qm=g.qm, rv=g.rv, L_prb=g.L_prb, n_prb=g.n_prb, n_dmrs2=g.n_dmrs2, tbs=g.tbs,
                        n_prb_slot1=g.n_prb_slot1 if g.hop else g.n_prb, flags=capi.UL_FLAG_SLOT1, nof_ack=g.nof_ack, ri_len=g.ri_len, cqi_len=g.cqi_len,
                        I_offset_ack=g.I_offset_ack, I_offset_ri=g.I_offset_ri, I_offset_cqi=g.I_offset_cqi)


def _run_ul_case(cell, ucfg, mutate, nsf=2, ngr=3, snr=30.0, seed=31, min_prb=3, table=1, llr_check=True):
    """sim -> product (GPU) and oracle for mutated grants: soft bits, chest figures, CRC and payload bit-exact; returns the number of CRC passes"""
    s = Sim(cell=cell, seed=seed, snr_db=snr, nof_ues=1)
    o = Oracle(cell)
    rng = np.random.default_rng(seed)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=nsf)
    phy.set_ul_cfg(ucfg.n_dmrs1, ucfg.delta_ss, ucfg.group_hopping, ucfg.seq_hopping)
    iq = np.zeros((nsf, s.sf_len), np.complex64)
    tti = np.arange(3, 3 + nsf, dtype=np.uint32)
    grants_o, pls, offs, grants_p = [], [], [], []
    for i in range(nsf):
        gr = ltelib.make_ul_grants(cell, rng, ngr, table=table, min_prb=min_prb)
        for g in gr:
            mutate(g, rng)
        x, pl, off = ltelib.sim_ul_subframe(s, int(tti[i]), ucfg, gr)
        iq[i] = x
        grants_o.append(gr), pls.append(pl), offs.append(off)
        grants_p += [_to_capi(i, g) for g in gr]
    res, ch, payload = phy.decode_ul(iq, tti, grants_p)
    tot = sum((ltelib.uci_layout(g).G + 7) & ~7 for gr in grants_o for g in gr)
    llr = phy.tap(capi.TAP_PDSCH_LLR, (tot,), np.int16) if llr_check else None
    k = nok = 0
    lo = 0
    for i in range(nsf):
        _, ref = ltelib.oracle_ul(o, ucfg, int(tti[i]), grants_o[i], iq[i], want_llr=True)
        for g, (r, opl, ocrc, och, ollr), off in zip(grants_o[i], ref, offs[i]):
            assert r == 0
            rr, nby, G = res[k], g.tbs // 8, ltelib.uci_layout(g).G
            if llr_check:
                assert np.array_equal(llr[lo:lo + G], ollr[:G]), describe_mismatch(llr[lo:lo + G], ollr[:G], "soft bits of grant %d" % k)
                lo += (G + 7) & ~7
            assert (ch[k].noise, ch[k].rsrp, ch[k].snr_db) == (och.noise, och.rsrp, och.snr_db), (k, ch[k].noise, och.noise)
            assert abs(ch[k].ta_us - och.ta_us) < 1e-3, (ch[k].ta_us, och.ta_us)       # atan2f of bit-identical sums, host libm on both sides
            assert abs(och.ta_us - g.ta_us) < 0.05
            assert rr.crc == ocrc and rr.payload_len == nby
            assert np.array_equal(payload[rr.payload_off:rr.payload_off + nby], opl[:nby])
            if rr.crc:
                assert np.array_equal(payload[rr.payload_off:rr.payload_off + nby], pls[i][off:off + nby])
                nok += 1
            k += 1
    phy.close()
    return nok, k


def test_pusch_uci_multiplexed(infra, phylib):
    """HARQ-ACK / RI / CQI multiplexed with the UL-SCH (36.212 5.2.2.6-8; PUSCH_Decoder::decode, src/src/UL_Sniffer_PUSCH.cc:429-450)"""
    cell = Cell(50, 1, 23, 1)
    ucfg = UlCfg(n_dmrs1=4, delta_ss=7)
    combos = [dict(nof_ack=1, I_offset_ack=9), dict(nof_ack=2, I_offset_ack=10, ri_len=1, I_offset_ri=8), dict(cqi_len=4, I_offset_cqi=8),
              dict(cqi_len=30, I_offset_cqi=6, ri_len=1, I_offset_ri=5, nof_ack=2, I_offset_ack=5), dict(cqi_len=11, I_offset_cqi=15, nof_ack=2, I_offset_ack=14)]
    for ci, cmb in enumerate(combos):
        def mut(g, rng):
            for kk, v in cmb.items():
                setattr(g, kk, v)
        nok, k = _run_ul_case(cell, ucfg, mut, seed=40 + ci, table=1 + (ci & 1))
        assert nok == k, (cmb, nok, k)


def test_pusch_hopping_group_hopping_timing(infra, phylib):
    """type-1 hopping (slot 1 elsewhere), DMRS group / sequence hopping, timing offsets: product == oracle, estimate == truth; at 50 and at 75 PRB"""
    cell = Cell(50, 1, 301, 1)
    import ctypes as C
    S = ltelib.sim()
    S.lte_ul_valid_prb.argtypes = [C.c_uint32]

    def hop(g, rng):
        lim = cell.nof_prb - g.L_prb
        g.hop, g.n_prb_slot1 = 1, int((g.n_prb + 17) % (lim + 1))
        g.ta_us = float(rng.uniform(-0.8, 0.8))
    for gh, sh in ((0, 0), (1, 0), (0, 1)):
        nok, k = _run_ul_case(cell, UlCfg(n_dmrs1=2, delta_ss=11, group_hopping=gh, seq_hopping=sh), hop, ngr=1, nsf=3, seed=60 + 2 * gh + sh, min_prb=6)
        assert nok == k == 3

    def ta_only(g, rng):
        g.ta_us = float(rng.uniform(-1.0, 1.0))
    nok, k = _run_ul_case(Cell(100, 1, 4, 1), UlCfg(n_dmrs1=0, delta_ss=0, group_hopping=1), ta_only, ngr=5, nsf=2, seed=70)
    assert nok == k
    cell = Cell(75, 1, 302, 1)                      # hop() reads the cell at call time
    nok, k = _run_ul_case(cell, UlCfg(n_dmrs1=1, delta_ss=5, group_hopping=1), hop, ngr=2, nsf=2, seed=71, min_prb=5)
    assert nok == k == 4


def test_pusch_every_dft_size(infra, phylib):
    """all 34 allocation sizes of valid_prb_ul from 3 PRB up (src/src/UL_Sniffer_PUSCH.cc:3-10): the mixed-radix IDFT equals the oracle's bit for bit"""
    cell = Cell(100, 1, 77, 1)
    import ctypes as C
    S = ltelib.sim()
    S.lte_ul_valid_prb.argtypes = [C.c_uint32]
    S.lte_ul_dci_to_grant.argtypes = [C.POINTER(Cell), C.POINTER(ltelib.Dci), C.c_int, C.POINTER(ltelib.UlGrant)]
    sizes = [L for L in range(3, 101) if S.lte_ul_valid_prb(L)]
    assert len(sizes) == 32 and sizes[-1] == 100
    ucfg = UlCfg(n_dmrs1=5, delta_ss=3)
    s = Sim(cell=cell, seed=8, snr_db=30.0, nof_ues=1)
    o = Oracle(cell)
    phy = capi.LtePhy(cell.nof_prb, 1, cell.cell_id, 1, max_subframes=1)
    phy.set_ul_cfg(5, 3)
    rng = np.random.default_rng(8)
    for n, L in enumerate(sizes):
        d = ltelib.Dci()
        st = int(rng.integers(0, 101 - L))
        d.format, d.rnti, d.alloc_type = 0, 0x1000 + L, 2
        d.riv = 100 * (L - 1) + st if (L - 1) <= 50 else 100 * (100 - L + 1) + (99 - st)
        d.mcs[0], d.n_dmrs = int(rng.integers(0, 27)), int(rng.integers(0, 8))
        g = ltelib.UlGrant()
        assert S.lte_ul_dci_to_grant(C.byref(cell), C.byref(d), 1, C.byref(g)) == 0 and g.L_prb == L and g.n_prb == st
        x, pl, off = ltelib.sim_ul_subframe(s, n, ucfg, [g])
        res, ch, payload = phy.decode_ul(x[None, :], np.array([n], np.uint32), [_to_capi(0, g)])
        llr = phy.tap(capi.TAP_PDSCH_LLR, (g.nof_bits,), np.int16)
        _, ref = ltelib.oracle_ul(o, ucfg, n, [g], x, want_llr=True)
        r, opl, ocrc, och, ollr = ref[0]
        assert np.array_equal(llr, ollr[:g.nof_bits]), (L, describe_mismatch(llr, ollr[:g.nof_bits], "L_prb %d" % L))
        assert res[0].crc == ocrc == 1 and np.array_equal(payload[:g.tbs // 8], pl[:g.tbs // 8])
    phy.close()


def test_pusch_symbols_kept_between_calls(infra, phylib):
    """iq_ul = NULL decodes the subframes of the previous call again (srsran_enb_ul_fft once, then decode_run per grant, UL_Sniffer_PUSCH.cc:392,456-570)"""
    cell = Cell(25, 1, 5, 1)
    ucfg = UlCfg(n_dmrs1=3, delta_ss=2)
    s = Sim(cell=cell, seed=3, snr_db=30.0, nof_ues=1)
    gr = ltelib.make_ul_grants(cell, np.random.default_rng(3), 3)
    x, pl, off = ltelib.sim_ul_subframe(s, 5, ucfg, gr)
    phy = capi.LtePhy(cell.nof_prb, 1, cell.cell_id, 1, max_subframes=1)
    phy.set_ul_cfg(3, 2)
    tti = np.array([5], np.uint32)
    res, ch, payload = phy.decode_ul(x[None, :], tti, [])
    for g, of in zip(gr, off):
        res, ch, payload = phy.decode_ul(None, tti, [_to_capi(0, g)])
        assert res[0].crc == 1 and np.array_equal(payload[:g.tbs // 8], pl[of:of + g.tbs // 8])
    with pytest.raises(RuntimeError):
        capi.LtePhy(cell.nof_prb, 1, cell.cell_id, 1, max_subframes=2).decode_ul(None, np.array([5, 6], np.uint32), [])
    phy.close()
