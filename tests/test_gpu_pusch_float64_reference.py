"""The CUDA PUSCH path against the float64 references of tests/ref64_ul.py (pytest -m gpu), and zero-filled uplink subframes through the kernel and
the oracle.

test_gpu_pusch.py holds pusch_kernel bit-exact to lteo_pusch_decode; a formula both restate wrongly passes there.  Here the numpy-synthesised subframes
of tests/test_pusch_float64_reference.py go through the product, each cell's cases in one decode_ul call (several subframes, several grants per
subframe, mixed M and so mixed IDFT pass counts under one shared-memory size), and the UL grid (TAP_UL_SYM), the channel-estimate fields of
ltephy_get_ul and the soft bits (TAP_PDSCH_LLR: the UL codewords in grant order, each padded to a multiple of 8) are compared with the reference, with
the bars of the CPU file.  The oracle is run on the same samples and must agree bit for bit."""
import numpy as np
import pytest

from ltelib import Oracle
from helpers import describe_mismatch
from test_pusch_float64_reference import (CASES, PINNED, ZERO_CELL, ZERO_KINDS, ZERO_UCFG, check_chest, check_grid, check_soft_bits, check_zero_chest,
                                          oracle_decode, synth, zero_subframe, zeroed_soft_bits)
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu


def to_capi(i, g):
    return capi.UlGrant(sf=i, rnti=g.rnti, qm=g.qm, rv=0, L_prb=g.L, n_prb=g.n_prb, n_dmrs2=g.n_dmrs2, tbs=g.tbs, n_prb_slot1=g.n_prb1,
                        flags=capi.UL_FLAG_SLOT1, nof_ack=g.uci["nof_ack"], ri_len=g.uci["ri_len"], cqi_len=g.uci["cqi_len"],
                        I_offset_ack=g.uci["I_ack"], I_offset_ri=g.uci["I_ri"], I_offset_cqi=g.uci["I_cqi"])


def run_product(cell, u, subs, iqs=None):
    """one decode_ul call over the subframes -> (results, chest, payload, UL grids [n][14 nsc], soft bits per grant)"""
    n = len(subs)
    phy = capi.LtePhy(cell.nof_prb, 1, cell.cell_id, 1, max_subframes=n, symbol_sz=cell.symbol_sz)
    phy.set_ul_cfg(u[0], u[1], u[2], u[3])
    iq = np.stack([s.iq for s in subs] if iqs is None else iqs)
    tti = np.array([10 + s.sf for s in subs], np.uint32)                  # tti % 10 = the subframe index each was synthesised for
    grants = [to_capi(i, g) for i, s in enumerate(subs) for g in s.grants]
    res, ch, payload = phy.decode_ul(iq, tti, grants)
    sym = phy.tap(capi.TAP_UL_SYM, (n, 14 * phy.nsc), np.complex64)
    Gs = [g.G for s in subs for g in s.grants]
    tap = phy.tap(capi.TAP_PDSCH_LLR, (sum((G + 7) & ~7 for G in Gs),), np.int16)
    phy.close()
    llr, lo = [], 0
    for G in Gs:
        llr.append(tap[lo:lo + G])
        lo += (G + 7) & ~7
    return res, ch, payload, sym, llr


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_kernel_pusch_equals_the_float64_reference(infra, phylib, case):
    cell, subs = synth(case)
    res, ch, payload, sym, llr = run_product(cell, case[2], subs)
    o = Oracle(cell)
    k = 0
    for i, s in enumerate(subs):
        osym, ores = oracle_decode(o, s)
        Y, ref = s.reference()
        check_grid(sym[i], Y, cell, (case[0], s.sf))
        assert np.array_equal(sym[i], osym), describe_mismatch(sym[i], osym, "UL grid sf %d" % s.sf)
        for g, (r, opl, ocrc, och, ollr), (info, rl, cond) in zip(s.grants, ores, ref):
            what = "%s sf %d L %d at %d qm %d" % (case[0], s.sf, g.L, g.n_prb, g.qm)
            check_chest(ch[k], info, what)
            check_soft_bits(llr[k], rl, cond, what)
            assert (ch[k].noise, ch[k].rsrp, ch[k].snr_db) == (och.noise, och.rsrp, och.snr_db), what
            assert abs(ch[k].ta_us - och.ta_us) < 1e-3, what
            assert np.array_equal(llr[k], ollr[:g.G]), describe_mismatch(llr[k], ollr[:g.G], what)
            assert res[k].crc == ocrc, what
            k += 1


@pytest.mark.parametrize("kind", ZERO_KINDS)
def test_kernel_on_zero_filled_subframes(infra, phylib, kind):
    """exactly-zero samples through the product: bit for bit the oracle, no NaN in the UL grid or the estimate fields, every soft bit of a zero-filled
    symbol 0; all_zero gives noise = RSRP = 0, snr_db NaN and ta_us 0; the pinned grants decode with symbols 11-13 lost"""
    s, iq, pls = zero_subframe(kind)
    res, ch, payload, sym, llr = run_product(ZERO_CELL, ZERO_UCFG, [s], [iq])
    o = Oracle(ZERO_CELL)
    osym, ores = oracle_decode(o, s, iq)
    assert not np.isnan(sym).any() and np.array_equal(sym[0], osym)
    _, ref = s.reference(iq)
    for k, (g, (r, opl, ocrc, och, ollr), (info, rl, cond)) in enumerate(zip(s.grants, ores, ref)):
        what = "%s grant %d qm %d" % (kind, k, g.qm)
        check_zero_chest(ch[k], kind, what)
        same = (ch[k].noise, ch[k].rsrp, ch[k].ta_us) == (och.noise, och.rsrp, och.ta_us)
        assert same and (ch[k].snr_db == och.snr_db or (np.isnan(ch[k].snr_db) and np.isnan(och.snr_db))), what
        assert np.array_equal(llr[k], ollr[:g.G]), describe_mismatch(llr[k], ollr[:g.G], what)
        z = zeroed_soft_bits(g, kind)
        assert np.all(llr[k][z] == 0), what
        check_soft_bits(llr[k], rl, cond, what)
        assert res[k].crc == ocrc, what
    if kind == "from_symbol_11":
        for i in PINNED:
            nby = s.grants[i].tbs // 8
            assert res[i].crc == 1 and np.array_equal(payload[res[i].payload_off:res[i].payload_off + nby], pls[i]), i
