"""MIB decode across the 40 ms PBCH period (DESIGN.md §2 "PBCH combining") on the CPU: the oracle combiner lteo_mib_* against lteo_pbch_decode
for one frame, against an independent Python statement of srsRAN's loop over lteo_dci_decode, and against what the simulated eNB broadcast."""
import numpy as np
import pytest

import ltelib
import mib_lib as M
from ltelib import Cell
from ref64 import gold

PBCH_CELLS = [(25, 1, 3, 1), (50, 2, 301, 2), (100, 2, 77, 2), (15, 1, 10, 1), (75, 2, 40, 2, 0, 3, 1)]


@pytest.mark.parametrize("cellp", PBCH_CELLS)
def test_one_frame_equals_pbch_decode(infra, cellp):
    """with one frame held and the cell's port count, the combiner is lteo_pbch_decode: found, bits, and dst = the frame position q"""
    cell = Cell(*cellp)
    o = ltelib.Oracle(cell)
    _, tti, fe = M.frames(cell, range(517, 522), 8.0, o=o)
    oc = M.OracleCombiner(cell)
    for t, f in zip(tti, fe):
        oc.reset()
        r = oc.decode(int(t), f)
        found, bits, nports, fq = o.pbch_decode(f["sym"], f["ce"])
        assert found == 1 and nports == cell.nof_ports
        assert r is not None and r[2] == 1 and r[5] == 1 and r[4] == fq and r[6] == tuple(int(b) for b in bits)
        assert r[7] == int(t) // 10 and r[0] == cell.nof_ports


@pytest.mark.parametrize("cellp,nant", [((25, 1, 3, 1), 1), ((15, 2, 11, 2), 1), ((15, 2, 11, 2), 2), ((50, 2, 301, 1), 2), ((100, 2, 77, 2), 2),
                                        ((75, 1, 12, 2), 1)])
@pytest.mark.parametrize("snr", [-8.0, 4.0])
def test_pbch_llr_equals_the_oracles_equalisers(infra, cellp, nant, snr):
    """lteo_pbch_llr == the equalisers lteo_pbch_decode uses (static in lte_oracle.c), bit for bit: the PBCH REs' samples and estimates are copied
    onto the first 240 PDCCH REs of an otherwise zero grid, lteo_pdcch_extract_llr equalises them with those functions (in pairs (2k, 2k + 1)
    for SFBC, as the PBCH does) and its PDCCH descrambling is undone, which only flips signs"""
    import ctypes as C
    cell = Cell(*cellp)
    ocell = Cell(cell.nof_prb, nant, cell.cell_id, cell.nof_rx)     # the port count the equaliser is run with
    o = ltelib.Oracle(ocell)
    _, _, fes = M.frames(cell, range(40, 43), snr, o=o)
    O = ltelib.oracle()
    O.lteo_pdcch_re_index.restype = C.c_uint32
    O.lteo_pdcch_re_index.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    idx = np.zeros(88 * 36, np.uint16)
    ncce = O.lteo_pdcch_re_index(o.h, 3, ltelib.ptr(idx), None)
    assert 36 * ncce >= 240
    ks, ls = np.zeros(240, np.uint16), np.zeros(240, np.uint8)
    S = ltelib.sim()
    S.lte_pbch_re.argtypes = [C.POINTER(ltelib.Cell), C.c_void_p, C.c_void_p]
    assert S.lte_pbch_re(C.byref(ocell), ltelib.ptr(ks), ltelib.ptr(ls)) == 240
    src = ls.astype(np.int64) * o.nsc + ks
    scr = gold(cell.cell_id, 8 * 9 * ncce).astype(bool)          # PDCCH scrambling of subframe 0: c_init = (0 << 9) + cell_id
    for fe in fes:
        sym, ce = np.zeros_like(fe["sym"]), np.zeros_like(fe["ce"])
        sym[:, idx[:240]], ce[:, idx[:240]] = fe["sym"][:, src], fe["ce"][:, src]
        llr = o.pdcch_llr(0, 3, sym, ce)
        ref = np.where(scr[:480], -llr[:480], llr[:480])
        got = M.pbch_llr(ocell, fe, nant)
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
        assert np.any(got != 0)


def _blocks(cell, o, plan, seed=5):
    """plan: [(first sfn, count, snr)] -> list of (tti, front-end dict) in that order"""
    out = []
    for k, (s0, n, snr) in enumerate(plan):
        _, tti, fe = M.frames(cell, range(s0, s0 + n), snr, seed=seed + k, o=o)
        out += list(zip([int(t) for t in tti], fe))
    return out


# SNR steps from -11 to 0 dB; consecutive blocks continue the SFN (state carries over), one gap, one SFN wrap
PLAN = [(1014, 6, -11.0), (1020, 6, -9.0), (2, 5, -7.0), (7, 6, -6.0), (40, 7, -5.0), (47, 4, -3.0), (51, 3, 0.0)]


@pytest.mark.parametrize("cellp", [(25, 1, 3, 1), (15, 2, 11, 2), (50, 2, 301, 1)])
@pytest.mark.parametrize("search_ports", [False, True])
def test_oracle_equals_python_statement(infra, cellp, search_ports):
    cell = Cell(*cellp)
    o = ltelib.Oracle(cell)
    seq = _blocks(cell, o, PLAN)
    oc, pc = M.OracleCombiner(cell), M.PyCombiner(cell)
    got, n_multi = 0, 0
    for i, (t, f) in enumerate(seq):
        if i == 20:                                   # srsran_ue_mib_reset in the middle of a run
            oc.reset(), pc.reset()
        a, b = oc.decode(t, f, search_ports), pc.decode(t, f, search_ports)
        assert a == b, (i, t, a, b)
        got += a is not None
        n_multi += a is not None and a[2] > 1
    assert got >= 5 and n_multi >= 1                  # the sequence reaches windows that combine several frames


def _single_and_combined(cell, o, sfns, snr, seed):
    _, tti, fe = M.frames(cell, sfns, snr, seed=seed, o=o)
    single = sum(o.pbch_decode(f["sym"], f["ce"])[0] for f in fe)
    oc = M.OracleCombiner(cell)
    return single, [(int(t), oc.decode(int(t), f)) for t, f in zip(tti, fe)]


def test_combining_reads_the_broadcast_mib_where_single_frames_fail(infra):
    """at an SNR where one frame alone decodes at most a quarter of the time, every MIB the combiner returns is the broadcast one with the SFN of
    the newest frame, some of them combine several frames, and this holds from every start position in the 40 ms period"""
    cell = Cell(25, 1, 3, 1, 512)
    o = ltelib.Oracle(cell)
    snr = None
    for s in (-6.0, -6.5, -7.0, -7.5, -8.0):         # calibration: the highest SNR at which single frames mostly fail
        single, _ = _single_and_combined(cell, o, range(700, 724), s, 11)
        if single <= 24 // 4:
            snr = s
            break
    assert snr is not None
    for start in range(4):
        sfns = range(800 + start, 800 + start + 24)
        single, res = _single_and_combined(cell, o, sfns, snr, 11)
        assert single <= len(sfns) // 4
        found = [(t, r) for t, r in res if r is not None]
        assert found and any(r[2] > 1 for _, r in found), (start, found)
        for t, r in found:
            sfn = t // 10
            assert r[7] == sfn and r[6] == M.broadcast(cell, sfn), (start, t, r)
            assert r[0] == 1 and 0 <= r[1] <= 6


def test_all_zero_frames(infra):
    cell = Cell(25, 2, 3, 2)
    o = ltelib.Oracle(cell)
    iq = np.zeros((6, cell.nof_rx, ltelib.Sim(cell=cell).sf_len), np.complex64)
    from helpers import oracle_frontend
    fe = oracle_frontend(o, iq, np.arange(0, 60, 10, dtype=np.uint32))
    oc = M.OracleCombiner(cell)
    for i, f in enumerate(fe):
        for nant in (1, 2):
            assert not np.isnan(M.pbch_llr(cell, f, nant)).any()
        assert oc.decode(10 * i, f, True) is None


@pytest.mark.parametrize("cellp", [(25, 1, 3, 1), (15, 2, 11, 2)])
def test_noise_only_frames(infra, cellp):
    """noise only: false MIBs are possible (up to 30 hypotheses x 2^-16 per frame and port count), so the two statements must only agree"""
    cell = Cell(*cellp)
    o = ltelib.Oracle(cell)
    seq = _blocks(cell, o, [(100, 24, -40.0)], seed=23)
    oc, pc = M.OracleCombiner(cell), M.PyCombiner(cell)
    for t, f in seq:
        assert oc.decode(t, f, True) == pc.decode(t, f, True)
