"""SURVEY 8f-1 (file mode): what srsran_ue_sync's file path and srsran_ue_mib_decode do before the hot path
(reference src/src/LTESniffer_Core.cc:252-262,365,382-396): constant carrier-frequency-offset correction of every subframe of samples,
and the PBCH / MIB decode of subframe 0 (bandwidth, PHICH configuration, SFN, antenna ports from the CRC mask)."""
import ctypes as C
import numpy as np
import pytest
import ltelib
from ltelib import Cell
from helpers import make_capture, oracle_frontend


def mib_fields(bits):
    S = ltelib.sim()
    S.lte_mib_unpack.argtypes = [C.c_void_p] + [C.POINTER(C.c_uint32)] * 4
    v = [C.c_uint32() for _ in range(4)]
    r = S.lte_mib_unpack(ltelib.ptr(np.ascontiguousarray(bits, np.uint8)), *[C.byref(x) for x in v])
    return r, [x.value for x in v]


@pytest.mark.parametrize("cellp,snr", [((25, 1, 3, 1), 8.0), ((50, 2, 301, 2), 6.0), ((100, 2, 77, 2), 10.0), ((15, 1, 10, 1), 12.0),
                                      ((75, 2, 40, 2, 0, 3, 1), 8.0)])
def test_oracle_decodes_the_simulators_pbch(infra, cellp, snr):
    cell = Cell(*cellp)
    tti0 = 10 * 517            # SFN 517 = 0b1000000101: 8 MSBs 129, position 1 in the 40 ms period
    sim, iq, tti, truths, payloads = make_capture(cell, 41, seed=5, cfi=3 if cell.phich_ext else 2, nof_ues=2, dl_min=1, dl_max=2, tm=1, snr_db=snr, pbch=1,
                                                  tti0=tti0)
    o = ltelib.Oracle(cell)
    seen = set()
    for i in range(0, 41, 10):
        fe = oracle_frontend(o, iq[i:i + 1], tti[i:i + 1])[0]
        found, mib, nports, fq = o.pbch_decode(fe["sym"], fe["ce"])
        sfn = (tti0 + i) // 10
        assert found == 1 and nports == cell.nof_ports and fq == sfn % 4
        r, (nof_prb, phich_ext, phich_res, sfn8) = mib_fields(mib)
        assert r == 0 and (nof_prb, phich_ext, phich_res) == (cell.nof_prb, cell.phich_ext, cell.phich_ng) and sfn8 == (sfn // 4) * 4
        seen.add(fq)
    assert seen == {0, 1, 2, 3}
    # a subframe without PBCH (subframe 1) must not produce a MIB
    fe = oracle_frontend(o, iq[1:2], tti[1:2])[0]
    assert o.pbch_decode(fe["sym"], fe["ce"])[0] == 0


def test_cfo_correction_restores_the_decode(infra):
    """a 2.5 kHz offset (17 % of the sub-carrier spacing) breaks the PDSCH decode; srsran_cfo_correct's rotation restores it"""
    cell = Cell(25, 1, 3, 1)
    kw = dict(seed=9, cfi=2, nof_ues=2, dl_min=2, dl_max=2, tm=1, mcs_min=24, mcs_max=24, snr_db=30.0, full_band=1)
    _, iq0, tti, truths, payloads = make_capture(cell, 3, **kw)
    _, iq1, _, _, _ = make_capture(cell, 3, cfo_hz=2500.0, **kw)
    o = ltelib.Oracle(cell)
    from helpers import truth_grants

    def crc_count(iq):
        fe = oracle_frontend(o, iq, tti)
        ok = 0
        for sf, d, g in truth_grants(cell, truths, tti):
            r, pl, c = o.pdsch_decode(int(tti[sf]) % 10, fe[sf]["cfi"], d.rnti, g, fe[sf]["sym"], fe[sf]["ce"])
            ok += c[0]
        return ok
    n = len(truth_grants(cell, truths, tti))
    assert crc_count(iq0) == n
    assert crc_count(iq1) < n // 2
    fixed = np.stack([o.cfo_correct(2500.0, iq1[i]) for i in range(3)])
    assert crc_count(fixed) == n
    assert np.abs(fixed - iq0).max() < 0.35        # same signal up to the (different) noise realisation


@pytest.mark.gpu
@pytest.mark.parametrize("cellp,snr", [((25, 1, 3, 1), 8.0), ((50, 2, 301, 2), 6.0), ((100, 2, 77, 2), 2.0), ((15, 1, 10, 1), 8.0), ((15, 2, 11, 2), 6.0),
                                      ((75, 1, 12, 1), 8.0), ((75, 2, 40, 2, 0, 3, 1), 6.0), ((25, 2, 150, 2, 0, 2, 1), 8.0), ((100, 1, 9, 1, 0, 1, 0), 8.0)])
def test_gpu_mib_matches_oracle(infra, phylib, cellp, snr):
    """ltephy_mib_decode == oracle PBCH decode on every subframe of the batch (found flag, port count, frame position, the 24 bits), and both
    equal what the simulated eNB broadcast, PHICH configuration included (cellp: nof_prb, ports, cell id, antennas[, symbol_sz, Ng, extended]);
    2 dB at 20 MHz: some frames fail in both"""
    from ltesniffer_b200 import capi
    cell = Cell(*cellp)
    tti0 = 10 * 1022
    sim, iq, tti, truths, payloads = make_capture(cell, 42, seed=5, cfi=3 if cell.phich_ext else 2, nof_ues=2, dl_min=1, dl_max=2, tm=1, snr_db=snr, pbch=1,
                                                  tti0=tti0)       # the extended duration spans three symbols: CFI 3
    o = ltelib.Oracle(cell)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=42, phich_resources=cell.phich_ng, phich_length=cell.phich_ext)
    phy.submit_iq(iq, tti)
    phy.get_phase_a(want_cands=False)
    mibs = phy.mib_decode()
    nfound = 0
    for i in range(42):
        m = mibs[i]
        if int(tti[i]) % 10:
            assert m.found == 0
            continue
        fe = oracle_frontend(o, iq[i:i + 1], tti[i:i + 1])[0]
        found, bits, nports, fq = o.pbch_decode(fe["sym"], fe["ce"])
        assert m.found == found
        if not found:
            continue
        nfound += 1
        packed = np.packbits(bits)
        assert (m.nof_ports, m.sfn_offset, bytes(m.bch_payload)) == (nports, fq, bytes(packed))
        sfn = (int(tti[i]) // 10) % 1024
        assert (m.nof_prb, m.phich_length, m.phich_resources, m.sfn) == (cell.nof_prb, cell.phich_ext, cell.phich_ng, sfn)
    assert nfound >= 3
    phy.close()


@pytest.mark.gpu
def test_gpu_cfo_correction_matches_oracle(infra, phylib):
    """ltephy_set_cfo: the OFDM kernel's rotation == the oracle's srsran_cfo_correct restatement followed by its FFT, bit for bit; and the pipeline
    decodes a capture with a 2.5 kHz offset only with the correction on"""
    from ltesniffer_b200 import capi
    cell = Cell(25, 1, 3, 1)
    kw = dict(seed=9, cfi=2, nof_ues=2, dl_min=2, dl_max=2, tm=1, mcs_min=24, mcs_max=24, snr_db=30.0, full_band=1)
    _, iq, tti, truths, payloads = make_capture(cell, 4, cfo_hz=2500.0, **kw)
    o = ltelib.Oracle(cell)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=4, flags=capi.FLAG_SKIP_LOW_POWER)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    info, dcis, tbs, pl = capi.decode_subframes(phy, srch, iq, tti)
    ok_off = sum(1 for i in range(2 * len(dcis)) if tbs[i].crc)
    phy.set_cfo(2500.0)
    phy.submit_iq(iq, tti)
    phy.get_phase_a(want_cands=False)
    g = 14 * 12 * cell.nof_prb
    sym = phy.tap(capi.TAP_SYM, (4, cell.nof_rx, g), np.complex64)
    for i in range(4):
        ref = o.ofdm(o.cfo_correct(2500.0, iq[i]))
        assert np.array_equal(sym[i].view(np.uint32), np.asarray(ref).reshape(cell.nof_rx, g).view(np.uint32))
    srch2 = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    info, dcis, tbs, pl = capi.decode_subframes(phy, srch2, iq, tti)
    ok_on = sum(1 for i in range(2 * len(dcis)) if tbs[i].crc)
    assert ok_on >= 5 and ok_off <= ok_on - 3      # a fresh RNTI history does not accept every DCI of the first subframes
    phy.set_cfo(0.0)
    phy.close()
