"""ltephy_mib_decode_combined on the GPU: every field of every result bit-exact against the oracle combiner lteo_mib_* (DESIGN.md §2 "PBCH
combining") over cells, SNRs, batch splits, gaps, the SFN wrap, reset and the port search; the one-frame case against ltephy_mib_decode;
invalid inputs; and the cell_search example on a capture whose first frame alone does not decode, and on one with no MIB to decode."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ltelib
import mib_lib as M
import sync_lib as S
from ltelib import Cell

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

GPU_MIB_CELLS = [(25, 1, 3, 1), (50, 2, 301, 2), (100, 2, 77, 2), (15, 1, 10, 1), (15, 2, 11, 2), (75, 1, 12, 1), (75, 2, 40, 2, 0, 3, 1),
                 (25, 2, 150, 2, 0, 2, 1), (100, 1, 9, 1, 0, 1, 0)]
# SNR steps from -11 to 0 dB over runs of consecutive frames, with a gap and the SFN wrap
PLAN = [(1016, 6, -11.0), (1022, 7, -8.0), (5, 6, -7.0), (30, 6, -5.0), (36, 5, -2.0), (41, 3, 0.0)]


def gpu_tuple(m):
    if not m.mib.found:
        return None
    bits = tuple(int(b) for b in np.unpackbits(np.frombuffer(bytes(m.mib.bch_payload), np.uint8)))
    return (m.mib.nof_ports, m.mib.sfn_offset, m.nof_frames, m.src, m.dst, m.window, bits, m.mib.sfn)


def expected(r):
    """what the GPU reports for an oracle result: a pass with a reserved bandwidth code is found = 0"""
    if r is None or r[6][0] * 4 + r[6][1] * 2 + r[6][2] >= 6:
        return None
    return r


def sequence(cell, plan, seed=5, ports=None):
    """frames of cell; the oracle front end estimates `ports` ports (a 1-port cell read by a 2-port handle has a port 1 estimate too)"""
    o = ltelib.Oracle(Cell(cell.nof_prb, ports or cell.nof_ports, cell.cell_id, cell.nof_rx, cell.symbol_sz, cell.phich_ng, cell.phich_ext))
    iqs, ttis, fes = [], [], []
    for k, (s0, n, snr) in enumerate(plan):
        iq, tti, fe = M.frames(cell, range(s0, s0 + n), snr, seed=seed + k, o=o)
        iqs.append(iq)
        ttis.append(tti)
        fes += fe
    return np.concatenate(iqs), np.concatenate(ttis), fes


def run_gpu(phy, iq, tti, batch, search_ports, reset_at=None):
    out = []
    for b0 in range(0, len(tti), batch):
        b1 = min(len(tti), b0 + batch)
        if reset_at is not None and b0 <= reset_at < b1:      # split the batch there
            out += run_gpu(phy, iq[b0:reset_at], tti[b0:reset_at], batch, search_ports) if reset_at > b0 else []
            phy.mib_reset()
            out += run_gpu(phy, iq[reset_at:b1], tti[reset_at:b1], batch, search_ports)
            continue
        phy.submit_iq(iq[b0:b1], tti[b0:b1])
        phy.get_phase_a(want_cands=False)
        out += [gpu_tuple(m) for m in phy.mib_decode_combined(search_ports)]
    return out


def run_oracle(cell, handle_ports, tti, fes, search_ports, reset_at=None):
    oc = M.OracleCombiner(Cell(cell.nof_prb, handle_ports, cell.cell_id, cell.nof_rx, cell.symbol_sz, cell.phich_ng, cell.phich_ext))
    out = []
    for i, (t, f) in enumerate(zip(tti, fes)):
        if i == reset_at:
            oc.reset()
        out.append(expected(oc.decode(int(t), f, search_ports)))
    return out


def _handle(cell, ports, n):
    from ltesniffer_b200 import capi
    return capi.LtePhy(cell.nof_prb, ports, cell.cell_id, cell.nof_rx, max_subframes=n, phich_resources=cell.phich_ng, phich_length=cell.phich_ext)


@pytest.mark.parametrize("cellp", GPU_MIB_CELLS)
def test_gpu_equals_oracle_combiner(infra, phylib, cellp):
    cell = Cell(*cellp)
    iq, tti, fes = sequence(cell, PLAN)
    n = len(tti)
    ref = run_oracle(cell, cell.nof_ports, tti, fes, False)
    phy = _handle(cell, cell.nof_ports, n)
    assert run_gpu(phy, iq, tti, n, False) == ref
    phy.close()
    assert sum(r is not None for r in ref) >= 4


@pytest.mark.parametrize("batch", [1, 3, 7, 64])
@pytest.mark.parametrize("cellp,ports,search", [((25, 1, 3, 1), 1, False), ((15, 2, 11, 2), 2, True), ((25, 1, 3, 1), 2, True),
                                                ((25, 1, 3, 1), 1, True), ((50, 2, 301, 1), 2, False)])
def test_gpu_batches_reset_and_port_search(infra, phylib, batch, cellp, ports, search):
    """the same frames in batches of 1, 3, 7 and all, with srsran_ue_mib_reset in the middle; a 1-port cell read by a 2-port handle searching the
    port count, and a 1-port handle with the flag"""
    cell = Cell(*cellp)
    iq, tti, fes = sequence(cell, PLAN, seed=17, ports=ports)
    n = len(tti)
    ref = run_oracle(cell, ports, tti, fes, search, reset_at=20)
    phy = _handle(cell, ports, min(batch, n))
    assert run_gpu(phy, iq, tti, batch, search, reset_at=20) == ref
    phy.close()


@pytest.mark.parametrize("cellp", [(25, 1, 3, 1), (15, 2, 11, 2)])
def test_gpu_noise_only_equals_oracle(infra, phylib, cellp):
    cell = Cell(*cellp)
    iq, tti, fes = sequence(cell, [(200, 40, -40.0)], seed=29)
    ref = run_oracle(cell, cell.nof_ports, tti, fes, True)
    phy = _handle(cell, cell.nof_ports, len(tti))
    assert run_gpu(phy, iq, tti, len(tti), True) == ref
    phy.close()


@pytest.mark.parametrize("cellp", [(25, 1, 3, 1), (50, 2, 301, 2), (75, 2, 40, 2, 0, 3, 1)])
def test_one_frame_windows_equal_mib_decode(infra, phylib, cellp):
    """every other frame: each window holds one frame, so the combined decode with the handle's port count is ltephy_mib_decode wherever the
    latter's CRC mask is the handle's"""
    cell = Cell(*cellp)
    iq, tti, _ = sequence(cell, [(500 + 2 * k, 1, s) for k, s in enumerate([-6.0, -3.0, 0.0, 4.0] * 4)])
    phy = _handle(cell, cell.nof_ports, len(tti))
    phy.submit_iq(iq, tti)
    phy.get_phase_a(want_cands=False)
    single = phy.mib_decode()
    comb = phy.mib_decode_combined()
    nmatch = 0
    for s, c in zip(single, comb):
        assert c.window == (1 if c.mib.found else 0)
        if s.found and s.nof_ports == cell.nof_ports:
            nmatch += 1
            assert c.mib.found and c.nof_frames == 1 and c.dst == s.sfn_offset
            for f in ("nof_ports", "sfn_offset", "phich_length", "phich_resources", "nof_prb", "sfn"):
                assert getattr(c.mib, f) == getattr(s, f), f
            assert bytes(c.mib.bch_payload) == bytes(s.bch_payload)
    assert nmatch >= 6
    phy.close()


def test_port0_estimate_does_not_depend_on_the_port_count(infra, phylib):
    """a 2-port handle equalises 1-port hypotheses with port 0 alone: its port 0 estimate is the 1-port handle's"""
    from ltesniffer_b200 import capi
    cell = Cell(25, 2, 150, 2)
    iq, tti, _ = sequence(cell, [(300, 3, 5.0)])
    g = 14 * 12 * cell.nof_prb
    ce = {}
    for p in (1, 2):
        phy = _handle(cell, p, 3)
        phy.submit_iq(iq, tti)
        phy.get_phase_a(want_cands=False)
        ce[p] = phy.tap(capi.TAP_CE, (3, p, cell.nof_rx, g), np.complex64)
        phy.close()
    assert np.array_equal(ce[2][:, 0].view(np.uint32), ce[1][:, 0].view(np.uint32))


def test_invalid_inputs(infra, phylib):
    from ltesniffer_b200 import capi
    cell = Cell(25, 1, 3, 1)
    phy = _handle(cell, 1, 4)
    L = phy.L
    L.ltephy_mib_decode_combined.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    out = (capi.MibComb * 4)()
    assert L.ltephy_mib_decode_combined(phy.h, 0, out) == -2           # nothing submitted
    iq, tti, _ = sequence(cell, [(10, 4, 5.0)])
    phy.submit_iq(iq, tti)
    assert L.ltephy_mib_decode_combined(phy.h, 0, None) == -2
    assert L.ltephy_mib_decode_combined(phy.h, 2, out) == -2           # unknown flag
    assert L.ltephy_mib_decode_combined(phy.h, capi.MIB_SEARCH_PORTS, out) == 0
    L.ltephy_mib_reset.argtypes = [C.c_void_p]
    assert L.ltephy_mib_reset(None) == -2
    phy.close()


def test_example_reads_the_mib_from_later_frames(infra, phylib, tmp_path):
    """a capture whose first frame alone does not decode (neither port count) but whose later frames do, combined: the example prints the
    simulator's truth line where it used to print "MIB not decoded\""""
    from ltesniffer_b200 import capi
    subprocess.run(["make", "-s", "-C", ROOT, "examples/cell_search"], check=True)
    N, off = 512, 4444
    cell = ltelib.Cell(25, 1, 71, 1, N)
    sfl = 15 * N
    chosen = None
    for seed in range(71, 83):
        s = S.sim(sync=1, cell=cell, seed=seed, pbch=1, snr_db=-7.0, nof_ues=1)
        x = np.concatenate([s.subframe(t)[0] for t in range(90)], axis=1)[:, off:].astype(np.complex64)
        cs = capi.CellSearch(N, 1, x.shape[1])
        c = cs.search(x)[0]
        cs.close()
        if not c.detected or c.pci != 71:
            continue
        fo = int(c.frame_offset)
        nf = (x.shape[1] - fo) // (10 * sfl)
        iq = np.stack([x[:, fo + 10 * f * sfl:fo + (10 * f + 1) * sfl] for f in range(nf)])
        tti = np.arange(nf, dtype=np.uint32) * 10
        first = []
        for p in (1, 2):
            phy = capi.LtePhy(15, p, 71, 1, max_subframes=nf, symbol_sz=N)
            phy.set_cfo(c.cfo_hz)
            phy.submit_iq(iq, tti)
            m = phy.mib_decode()[0]
            first.append(m.found and m.nof_ports == p)
            phy.close()
        if not any(first):
            chosen = (x, c, (off + fo) // sfl)
            break
    assert chosen is not None
    x, c, k0 = chosen
    f = tmp_path / "cap.cf32"
    x.tofile(str(f))
    r = subprocess.run([os.path.join(ROOT, "examples", "cell_search"), str(f), str(N), "1"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    w = r.stdout.split()
    assert int(w[1]) == 71 and int(w[3]) == c.frame_offset
    assert (int(w[7]), int(w[9]), int(w[11]), int(w[13]), int(w[15])) == (25, 1, 0, 0, k0 // 10)


def test_example_reports_an_undecoded_mib(infra, phylib, tmp_path):
    """a cell the search finds but whose MIB no window decodes (this capture carries no PBCH at all): the example says so on stderr and exits
    with 3 instead of printing a result line"""
    from ltesniffer_b200 import capi
    subprocess.run(["make", "-s", "-C", ROOT, "examples/cell_search"], check=True)
    N = 512
    cell = ltelib.Cell(25, 1, 71, 1, N)
    s = S.sim(sync=1, cell=cell, seed=81, pbch=0, snr_db=20.0, nof_ues=1)
    x = np.concatenate([s.subframe(t)[0] for t in range(60)], axis=1)[:, 4444:].astype(np.complex64)
    cs = capi.CellSearch(N, 1, x.shape[1])
    c = cs.search(x)[0]
    cs.close()
    assert c.detected and c.pci == 71
    f = tmp_path / "cap.cf32"
    x.tofile(str(f))
    r = subprocess.run([os.path.join(ROOT, "examples", "cell_search"), str(f), str(N), "1"], capture_output=True, text=True)
    assert r.returncode == 3 and r.stdout == ""
    assert r.stderr.strip() == "cell 71 found, MIB not decoded"
