"""The numpy eNB of tests/ref64_ctrl.py (control region and PBCH placed from 36.211 alone) through the product (pytest -m gpu).  The kernels only gather
through the host-built control-region table and the PBCH table of the device handle, so these tests pin both tables against the standard where
tests/test_control_region_36211.py cannot reach them:
  * the PDCCH LLRs (TAP_LLR), PCFICH correlations, CFI and per-CCE power against ref64 on the spec's indices;
  * the phase-A candidate table at every planted (location, size): planted bits and RNTI, aggregation levels 1 / 2 / 4 / 8, two DCI sizes;
  * ltephy_mib_decode / ltephy_mib_decode_combined: bandwidth, Ng, duration, SFN and port count at every SFN mod 4, found = 0 for a reserved code;
  * the PBCH soft bits (TAP_PBCH_LLR) against a float64 MRC / SFBC on the spec's 240 resource elements."""
import numpy as np
import pytest

import ref64
import ref64_ctrl
from ltelib import Cell
from test_control_region_36211 import plant
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu

# (nof_prb, ports, pci, rx, symbol_sz, phich_ng, phich_ext): every bandwidth, 1 / 2 ports x 1 / 2 antennas, each Ng with both durations, PCI mod 3
# = 0 / 1 / 2, PCIs above 2 N and above M_quad
GPU_CELLS = [(15, 1, 0, 1, 0, 0, 0), (15, 2, 31, 2, 0, 1, 1), (25, 1, 151, 2, 0, 2, 0), (25, 2, 53, 1, 0, 3, 1), (50, 2, 302, 2, 0, 0, 1),
             (50, 1, 100, 1, 0, 1, 0), (75, 1, 500, 2, 0, 2, 1), (75, 2, 17, 1, 1536, 3, 0), (100, 2, 7, 2, 0, 0, 0), (100, 1, 205, 1, 0, 3, 1)]
SFN0 = 513                                   # frames SFN0 .. SFN0 + 3: every SFN mod 4


def batch(cell, phy, rng, chan, bw_code=None):
    """subframes 0..9 of frame SFN0 and subframe 0 of the next three frames -> (iq [13][rx][sf_len], tti, [(sf, cfi, truth, Y)])"""
    sizes, sidx = phy.sizes()
    distinct = sorted({sidx[f]: sizes[f] for f in range(capi.NOF_FORMATS)}.items(), key=lambda x: x[1])
    use = [distinct[0], distinct[-1]]
    H = ref64.channel(chan, cell.nof_rx, cell.nof_ports, 12 * cell.nof_prb, taps=5.0)
    tti = [10 * SFN0 + k for k in range(10)] + [10 * (SFN0 + f) for f in (1, 2, 3)]
    iq, subs = [], []
    for t in tti:
        sf, sfn = t % 10, t // 10
        cfi = 3 if cell.phich_ext else 1 + (t + sfn) % 3
        nc, Ls = phy.locations(cfi)
        dcis = plant(phy.nof_cce(cfi), rng, [s for _, s in use], locs=[(int(n), 1 << int(L)) for n, L in zip(nc, Ls)], first=t)
        grids, truth = ref64_ctrl.enb_subframe(cell, sf, cfi, dcis, rng, sfn=sfn, spare=int(rng.integers(0, 1024)), bw_code=bw_code)
        _, x = ref64_ctrl.capture(cell, grids, H, 3e-3, rng)
        Y = np.stack([ref64.ofdm_demodulate(cell, x[a]) for a in range(cell.nof_rx)])     # the receiver's view of the complex64 samples
        iq.append(x)
        subs.append((sf, cfi, truth, Y, {s: i for i, s in use}))
    return np.stack(iq), np.array(tti, np.uint32), subs


@pytest.mark.parametrize("cellp", GPU_CELLS, ids=lambda c: "x".join(map(str, c)))
def test_product_decodes_the_numpy_enb(infra, phylib, cellp):
    cell = Cell(*cellp)
    rng = np.random.default_rng(cellp[2] + 7 * cellp[0])
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=13, turbo_max_iter=1, symbol_sz=cell.symbol_sz,
                      phich_resources=cell.phich_ng, phich_length=cell.phich_ext)
    iq, tti, subs = batch(cell, phy, rng, "delay" if cellp[0] == 50 and cellp[1] == 1 else "selective")
    n = len(tti)
    phy.submit_iq(iq, tti)
    info, cands = phy.get_phase_a()
    llr = phy.tap(capi.TAP_LLR, (n, capi.LLR_STRIDE), np.float32)
    Ls = set()
    for i, (sf, cfi, truth, Y, size_index) in enumerate(subs):
        inf = info[i]
        ce, _ = ref64.chest(cell, sf, Y)
        m = ref64_ctrl.cell_map(cell, cfi)
        assert inf.cfi == cfi, (i, inf.cfi, cfi)
        rc = ref64.pcfich_corr(cell, sf, ce, Y, m.pcfich)
        assert np.abs(np.array(inf.pcfich_corr[:]) - rc).max() <= 1e-5 * np.abs(rc).max(), (i, list(inf.pcfich_corr), rc)
        rl = ref64.pdcch_llr(cell, sf, ce, Y, m.pdcch.ravel(), (sf << 9) + cell.cell_id)
        assert inf.nof_cce == m.ncce, (i, inf.nof_cce, m.ncce)
        assert np.abs(llr[i, :len(rl)] - rl).max() <= 1e-5 * np.abs(rl).max(), (i, np.abs(llr[i, :len(rl)] - rl).max() / np.abs(rl).max())
        rp = np.abs(rl).reshape(-1, 72).mean(1)
        assert np.abs(np.array(inf.cce_power[:inf.nof_cce]) - rp).max() <= 1e-5 * rp.max(), i
        nc, Lg = phy.locations(cfi)
        where = {(int(a), 1 << int(b)): j for j, (a, b) in enumerate(zip(nc, Lg))}
        for bits, rnti, L, first in truth.dcis:
            c = cands[i, where[(first, L)], size_index[len(bits)]]
            assert c["valid"] == 1 and int(c["rnti"]) == rnti and np.array_equal(capi.cand_bits(c["bits"], len(bits)), bits), (i, first, L, len(bits), hex(rnti))
            Ls.add(L)
        assert max(first + L for _, _, L, first in truth.dcis) == max(int(a) + (1 << int(b)) for a, b in zip(nc, Lg))      # the last CCE searched
    if cell.nof_prb >= 25:
        assert Ls == {1, 2, 4, 8}, Ls
    # the MIB, one frame at a time, and the PBCH soft bits of the handle's port count
    frames = [i for i, s in enumerate(subs) if s[0] == 0]
    assert len(frames) == 4
    mib = phy.mib_decode()
    pb = phy.tap(capi.TAP_PBCH_LLR, (4, 2, 480), np.float32)
    for f, i in enumerate(frames):
        sf, cfi, truth, Y, _ = subs[i]
        r = mib[i]
        bw, ext, ng, msb, _ = ref64_ctrl.mib_fields(truth.mib)
        assert (r.found, r.nof_ports, r.nof_prb, r.phich_length, r.phich_resources, r.sfn) == (1, cell.nof_ports, cell.nof_prb, ext, ng, truth.sfn), \
            (f, r.found, r.nof_ports, r.nof_prb, r.phich_length, r.phich_resources, r.sfn, truth.sfn)
        assert bytes(r.bch_payload) == np.packbits(truth.mib).tobytes()
        ce, _ = ref64.chest(cell, 0, Y)
        ref = ref64_ctrl.pbch_llr(cell, ce, Y, cell.nof_ports)
        got = pb[f, cell.nof_ports - 1]
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max(), (f, np.abs(got - ref).max() / np.abs(ref).max())
    assert all(mib[i].found == 0 for i in range(n) if i not in frames)
    # with soft combining: every frame decodes on its own at this SNR; both port-count halves of the soft bits are written
    phy.mib_reset()
    comb = phy.mib_decode_combined(search_ports=True)
    pb = phy.tap(capi.TAP_PBCH_LLR, (4, 2, 480), np.float32)
    for f, i in enumerate(frames):
        sf, cfi, truth, Y, _ = subs[i]
        r = comb[i].mib
        _, ext, ng, _, _ = ref64_ctrl.mib_fields(truth.mib)
        assert (r.found, r.nof_ports, r.nof_prb, r.phich_length, r.phich_resources, r.sfn) == (1, cell.nof_ports, cell.nof_prb, ext, ng, truth.sfn), \
            (f, r.found, r.nof_ports, r.nof_prb, r.sfn, truth.sfn)
        ce, _ = ref64.chest(cell, 0, Y)
        for p in range(1, cell.nof_ports + 1):
            ref = ref64_ctrl.pbch_llr(cell, ce, Y, p)
            assert np.abs(pb[f, p - 1] - ref).max() <= 1e-5 * np.abs(ref).max(), (f, p)
    phy.close()


@pytest.mark.parametrize("code", [6, 7])
def test_reserved_bandwidth_code_is_not_a_mib(infra, phylib, code):
    """a PBCH that passes its CRC with dl-Bandwidth 6 or 7 (not in the 36.331 enumeration) is no MIB"""
    cell = Cell(25, 2, 77, 2)
    rng = np.random.default_rng(code)
    phy = capi.LtePhy(25, 2, 77, 2, max_subframes=13, turbo_max_iter=1)
    iq, tti, subs = batch(cell, phy, rng, "selective", bw_code=code)
    phy.submit_iq(iq, tti)
    phy.get_phase_a(want_cands=False)
    assert all(m.found == 0 for m in phy.mib_decode())
    assert all(c.mib.found == 0 for c in phy.mib_decode_combined())
    pb = phy.tap(capi.TAP_PBCH_LLR, (4, 2, 480), np.float32)
    assert np.abs(pb[:, 1]).max() > 0                                       # the frames were there: their soft bits fail only the unpack
    phy.close()
