"""Every handle gives its device memory back when it is destroyed (pytest -m gpu).  For each handle type -- LtePhy, CellSearch, Tracker and,
when NCCL loads, a Shard of world size 1 -- a few cycles of create -> exercise -> destroy must leave the device's free memory within half of
one live handle's footprint F of where it was.  Each cycle also has to give the results of the first.

Free memory is a device-wide reading that other work on the device moves, so the handles are sized to F >= 0.5 GB and the check allows F / 2.
The first cycle is not counted: it loads the kernels (and NCCL's one-time state), and it is where F is read."""
import ctypes as C

import numpy as np
import pytest

import ltelib

pytestmark = pytest.mark.gpu

GB = 1 << 30
CYCLES = 3


def _free():
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()  # the tracker's results are torch copies: their cached blocks are not the handle's
    return torch.cuda.mem_get_info(0)[0]


def _cycles(make, exercise):
    f_start = _free()
    h = make()
    first = exercise(h)
    F = f_start - _free()
    h.close()
    assert F >= 0.5 * GB, "a live handle takes %.2f GB: too small to tell a leak from other work on the device" % (F / GB)
    f0 = _free()
    for _ in range(CYCLES):
        h = make()
        assert exercise(h) == first
        h.close()
    drop = f0 - _free()
    assert drop < F / 2, "%d cycles lost %.1f MB of device memory; one handle takes %.1f MB" % (CYCLES, drop / 2 ** 20, F / 2 ** 20)


# ---------------------------------------------------------------------------------------------------- LtePhy
PHY_CELL = (100, 2, 4, 2)
PHY_SUBFRAMES = 10


def _phy_inputs():
    """a busy 100-PRB 2 x 2 capture with its truth grants, and uplink grants of every size, n_DMRS^(2) and slot: their DMRS / IDFT tables
    outgrow the uplink table pool's first reservation, so every cycle grows it"""
    from helpers import make_capture, to_phy_grant, truth_grants
    from test_gpu_phase_b import UL_POOL_FLOAT2, _ul_table_float2
    cell = ltelib.Cell(*PHY_CELL)
    sim, iq, tti, truths, _ = make_capture(cell, PHY_SUBFRAMES, seed=31, cfi=3, nof_ues=12, dl_min=4, dl_max=6, tm=3, mcs_min=14, mcs_max=28,
                                           snr_db=25.0, full_band=1)
    grants = [to_phy_grant(sf, d.rnti, g) for sf, d, g in truth_grants(cell, truths, tti)]
    S = ltelib.sim()
    S.lte_ul_valid_prb.argtypes = [C.c_uint32]
    S.lte_ul_dci_to_grant.argtypes = [C.POINTER(ltelib.Cell), C.POINTER(ltelib.Dci), C.c_int, C.POINTER(ltelib.UlGrant)]
    sizes = [L for L in range(3, 101) if S.lte_ul_valid_prb(L)]
    assert _ul_table_float2(cell.cell_id, ltelib.UlCfg(n_dmrs1=0, delta_ss=0, group_hopping=1), sizes) > UL_POOL_FLOAT2
    tbs = {}
    for L in sizes:                                   # MCS 0 from PRB 0
        d, g = ltelib.Dci(), ltelib.UlGrant()
        d.format, d.rnti, d.alloc_type = 0, 0x1000 + L, 2
        d.riv = 100 * (L - 1) if (L - 1) <= 50 else 100 * (100 - L + 1) + 99
        assert S.lte_ul_dci_to_grant(C.byref(cell), C.byref(d), 1, C.byref(g)) == 0
        tbs[L] = (g.qm, g.tbs)
    rng = np.random.default_rng(5)
    ul_iq = (rng.standard_normal((PHY_SUBFRAMES, iq.shape[2])) + 1j * rng.standard_normal((PHY_SUBFRAMES, iq.shape[2]))).astype(np.complex64)
    turbo_in = rng.integers(-40, 40, (4, 3 * (6144 + 4))).astype(np.int16)
    return iq, tti, grants, sizes, tbs, ul_iq, turbo_in


def test_ltephy_cycles(infra, phylib):
    from ltesniffer_b200 import capi
    iq, tti, grants, sizes, tbs, ul_iq, turbo_in = _phy_inputs()

    def exercise(phy):
        phy.set_cfo(150.0)
        phy.set_cfo(0.0)
        phy.harq_reserve(8)
        phy.submit_iq(iq, tti)
        phy.get_phase_a()
        mib = phy.mib_decode_combined(search_ports=True)
        phy.submit_grants(grants)
        res, pl = phy.get_phase_b()
        assert sum(r.crc for r in res) > 0
        out = [bytes(res), pl.tobytes(), bytes(mib)]
        phy.set_ul_cfg(0, 0, 1, 0)
        phy.set_ul_cfo(-80.0)
        for n_dmrs2 in range(8):
            ul = [capi.UlGrant(sf=sf, rnti=0x1000 + L, qm=tbs[L][0], rv=0, L_prb=L, n_prb=0, n_dmrs2=n_dmrs2, tbs=tbs[L][1])
                  for sf in range(PHY_SUBFRAMES) for L in sizes]
            ures, uch, upl = phy.decode_ul(ul_iq if n_dmrs2 == 0 else None, tti, ul)
            out += [bytes(ures), upl.tobytes()]
        out += [a.tobytes() for a in phy.turbo_batch(turbo_in, 6144, 4, 1)]
        return out

    # 700 subframes of 100 PRB and 2 antennas: about 0.7 GB of phase-A buffers, and the uplink's about 0.3 GB more
    _cycles(lambda: capi.LtePhy(*PHY_CELL, max_subframes=700, turbo_max_iter=8), exercise)


# ---------------------------------------------------------------------------------------------------- CellSearch
def test_cell_search_cycles(infra, phylib):
    from ltesniffer_b200 import capi
    from test_cell_search import sim_capture
    N, pci = 2048, 333
    x = sim_capture(N, pci, 22, N * 13 // 2, 75 * N + N + 100, nrx=2, snr=20.0, seed=9)

    def exercise(cs):
        got = cs.search(x)
        assert any(c.detected and c.pci == pci for c in got)
        return [bytes(c) for c in got]

    # 32 Mi samples on each of 2 antennas: about 0.7 GB
    _cycles(lambda: capi.CellSearch(N, 2, 32 << 20), exercise)


# ---------------------------------------------------------------------------------------------------- Tracker
def test_tracker_cycles(phylib):
    from ltesniffer_b200 import capi
    import track_reacq_lib as Q
    from test_track_reacquire import PCI, T0, drop_capture
    N = 384
    x, _, _, _, lead = drop_capture(N, 1, 20.0, "37SF+1234")
    xu = Q.noise(np.random.default_rng(5), 1, x.shape[1], 1.0)[0]

    def exercise(tr):
        got = tr.push_ul(x, xu, 0)
        assert got["finds"] == 1                      # the tracker's own cell search ran
        return [got["sf"].tobytes(), got["hf"].tobytes(), got["iq"].cpu().numpy().tobytes(), got["ul_iq"].cpu().numpy().tobytes()]

    # 6000 subframes of cut on the downlink and the uplink: about 0.7 GB
    _cycles(lambda: capi.Tracker(N, 1, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=capi.TRACK_REACQUIRE, max_subframes=6000,
                                 ul=dict(cfo_ratio=0.95, ul_offset=-(3 * N + 5))), exercise)


# ---------------------------------------------------------------------------------------------------- Shard
class _ShardedPipeline:
    """a Shard of world size 1 with the LtePhy and Search it decodes with, destroyed together"""

    def __init__(self, capi, cell, max_subframes):
        self.phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=max_subframes, turbo_max_iter=8,
                               flags=capi.FLAG_SKIP_LOW_POWER)
        self.srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
        self.sh = capi.Shard(capi.Shard.unique_id(), 0, 1, 0)

    def close(self):
        self.sh.close()
        self.srch.close()
        self.phy.close()


def test_shard_cycles(infra, phylib):
    from ltesniffer_b200 import capi
    from helpers import make_capture
    from test_gpu_shard import CELL, SIM_KW, _sharded_decode, _tb_table
    try:
        capi.Shard.unique_id()
    except RuntimeError as e:
        pytest.skip("NCCL cannot be loaded: %s" % e)
    cell = ltelib.Cell(*CELL)
    n = 16
    _, iq, tti, _, _ = make_capture(cell, n, **SIM_KW)

    def exercise(p):
        out = []
        for seq, (a, b) in enumerate([(0, 8), (8, 16)]):
            info, dcis, tbs, pl, st = _sharded_decode(capi, p.sh, p.phy, p.srch, iq[a:b], tti[a:b], seq, 32 * n, 1)
            out.append(_tb_table(dcis, tbs, pl))
        p.phy.submit_iq(iq[:8], tti[:8])              # and ltephy_pack_phase_a, which packs into a slot of its own
        p.phy.get_phase_a_compact()
        rec, offs = capi.pack_phase_a(p.phy)
        return out + [rec.tobytes(), offs.tobytes()]

    # 1000 subframes of 50 PRB and 2 antennas: about 0.6 GB, nearly all of it the LtePhy's
    _cycles(lambda: _ShardedPipeline(capi, cell, 1000), exercise)
