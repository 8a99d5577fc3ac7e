"""Phase-B state shared by the downlink, uplink and stand-alone turbo entry points (pytest -m gpu).

* The PUSCH DMRS / IDFT table pool grows past its first reservation and keeps every table built before the growth valid: one handle
  builds the tables of every allocation size, every n_DMRS^(2) and every slot of a 100-PRB cell with group hopping, then decodes a
  simulated capture bit-exactly against the oracle.
* ltephy_turbo_batch starts a new batch like the other submits, so a later ltephy_get_phase_b reports no transport block."""
import ctypes as C

import numpy as np
import pytest

import ltelib
from helpers import make_capture, to_phy_grant, truth_grants
from ltesniffer_b200 import capi
from ref64 import gold
from test_gpu_pusch import _run_ul_case

pytestmark = pytest.mark.gpu

UL_POOL_FLOAT2 = (1 << 20) + (1 << 18) + 1024        # the pool's first reservation: DevBuf::reserve(1 Mi) rounds up by a quarter + 1024
N_DMRS1_OF = [0, 2, 3, 4, 6, 8, 9, 10]                # cyclicShift -> n_DMRS^(1), 36.211 Table 5.5.2.1.1-2


def _ul_table_float2(cell_id, ucfg, sizes):
    """float2 of the distinct DMRS (M, n_cs, u, v) and IDFT (M) tables that grants of every size, every n_DMRS^(2) and every slot
    ask for under group hopping (v = 0): n_PRS(ns) from 36.211 5.5.2.1.1, f_gh(ns) from 5.5.1.3, as in ltephy_set_ul_cfg"""
    assert ucfg.group_hopping and not ucfg.seq_hopping
    fss = (cell_id % 30 + ucfg.delta_ss) % 30
    c = gold((cell_id // 30) * 32 + fss, 8 * 7 * 20 + 8)
    cg = gold(cell_id // 30, 8 * 20 + 8)
    keys = set()
    for ns in range(20):
        n_prs = sum(int(c[8 * 7 * ns + i]) << i for i in range(8))
        u = (sum(int(cg[8 * ns + i]) << i for i in range(8)) % 30 + fss) % 30
        for n_dmrs2 in range(8):
            for L in sizes:
                keys.add((12 * L, (N_DMRS1_OF[ucfg.n_dmrs1] + n_dmrs2 + n_prs) % 12, u))
    return sum(M for M, _, _ in keys) + sum(12 * L for L in sizes)


def test_pusch_tables_grow_past_first_pool(infra, phylib):
    cell = ltelib.Cell(100, 1, 4, 1)
    ucfg = ltelib.UlCfg(n_dmrs1=0, delta_ss=0, group_hopping=1)
    S = ltelib.sim()
    S.lte_ul_valid_prb.argtypes = [C.c_uint32]
    S.lte_ul_dci_to_grant.argtypes = [C.POINTER(ltelib.Cell), C.POINTER(ltelib.Dci), C.c_int, C.POINTER(ltelib.UlGrant)]
    sizes = [L for L in range(3, 101) if S.lte_ul_valid_prb(L)]
    assert len(sizes) == 32
    need = _ul_table_float2(cell.cell_id, ucfg, sizes)
    assert need > UL_POOL_FLOAT2, need
    tbs = {}
    for L in sizes:                                   # MCS 0 from PRB 0: the smallest transport block of each size
        d, g = ltelib.Dci(), ltelib.UlGrant()
        d.format, d.rnti, d.alloc_type = 0, 0x1000 + L, 2
        d.riv = 100 * (L - 1) if (L - 1) <= 50 else 100 * (100 - L + 1) + 99
        assert S.lte_ul_dci_to_grant(C.byref(cell), C.byref(d), 1, C.byref(g)) == 0 and (g.L_prb, g.n_prb) == (L, 0)
        tbs[L] = (g.qm, g.tbs)
    nsf = 10
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=nsf)
    try:
        phy.set_ul_cfg(ucfg.n_dmrs1, ucfg.delta_ss, ucfg.group_hopping, ucfg.seq_hopping)
        rng = np.random.default_rng(5)
        noise = (rng.standard_normal((nsf, phy.sf_len)) + 1j * rng.standard_normal((nsf, phy.sf_len))).astype(np.complex64)
        tti = np.arange(nsf, dtype=np.uint32)
        for n_dmrs2 in range(8):                      # one batch per n_DMRS^(2): every size in every subframe
            grants = [capi.UlGrant(sf=sf, rnti=0x1000 + L, qm=tbs[L][0], rv=0, L_prb=L, n_prb=0, n_dmrs2=n_dmrs2, tbs=tbs[L][1])
                      for sf in range(nsf) for L in sizes]
            res, ch, payload = phy.decode_ul(noise if n_dmrs2 == 0 else None, tti, grants)
            assert all(res[i].payload_len == tbs[g.L_prb][1] // 8 for i, g in enumerate(grants))

        def ta_only(g, rng):
            g.ta_us = float(rng.uniform(-1.0, 1.0))
        nok, k = _run_ul_case(cell, ucfg, ta_only, ngr=5, nsf=2, seed=70, phy=phy)   # tables built before and after the growth
        assert nok == k
    finally:
        phy.close()


def test_get_phase_b_after_turbo_batch_reports_nothing(infra, phylib):
    cell = ltelib.Cell(25, 1, 5, 1)
    sim, iq, tti, truths, payloads = make_capture(cell, 2, seed=11, cfi=2, nof_ues=4, dl_min=2, dl_max=3, tm=1, mcs_min=2, mcs_max=12, snr_db=30.0)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=2)
    try:
        phy.submit_iq(iq, tti)
        phy.get_phase_a()
        grants = [to_phy_grant(sf, d.rnti, g) for sf, d, g in truth_grants(cell, truths, tti)]
        assert grants
        phy.submit_grants(grants)
        res, pl = phy.get_phase_b()
        assert sum(1 for r in res[:2 * len(grants)] if r.crc) > 0
        K = 40
        bits, iters, ok = phy.turbo_batch(np.zeros((3, 3 * (K + 4)), np.int16), K, 2, 0)
        assert bits.shape == (3, K)
        out = (capi.TbResult * (2 * len(grants)))()
        for r in out:
            r.crc, r.payload_len = 0xAB, 0xFFFFFFFF
        buf = np.zeros(1 << 16, np.uint8)
        assert phy.L.ltephy_get_phase_b(phy.h, out, buf.ctypes.data, buf.nbytes) == 0
        assert all(r.crc == 0xAB and r.payload_len == 0xFFFFFFFF for r in out)   # no result slot: nothing written
        assert phy.turbo_work()[2] == 0                                             # and no transport block in the batch
    finally:
        phy.close()
