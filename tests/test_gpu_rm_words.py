"""GPU: the turbo input streams the rate de-matcher writes (LTEPHY_TAP_TURBO_IN) equal, word for word, the numpy restatement of the
per-word rule (tests/rm_ref.py) fed with the soft bits of LTEPHY_TAP_PDSCH_LLR: every DL transmission scheme, QPSK to 256QAM, filler
bits, ragged K, single-code-block pairs, HARQ first transmissions and retransmissions (one slot used twice in a batch), and the UL path."""
import numpy as np
import pytest

import ltelib
import rm_ref
from helpers import make_capture, to_phy_grant, truth_grants
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu

# (tx scheme, TBs as (tbs, qm, rv)): C = 1 with fillers (528 -> K 560, F 8, ragged), C = 1 without (40 -> K 64), several code blocks of
# two sizes (K- / K+), the largest K, 256QAM
SCHEMES = [
    (capi.TX_PORT0, [(528, 2, 0)]),
    (capi.TX_PORT0, [(14112, 4, 1)]),
    (capi.TX_DIVERSITY, [(2088, 6, 2)]),
    (capi.TX_DIVERSITY, [(40, 2, 3)]),
    (capi.TX_CDD, [(9528, 6, 0), (528, 4, 2)]),
    (capi.TX_CDD, [(25456, 8, 3), (3496, 8, 1)]),
    (capi.TX_SPATIALMUX, [(6968, 8, 2)]),
    (capi.TX_SPATIALMUX, [(11064, 6, 1), (1800, 2, 3)]),
]


@pytest.fixture(scope="module")
def dl_case(infra, phylib):
    cell = ltelib.Cell(50, 2, 3, 2)
    sim, iq, tti, truths, payloads = make_capture(cell, 3, seed=11, cfi=2, nof_ues=6, dl_min=3, dl_max=4, tm=3, mcs_min=4, mcs_max=16, snr_db=26.0)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=3)
    phy.submit_iq(iq, tti)
    phy.get_phase_a()
    tg = truth_grants(cell, truths, tti)
    assert len(tg) >= 8
    yield cell, phy, tg
    phy.close()


def _grant(sf, d, g, k, harq=None):
    """the truth grant's resource allocation with scheme / transport blocks of SCHEMES[k]; harq: [(op, slot)] per TB"""
    scheme, tbs = SCHEMES[k % len(SCHEMES)]
    pg = to_phy_grant(sf, d.rnti, g)
    pg.tx_scheme, pg.nof_tb, pg.pmi = scheme, len(tbs), 0
    for t in range(2):
        pg.tb[t].enabled = t < len(tbs)
        if t < len(tbs):
            pg.tb[t].tbs, pg.tb[t].qm, pg.tb[t].rv, pg.tb[t].cw_idx = tbs[t][0], tbs[t][1], tbs[t][2], t
            pg.tb[t].harq_op, pg.tb[t].harq_slot = harq[t] if harq else (0, 0)
    return pg


def _expect_dl(model, grants):
    model.begin()
    llr = 0
    for pg in grants:
        for t in range(2):
            if not pg.tb[t].enabled:
                continue
            G = pg.nof_re * pg.tb[t].qm
            model.add_tb(pg.tb[t].tbs, G, pg.tb[t].qm, pg.tb[t].rv, 2 if pg.tx_scheme == capi.TX_DIVERSITY else 1, llr, pg.tb[t].harq_op,
                         pg.tb[t].harq_slot)
            llr += (G + 7) & ~7
    return llr


def _check(phy, model, nllr):
    llr = phy.tap(capi.TAP_PDSCH_LLR, (nllr,), np.int16)
    got = phy.tap(capi.TAP_TURBO_IN, (2 * model.words,), np.int16)
    want = model.expected(llr)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "%d of %d int16 differ, first at %d: got %d want %d" % (bad.size, got.size, bad[0], got[bad[0]], want[bad[0]])
    return model


def test_dl_schemes_and_sizes(dl_case, phylib):
    cell, phy, tg = dl_case
    model = rm_ref.PhaseB(phylib)
    grants = [_grant(sf, d, g, k) for k, (sf, d, g) in enumerate(tg)]
    nllr = _expect_dl(model, grants)
    phy.submit_grants(grants)
    phy.get_phase_b()
    _check(phy, model, nllr)
    assert any(len(p["cbs"]) == 1 for p in model.pairs) and any(len(p["cbs"]) == 2 for p in model.pairs)
    assert any(cb["F"] > 0 for cb in model.cbs) and any(cb["K"] % 32 for cb in model.cbs)
    assert {cb["rv"] for cb in model.cbs} == {0, 1, 2, 3}


def test_dl_harq_first_transmission_and_retransmissions(dl_case, phylib):
    cell, phy, tg = dl_case
    phy.harq_reserve(16)
    model = rm_ref.PhaseB(phylib)
    # batch 1: every TB a first transmission in its own slot, except that grant 1 retransmits grant 0's first TB into the same slot in the
    # same batch (a second generation)
    first = []
    for k, (sf, d, g) in enumerate(tg[:6]):
        first.append(_grant(sf, d, g, 0 if k < 2 else k, [(rm_ref.HARQ_NEW, 2 * k), (rm_ref.HARQ_NEW, 2 * k + 1)]))
    first[1].tb[0].harq_op, first[1].tb[0].harq_slot, first[1].tb[0].rv = rm_ref.HARQ_RETX, 0, 2
    nllr = _expect_dl(model, first)
    assert any(cb["gen"] == 1 for cb in model.cbs)
    phy.submit_grants(first)
    phy.get_phase_b()
    _check(phy, model, nllr)
    # batch 2: the same transport blocks again, other redundancy versions and other soft bits, added to the slots
    second = []
    for k, (sf, d, g) in enumerate(tg[2:8]):
        pg = _grant(sf, d, g, k + 2, [(rm_ref.HARQ_RETX, 2 * k + 4), (rm_ref.HARQ_RETX, 2 * k + 5)])
        for t in range(2):
            pg.tb[t].rv = (pg.tb[t].rv + 2) & 3
        second.append(pg)
    nllr = _expect_dl(model, second)
    phy.submit_grants(second)
    phy.get_phase_b()
    _check(phy, model, nllr)


def test_ul_path(infra, phylib):
    cell = ltelib.Cell(50, 1, 9, 1)
    ucfg = ltelib.UlCfg(n_dmrs1=3, delta_ss=2)
    s = ltelib.Sim(cell=cell, seed=5, snr_db=25.0, nof_ues=1)
    rng = np.random.default_rng(5)
    iq = np.zeros((2, s.sf_len), np.complex64)
    grants, capi_grants = [], []
    for i in range(2):
        gr = [g for g in ltelib.make_ul_grants(cell, rng, 4, table=1)]
        iq[i] = ltelib.sim_ul_subframe(s, i, ucfg, gr)[0]
        grants += gr
        capi_grants += [capi.UlGrant(sf=i, rnti=g.rnti, qm=g.qm, rv=g.rv, L_prb=g.L_prb, n_prb=g.n_prb, n_dmrs2=g.n_dmrs2, tbs=g.tbs, n_prb_slot1=g.n_prb,
                                     flags=capi.UL_FLAG_SLOT1, nof_ack=g.nof_ack, ri_len=g.ri_len, cqi_len=g.cqi_len, I_offset_ack=g.I_offset_ack,
                                     I_offset_ri=g.I_offset_ri, I_offset_cqi=g.I_offset_cqi) for g in gr]
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=2)
    try:
        phy.set_ul_cfg(3, 2)
        phy.decode_ul(iq, np.arange(2, dtype=np.uint32), capi_grants)
        model = rm_ref.PhaseB(phylib)
        model.begin()
        llr = 0
        for g in grants:
            G = ltelib.uci_layout(g).G
            model.add_tb(g.tbs, G, g.qm, g.rv, 1, llr)
            llr += (G + 7) & ~7
        _check(phy, model, llr)
    finally:
        phy.close()
