"""Uplink receive diversity on the CPU (DESIGN.md §2, "uplink receive diversity"): the two-antenna PUSCH oracle lteo_pusch_decode_rx against the
one-antenna oracle lteo_pusch_decode and against float64 references, the gain of the second antenna, the simulator's multi-antenna uplink and the
oracle tracker's multi-antenna UL cut."""
import numpy as np
import pytest

import ltelib
import pusch_rx_lib as X
import ref64_ul
from ltelib import Cell, Oracle, Sim, UlCfg
from test_pusch_float64_reference import G, check_chest, check_soft_bits, to_oracle, ul_cfg


def _grants(cell, rng, n, table, mutate=None, min_prb=3):
    gr = ltelib.make_ul_grants(cell, rng, n, table=table, min_prb=min_prb)
    for g in gr:
        if mutate:
            mutate(cell, g, rng)
    return gr


def _uci(cell, g, rng):
    k = int(rng.integers(0, 3))
    if k == 0:
        g.nof_ack, g.I_offset_ack = 2, 10
    elif k == 1:
        g.cqi_len, g.I_offset_cqi, g.ri_len, g.I_offset_ri, g.nof_ack, g.I_offset_ack = 30, 6, 1, 5, 1, 9
    else:
        g.ri_len, g.I_offset_ri = 2, 8


def _hop(cell, g, rng):
    g.hop, g.n_prb_slot1 = 1, int((g.n_prb + 17) % (cell.nof_prb - g.L_prb + 1))
    g.ta_us = float(rng.uniform(-0.8, 0.8))


# (cell, UL configuration, table (2: Qm up to 8), grant mutation, grants per subframe, minimum L_prb)
CASES = [
    ("qm2-6", Cell(50, 1, 17, 1), UlCfg(n_dmrs1=3, delta_ss=2), 1, None, 4, 3),
    ("qm8", Cell(25, 1, 5, 1), UlCfg(n_dmrs1=1, delta_ss=9), 2, None, 3, 3),
    ("uci", Cell(50, 1, 23, 1), UlCfg(n_dmrs1=4, delta_ss=7), 1, _uci, 3, 3),
    ("hop_gh", Cell(50, 1, 301, 1), UlCfg(n_dmrs1=2, delta_ss=11, group_hopping=1), 1, _hop, 1, 6),
    ("hop_sh", Cell(75, 1, 302, 1), UlCfg(n_dmrs1=5, delta_ss=3, seq_hopping=1), 2, _hop, 1, 6),
]


def _subframes(case, nsf=3, snr=24.0, nof_rx=2, seed=11):
    cid, cell, ucfg, table, mut, ngr, min_prb = case
    s = Sim(cell=Cell(cell.nof_prb, 1, cell.cell_id, 2), seed=seed, snr_db=snr, nof_ues=1, chan_delay=3)
    rng = np.random.default_rng(seed)
    out = []
    for i in range(nsf):
        gr = _grants(cell, rng, ngr, table, mut, min_prb)
        iq, pl, off = X.sim_ul_rx(s, 3 + i, ucfg, gr, nof_rx)
        out.append((3 + i, gr, iq, pl, off))
    return cell, ucfg, out


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_one_antenna_equals_the_one_antenna_oracle(infra, case):
    """lteo_pusch_decode_rx with nof_rx = 1 equals lteo_pusch_decode bit for bit: soft bits, payload, CRC and every chest figure"""
    cell, ucfg, sfs = _subframes(case)
    o = Oracle(cell)
    qms = set()
    for tti, gr, iq, _, _ in sfs:
        _, ref = ltelib.oracle_ul(o, ucfg, tti, gr, iq[0], want_llr=True)
        _, got = X.oracle_ul_rx(o, ucfg, tti, gr, iq[:1])
        for g, (r, pl, ok, ch, llr), (r2, pl2, ok2, ch2, llr2, _) in zip(gr, ref, got):
            G_ = ltelib.uci_layout(g).G
            assert r == r2 == 0
            assert np.array_equal(llr[:G_], llr2)
            assert ok == ok2 and np.array_equal(pl[:g.tbs // 8], pl2[:g.tbs // 8])
            assert (ch.noise, ch.rsrp, ch.snr_db, ch.ta_us) == (ch2.noise, ch2.rsrp, ch2.snr_db, ch2.ta_us)
            qms.add(g.qm)
    assert qms


def test_case_matrix_covers_every_modulation():
    qms = set()
    for case in CASES:
        cell, _, sfs = _subframes(case, nsf=3)
        qms |= {g.qm for _, gr, *_ in sfs for g in gr}
    assert qms == {2, 4, 6, 8}


@pytest.mark.parametrize("case", CASES[:3], ids=[c[0] for c in CASES[:3]])
def test_same_antenna_twice_and_a_silent_second_antenna(infra, case):
    """the same grid twice: numerator and denominator are doubled, which is exact, so soft bits and payload equal one antenna's; noise / RSRP agree to
    the rounding of the longer sum (antenna-major, then slot: ((s0 + s1) + s0) + s1 is not 2 (s0 + s1) bit for bit).  A second antenna of zeros adds exact zeros to both sums: soft bits equal antenna 0's alone, noise and RSRP are halved"""
    cell, ucfg, sfs = _subframes(case)
    o = Oracle(cell)
    for tti, gr, iq, _, _ in sfs:
        sym = X.ul_ofdm(o, iq[:1])
        for g in gr:
            r1, pl1, ok1, ch1, llr1, eq1 = X.decode_rx(cell, ucfg, tti % 10, g, [sym[0]])
            r2, pl2, ok2, ch2, llr2, eq2 = X.decode_rx(cell, ucfg, tti % 10, g, [sym[0], sym[0]])
            r3, pl3, ok3, ch3, llr3, eq3 = X.decode_rx(cell, ucfg, tti % 10, g, [sym[0], np.zeros_like(sym[0])])
            nb = g.tbs // 8
            for llr, pl, ok, eq in ((llr2, pl2, ok2, eq2), (llr3, pl3, ok3, eq3)):
                assert np.array_equal(llr, llr1) and ok == ok1 and np.array_equal(pl[:nb], pl1[:nb]) and np.array_equal(eq, eq1)
            assert abs(ch2.noise - ch1.noise) <= 1e-6 * ch1.noise and abs(ch2.rsrp - ch1.rsrp) <= 1e-6 * ch1.rsrp
            assert (ch3.noise, ch3.rsrp) == (ch1.noise / 2, ch1.rsrp / 2)


def _rx_cases():
    """(id, cell, UL configuration, [(sf, grants)], per-antenna (channel, delay))"""
    fade = lambda nsc: ref64_ul.channel("selective", nsc) * 10 ** (-30 / 20)
    flat2 = lambda nsc: np.exp(-1.9j) * 0.7 * np.ones((14, nsc), complex)
    return [
        ("flat", (25, 1, 150, 2, 0), (1, 3, 1, 0), [(2, [G(25, 0, 8, n_dmrs2=4, rnti=0x3001)]), (3, [G(5, 0, 2, ri_len=2, I_ri=5), G(20, 5, 4, nof_ack=2, I_ack=10)])],
         [(lambda nsc: ref64_ul.channel("flat", nsc), 0), (flat2, 0)]),
        ("delayed", (50, 1, 301, 2, 768), (2, 7, 0, 1), [(4, [G(48, 0, 6, n_dmrs2=10)]), (5, [G(6, 0, 4, n_dmrs2=9), G(40, 10, 8, ri_len=1, I_ri=2)])],
         [(lambda nsc: ref64_ul.channel("flat", nsc), 3), (flat2, -4)]),
        ("faded", (100, 1, 7, 2, 0), (4, 0, 0, 0), [(8, [G(100, 0, 4, n_dmrs2=6)]), (9, [G(20, 0, 6, n_prb1=55, nof_ack=2, I_ack=3), G(27, 60, 2)])],
         [(lambda nsc: ref64_ul.channel("selective", nsc), 0), (fade, 0)]),
    ]


@pytest.mark.parametrize("case", _rx_cases(), ids=[c[0] for c in _rx_cases()])
def test_two_antennas_equal_the_float64_reference(infra, case):
    """independent channels per antenna (flat, delayed by whole samples, one antenna 30 dB down on a selective channel): the equalised symbols within
    3e-5 of the float64 combiner's relative to the symbol's largest magnitude, the chest figures within check_chest's bars, the soft bits within
    check_soft_bits'"""
    cid, cellp, u, sfs, chans = case
    cell = Cell(*cellp)
    o = Oracle(cell)
    nsc = 12 * cell.nof_prb
    for i, (sf, grants) in enumerate(sfs):
        rng = np.random.default_rng(100 + i)
        grid = np.zeros((14, nsc), complex)
        for g in grants:
            grid += ref64_ul.transmit(cell, g, sf, u, None, rng)[0]
        iq = np.array([ref64_ul.scfdma_modulate(cell, ref64_ul.receive(grid, H(nsc), 3e-3, rng), d) for H, d in chans]).astype(np.complex64)
        Ys = [ref64_ul.ul_grid(cell, iq[a]) for a in range(2)]
        sym = X.ul_ofdm(o, iq)
        for g in grants:
            what = "%s sf %d L %d" % (cid, sf, g.L)
            r, _, _, ch, llr, eq = X.decode_rx(cell, ul_cfg(u), sf, to_oracle(g), sym)
            assert r == 0
            info, eq_ref, llr_ref, cond = X.decode_ref_rx(cell, Ys, g, sf, u)
            check_chest(ch, info, what)
            err = np.abs(eq - eq_ref).max(axis=1) / np.abs(eq_ref).max(axis=1)
            assert err.max() <= 3e-5, (what, err.max())
            check_soft_bits(llr, llr_ref, cond, what)


SNR_GAIN_DB = 10.0   # noise power 10 dB below the unit-power channel: antenna 0 alone decodes about half of the grants


def test_second_antenna_decodes_more_grants_under_rayleigh_fading(infra):
    """per-grant Rayleigh flat channels, independent per antenna, at an SNR where antenna 0 alone decodes about half of 240 grants: both antennas
    decode strictly more.  Measured: 117 of 240 with antenna 0, 179 with both (10 dB below the unit-power channel); pinned with a margin."""
    cell = Cell(25, 1, 41, 2)
    ucfg = UlCfg(n_dmrs1=2, delta_ss=4)
    s = Sim(cell=cell, seed=3, snr_db=300.0, nof_ues=1)        # noiseless: the channel and the noise are drawn here
    o = Oracle(cell)
    rng = np.random.default_rng(77)
    ok1 = ok2 = n = 0
    sigma = 10 ** (-SNR_GAIN_DB / 20) * np.sqrt(0.5)
    for i in range(240):
        g = _grants(cell, rng, 1, 1)[0]
        x, pl, off = X.sim_ul_rx(s, i, ucfg, [g], 1)
        h = (rng.standard_normal(2) + 1j * rng.standard_normal(2)) * np.sqrt(0.5)
        y = (h[:, None] * x[0][None, :] + sigma * (rng.standard_normal((2, x.shape[1])) + 1j * rng.standard_normal((2, x.shape[1])))).astype(np.complex64)
        sym = X.ul_ofdm(o, y)
        a = X.decode_rx(cell, ucfg, i % 10, g, sym[:1])
        b = X.decode_rx(cell, ucfg, i % 10, g, sym)
        ok1 += a[2]
        ok2 += b[2]
        n += 1
    assert 100 <= ok1 <= 140, ok1
    assert ok2 >= ok1 + 45 and ok2 >= 165, (ok1, ok2)



def test_simulator_antenna_zero_is_the_one_antenna_subframe(infra):
    """lte_sim_ul_subframe_rx: antenna 0 equals lte_sim_ul_subframe bit for bit (antenna 1's noise is drawn after antenna 0's); antenna 1 differs"""
    cell = Cell(25, 1, 5, 2)
    ucfg = UlCfg(n_dmrs1=3, delta_ss=2)
    for seed in (1, 2):
        gr = ltelib.make_ul_grants(cell, np.random.default_rng(seed), 3)
        one = ltelib.sim_ul_subframe(Sim(cell=cell, seed=seed, snr_db=20.0, nof_ues=1, chan_delay=4), 7, ucfg, gr)
        two = X.sim_ul_rx(Sim(cell=cell, seed=seed, snr_db=20.0, nof_ues=1, chan_delay=4), 7, ucfg, gr, 2)
        assert one[0].tobytes() == two[0][0].tobytes() and np.array_equal(one[1], two[1]) and np.array_equal(one[2], two[2])
        assert not np.array_equal(two[0][0], two[0][1])


def test_oracle_tracker_cuts_each_ul_antenna_as_a_one_antenna_tracker():
    """lteo_track_set_ul_rx with two UL antennas: UL antenna a of the cut equals the UL cut of a one-antenna tracker fed antenna a, records and DL
    cut unchanged; nof_rx 3 is refused"""
    import track_lib as T
    N = 256
    x = T.capture(N, 33, 40, nrx=2, ppm=20.0, cfo=700.0, ramp=500.0, snr=12.0, lead=1234, seed=4)[0]
    rng = np.random.default_rng(9)
    xu = (rng.standard_normal((2, x.shape[1])) + 1j * rng.standard_normal((2, x.shape[1]))).astype(np.complex64)
    got = T.Oracle(N, 2, 33, 1234, cfo_hz=650.0, ul=dict(cfo_ratio=0.948, ul_offset=-200, nof_rx=2)).push_ul(x, xu, 0)
    assert len(got["sf"]) >= 35
    for a in range(2):
        one = T.Oracle(N, 2, 33, 1234, cfo_hz=650.0, ul=dict(cfo_ratio=0.948, ul_offset=-200)).push_ul(x, xu[a], 0)
        assert got["sf"].tobytes() == one["sf"].tobytes() and got["hf"].tobytes() == one["hf"].tobytes() and got["iq"].tobytes() == one["iq"].tobytes()
        assert np.ascontiguousarray(got["ul_iq"][:, a]).tobytes() == one["ul_iq"].tobytes()
    t = T.Oracle(N, 2, 33, 1234)
    assert T.lib().lteo_track_set_ul_rx(t.t, 1.0, 0, 3) == -2


def test_three_ul_antennas_are_refused_without_a_gpu(phylib):
    """ltephy_create checks ul_nof_rx before it looks for a device"""
    from ltesniffer_b200 import capi
    with pytest.raises(RuntimeError, match=r"\(-2\)"):
        capi.LtePhy(25, 1, 5, 1, max_subframes=1, ul_nof_rx=3)
