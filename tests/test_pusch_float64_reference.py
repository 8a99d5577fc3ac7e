"""The CPU oracle's PUSCH receive path against the float64 references of tests/ref64_ul.py (written from 36.211 / 36.212 / 36.213 and DESIGN.md
section 2, not from lte_oracle.c).  test_gpu_pusch.py holds the kernel bit-exact to lteo_pusch_decode, and simulator captures at 20-34 dB pass their
CRC with a wrong interpolation weight or scale just as well; so a formula the oracle and the kernel both restate wrongly -- the weight of an
extrapolated symbol, the 1 / sqrt M of the IDFT, the scrambling bit index, which control symbols are dropped or erased, the noise normalisation, the
sign of the timing offset -- is invisible to them.  These tests pin the oracle from outside; tests/test_gpu_pusch_float64_reference.py runs the same
cases against the kernels.

Inputs are synthesised in numpy (ref64_ul's transmitter: DMRS, interleaver, scrambling, transform precoding, a designed channel, the SC-FDMA
modulator), so nothing here goes through the simulator's transmitter, which shares the DMRS and the control-information map with the oracle."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import ltelib
import ref64
import ref64_ul
from ref64_ul import Grant
from ltelib import Cell, Oracle, UlCfg
from test_float64_reference import check_llr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import check_tables  # noqa: E402

_TBS = np.array(check_tables.load()[2]).reshape(-1, 110)
ITBS = {2: 6, 4: 14, 6: 20, 8: 26}                                         # a transport block size of each modulation's own range


def tbs(L, qm, itbs=None):
    return int(_TBS[ITBS[qm] if itbs is None else itbs, L - 1])


def G(L, n_prb, qm, **kw):
    return Grant(L, n_prb, qm, kw.pop("tbs", None) or tbs(L, qm), **kw)


# ------------------------------------------------------------------------------------------------ the case matrix
# (id, cell (nof_prb, ports, cell_id, rx, symbol_sz), UL configuration (cyclicShift, delta_ss, group hopping, sequence hopping),
#  subframes [(sf_idx, channel, delay in samples, grants)]).  Between them: every subframe index and cyclicShift, 15 / 25 / 50 / 75 / 100 PRB with
#  384, 768 and 1536-point symbols, L_prb 3 (M = 36), 25 (M = 300: 8 + 4 symbols per IDFT pass), 75 (3 * 5^2) and 100 (M = 1200: 2 symbols per pass),
#  allocations at PRB 0 and at the top edge, Qm 2 / 4 / 6 / 8, group and sequence hopping, type-1 hopping, ACK over data and over CQI, 2-bit RI,
#  long CQI, a deep fade and whole-sample delays of both signs
def cell_cases():
    return [
        ("p15_384", (15, 1, 31, 1, 384), (0, 0, 0, 0), [
            (0, "selective", 0, [G(3, 0, 2), G(12, 3, 4, n_dmrs2=6, nof_ack=1, I_ack=9, rnti=0x2001)]),
            (1, "late_change", 0, [G(15, 0, 6, n_dmrs2=3, rnti=0x2002)])]),
        ("p25_gh", (25, 1, 150, 1, 0), (1, 3, 1, 0), [
            (2, "selective", 0, [G(25, 0, 8, n_dmrs2=4, rnti=0x3001)]),
            (3, "linear_l", 0, [G(5, 0, 2, n_dmrs2=2, ri_len=2, I_ri=5, rnti=0x3002),
                                G(20, 5, 4, n_dmrs2=8, nof_ack=2, I_ack=10, cqi_len=30, I_cqi=6, rnti=0x3003)])]),
        ("p50_768_sh", (50, 1, 301, 1, 768), (2, 7, 0, 1), [
            (4, "selective", 0, [G(48, 0, 6, n_dmrs2=10, rnti=0x4001)]),
            (5, "flat", 0, [G(6, 0, 4, n_dmrs2=9, rnti=0x4002), G(4, 6, 2, rnti=0x4003), G(40, 10, 8, rnti=0x4004, ri_len=1, I_ri=2)])]),
        ("p75_gh_hop", (75, 1, 77, 1, 0), (3, 11, 1, 0), [
            (6, "linear_l", 0, [G(75, 0, 4, n_dmrs2=3, rnti=0x5001)]),
            (7, "per_slot", 0, [G(20, 0, 6, n_prb1=55, rnti=0x5002, nof_ack=2, I_ack=3), G(27, 20, 2, n_prb1=0, n_dmrs2=6, rnti=0x5003)])]),
        ("p100", (100, 1, 7, 1, 0), (4, 0, 0, 0), [
            (8, "selective", 0, [G(100, 0, 8, n_dmrs2=6, rnti=0x6001)]),
            (9, "selective", 0, [G(3, 97, 2, tbs=tbs(3, 2, 0), cqi_len=30, I_cqi=2, nof_ack=2, I_ack=14, rnti=0x6002),
                                 G(45, 0, 6, n_dmrs2=2, ri_len=1, I_ri=8, nof_ack=1, I_ack=6, cqi_len=11, I_cqi=9, rnti=0x6003),
                                 G(36, 50, 4, n_dmrs2=9, rnti=0x6004)])]),
        ("p100_1536_fade", (100, 1, 1, 1, 1536), (5, 29, 1, 0), [
            (0, "fade", 0, [G(50, 0, 4, rnti=0x7001), G(50, 50, 6, n_dmrs2=8, rnti=0x7002)]),
            (1, "flat", 7, [G(32, 4, 2, rnti=0x7003), G(64, 36, 4, n_dmrs2=4, rnti=0x7004)])]),
        ("p50_sh_delay", (50, 1, 9, 1, 0), (6, 2, 0, 1), [
            (2, "flat", -5, [G(30, 20, 6, n_dmrs2=4, rnti=0x8001), G(16, 0, 8, n_dmrs2=10, rnti=0x8002)])]),
        ("p25_hop", (25, 1, 5, 1, 0), (7, 5, 0, 0), [
            (3, "selective", 0, [G(9, 16, 4, n_dmrs2=10, rnti=0x9001), G(8, 0, 8, rnti=0x9002)]),
            (4, "per_slot", 0, [G(10, 0, 8, n_prb1=15, rnti=0x9003)])]),
    ]


FADE_PRBS = list(range(4)) + list(range(20, 24)) + list(range(96, 100))


def ul_cfg(u):
    return UlCfg(n_dmrs1=u[0], delta_ss=u[1], group_hopping=u[2], seq_hopping=u[3], n_rb_ho=0)


def to_oracle(g):
    """the ref64_ul grant as lteo_pusch_decode takes it"""
    o = ltelib.UlGrant(rnti=g.rnti, L_prb=g.L, n_prb=g.n_prb, qm=g.qm, rv=0, tbs=g.tbs, n_dmrs2=g.n_dmrs2, hop=int(g.hop), n_prb_slot1=g.n_prb1,
                       nof_ack=g.uci["nof_ack"], ri_len=g.uci["ri_len"], cqi_len=g.uci["cqi_len"], I_offset_ack=g.uci["I_ack"],
                       I_offset_ri=g.uci["I_ri"], I_offset_cqi=g.uci["I_cqi"])
    o.nof_re, o.nof_bits = 12 * g.M, g.G
    return o


class Subframe:
    """one synthesised uplink subframe: the grants' grids through a designed channel (or a pure delay), AWGN per RE, SC-FDMA.
    iq complex64 [sf_len]; bits: the UL-SCH bits of each grant (None: random); H: the channel [14][nsc] (default: the kind's)"""

    def __init__(self, cell, sf, ucfg, grants, chan="selective", delay=0, noise_var=3e-3, seed=0, bits=None, H=None):
        rng = np.random.default_rng(seed)
        self.cell, self.sf, self.ucfg, self.grants, self.delay = cell, sf, ucfg, grants, delay
        nsc = 12 * cell.nof_prb
        grid = np.zeros((14, nsc), complex)
        self.d = []
        for i, g in enumerate(grants):
            gg, d = ref64_ul.transmit(cell, g, sf, ucfg, None if bits is None else bits[i], rng)
            grid += gg
            self.d.append(d)
        self.H = H if H is not None else ref64_ul.channel(chan, nsc, prbs=FADE_PRBS)
        Y = ref64_ul.receive(grid, self.H, noise_var, rng)
        self.iq = ref64_ul.scfdma_modulate(cell, Y, delay).astype(np.complex64)

    def reference(self, iq=None):
        """float64 receive chain from the complex64 samples -> (grid, [(chest, llr, cond)] per grant)"""
        Y = ref64_ul.ul_grid(self.cell, self.iq if iq is None else iq)
        return Y, [ref64_ul.decode(self.cell, Y, g, self.sf, self.ucfg) for g in self.grants]


def synth(case):
    """noise variance 3e-3 per RE; 3e-7 under the deep fade, whose estimate must be deeper than the noise to saturate"""
    cid, cellp, u, sfs = case
    cell = Cell(*cellp)
    return cell, [Subframe(cell, sf, u, grants, chan=chan, delay=delay, noise_var=3e-7 if chan == "fade" else 3e-3, seed=100 * i + sf)
                  for i, (sf, chan, delay, grants) in enumerate(sfs)]


def check_chest(got, ref, what):
    """noise / RSRP within 1e-5 relative, snr_db within 1e-4 dB, ta_us within 1e-3 us"""
    assert abs(got.noise - ref["noise"]) <= 1e-5 * ref["noise"], (what, got.noise, ref["noise"])
    assert abs(got.rsrp - ref["rsrp"]) <= 1e-5 * ref["rsrp"], (what, got.rsrp, ref["rsrp"])
    assert abs(got.snr_db - ref["snr_db"]) <= 1e-4, (what, got.snr_db, ref["snr_db"])
    assert abs(got.ta_us - ref["ta_us"]) <= 1e-3, (what, got.ta_us, ref["ta_us"])


ILL_SIGN_BAR = 1024


def check_soft_bits(got, ref, cond, what):
    """check_llr's bar (test_float64_reference.py) with cond = max |h|^2 / min |h|^2 over the data symbol of each soft bit: where cond <= 100, |diff| <= 1,
    >= 99.5 % exactly equal, saturated values exact.  Above 100 the signs where |ref| > ILL_SIGN_BAR, not 64: the IDFT puts the float32 rounding of the
    deepest RE's quotient into every sample of the symbol, and the fold bits of large samples are differences of large numbers (the deep fade, cond
    2e7 - 2e9: |diff| up to 578, no sign flip above 256)"""
    got = np.asarray(got, np.int64)[:len(ref)]
    well = cond <= 100
    check_llr(got[well], ref[well], cond[well], 1, what)
    strong = ~well & (np.abs(ref) > ILL_SIGN_BAR)
    assert np.all(np.sign(got[strong]) == np.sign(ref[strong])), "%s: %d sign flips on ill-conditioned symbols" % (what, int(np.sum(np.sign(got[strong]) != np.sign(ref[strong]))))


def check_grid(got, Y, cell, what):
    N = ref64.fft_size(cell)
    err = np.abs(np.asarray(got).reshape(Y.shape) - Y).max()
    assert err <= 2e-5 * np.sqrt(N), (what, err, 2e-5 * np.sqrt(N))


def oracle_decode(o, s, iq=None, max_iter=8):
    """lteo_ul_ofdm + lteo_pusch_decode of every grant of the subframe -> (UL grid, [(ret, payload, crc, chest, llr)])"""
    return ltelib.oracle_ul(o, ul_cfg(s.ucfg), s.sf, [to_oracle(g) for g in s.grants], s.iq if iq is None else iq, max_iter=max_iter, want_llr=True)


CASES = cell_cases()


def test_case_matrix_covers_the_edges():
    sfs = [(cellp, sf, chan, delay, g) for _, cellp, u, subs in CASES for sf, chan, delay, grants in subs for g in grants]
    assert {sf for _, sf, _, _, _ in sfs} == set(range(10))
    assert {u[0] for _, _, u, _ in CASES} == set(range(8))
    assert {c[0] for _, c, _, _ in CASES} == {15, 25, 50, 75, 100} and {c[4] for _, c, _, _ in CASES} >= {384, 768, 1536}
    Ls = {g.L for *_, g in sfs}
    assert {3, 25, 75, 100} <= Ls
    assert {g.qm for *_, g in sfs} == {2, 4, 6, 8}
    assert any(g.n_prb == 0 for *_, g in sfs) and any(g.n_prb + g.L == c[0] for c, *_, g in sfs)
    assert {(u[2], u[3]) for _, _, u, _ in CASES} == {(0, 0), (1, 0), (0, 1)}
    assert any(g.hop for *_, g in sfs)
    kinds = set().union(*(set(np.unique(g.kind).tolist()) for *_, g in sfs))
    assert kinds == {ref64_ul.DATA, ref64_ul.CQI, ref64_ul.RI, ref64_ul.ACK_DATA, ref64_ul.ACK_CQI}
    assert any(g.uci["ri_len"] == 2 for *_, g in sfs) and any(g.uci["cqi_len"] > 11 for *_, g in sfs)
    assert {d for *_, d, _ in sfs} >= {-5, 0, 7}
    assert all(g.G > 0 for *_, g in sfs)                                   # the product refuses a grant whose control information fills it
    for _, cellp, _, subs in CASES:                                         # grants of one subframe never share a PRB in a slot
        for sf, _, _, grants in subs:
            for sl in range(2):
                used = np.concatenate([np.arange(g.k0(sl) // 12, g.k0(sl) // 12 + g.L) for g in grants])
                assert len(set(used.tolist())) == len(used) and used.max() < cellp[0], (cellp, sf, sl)


# ------------------------------------------------------------------------------------------------ primitives of the reference against the shared C
def test_reference_layout_and_map_equal_the_shared_primitives(infra):
    """the reference's Q' / G (exact rationals) and interleaver map against lte_uci_layout / lte_uci_map, on every grant of the matrix and on a sweep of
    beta offsets: a disagreement here would be one the oracle's soft-bit comparison cannot localise"""
    S = ltelib.sim()
    S.lte_uci_map.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    grants = [g for _, _, _, subs in CASES for *_, grants in subs for g in grants]
    rng = np.random.default_rng(12)
    for _ in range(60):
        L = int(rng.choice([3, 4, 5, 6, 8, 10, 15, 25, 48, 100]))
        qm = int(rng.choice([2, 4, 6, 8]))
        grants.append(G(L, 0, qm, tbs=tbs(L, qm, int(rng.integers(0, 27))), nof_ack=int(rng.integers(0, 3)), ri_len=int(rng.integers(0, 3)),
                        cqi_len=int(rng.choice([0, 4, 11, 12, 40, 66])), I_ack=int(rng.integers(0, 15)), I_ri=int(rng.integers(0, 13)),
                        I_cqi=int(rng.integers(2, 16))))
    for g in grants:
        L = ltelib.uci_layout(to_oracle(g))
        assert (L.Qp_ack, L.Qp_ri, L.Qp_cqi, L.G) == (g.qa, g.qr, g.qc, g.G), (g.L, g.qm, g.tbs, g.uci)
        kind = np.zeros(12 * g.M, np.uint8)
        dpos = np.zeros(12 * g.M, np.uint32)
        S.lte_uci_map(g.M, C.byref(L), ltelib.ptr(kind), ltelib.ptr(dpos))
        assert np.array_equal(kind.reshape(g.M, 12), g.kind)
        sel = np.isin(g.kind, (ref64_ul.DATA, ref64_ul.ACK_DATA, ref64_ul.CQI))
        assert np.array_equal(dpos.reshape(g.M, 12)[sel], g.pos[sel])


def test_reference_dmrs_equals_the_shared_primitive(infra):
    S = ltelib.sim()
    S.lte_pusch_dmrs.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    for _, cellp, u, subs in CASES:
        cell = Cell(*cellp)
        for sf, _, _, grants in subs:
            for g in grants:
                for sl in range(2):
                    r = np.zeros(g.M, np.complex64)
                    assert S.lte_pusch_dmrs(C.byref(cell), C.byref(ul_cfg(u)), 2 * sf + sl, g.n_dmrs2, g.M, ltelib.ptr(r)) == 0
                    assert np.abs(r - ref64_ul.dmrs(cell.cell_id, u, 2 * sf + sl, g.n_dmrs2, g.M)).max() < 2e-4, (cellp, sf, g.L)


# ------------------------------------------------------------------------------------------------ the oracle against the reference
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_pusch_equals_the_float64_reference(infra, case):
    cell, subs = synth(case)
    o = Oracle(cell)
    nsat = 0
    for s in subs:
        sym, res = oracle_decode(o, s)
        Y, ref = s.reference()
        check_grid(sym, Y, cell, (case[0], s.sf))
        for g, (r, _, _, ch, llr), (info, rl, cond) in zip(s.grants, res, ref):
            what = "%s sf %d L %d at %d qm %d" % (case[0], s.sf, g.L, g.n_prb, g.qm)
            assert r == 0, (what, r)
            check_chest(ch, info, what)
            check_soft_bits(llr[:g.G], rl, cond, what)
            nsat += int(np.sum(np.abs(rl) == 32767))
            if s.delay:                                                    # the designed delay dominates the estimate's phase slope
                assert abs(info["ta_us"] - s.delay / (ref64.fft_size(cell) * 15e-3)) < 0.05, (what, info["ta_us"])
    if case[0].endswith("fade"):
        assert nsat > 0, "the deep fade drives the int16 clamp"


# ------------------------------------------------------------------------------------------------ physics anchors
@pytest.mark.parametrize("chan", ["flat", "linear_l"])
def test_noiseless_estimate_is_the_channel_and_soft_bits_are_the_transmitted_points(infra, chan):
    """without noise the smoothed estimate is exact for a channel flat in frequency, and the time interpolation is exact for one linear in time on
    every data symbol, extrapolated ones (0-2, 11-13) included: RSRP = mean |h|^2 of the two reference symbols, noise ~ 0, and the soft bits are the
    int16 demodulation of the transmitted modulation symbols"""
    cell = Cell(50, 1, 301, 1)
    u = (3, 0, 1, 0)
    grants = [G(25, 0, 4, n_dmrs2=3), G(20, 25, 8, nof_ack=2, I_ack=8, rnti=0x4321), G(5, 45, 2, ri_len=1, I_ri=4, rnti=0x1111)]
    s = Subframe(cell, 7, u, grants, chan=chan, noise_var=0.0, seed=5)
    o = Oracle(cell)
    _, res = oracle_decode(o, s)
    rsrp = np.mean(np.abs(s.H[[3, 10], 0]) ** 2)
    for g, (r, _, _, ch, llr), d in zip(grants, res, s.d):
        assert r == 0
        assert abs(ch.rsrp - rsrp) <= 1e-5 * rsrp, (ch.rsrp, rsrp)
        assert ch.noise <= 1e-9 * rsrp, ch.noise
        want, _ = ref64_ul.soft_bits(cell, d, g, s.sf)
        assert np.abs(llr[:g.G].astype(np.int64) - want).max() <= 1, (chan, g.L, g.qm)


def test_noise_and_snr_estimates_on_a_flat_channel(infra):
    """flat channel, AWGN of variance s2 per RE, 100-PRB grants over 6 subframes: 6 x 2 x 1200 = 14 400 LS residuals, whose mean has a relative
    standard deviation near 1 %: the +-5 % bar on the noise and the +-0.3 dB bar on the SNR are more than 4 sigma wide"""
    cell = Cell(100, 1, 7, 1)
    o = Oracle(cell)
    s2 = 10 ** (-15 / 10)
    H = np.ones((14, 1200), complex) * np.exp(0.4j)
    nsum = rsum = 0.0
    for sf in range(6):
        s = Subframe(cell, sf, (1, 4, 0, 0), [G(100, 0, 4, rnti=0x100 + sf)], H=H, noise_var=s2, seed=70 + sf)
        _, res = oracle_decode(o, s)
        nsum += res[0][3].noise
        rsum += res[0][3].rsrp
    assert abs(nsum / 6 / s2 - 1) < 0.05, nsum / 6 / s2
    assert abs(10 * np.log10(rsum / nsum) - 15.0) < 0.3, 10 * np.log10(rsum / nsum)


@pytest.mark.parametrize("cellp,delay", [((25, 1, 5, 1, 0), 9), ((25, 1, 5, 1, 0), -9), ((50, 1, 9, 1, 768), 4), ((100, 1, 1, 1, 0), -30),
                                         ((100, 1, 1, 1, 1536), 21)], ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_timing_offset_of_a_pure_delay(infra, cellp, delay):
    """a delay of d whole samples (|d| < CP) is a phase slope of 2 pi d / N per subcarrier: ta_us = d / (N 15 kHz), with its sign -- a late UE is positive"""
    cell = Cell(*cellp)
    o = Oracle(cell)
    N = ref64.fft_size(cell)
    want = delay / (N * 15e-3)
    s = Subframe(cell, 4, (2, 1, 0, 0), [G(cell.nof_prb // 5, 0, 2), G(cell.nof_prb // 2, cell.nof_prb // 2, 4, rnti=0x999)], chan="flat",
                 delay=delay, noise_var=1e-3, seed=delay & 0xFF)
    _, res = oracle_decode(o, s)
    _, ref = s.reference()
    for (_, _, _, ch, _), (info, _, _) in zip(res, ref):
        assert abs(ch.ta_us - want) < 0.01, (ch.ta_us, want)
        assert abs(ch.ta_us - info["ta_us"]) <= 1e-3


# ------------------------------------------------------------------------------------------------ zero-filled samples
ZERO_CELL = Cell(50, 1, 23, 1)
ZERO_UCFG = (3, 2, 0, 0)
ZERO_KINDS = ["all_zero", "from_symbol_11", "slot1_under_hopping"]
PINNED = (2, 3)                                                             # decode from_symbol_11; with the fold thresholds as soft bits they do not


def zero_grants(kind):
    """grants of Qm 2 / 4 / 6 / 8 at code rates 0.40 - 0.48; PINNED are the 64QAM and 256QAM ones.  Under slot1_under_hopping every grant hops"""
    hop = kind == "slot1_under_hopping"
    gs = [G(10, 0, 4, tbs=tbs(10, 4, 12), rnti=0x3101),
          G(8, 10, 2, tbs=tbs(8, 2, 8), rnti=0x3102, nof_ack=1, I_ack=4),
          G(12, 18, 6, tbs=tbs(12, 6, 17), rnti=0x3103, ri_len=1, I_ri=3),
          G(20, 30, 8, tbs=tbs(20, 8, 22), rnti=0x3104)]
    if hop:
        for g, s1 in zip(gs, (40, 32, 0, 12)):
            gs[gs.index(g)] = Grant(g.L, g.n_prb, g.qm, g.tbs, rnti=g.rnti, n_prb1=s1, **{k: v for k, v in g.uci.items()})
    return gs


def encode(g, rng):
    """a transport block of g.tbs random bits through the UL-SCH coding of the simulator (CRC, segmentation, turbo, rate matching to G): the CRC case
    needs real code bits, everything else of the subframe is ref64_ul's"""
    S = ltelib.sim()
    pl = rng.integers(0, 256, g.tbs // 8).astype(np.uint8)
    e = np.zeros(g.G, np.uint8)
    assert S.lte_sim_dlsch_encode(ltelib.ptr(pl), g.tbs, 0, g.G, g.qm, 1, ltelib.ptr(e)) == 0
    return pl, e


def zero_fill(iq, kind, cell):
    out = iq.copy()
    N = ref64.fft_size(cell)
    start = [sum(ref64.cp_len(N, j) + N for j in range(l)) for l in range(15)]
    if kind == "all_zero":
        out[:] = 0
    elif kind == "from_symbol_11":                                            # data symbols 11-13; both reference symbols intact
        out[start[11]:] = 0
    elif kind == "slot1_under_hopping":                                       # all of slot 1: its estimate is 0 and |h|^2 = 0
        out[start[7]:] = 0
    return out


def zero_subframe(kind):
    """-> (Subframe with encoded UL-SCH bits at 30 dB, zero-filled iq, payloads)"""
    rng = np.random.default_rng(17)
    grants = zero_grants(kind)
    enc = [encode(g, rng) for g in grants]
    s = Subframe(ZERO_CELL, 6, ZERO_UCFG, grants, chan="selective", noise_var=1e-3, seed=23, bits=[e for _, e in enc])
    return s, zero_fill(s.iq, kind, ZERO_CELL), [p for p, _ in enc]


def zeroed_columns(kind):
    """the interleaver columns (data symbols) whose samples are all zero"""
    return {"all_zero": range(12), "from_symbol_11": range(9, 12), "slot1_under_hopping": range(6, 12)}[kind]


def zeroed_soft_bits(g, kind):
    """mask over the G soft bits of the grant that come from a zero-filled data symbol"""
    cols = np.zeros(12, bool)
    cols[list(zeroed_columns(kind))] = True
    m = np.zeros(g.G // g.qm, bool)
    for kd in (ref64_ul.DATA, ref64_ul.ACK_DATA):
        k, c = np.nonzero(g.kind == kd)
        m[g.pos[k, c]] = cols[c]
    return np.repeat(m, g.qm)


def check_zero_chest(ch, kind, what):
    assert not np.isnan(ch.noise) and not np.isnan(ch.rsrp) and not np.isnan(ch.ta_us), what
    if kind == "all_zero":
        assert ch.noise == 0 and ch.rsrp == 0 and np.isnan(ch.snr_db) and ch.ta_us == 0, (what, ch.noise, ch.rsrp, ch.snr_db, ch.ta_us)
    else:
        assert not np.isnan(ch.snr_db), what


@pytest.mark.parametrize("kind", ZERO_KINDS)
def test_oracle_on_zero_filled_subframes(infra, kind):
    """exactly-zero samples: no NaN anywhere, every soft bit of a zero-filled symbol 0 (an erasure, not the -252 / -432 / -613 fold thresholds of a zero
    sample, nor the spread 0/0 of a zero channel), the rest within the reference's bars; the pinned 16QAM grant at code rate <= 0.6 decodes with
    symbols 11-13 lost"""
    s, iq, pls = zero_subframe(kind)
    o = Oracle(ZERO_CELL)
    sym, res = oracle_decode(o, s, iq)
    assert not np.isnan(sym).any()
    Y, ref = s.reference(iq)
    for i, (g, (r, pl, crc, ch, llr), (info, rl, cond)) in enumerate(zip(s.grants, res, ref)):
        what = "%s grant %d qm %d" % (kind, i, g.qm)
        assert r == 0
        check_zero_chest(ch, kind, what)
        z = zeroed_soft_bits(g, kind)
        assert z.any() and np.all(llr[:g.G][z] == 0), (what, int(np.sum(llr[:g.G][z] != 0)))
        assert np.all(rl[z] == 0)
        check_soft_bits(llr[:g.G], rl, cond, what)
        if kind != "all_zero":
            assert abs(ch.noise - info["noise"]) <= 1e-5 * info["noise"] and abs(ch.rsrp - info["rsrp"]) <= 1e-5 * info["rsrp"], what
    if kind == "from_symbol_11":
        for i in PINNED:
            g = s.grants[i]
            assert g.qm >= 6 and g.tbs / g.G <= 0.6
            assert res[i][2] == 1 and np.array_equal(res[i][1][:g.tbs // 8], pls[i]), "grant %d decodes without symbols 11-13" % i
