"""The channeliser's whole plan space on the CPU (DESIGN.md §2 "channeliser", "channeliser, rational carriers"): ltephy_chan_design accepts a
carrier exactly when the float64 rule of chan_rational_lib.geometry does, for every integer plan, for every capture rate on the 1 kHz grid at
offset 0, for seeded random rates in whole Hz, at the band-edge offsets and at the boundary plans of the limits.  Every accepted plan it checks in
full has finite tables equal to lteo_chan_design_poly's bit for bit, Tp = kaiserord(70, w) | 1, and a prototype hp / L with at least 65 dB of
stop band from min(fs_in, fs_out) - f_pass up and at most 0.02 dB of ripple on [0, f_pass], measured by a float64 FFT at rate L fs_in."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.signal as ss

import chan_lib as CH
import chan_rational_lib as R

MAX_FS = 245760000
GEO = ("L", "M", "Tp", "Kp", "Ka", "Kb", "P")


class _Design:
    """ltephy_chan_design on one reused plan: geometry only, or None when refused"""

    def __init__(self, phylib):
        from ltesniffer_b200 import capi
        capi._bind_chan(phylib)
        self.L, self.q = phylib, capi.ChanPoly()
        self.cfg = capi.chan_cfg(1, [(0, 128)], flags=R.RATIONAL)

    def __call__(self, fs, off, N, flags=R.RATIONAL):
        self.cfg.fs_in, self.cfg.flags = fs, flags
        self.cfg.carrier[0].offset_hz, self.cfg.carrier[0].symbol_sz = off, N
        r = self.L.ltephy_chan_design(C.byref(self.cfg), 0, C.byref(self.q), None, None, None)
        assert r in (0, -2), r
        return {k: getattr(self.q, k) for k in GEO} if r == 0 else None


def _amax(fs, N):
    """the largest offset on the 1 kHz grid whose band fits in the capture: 2 (|offset| + f_pass) <= fs_in"""
    return (fs - 2 * 90000 * CH.MAX_PRB[N]) // 2000 * 1000


def _offsets(fs, N):
    """0, +-1 kHz, +-the band edge, all accepted by the band check, and one kHz beyond the edge, refused"""
    a = _amax(fs, N)
    return sorted({o for o in (0, 1000, -1000, a, -a) if abs(o) <= a}), [a + 1000, -a - 1000]


def _same_rule(design, fs, off, N, flags=R.RATIONAL):
    """the library and the rule agree on acceptance and geometry; -> the rule's geometry or None"""
    geo = R.geometry(fs, off, N) if flags else CH.geometry(fs, off, N)
    got = design(fs, off, N, flags)
    assert (got is None) == (geo is None), (fs, off, N, flags, got, geo)
    if geo is None:
        return None
    if not flags:     # (T, D, P, f_pass): the integer rule
        T_, D, P, _ = geo
        geo = R.geometry(fs, off, N)
        assert (geo["L"], geo["M"], geo["Tp"], geo["P"]) == (1, D, T_, P)
    for k in GEO:
        assert got[k] == geo[k], (fs, off, N, k, got[k], geo[k])
    if geo["L"] > 2 * geo["M"]:
        raise AssertionError("a plan above 2x upsampling passed the band check", fs, N)
    return geo


def _full_check(fs, off, N, flags=R.RATIONAL):
    """tables of the library == the oracle's bit for bit, all finite; Tp from kaiserord; stop band and ripple of hp / L by a float64 FFT"""
    from ltesniffer_b200 import capi
    d = capi.chan_design(fs, [(off, N)], 0, rational=bool(flags))
    o = R.design(fs, off, N, flags)
    geo = R.geometry(fs, off, N)
    for k in GEO:
        assert d[k] == o[k] == geo[k], (fs, off, N, k)
    for k in ("hp", "g", "rot"):
        assert np.isfinite(d[k].view(np.float32)).all(), (fs, off, N, k)
        assert d[k].tobytes() == o[k].tobytes(), (fs, off, N, k)
    assert d["Tp"] == ss.kaiserord(CH.ATTEN, geo["w"])[0] | 1
    assert d["L"] * d["Kp"] <= R.MAX_TABLE and d["Kp"] == d["Ka"] + d["Kb"] + 1
    L, f_pass, fo = d["L"], geo["f_pass"], 15000 * N
    h = d["hp"].astype(np.float64) / L
    nfft = 1 << max(15, int(16 * len(h) - 1).bit_length())
    mag = 20 * np.log10(np.maximum(np.abs(np.fft.rfft(h, nfft)), 1e-300))
    f = np.arange(len(mag)) * (L * fs / nfft)
    stop = f >= min(fs, fo) - f_pass
    assert not stop.any() or mag[stop].max() <= -65.0, (fs, off, N, mag[stop].max())
    assert np.abs(mag[f <= f_pass]).max() <= 0.02, (fs, off, N, np.abs(mag[f <= f_pass]).max())
    return d


@pytest.mark.parametrize("N", CH.SYMBOL_SIZES)
def test_every_integer_plan(phylib, N):
    """D = 1..128 and the first D past 245.76 MHz, with and without the flag: the library's verdict and geometry are the rule's; every accepted
    integer plan (D >= 2) passes the full check at offset 0 and at the band edge, and one kHz past the edge is refused"""
    design = _Design(phylib)
    plans = 0
    for D in range(1, 130):
        fs = 15000 * N * D
        for flags in (0, R.RATIONAL):
            _same_rule(design, fs, 0, N, flags)
        if D == 1 or D > 128 or fs > MAX_FS:
            continue
        plans += 1
        ok, bad = _offsets(fs, N)
        for off in ok:
            for flags in (0, R.RATIONAL):
                assert _same_rule(design, fs, off, N, flags) is not None, (fs, off)
        for off in bad:
            for flags in (0, R.RATIONAL):
                assert _same_rule(design, fs, off, N, flags) is None, (fs, off)
        for off in (0, ok[-1]):
            d = _full_check(fs, off, N, flags=0)
            assert (d["L"], d["M"]) == (1, D)
    assert plans == len([D for D in range(2, 129) if 15000 * N * D <= MAX_FS])


_SPACE = None


def _space():
    global _SPACE
    if _SPACE is None:
        _SPACE = R.plan_space()
    return _SPACE


def test_integer_plan_count():
    """313 integer (N, D) plans, and the rational plan space at offset 0 on the 1 kHz grid"""
    assert sum(1 for N in CH.SYMBOL_SIZES for D in range(2, 129) if 15000 * N * D <= MAX_FS) == 313
    space = _space()
    assert len(space) > 139000 and len({(d["L"], d["M"], d["Kp"], d["R"]) for d in space}) > 84000


@pytest.mark.parametrize("N", CH.SYMBOL_SIZES)
def test_rational_grid(phylib, N):
    """every capture rate on the 1 kHz grid up to 245.76 MHz at offset 0, plus 2 f_pass and its neighbours in Hz: the library accepts exactly
    the plans of the rule, with the rule's geometry.  Every 40th accepted plan also gets the band-edge offsets and the full check"""
    design = _Design(phylib)
    f2 = 2 * 90000 * CH.MAX_PRB[N]
    space = {d["fs"]: d for d in _space() if d["N"] == N}
    for fs in range(1000, MAX_FS + 1, 1000):
        got = design(fs, 0, N)
        d = space.get(fs)
        assert (got is None) == (d is None), (fs, N, got)
        if d is not None:
            assert all(got[k] == d[k] for k in GEO), (fs, N, got, d)
    for fs in (f2 - 1, f2, f2 + 1):
        _same_rule(design, fs, 0, N)
    assert design(f2, 0, N) is None        # no transition band
    accepted = sorted(space)
    for fs in accepted[::40] + accepted[-1:]:
        ok, bad = _offsets(fs, N)
        for off in ok:
            assert _same_rule(design, fs, off, N) is not None, (fs, off)
        for off in bad:
            assert _same_rule(design, fs, off, N) is None, (fs, off)
    for fs in accepted[::len(accepted) // 12] + accepted[-1:]:
        for off in (0, _offsets(fs, N)[0][-1]):
            _full_check(fs, off, N)


@pytest.mark.parametrize("N", CH.SYMBOL_SIZES)
def test_rational_random_rates(phylib, N):
    """seeded random capture rates in whole Hz, and on the 1 kHz grid, at the offsets of _offsets(): the library's verdict and geometry are the
    rule's, and every accepted plan passes the full check"""
    design = _Design(phylib)
    rng = np.random.default_rng(N)
    rates = [int(f) for f in rng.integers(1, MAX_FS + 1, 300)] + [int(f) * 1000 for f in rng.integers(1, MAX_FS // 1000 + 1, 300)]
    f2 = 2 * 90000 * CH.MAX_PRB[N]
    rates += [int(f) for f in rng.integers(f2 - 2000, f2 + 2000, 50)]
    full = 0
    for fs in rates:
        if _same_rule(design, fs, 0, N) is None:
            continue
        ok, bad = _offsets(fs, N)
        for off in ok:
            assert _same_rule(design, fs, off, N) is not None, (fs, off)
        for off in bad:
            assert _same_rule(design, fs, off, N) is None, (fs, off)
        if full < 12:
            _full_check(fs, ok[-1], N)
            full += 1


# (fs_in, N, what it reaches): checked against the geometry of ltephy_chan_design
BOUNDARY = [
    (49395000, 128, dict(L=128, M=3293), "L Kp = 2^15 exactly"),
    (10425000, 1024, dict(L=1024), "L = 1024 and L Kp = 2^15"),
    (245680000, 128, dict(L=24, M=3071, Kp=1266), "the largest M / L"),
    (6134000, 128, dict(L=960, M=3067, R=3), "the smallest R"),
    (15360000, 1024, dict(L=1, M=1), "L = M = 1"),
]


@pytest.mark.parametrize("fs,N,want,why", BOUNDARY, ids=[b[3] for b in BOUNDARY])
def test_boundary_plans(phylib, fs, N, want, why):
    design = _Design(phylib)
    geo = _same_rule(design, fs, 0, N)
    assert geo is not None
    geo["R"] = R.tile_rows(geo["L"], geo["M"], geo["Kp"])
    for k, v in want.items():
        assert geo[k] == v, (k, geo[k], v)
    space = _space()
    if why == "L Kp = 2^15 exactly" or why == "L = 1024 and L Kp = 2^15":
        assert geo["L"] * geo["Kp"] == R.MAX_TABLE == max(d["L"] * d["Kp"] for d in space)
    if why == "L = 1024 and L Kp = 2^15":
        assert geo["L"] == R.MAX_L
    if why == "the largest M / L":
        assert max((d for d in space if d["L"] > 1), key=lambda d: d["M"] / d["L"])["fs"] == fs
    if why == "the smallest R":
        assert min(d["R"] for d in space) == 3
    ok, bad = _offsets(fs, N)
    for off in ok:
        assert _same_rule(design, fs, off, N) is not None
        _full_check(fs, off, N)
    for off in bad:
        assert _same_rule(design, fs, off, N) is None


def test_upsampling_limit_only_names_the_refusal():
    """for every N, fs_out / 2 < 2 f_pass: a plan above 2x upsampling (fs_in < fs_out / 2) also fails the band check, so the 2x limit only
    decides which message a refusal gives"""
    for N in CH.SYMBOL_SIZES:
        assert 15000 * N / 2 < 2 * 90000 * CH.MAX_PRB[N]
