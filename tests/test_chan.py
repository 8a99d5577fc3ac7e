"""Channeliser on the CPU (DESIGN.md §2 "channeliser"): the filter design of ltephy_chan_taps against scipy and float64 numpy, the oracle's tables
equal to the library's bit for bit, the oracle lteo_chan_run against a float64 restatement of the rule and against scipy.signal.upfirdn, chunking
invariance, cell search through the oracles on a three-carrier capture, and the configurations the library refuses without a device."""
import ctypes as C

import numpy as np
import pytest
import scipy.signal as ss

import chan_lib as CH
import sync_lib as S

FS_CASES = [(fs, N) for N in CH.SYMBOL_SIZES for D in (2, 3, 8, 64, 128) for fs in [15000 * N * D] if fs <= 245760000]


def _taps(fs, off, N):
    from ltesniffer_b200 import capi
    return capi.chan_taps(fs, [(off, N)], 0)


@pytest.mark.parametrize("fs,N", FS_CASES)
def test_filter_design(phylib, fs, N):
    """the prototype is scipy's Kaiser-windowed sinc of kaiserord's length (made odd), with >= 65 dB stop band and <= 0.02 dB pass-band ripple"""
    T_, D, P, f_pass = CH.geometry(fs, 0, N)
    t = _taps(fs, 0, N)
    assert (t["T"], t["D"], t["P"]) == (T_, D, 1)
    ref = ss.firwin(T_, 7500.0 * N, window=("kaiser", CH.BETA), fs=fs)
    h = t["h"].astype(np.float64)
    assert np.abs(h - ref).max() <= 2 ** -23 * np.abs(ref).max() * 4
    fo = 15000 * N
    w, H = ss.freqz(h, worN=np.linspace(0, fs / 2, 8192), fs=fs)
    mag = 20 * np.log10(np.maximum(np.abs(H), 1e-300))
    assert mag[w >= fo - f_pass].max() <= -65.0, mag[w >= fo - f_pass].max()
    assert np.abs(mag[w <= f_pass]).max() <= 0.02


@pytest.mark.parametrize("fs,off,N", [(30720000, -7500000, 1024), (30720000, 5000000, 512), (30720000, 11000000, 256), (46080000, 13000, 1536),
                                      (245760000, -101377000, 256), (245760000, 99999000, 128), (61440000, 19800000, 2048)])
def test_complex_taps_and_rotation(phylib, fs, off, N):
    """g[k] = h[k] e^{j w k} and r[i] = e^{-j w i D} within float rounding of float64 numpy; the oracle's tables equal ltephy_chan_taps"""
    t = _taps(fs, off, N)
    T_, D, P = t["T"], t["D"], t["P"]
    H = (T_ - 1) // 2
    k = np.arange(-H, H + 1)
    g64 = t["h"].astype(np.float64) * np.exp(2j * np.pi * ((off * k) % fs) / fs)
    assert np.abs(t["g"] - g64).max() <= 2 ** -23 * np.abs(t["h"]).max() * 2
    i = np.arange(P)
    assert P == fs // np.gcd((D * off) % fs, fs) and P <= fs // 1000
    r64 = np.exp(-2j * np.pi * ((D * off * i) % fs) / fs)
    assert np.abs(t["rot"] - r64).max() <= 2 ** -23 * 2
    o = CH.design(fs, off, N)
    assert (o["T"], o["D"], o["P"]) == (T_, D, P)
    for key in ("h", "g", "rot"):
        assert o[key].tobytes() == t[key].tobytes(), key


def _signal(n, nrx, fs, seed):
    """random complex noise plus a few tones across the band"""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((nrx, n)) + 1j * rng.standard_normal((nrx, n))) * 0.3
    t = np.arange(n)
    for f in rng.uniform(-0.45, 0.45, 4) * fs:
        x += np.exp(2j * np.pi * f * t / fs)[None, :] * rng.uniform(0.2, 1.0)
    return x.astype(np.complex64)


@pytest.mark.parametrize("fs,carriers", [(30720000, [(-7500000, 1024), (5000000, 512), (11000000, 256)]),
                                         (46080000, [(1000, 1536), (-15000000, 768)]),
                                         (245760000, [(-101377000, 256), (99999000, 128)])])
def test_oracle_against_float64_and_upfirdn(fs, carriers):
    """every output of lteo_chan_run within 2e-5 of the output's RMS of the float64 rule; the same against scipy.signal.upfirdn on the signal
    mixed down by the carrier offset"""
    x = _signal(60000, 1, fs, 3)
    outs, _ = CH.run(fs, carriers, x, 0)
    for (off, N), o in zip(carriers, outs):
        assert o["first"] == 0 and o["count"] > 100
        y = o["iq"][0].astype(np.complex128)
        ms = np.arange(o["count"])
        ref = CH.reference(fs, off, N, x[0], ms)
        rms = np.sqrt(np.mean(np.abs(ref) ** 2))
        assert np.abs(y - ref).max() <= 2e-5 * rms, (off, N, np.abs(y - ref).max() / rms)
        t = CH.design(fs, off, N)
        H, D = (t["T"] - 1) // 2, t["D"]
        n = np.arange(x.shape[1])
        mixed = x[0].astype(np.complex128) * np.exp(-2j * np.pi * ((off * n) % fs) / fs)
        full = ss.upfirdn(t["h"].astype(np.float64), mixed)
        assert np.abs(y - full[ms * D + H]).max() <= 2e-5 * rms


CHUNKINGS = [[10 ** 9], [1, 1, 1, 2, 3, 5000], [777, 4111, 13], [1500], [60, 61, 62, 63, 64, 65]]


@pytest.mark.parametrize("sizes", CHUNKINGS)
def test_chunking_invariance(sizes):
    """the outputs, with repeated ones dropped, and the final next_sample do not depend on how the capture is split"""
    fs, carriers = 30720000, [(-7500000, 1024), (5000000, 512), (11000000, 256)]
    x = _signal(9000, 2, fs, 5)
    one, nxt = CH.run(fs, carriers, x, 0)
    got, nexts = CH.stream(lambda xx, f: CH.run(fs, carriers, xx, f), x, sizes)
    assert nexts[-1] == nxt
    assert all(b >= a for a, b in zip(nexts, nexts[1:]))
    for a, b in zip(one, got):
        assert b["first"] == 0 and a["iq"].tobytes() == b["iq"].tobytes()


def test_first_call_from_zero_and_later_starts():
    """with first = 0, output 0 exists (samples before 0 count as zero); a call from first > 0 starts at the first output whose window lies
    inside it, and next_sample is the lowest sample any carrier still needs"""
    fs, carriers = 30720000, [(-7500000, 1024), (11000000, 256)]
    x = _signal(3000, 1, fs, 9)
    outs, nxt = CH.run(fs, carriers, x, 0)
    ref0 = CH.reference(fs, carriers[0][0], carriers[0][1], x[0], [0])
    assert outs[0]["first"] == 0 and abs(outs[0]["iq"][0, 0] - ref0[0]) <= 1e-5 * abs(ref0[0]) + 1e-7
    needs = []
    for (off, N), o in zip(carriers, outs):
        t = CH.design(fs, off, N)
        H, D = (t["T"] - 1) // 2, t["D"]
        last = o["first"] + o["count"] - 1
        assert last * D + H <= 2999 < (last + 1) * D + H
        needs.append((last + 1) * D - H)
    assert nxt == min(needs)
    later, _ = CH.run(fs, carriers, x[:, nxt:], nxt)
    for (off, N), o in zip(carriers, later):
        t = CH.design(fs, off, N)
        H, D = (t["T"] - 1) // 2, t["D"]
        assert o["first"] == -(-(nxt + H) // D)


def test_cell_search_through_the_oracles():
    """30.72 Msps, three carriers (50 PRB at -7.5 MHz, 25 PRB at +5 MHz, 15 PRB at +11 MHz, the middle one 20 dB weaker), each with its own PCI,
    carrier offset and lead, the clock 20 ppm off: lteo_cell_search on each channelised stream finds the PCI at the truth frame timing in carrier
    samples, as closely as on the carrier's own narrowband capture"""
    fs = 30720000
    spec = [dict(offset_hz=-7500000, N=1024, pci=101, cfo=900.0, lead=3000, gain_db=0.0),
            dict(offset_hz=5000000, N=512, pci=257, cfo=-1700.0, lead=777, gain_db=-20.0),
            dict(offset_hz=11000000, N=256, pci=44, cfo=300.0, lead=2500, gain_db=0.0)]
    x, truths = CH.compose(fs, spec, 12, nrx=1, ppm=20.0, noise_db=-35.0, seed=2)
    outs, _ = CH.run(fs, [(c["offset_hz"], c["N"]) for c in spec], x, 0)
    for c, o, tr in zip(spec, outs, truths):
        N = c["N"]
        fo_truth = tr["truth"][0]
        r, cells, _ = S.cell_search(N, o["iq"])
        rn, cells_n, _ = S.cell_search(N, tr["narrow"])
        assert r == 0 and rn == 0
        best, best_n = cells[0], cells_n[0]
        assert best.detected and best.pci == c["pci"], (c, best.pci, best.psr, best.sss_ratio)
        assert best_n.detected and best_n.pci == c["pci"]
        tol = max(1.0, abs(best_n.frame_offset - fo_truth)) + 0.5
        assert abs(best.frame_offset - fo_truth) <= tol, (best.frame_offset, fo_truth, best_n.frame_offset)
        assert abs(best.cfo_hz - c["cfo"]) <= abs(best_n.cfo_hz - c["cfo"]) + 100.0


REFUSED = [
    (25000000, 1, [(0, 1024)], "non-integer D"),
    (15360000, 1, [(0, 1024)], "D < 2"),
    (247680000, 1, [(0, 128)], "D > 128"),
    (30720000, 1, [(12000000, 1024)], "band outside the capture"),
    (30720000, 1, [(-11000000, 1024)], "band outside the capture (below)"),
    (30720000, 1, [(500, 1024)], "offset off the 1 kHz grid"),
    (30720000, 1, [], "no carriers"),
    (30720000, 1, [(0, 256)] * 9, "nine carriers"),
    (30720000, 1, [(0, 1000)], "unknown N"),
    (30720000, 3, [(0, 1024)], "three antennas"),
    (276480000, 1, [(0, 2048)], "fs_in above 245.76 MHz"),
]


@pytest.mark.parametrize("fs,nrx,carriers,why", REFUSED, ids=[r[3] for r in REFUSED])
def test_invalid_configurations_are_refused_without_a_device(phylib, fs, nrx, carriers, why):
    from ltesniffer_b200 import capi
    capi._bind_chan(phylib)
    cfg = capi.chan_cfg(fs, carriers, nrx, max_samples=100000)
    h = C.c_void_p()
    assert phylib.ltephy_chan_create(C.byref(cfg), C.byref(h)) == -2, why
    assert not h.value
    if nrx == 1 and 1 <= len(carriers) <= 8:
        assert CH.design(fs, carriers[0][0], carriers[0][1]) is None
        T_, D, P = C.c_uint32(), C.c_uint32(), C.c_uint32()
        assert phylib.ltephy_chan_taps(C.byref(cfg), 0, None, None, None, C.byref(T_), C.byref(D), C.byref(P)) == -2


def test_max_samples_and_null_config_are_refused(phylib):
    from ltesniffer_b200 import capi
    capi._bind_chan(phylib)
    h = C.c_void_p()
    for ms in (0, 2 ** 31 + 1):
        cfg = capi.chan_cfg(30720000, [(0, 1024)], 1, max_samples=ms)
        assert phylib.ltephy_chan_create(C.byref(cfg), C.byref(h)) == -2
        assert b"max_samples" in phylib.ltephy_last_error()
    assert phylib.ltephy_chan_create(None, C.byref(h)) == -2


def test_oracle_receiver_decodes_every_carrier():
    """the three-carrier capture with PDSCH on every carrier (the middle one 20 dB weaker, 20 ppm clock, each its own carrier offset): after
    lteo_chan_run, the oracle receiver decodes every truth transport block of every carrier from subframes cut at the truth timing in carrier
    samples and corrected by the truth carrier offset, with the simulator's bytes"""
    import ltelib
    from helpers import oracle_frontend, truth_grants
    fs = 30720000
    spec = [dict(offset_hz=-7500000, N=1024, pci=101, cfo=900.0, lead=3000, gain_db=0.0, decode=True),
            dict(offset_hz=5000000, N=512, pci=257, cfo=-1700.0, lead=777, gain_db=-20.0, decode=True),
            dict(offset_hz=11000000, N=256, pci=44, cfo=300.0, lead=2500, gain_db=0.0, decode=True)]
    x, truths = CH.compose(fs, spec, 12, nrx=2, ppm=20.0, noise_db=-35.0, seed=2)   # two antennas: the simulator sends two-layer blocks too
    outs, _ = CH.run(fs, [(c["offset_hz"], c["N"]) for c in spec], x, 0)
    for c, o, tr in zip(spec, outs, truths):
        N, SF = c["N"], 15 * c["N"]
        cell = ltelib.Cell(CH.MAX_PRB[N], 2, c["pci"], 2, N)
        y = o["iq"].astype(np.complex128)
        ks = [k for k in range(len(tr["truth"])) if int(round(tr["truth"][k])) + SF <= y.shape[1]]
        assert len(ks) >= 10
        n = np.arange(SF)
        iq = np.zeros((len(ks), 2, SF), np.complex64)
        for i, k in enumerate(ks):
            s0 = int(round(tr["truth"][k]))
            iq[i] = y[:, s0:s0 + SF] * np.exp(-2j * np.pi * c["cfo"] * (s0 + n) / (15000.0 * N))
        tti = np.array(ks, np.uint32)
        orc = ltelib.Oracle(cell)
        ref = oracle_frontend(orc, iq, tti)
        subs = [tr["sub"][k] for k in ks]
        assert [r["cfi"] for r in ref] == [s[1].cfi for s in subs]
        ok = 0
        for sf, d, g in truth_grants(cell, [s[1] for s in subs], tti):
            _, opl, ook = orc.pdsch_decode(int(tti[sf]) % 10, ref[sf]["cfi"], d.rnti, g, ref[sf]["sym"], ref[sf]["ce"], 8)
            for t in range(2):
                if g.tb[t].enabled:
                    nb = g.tb[t].tbs // 8
                    assert ook[t] and bytes(opl[t][:nb]) == bytes(subs[sf][2][d.payload_off[t]:d.payload_off[t] + nb]), (c, int(tti[sf]), d.rnti, t)
                    ok += 1
        assert ok >= 20, (c, ok)
