"""Rational carriers and integer samples of the channeliser on the CPU (DESIGN.md §2 "channeliser"): the polyphase prototype against scipy, the
oracle's tables equal to ltephy_chan_design bit for bit, the oracle lteo_chan_run_poly against a float64 restatement of the rule and against
scipy.signal.resample_poly, chunking invariance, sc16 / sc8 input, the plans the library refuses without a device, and the oracle receiver on a
two-carrier 25 Msps capture."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.signal as ss

import chan_lib as CH
import chan_rational_lib as R
import sync_lib as S
from test_chan import CHUNKINGS, _signal

# (fs_in, N, L * Kp): the plans of DESIGN.md §2's table, then 56 Msps, 10 Msps, 3 / 8 and 1 / 1
DESIGNS = [(20000000, 1024, 1344), (20000000, 2048, 8448), (25000000, 1024, 6912), (25000000, 2048, 12288), (100000000, 2048, 6528),
           (200000000, 128, 6180), (56000000, 2048, None), (10000000, 512, None), (61440000, 1536, None), (15360000, 1024, None)]


@pytest.mark.parametrize("fs,N,table", DESIGNS)
def test_filter_design(phylib, fs, N, table):
    """Tp is kaiserord's length made odd, hp / L is scipy's firwin at rate L fs_in, >= 65 dB stop band and <= 0.02 dB pass-band ripple"""
    from ltesniffer_b200 import capi
    geo = R.geometry(fs, 0, N)
    d = capi.chan_design(fs, [(0, N)], 0)
    for k in ("L", "M", "Tp", "Kp", "Ka", "Kb", "P"):
        assert d[k] == geo[k], (k, d[k], geo[k])
    if table is not None:
        assert d["L"] * d["Kp"] == table
    L, Tp = d["L"], d["Tp"]
    fo = 15000 * N
    assert (L, d["M"]) == (fo // math.gcd(fo, fs), fs // math.gcd(fo, fs))
    if min(fs, fo) < L * fs:
        ref = ss.firwin(Tp, min(fs, fo) / 2, window=("kaiser", CH.BETA), fs=L * fs)
    else:   # 1 / 1: the cutoff is the Nyquist rate, which firwin refuses; its own expression, a windowed sinc of unit step, normalised
        ref = np.sinc(np.arange(Tp) - (Tp - 1) / 2) * ss.get_window(("kaiser", CH.BETA), Tp, fftbins=False)
        ref /= ref.sum()
    h = d["hp"].astype(np.float64) / L
    assert np.abs(h - ref).max() <= 2 ** -23 * np.abs(ref).max() * 4
    f_pass = geo["f_pass"]
    w, H = ss.freqz(h, worN=np.linspace(0, L * fs / 2, 16384), fs=L * fs)
    mag = 20 * np.log10(np.maximum(np.abs(H), 1e-300))
    stop = w >= min(fs, fo) - f_pass
    assert not stop.any() or mag[stop].max() <= -65.0, mag[stop].max()
    assert np.abs(mag[w <= f_pass]).max() <= 0.02


TABLES = [(20000000, -3000000, 1024), (25000000, 5000000, 512), (200000000, -60000000, 128), (15360000, 0, 1024), (100000000, 30000000, 2048),
          (20000000, 1000, 2048), (30720000, -7500000, 1024), (245760000, 99999000, 128)]


@pytest.mark.parametrize("fs,off,N", TABLES)
def test_tables_equal_the_oracle(phylib, fs, off, N):
    """ltephy_chan_design equals lteo_chan_design_poly bit for bit; for an integer carrier (L = 1) both equal ltephy_chan_taps, and the taps of
    a rational carrier are the rule's within float rounding of float64 numpy"""
    from ltesniffer_b200 import capi
    d = capi.chan_design(fs, [(off, N)], 0)
    o = R.design(fs, off, N)
    for k in ("L", "M", "Tp", "Kp", "Ka", "Kb", "P"):
        assert d[k] == o[k], k
    for k in ("hp", "g", "rot"):
        assert d[k].tobytes() == o[k].tobytes(), k
    fo = 15000 * N
    if fs % fo == 0 and 2 <= fs // fo <= 128:
        t = capi.chan_taps(fs, [(off, N)], 0)
        assert (d["L"], d["M"], d["Tp"], d["Ka"], d["Kb"], d["P"]) == (1, t["D"], t["T"], t["T"] // 2, t["T"] // 2, t["P"])
        assert d["hp"].tobytes() == t["h"].tobytes() and d["g"][0].tobytes() == t["g"].tobytes() and d["rot"].tobytes() == t["rot"].tobytes()
        return
    L, Tp, Ka, Kb = d["L"], d["Tp"], d["Ka"], d["Kb"]
    Hp = (Tp - 1) // 2
    ph, k = np.arange(L)[:, None], np.arange(-Kb, Ka + 1)[None, :]
    idx = Hp + ph + L * k
    tap = np.where((idx >= 0) & (idx < Tp), d["hp"].astype(np.float64)[np.clip(idx, 0, Tp - 1)], 0.0)
    g64 = tap * np.exp(2j * np.pi * ((off * (ph + L * k)) % (L * fs)) / (L * fs))
    assert np.abs(d["g"] - g64).max() <= 2 ** -23 * np.abs(d["hp"]).max() * 2
    i = np.arange(d["P"])
    assert d["P"] == fo // math.gcd(off % fo, fo)
    assert np.abs(d["rot"] - np.exp(-2j * np.pi * ((off * i) % fo) / fo)).max() <= 2 ** -23 * 2


ACCURACY = [(25000000, [(-6000000, 1024), (5000000, 512)], 1), (20000000, [(0, 2048)], 2), (20000000, [(1000000, 1536), (-5000000, 1024)], 1),
            (56000000, [(-18000000, 2048), (13000000, 1024)], 2), (200000000, [(-60000000, 128), (40000000, 2048)], 1), (15360000, [(1000, 1024)], 1),
            (61440000, [(-19000000, 1536)], 1)]


@pytest.mark.parametrize("fs,carriers,nrx", ACCURACY)
def test_oracle_against_float64_and_resample_poly(fs, carriers, nrx):
    """every output of lteo_chan_run_poly within 2e-5 of the RMS of the float64 rule, and of scipy.signal.resample_poly(x e^{-j w i}, L, M,
    window=hp / L), whose alignment an impulse checks first (the output rotation r undoes the mixing of the taps g_phi, so the rule's output is
    the mixed-down capture resampled)"""
    n = 40000 if fs < 100000000 else 120000
    x = _signal(n, nrx, fs, 3)
    outs, _ = R.run(fs, carriers, x, 0)
    for (off, N), o in zip(carriers, outs):
        d = R.design(fs, off, N)
        L, M = d["L"], d["M"]
        assert o["first"] == 0 and o["count"] > 100
        win = d["hp"].astype(np.float64) / L
        imp = np.zeros((1, 4 * d["Tp"] // L + 4 * M + 64), np.complex64)
        imp[0, 2 * (d["Kb"] + M)] = 1.0
        io, _ = R.run(fs, [(0, N)], imp, 0)
        ri = ss.resample_poly(imp[0].astype(np.complex128), L, M, window=win)
        assert np.abs(io[0]["iq"][0] - ri[:io[0]["count"]]).max() <= 1e-6       # no lag between the two
        ms = np.arange(o["count"])
        for a in range(nrx):
            y = o["iq"][a].astype(np.complex128)
            ref = R.reference(fs, off, N, x[a], ms)
            rms = np.sqrt(np.mean(np.abs(ref) ** 2))
            assert np.abs(y - ref).max() <= 2e-5 * rms, (off, N, np.abs(y - ref).max() / rms)
            i = np.arange(n)
            mixed = x[a].astype(np.complex128) * np.exp(-2j * np.pi * ((off * i) % fs) / fs)
            rp = ss.resample_poly(mixed, L, M, window=win)[:o["count"]]
            assert np.abs(y - rp).max() <= 2e-5 * rms, (off, N, np.abs(y - rp).max() / rms)


MIXED = (30720000, [(-7500000, 1024), (3000000, 1536), (9000000, 256)])   # D = 2, 3 / 4, D = 8


@pytest.mark.parametrize("sizes", CHUNKINGS)
def test_chunking_invariance(sizes):
    """a plan mixing integer and rational carriers: the outputs, with repeats dropped, and the final next_sample do not depend on the split"""
    fs, carriers = MIXED
    x = _signal(9000, 2, fs, 5)
    one, nxt = R.run(fs, carriers, x, 0)
    got, nexts = CH.stream(lambda xx, f: R.run(fs, carriers, xx, f), x, sizes)
    assert nexts[-1] == nxt
    assert all(b >= a for a, b in zip(nexts, nexts[1:]))
    for a, b in zip(one, got):
        assert b["first"] == 0 and a["iq"].tobytes() == b["iq"].tobytes()


def test_call_range_and_next_sample():
    """a rational carrier's outputs are those whose window [n - Ka, n + Kb] lies in the call, next_sample the least max(0, n(m') - Ka); the
    integer carriers of the plan are lteo_chan_run's to the bit"""
    fs, carriers = MIXED
    x = _signal(5000, 1, fs, 9)
    outs, nxt = R.run(fs, carriers, x, 0)
    ref, nref = CH.run(fs, [carriers[0], carriers[2]], x, 0)
    assert outs[0]["iq"].tobytes() == ref[0]["iq"].tobytes() and outs[2]["iq"].tobytes() == ref[1]["iq"].tobytes()
    needs = []
    for (off, N), o in zip(carriers, outs):
        d = R.design(fs, off, N)
        L, M, Ka, Kb = d["L"], d["M"], d["Ka"], d["Kb"]
        last = o["first"] + o["count"] - 1
        assert last * M // L + Kb <= 4999 < (last + 1) * M // L + Kb
        needs.append(max(0, (last + 1) * M // L - Ka))
    assert nxt == min(needs)
    later, _ = R.run(fs, carriers, x[:, nxt:], nxt)
    for (off, N), o, o1 in zip(carriers, later, outs):
        d = R.design(fs, off, N)
        L, M, Ka = d["L"], d["M"], d["Ka"]
        assert o["first"] == -(-(nxt + Ka) * L // M)
        k = o1["first"] + o1["count"] - o["first"]
        assert o["iq"][:, :max(0, k)].tobytes() == o1["iq"][:, o["first"]:].tobytes()


@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
@pytest.mark.parametrize("fs,carriers", [MIXED, (25000000, [(-6000000, 1024), (5000000, 512)])])
def test_integer_samples_equal_cf32(fs, carriers, fmt):
    """sc16 and sc8 inputs give the bits of a cf32 run on the converted samples, for integer and rational carriers alike"""
    x = _signal(7000, 2, fs, 4) / 4.0
    q, xf = R.to_format(x, fmt)
    a, na = R.run(fs, carriers, q, 0, fmt)
    b, nb = R.run(fs, carriers, xf, 0)
    assert na == nb
    for u, v in zip(a, b):
        assert u["first"] == v["first"] and u["iq"].tobytes() == v["iq"].tobytes()


def _table_only_plan():
    """a plan (fs_in, N 128) the rational rule refuses only for its phase table: L <= 1024, M <= 128 L, but L Kp > 2^15"""
    fo = 15000 * 128
    for L in (8, 16, 32, 64):
        for M in range(3000, 128 * L + 1):
            fs = fo * M // L
            if math.gcd(L, M) != 1 or fo * M % L or fs > 245760000:
                continue
            w = (fo - 2 * 540000) / (L * fs / 2)
            Hp = (ss.kaiserord(CH.ATTEN, w)[0] | 1) // 2
            if L * (Hp // L + -(-Hp // L) + 1) > R.MAX_TABLE:
                return fs
    raise AssertionError("no such plan")


REFUSED = [
    (30720001, [(0, 1024)], 1, 0, "L above 1024", b"above 1024"),
    (5000000, [(0, 1024)], 1, 0, "upsampling beyond 2x", b"upsamples"),
    (None, [(0, 128)], 1, 0, "phase table over 2^15 taps", b"phase table"),
    (25000000, [(10000000, 1024)], 1, 0, "band outside the capture", b"outside the capture"),
    (25000000, [(0, 1024)], 3, 0, "unknown flag bits", b"flags"),
    (25000000, [(0, 1024)], 1, 3, "unknown format", b"iq_format"),
] + [  # fs_in = 2 f_pass < fs_out: the band check holds with equality, and the transition band [f_pass, fs_in - f_pass] is empty
    (fs, [(0, N)], 1, 0, "no transition band at %g Msps, N %d" % (fs / 1e6, N), b"no transition band")
    for fs, N in ((18000000, 1536), (18000000, 2048), (9000000, 768), (9000000, 1024), (4500000, 384), (4500000, 512), (2700000, 256), (1080000, 128))
]


@pytest.mark.parametrize("fs,carriers,flags,fmt,why,msg", REFUSED, ids=[r[4] for r in REFUSED])
def test_refused_without_a_device(phylib, fs, carriers, flags, fmt, why, msg):
    from ltesniffer_b200 import capi
    capi._bind_chan(phylib)
    fs = fs or _table_only_plan()
    cfg = capi.chan_cfg(fs, carriers, 1, max_samples=100000, flags=flags, iq_format=fmt)
    h = C.c_void_p()
    assert phylib.ltephy_chan_create(C.byref(cfg), C.byref(h)) == -2, why
    assert not h.value and msg in phylib.ltephy_last_error(), phylib.ltephy_last_error()
    if fmt == 0:
        q = capi.ChanPoly()
        assert phylib.ltephy_chan_design(C.byref(cfg), 0, C.byref(q), None, None, None) == -2
        assert R.design(fs, carriers[0][0], carriers[0][1], flags) is None
        if flags == 1:
            assert R.geometry(fs, carriers[0][0], carriers[0][1]) is None


def test_rational_plans_need_the_flag(phylib):
    """without LTEPHY_CHAN_RATIONAL a rational carrier is refused as before; with it ltephy_chan_taps refuses it and names ltephy_chan_design"""
    from ltesniffer_b200 import capi
    capi._bind_chan(phylib)
    h = C.c_void_p()
    T_, D, P = C.c_uint32(), C.c_uint32(), C.c_uint32()
    cfg = capi.chan_cfg(25000000, [(0, 1024)], 1, max_samples=1000)
    assert phylib.ltephy_chan_create(C.byref(cfg), C.byref(h)) == -2 and b"integer decimation" in phylib.ltephy_last_error()
    cfg = capi.chan_cfg(25000000, [(0, 1024)], 1, max_samples=1000, flags=capi.CHAN_RATIONAL)
    assert phylib.ltephy_chan_taps(C.byref(cfg), 0, None, None, None, C.byref(T_), C.byref(D), C.byref(P)) == -2
    assert b"ltephy_chan_design" in phylib.ltephy_last_error()
    assert R.design(25000000, 0, 1024, flags=0) is None


SPEC = [dict(offset_hz=-6000000, N=1024, pci=101, cfo=900.0, lead=3000, gain_db=0.0, decode=True),
        dict(offset_hz=5000000, N=512, pci=257, cfo=-1700.0, lead=777, gain_db=-20.0, decode=True)]


def test_oracle_receiver_on_a_rational_capture():
    """25 Msps, N 1024 at -6 MHz and N 512 at +5 MHz (20 dB weaker), 20 ppm clock, composed with a long scipy resampler: lteo_cell_search on each
    channelised stream finds the PCI at the truth timing in carrier samples, and the oracle receiver decodes every truth transport block"""
    import ltelib
    from helpers import oracle_frontend, truth_grants
    fs = 25000000
    x, truths = R.compose(fs, SPEC, 12, nrx=2, ppm=20.0, noise_db=-35.0, seed=2)
    outs, _ = R.run(fs, [(c["offset_hz"], c["N"]) for c in SPEC], x, 0)
    for c, o, tr in zip(SPEC, outs, truths):
        N, SF = c["N"], 15 * c["N"]
        r, cells, _ = S.cell_search(N, o["iq"][:1])
        rn, cells_n, _ = S.cell_search(N, tr["narrow"][:1])
        assert r == 0 and rn == 0 and cells[0].detected and cells[0].pci == c["pci"], (c, cells[0].pci)
        tol = max(1.0, abs(cells_n[0].frame_offset - tr["truth"][0])) + 0.5
        assert abs(cells[0].frame_offset - tr["truth"][0]) <= tol, (cells[0].frame_offset, tr["truth"][0])
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
        assert [q["cfi"] for q in ref] == [s[1].cfi for s in subs]
        ok = 0
        for sf, d, g in truth_grants(cell, [s[1] for s in subs], tti):
            _, opl, ook = orc.pdsch_decode(int(tti[sf]) % 10, ref[sf]["cfi"], d.rnti, g, ref[sf]["sym"], ref[sf]["ce"], 8)
            for t in range(2):
                if g.tb[t].enabled:
                    nb = g.tb[t].tbs // 8
                    assert ook[t] and bytes(opl[t][:nb]) == bytes(subs[sf][2][d.payload_off[t]:d.payload_off[t] + nb]), (c, int(tti[sf]), d.rnti, t)
                    ok += 1
        assert ok >= 20, (c, ok)
