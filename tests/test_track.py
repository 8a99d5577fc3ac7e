"""Tracker on the CPU (DESIGN.md §2, "tracking"): the oracle lteo_track_* against the float64 restatement in ref64_track.py, its physics on
captures with a sampling-clock offset, a carrier-offset ramp, a zero-filled gap and noise only, chunking invariance, and the C-ABI's checks of
its configuration."""
import ctypes as C

import numpy as np
import pytest

import ref64_track as F
import track_lib as T


def test_resampler_in_band_error():
    """the windowed-sinc resampler delays in-band tones (up to 0.3 cycles per sample, the widest occupied band here) with error below -60 dB"""
    rng = np.random.default_rng(0)
    M, ppm = 20000, 137.0
    fr = rng.uniform(-0.3, 0.3, 16)
    ph = rng.uniform(0, 2 * np.pi, 16)
    sig = lambda t: np.exp(2j * np.pi * fr[:, None] * t[None, :] + 1j * ph[:, None]).sum(0)
    y = T.resample(sig(np.arange(M, dtype=float))[None, :], ppm, M - 200)[0]
    t = np.arange(M - 200) * (1 + ppm * 1e-6)
    ref = sig(t)
    sl = slice(100, M - 300)                       # away from the zero padding at both ends
    err = 10 * np.log10(np.mean(np.abs(y[sl] - ref[sl]) ** 2) / np.mean(np.abs(ref[sl]) ** 2))
    assert err < -60, err


@pytest.mark.parametrize("N,nrx,snr,delay,ppm", [(128, 1, 25.0, 0, 0.0), (256, 2, 10.0, 3, 20.0), (384, 1, 0.0, 0, -20.0), (512, 2, 25.0, 5, 2.0),
                                                 (768, 1, 15.0, 2, 50.0), (1536, 2, 5.0, 0, -5.0), (2048, 1, 20.0, 4, 20.0)])
def test_oracle_equals_float64_reference(N, nrx, snr, delay, ppm):
    """identical argmax, lock and timing decisions, and S within 1e-5 relative, on 3 frames (6 half-frames, a timing correction)"""
    x, truth, _ = T.capture(N, 301, 32, nrx=nrx, ppm=ppm, cfo=1500.0, snr=snr, lead=7 * N, seed=N + nrx, chan_delay=delay, t0=3)
    o = T.Oracle(N, nrx, 301, 7 * N, cfo_hz=1400.0, first_tti=3).push(x, 0)
    f = F.track(N, x, 301, 7 * N, 1400.0, first_tti=3)
    assert len(o["hf"]) >= 5
    np.testing.assert_array_equal(o["sf"]["start"], f["start"])
    np.testing.assert_array_equal(o["sf"]["flags"], f["flags"])
    np.testing.assert_array_equal(o["hf"]["delta"], f["delta"])
    np.testing.assert_array_equal((o["hf"]["flags"] & T.LOCKED) != 0, f["locked"])
    np.testing.assert_allclose(o["hf"]["peak"], f["peak"], rtol=1e-4)
    S = o["hf"]["s_re"] + 1j * o["hf"]["s_im"]
    np.testing.assert_allclose(S, f["S"], rtol=1e-5, atol=1e-5 * np.abs(f["S"]).max())
    np.testing.assert_allclose(o["sf"]["cfo_hz"], f["cfo"], rtol=0, atol=0.05)


@pytest.mark.parametrize("nof_ues,cfo_tol", [(1, 50.0), (3, 75.0)])
@pytest.mark.parametrize("ppm", [0.0, 2.0, -2.0, 20.0, -20.0])
def test_tracks_clock_offset_and_cfo_ramp(ppm, nof_ues, cfo_tol):
    """25 PRB, 2 antennas, 400 ms, carrier offset 1 kHz + 200 Hz/s: every start within 2 samples of the truth after 40 ms, and the carrier offset
    within cfo_tol of the truth after 200 ms.  The data sharing the PSS symbol is what spreads each half-frame's f_meas (about +-100 Hz with a
    full load), and the loop's lag on the ramp is 200 Hz/s * 5 ms / 0.05 = 20 Hz: within 50 Hz with one scheduled UE, within 75 Hz at the full
    load of three (53 to 61 Hz measured, DESIGN.md §7)."""
    N = 512
    x, truth, ft = T.capture(N, 77, 400, nrx=2, ppm=ppm, cfo=1000.0, ramp=200.0, snr=20.0, lead=1000, seed=3, nof_ues=nof_ues)
    r = T.Oracle(N, 2, 77, 1000, cfo_hz=900.0).push(x, 0, cut=False)
    k = r["sf"]["index"]
    assert len(k) >= 390
    err = r["sf"]["start"] - truth[k]
    assert np.abs(err[k >= 40]).max() <= 2, np.abs(err[k >= 40]).max()
    assert np.abs(r["sf"]["cfo_hz"] - ft[k])[k >= 200].max() <= cfo_tol
    assert (r["hf"]["flags"] & T.LOCKED).all() and not (r["sf"]["flags"] & T.LOST).any()


def test_no_clock_offset_gives_the_fixed_cut():
    N = 384
    x, truth, _ = T.capture(N, 5, 120, nrx=1, cfo=-2500.0, snr=15.0, lead=333, seed=8)
    r = T.Oracle(N, 1, 5, 333, cfo_hz=-2500.0).push(x, 0, cut=False)
    np.testing.assert_array_equal(r["sf"]["start"], 333 + np.arange(len(r["sf"])) * 15 * N)


def test_gap_is_flagged_lost_and_relocks():
    """100 ms of zeros at 20 ppm: flagged lost after 4 misses, cut continues at the predicted starts, relocks after it and keeps the timing"""
    N = 256
    x, truth, _ = T.capture(N, 100, 400, nrx=1, ppm=20.0, snr=20.0, lead=500, seed=4, gap=(150 * 15 * N, 100 * 15 * N))
    r = T.Oracle(N, 1, 100, 500).push(x, 0, cut=False)
    sf, hf = r["sf"], r["hf"]
    lost = (sf["flags"] & T.LOST) != 0
    assert lost.any()
    assert not lost[sf["index"] < 150].any() and not lost[sf["index"] >= 260].any()
    assert (hf["flags"][hf["index"] >= 260] & T.LOCKED).all()
    k = sf["index"]
    assert np.abs(sf["start"] - truth[k])[k >= 290].max() <= 2


@pytest.mark.parametrize("N,nrx", [(128, 1), (512, 2), (2048, 1)])
def test_no_lock_on_noise(N, nrx):
    rng = np.random.default_rng(N)
    L = 15 * N * 200
    x = ((rng.standard_normal((nrx, L)) + 1j * rng.standard_normal((nrx, L))) * 0.3).astype(np.complex64)
    r = T.Oracle(N, nrx, 0, 0).push(x, 0, cut=False)
    assert len(r["hf"]) == 40
    assert not (r["hf"]["flags"] & T.LOCKED).any(), r["hf"]["peak"].max() * N
    assert (r["hf"]["peak"] * N).max() < 0.6 * F.LOCK_K


def chunk_cases(N):
    SF = 15 * N
    return [[10 ** 9], [SF], [SF + 1], [7919, 3 * SF + 17, 104729], [13 * N // 2 + 3, SF - 5]]


@pytest.mark.parametrize("sizes_i", range(5))
def test_chunking_invariance(sizes_i):
    N = 256
    x, _, _ = T.capture(N, 33, 120, nrx=2, ppm=-20.0, cfo=700.0, ramp=500.0, snr=12.0, lead=1234, seed=6)
    ref = T.Oracle(N, 2, 33, 1234, cfo_hz=650.0).push(x, 0)
    got = T.run_chunks(T.Oracle(N, 2, 33, 1234, cfo_hz=650.0), x, chunk_cases(N)[sizes_i])
    assert got["sf"].tobytes() == ref["sf"].tobytes() and got["hf"].tobytes() == ref["hf"].tobytes()
    assert got["iq"].tobytes() == ref["iq"].tobytes()


def test_fixed_cut_loses_the_end_at_20ppm():
    """why tracking is needed: at 20 ppm the fixed cut of a 2 s capture leaves the cyclic prefix (144 N / 2048 samples) in the last second, while
    the tracked starts stay within 2 samples"""
    N = 256
    x, truth, _ = T.capture(N, 12, 2000, nrx=1, ppm=20.0, snr=20.0, lead=100, seed=2, nof_ues=1)
    r = T.Oracle(N, 1, 12, 100).push(x, 0, max_sf=2000, cut=False)
    k = r["sf"]["index"]
    assert len(k) >= 1990
    fixed = 100 + k * 15 * N
    assert np.abs(fixed - truth[k])[k >= 1000].min() > 9 * N / 128
    assert np.abs(r["sf"]["start"] - truth[k])[k >= 40].max() <= 2


def test_invalid_configs_are_rejected(phylib):
    from ltesniffer_b200 import capi
    good = dict(symbol_sz=512, nof_rx=1, pci=1, first_tti=0, frame_offset=0, cfo_hz=0.0, max_ppm=50.0, max_subframes=10, flags=0, device=0)
    h = C.c_void_p()
    phylib.ltephy_track_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    for bad in [dict(symbol_sz=500), dict(nof_rx=3), dict(nof_rx=0), dict(pci=504), dict(first_tti=10240), dict(cfo_hz=8000.0), dict(cfo_hz=float("nan")),
                dict(max_ppm=-1.0), dict(max_subframes=0), dict(flags=8)]:
        cfg = capi.TrackCfg(**{**good, **bad})
        assert phylib.ltephy_track_create(C.byref(cfg), C.byref(h)) == -2, bad
    assert phylib.ltephy_track_create(None, C.byref(h)) == -2
    phylib.ltephy_track_push.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]
    assert phylib.ltephy_track_push(None, None, 0, 0, None) == -2
