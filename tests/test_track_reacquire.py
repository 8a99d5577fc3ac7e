"""The tracker's find state on the CPU (LTEPHY_TRACK_REACQUIRE, DESIGN.md §2 "tracking"), on the oracle lteo_track_*: a receiver that drops
samples is lost, searched again frame by frame and resumed at the new timing with the right subframe numbers; a zero-filled fade resumes at the
old timing with a continuous SFN; noise is never taken for the cell; the result does not depend on how the recording is split; the uplink cut
follows the new timing."""
import numpy as np
import pytest

import track_lib as T
import track_reacq_lib as Q

PCI, T0, CFO = 301, 3, 1000.0
DROP_CASES = [  # N, nrx, snr, drop
    (128, 1, 10.0, "3N+17"), (128, 2, 25.0, "37SF+1234"),
    (512, 2, 15.0, "3N+17"), (512, 1, 20.0, "37SF+1234"),
    (1536, 1, 25.0, "3N+17"), (1536, 2, 12.0, "37SF+1234"),
]


def drop_capture(N, nrx, snr, drop, seed=None):
    """a tracker's first timing correction before the drop (40 subframes in), then at least 60 subframes after it; 20 ppm"""
    SF, lead = 15 * N, 5 * N + 7
    cnt = Q.drop_cases(N)[drop] if isinstance(drop, str) else drop
    nsf = 40 + -(-cnt // SF) + 60
    x, truth, ft, num = Q.capture(N, PCI, nsf, drop=(lead + 40 * SF + 333, cnt), nrx=nrx, ppm=20.0, cfo=CFO, snr=snr, lead=lead,
                                  seed=N + nrx, t0=T0)
    return x, truth, ft, num, lead


def check_reacquired(r, truth, ft, num, drop_at, N, cfo_tol=200.0):
    """the records of one drop: lost, then nothing until the re-acquired subframe at the truth timing and subframe number, then locked.  The
    found start is within 1 sample of the truth plus what a 20 ppm clock moves over the frame the cell search averages (4.6 samples at N = 1536),
    until the tracker's first timing correction after it; then within 2 (3.3 at N = 1536, where the clock moves 9 samples between corrections).  The
    carrier offset restarts from the find's estimate over two or three PSS (up to 177 Hz off at 10 dB on one antenna of 6 PRB), which the loop,
    with its 100 ms time constant, has not yet refined to test_track's 50 / 75 Hz within the 60 subframes these captures have after the drop."""
    sf, hf = r["sf"], r["hf"]
    k = sf["index"].astype(np.int64)
    assert (np.diff(k) > 0).all()
    lost = np.flatnonzero(hf["flags"] & T.LOST)
    assert len(lost), "never lost"
    ire = np.flatnonzero(sf["flags"] & Q.REACQUIRED)
    assert len(ire) == 1, ire
    i = ire[0]
    assert sf["flags"][i] & T.LOCKED and not sf["flags"][i] & T.LOST
    assert sf["index"][i - 1] == hf["index"][lost[0]], "subframes were cut in the find state"
    assert not (sf["flags"][:i] & Q.REACQUIRED).any()
    j = int(np.argmin(np.abs(truth - sf["start"][i])))
    tol = 1 + 20e-6 * 150 * N
    assert truth[j] >= drop_at and abs(sf["start"][i] - truth[j]) <= tol, (sf["start"][i], truth[j])
    assert sf["tti"][i] % 10 == (T0 + num[j]) % 10
    after = sf[i:]
    jj = j + (after["index"].astype(np.int64) - int(sf["index"][i]))
    ok = jj < len(truth)
    assert ok.sum() >= 30
    err = np.abs(after["start"][ok] - truth[jj[ok]])
    assert err.max() <= tol and err[after["index"][ok] >= sf["index"][i] + 25].max() <= max(2.0, tol / 2 + 1)
    assert ((after["tti"][ok] - (T0 + num[jj[ok]])) % 10 == 0).all()
    assert np.abs(after["cfo_hz"][ok] - ft[jj[ok]]).max() <= cfo_tol
    later = hf["index"] >= sf["index"][i]
    assert later.sum() >= 6 and (hf["flags"][later] & T.LOCKED).all() and not (hf["flags"][later] & T.LOST).any()
    assert not (after["flags"] & T.LOST).any()
    return i


@pytest.mark.parametrize("case", range(len(DROP_CASES)))
def test_drop_is_reacquired(case):
    N, nrx, snr, drop = DROP_CASES[case]
    x, truth, ft, num, lead = drop_capture(N, nrx, snr, drop)
    r = T.Oracle(N, nrx, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE).push(x, 0, cut=False)
    i = check_reacquired(r, truth, ft, num, lead + 40 * 15 * N + 333, N)
    # the first window starts at the subframe after the lost one, 20 ms after the drop: wholly after it, so one window finds the cell
    assert r["finds"] == 1
    assert 0 <= r["sf"]["start"][i] - (r["sf"]["start"][i - 1] + 15 * N) < 15 * N + 2
    # without the flag the tracker never locks again
    r0 = T.Oracle(N, nrx, PCI, lead, cfo_hz=900.0, first_tti=T0).push(x, 0, cut=False)
    n = len(r["sf"]) and int(r["sf"]["index"][i])
    assert (r0["sf"]["flags"][r0["sf"]["index"] >= n] & T.LOST).all()


@pytest.mark.parametrize("N", [128, 512, 1536])
def test_drop_of_whole_frames_keeps_the_timing(N):
    """12 frames dropped move every later PSS by only what the 20 ppm clock moved over them (4.6 samples at N = 128), inside the tracker's
    +-9 N / 128: nothing is lost and no window is searched, and the subframe numbers stay right, but the SFN is 12 frames ahead of the count --
    only the MIB can tell"""
    x, truth, ft, num, lead = drop_capture(N, 2, 15.0, 12 * 150 * N)
    r = T.Oracle(N, 2, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE).push(x, 0, cut=False)
    sf = r["sf"]
    assert r["finds"] == 0 and not (sf["flags"] & (T.LOST | Q.REACQUIRED)).any()
    k = sf["index"]
    assert np.abs(sf["start"] - truth[k]).max() <= 9 * N // 128
    assert ((sf["tti"] - (T0 + num[k])) % 10 == 0).all()
    assert ((T0 + num[k] - sf["tti"])[k >= 60] == 120).all()


def test_fade_reacquires_at_the_old_timing():
    """the 100 ms zero-filled gap of test_track.test_gap_is_flagged_lost_and_relocks, with the flag: found again at the old timing (at the first
    subframe boundary of the window that detects the cell, which may still lie in the gap), and every tti is the truth tti because no sample
    was dropped"""
    N = 256
    x, truth, _ = T.capture(N, 100, 400, nrx=1, ppm=20.0, snr=20.0, lead=500, seed=4, gap=(150 * 15 * N, 100 * 15 * N))
    r = T.Oracle(N, 1, 100, 500, flags=Q.REACQUIRE).push(x, 0, cut=False)
    sf = r["sf"]
    ire = np.flatnonzero(sf["flags"] & Q.REACQUIRED)
    assert len(ire) == 1 and r["finds"] >= 1
    k = sf["index"]
    assert np.abs(sf["start"][ire[0]] - truth[k[ire[0]]]) <= 1
    assert np.abs(sf["start"] - truth[k])[k >= 290].max() <= 2
    np.testing.assert_array_equal(sf["tti"], k % 10240)
    assert not (sf["flags"][ire[0]:] & T.LOST).any()


NOISE_CASES = [(128, 1, 60), (128, 2, 40), (512, 1, 30), (512, 2, 30), (1536, 1, 20), (1536, 2, 20)]  # N, nrx, windows: 200 in all


@pytest.mark.parametrize("case", range(len(NOISE_CASES)))
def test_noise_is_never_found(case):
    """the cell for 30 subframes, then noise of the same power: no find succeeds, nothing is cut, next_sample steps one frame per window"""
    N, nrx, nwin = NOISE_CASES[case]
    SF, FR = 15 * N, 150 * N
    x, _, _ = T.capture(N, PCI, 30, nrx=nrx, snr=20.0, lead=N, seed=case)
    rms = np.sqrt(np.mean(np.abs(x[:, N:]) ** 2))
    x = np.concatenate([x, Q.noise(np.random.default_rng(case), nrx, (nwin + 3) * FR, rms)], axis=1)
    tr = T.Oracle(N, nrx, PCI, N, flags=Q.REACQUIRE)
    r = tr.push(x[:, :N + 30 * SF], 0, cut=False)           # locked up to the end of the cell
    assert r["finds"] == 0 and not (r["sf"]["flags"] & T.LOST).any()
    total, nxt = 0, tr.next_sample
    for e in range(N + 31 * SF, x.shape[1] + 1, FR // 2):   # the rest half a frame at a time
        r = tr.push(x[:, tr.next_sample:e], tr.next_sample, cut=False)
        if total == 0 and len(r["sf"]):
            assert (r["sf"]["flags"] & T.LOST).sum() <= 5 and not (r["sf"]["flags"] & Q.REACQUIRED).any()
            nxt = tr.next_sample
        else:
            assert len(r["sf"]) == 0
            assert tr.next_sample == nxt + r["finds"] * FR
            nxt = tr.next_sample
        total += r["finds"]
    assert total >= nwin, total


def test_chunking_inside_and_at_find_windows():
    N, nrx = 128, 2
    SF, FR = 15 * N, 150 * N
    x, truth, ft, num, lead = drop_capture(N, nrx, 15.0, "37SF+1234")
    mk = lambda: T.Oracle(N, nrx, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE)
    ref = mk().push(x, 0)
    assert ref["finds"] == 1
    for sizes in [[FR + N], [FR], [FR // 3], [SF - 1, FR + N + 1], [7919, 3 * SF + 17, 104729]]:
        got = T.run_chunks(mk(), x, sizes)
        assert got["sf"].tobytes() == ref["sf"].tobytes() and got["hf"].tobytes() == ref["hf"].tobytes(), sizes
        assert got["iq"].tobytes() == ref["iq"].tobytes() and got["finds"] == ref["finds"], sizes


@pytest.mark.parametrize("ul_offset", [-(3 * 128 + 5), 2 * 128 + 1])
def test_uplink_cut_follows_the_new_timing(ul_offset):
    """OracleUl with the flag: the DL records are those without the uplink, and each UL subframe after the re-acquisition is x_ul from
    start + ul_offset, rotated by f_ul = cfo_hz cfo_ratio"""
    N, rho = 128, 0.95
    x, truth, ft, num, lead = drop_capture(N, 1, 20.0, "37SF+1234")
    xu = Q.noise(np.random.default_rng(5), 1, x.shape[1], 1.0)[0]
    dl = T.Oracle(N, 1, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE).push(x, 0, cut=False)
    tr = T.Oracle(N, 1, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE, ul=dict(cfo_ratio=rho, ul_offset=ul_offset))
    r = tr.push_ul(x, xu, 0)
    assert r["sf"].tobytes() == dl["sf"].tobytes() and r["finds"] == dl["finds"] == 1
    i = int(np.flatnonzero(r["sf"]["flags"] & Q.REACQUIRED)[0])
    n = np.arange(15 * N)
    for q in range(i, len(r["sf"])):
        s, f = int(r["sf"]["start"][q]) + ul_offset, float(np.float32(r["sf"]["cfo_hz"][q] * rho))
        want = xu[s:s + 15 * N] * np.exp(-2j * np.pi * f * n / (15000.0 * N))
        np.testing.assert_allclose(r["ul_iq"][q], want, rtol=0, atol=1e-5 * np.abs(want).max())


@pytest.mark.parametrize("case", [0, 1, 3])
def test_oracle_equals_float64_reference(case):
    """the find rule restated in float64 (ref64_track_find, on ref64_sync.search): identical starts, ttis, flags and find count on the drop
    captures -- the exact re-acquired start, subframe number and drift rebase, not only their distance from the truth"""
    import ref64_track_find as F
    N, nrx, snr, drop = DROP_CASES[case]
    x, _, _, _, lead = drop_capture(N, nrx, snr, drop)
    o = T.Oracle(N, nrx, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE).push(x, 0, cut=False)
    f = F.track(N, x, PCI, lead, 900.0, first_tti=T0)
    assert (o["sf"]["flags"] & Q.REACQUIRED).any() and o["finds"] == f["finds"] == 1
    np.testing.assert_array_equal(o["sf"]["start"], f["start"])
    np.testing.assert_array_equal(o["sf"]["tti"], f["tti"])
    np.testing.assert_array_equal(o["sf"]["flags"], f["flags"])
