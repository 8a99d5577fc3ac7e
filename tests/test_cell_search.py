"""Cell search on the CPU: the PSS / SSS the simulator maps against a numpy statement of 36.211 6.11, and the oracle's lteo_cell_search
(DESIGN.md §2, "cell search") on captures cut at random offsets, with CFO, noise, multipath, two cells and the edge cases of the timing rules;
its intermediates against the float64 reference in ref64_sync.py; and the PBCH decoded at the timing it finds."""
import numpy as np
import pytest

import ltelib
import sync_lib as S
import ref64_sync as R

NS = [128, 256, 384, 512, 768, 1024, 1536, 2048]
PRB_OF = {256: 15, 384: 25, 512: 25, 768: 50, 1024: 50, 1536: 75, 2048: 100}


def truth_offset(N, off, t0=0):
    """first sample of a subframe 0 in a capture cut at sample off of a recording whose first subframe is t0"""
    return (-(t0 % 10) * 15 * N - off) % (150 * N)


def sim_capture(N, pci, nsf, off, L, nrx=1, cfo=0.0, snr=60.0, t0=0, seed=1, chan_delay=0, nof_ports=1, pbch=0, frac=False, nof_ues=3):
    """sync = 1 subframes t0 .. t0 + nsf - 1 per antenna, concatenated, cut to [off, off + L), a continuous CFO applied in float64"""
    if N == 128:
        rng = np.random.default_rng(seed)
        full = np.array([R.synth(N, pci, nsf, rng, t0) for _ in range(nrx)])
        full = full + (rng.standard_normal(full.shape) + 1j * rng.standard_normal(full.shape)) * np.sqrt(0.5 * 10 ** (-snr / 10))
    else:
        cell = ltelib.Cell(PRB_OF[N], nof_ports, pci, nrx, N)
        s = S.sim(sync=1, cell=cell, seed=seed, pbch=pbch, snr_db=snr, nof_ues=nof_ues, dl_min=1, dl_max=3, chan_delay=chan_delay)
        full = np.concatenate([s.subframe(t0 + i)[0] for i in range(nsf)], axis=1).astype(np.complex128)
    if frac:   # half a sample of delay as a phase ramp over the whole recording
        F = np.fft.fftfreq(full.shape[1])
        full = np.fft.ifft(np.fft.fft(full, axis=1) * np.exp(-2j * np.pi * F * 0.5), axis=1)
    x = full[:, off:off + L]
    n = np.arange(off, off + x.shape[1])
    return (x * np.exp(2j * np.pi * cfo * n / (15000 * N))).astype(np.complex64)


def best(out):
    return out[0]


def test_pss_sss_sequences_match_the_simulator():
    """the numpy PSS / SSS for all 504 PCIs and both SSS subframes equal the REs the simulator maps, read back through lteo_ofdm_rx"""
    f = R.subcarriers()
    for pci in range(504):
        cell = ltelib.Cell(15, 1, pci, 1, 256)
        s = S.sim(sync=1, cell=cell, seed=pci, snr_db=300.0, nof_ues=0)
        o = ltelib.Oracle(cell)
        for sf in (0, 5):
            sym = o.ofdm(s.subframe(sf)[0]).reshape(14, 180)
            k = f + 90 - (f > 0)          # grid index of sub-carrier f: 90 + f below DC, 89 + f above
            g = sym[6, k[0]] / R.pss(pci % 3)[0]   # the channel of port 0 and the sqrt(N) of the unscaled DFT
            assert abs(abs(g) - 16.0) < 1e-3
            np.testing.assert_allclose(sym[6, k] / g, R.pss(pci % 3), atol=2e-5)
            np.testing.assert_allclose(sym[5, k] / g, R.sss(pci // 3, pci % 3, sf == 5), atol=2e-5)


def test_pss_unit_modulus_and_low_cross_correlation():
    d = [R.pss(u) for u in range(3)]
    for u in range(3):
        np.testing.assert_allclose(np.abs(d[u]), 1.0, atol=1e-12)
    p = R.replicas(2048)
    for a in range(3):
        for b in range(3):
            if a != b:   # largest circular cross-correlation of two roots at any lag against the autocorrelation at lag 0 (0.19 .. 0.39)
                xc = np.abs(np.fft.ifft(np.fft.fft(p[a]) * np.conj(np.fft.fft(p[b])))).max()
                assert xc < 0.4 * np.abs(np.vdot(p[a], p[a]))


def test_sync_off_leaves_the_samples_unchanged():
    cell = ltelib.Cell(25, 2, 77, 2, 0)
    a = ltelib.Sim(cell=cell, seed=4, nof_ues=4, dl_min=2, dl_max=3).subframe(5)[0]
    b = S.sim(sync=0, cell=cell, seed=4, nof_ues=4, dl_min=2, dl_max=3).subframe(5)[0]
    c = S.sim(sync=1, cell=cell, seed=4, nof_ues=4, dl_min=2, dl_max=3).subframe(5)[0]
    assert a.tobytes() == b.tobytes() and a.tobytes() != c.tobytes()


def test_all_504_pcis_at_128():
    rng = np.random.default_rng(7)
    for pci in range(504):
        off = int(rng.integers(0, 150 * 128))
        x = sim_capture(128, pci, 22, off, 75 * 128 * 2 + 128, seed=pci)
        r, out, _ = S.cell_search(128, x)
        assert r == 0
        c = best(out)
        assert c.detected and c.pci == pci and c.frame_offset == truth_offset(128, off), (pci, c.pci, c.frame_offset)


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("nrx", [1, 2])
def test_every_symbol_size(N, nrx):
    rng = np.random.default_rng(N + nrx)
    pci, off = int(rng.integers(0, 504)), int(rng.integers(0, 150 * N))
    x = sim_capture(N, pci, 22, off, 75 * N * 2 + N, nrx=nrx, seed=N)
    r, out, _ = S.cell_search(N, x)
    c = best(out)
    assert r == 0 and c.detected and c.pci == pci and c.frame_offset == truth_offset(N, off)
    assert c.nof_half_frames >= 1 and sorted([o.n_id_2 for o in out]) == [0, 1, 2]
    assert all(out[i].pss_peak >= out[i + 1].pss_peak for i in range(2))


@pytest.mark.parametrize("cfo", [0.0, 1200.0, -1200.0, 4000.0, -4000.0])
@pytest.mark.parametrize("N", [256, 768])
def test_cfo(N, cfo):
    """noiseless flat channel: within 30 Hz when the PSS symbol carries nothing else; within 100 Hz with PDSCH on the other sub-carriers, whose
    leakage into the half-symbol correlations is the error that remains"""
    off = 3 * N + 17
    for ues, tol in ((0, 30.0), (3, 100.0)):
        x = sim_capture(N, 211, 32, off, 75 * N * 4, cfo=cfo, seed=3, nof_ues=ues)
        r, out, _ = S.cell_search(N, x)
        c = best(out)
        assert c.detected and c.pci == 211 and c.frame_offset == truth_offset(N, off)
        assert abs(c.cfo_hz - cfo) <= tol, (ues, c.cfo_hz)


@pytest.mark.parametrize("snr", [20.0, 0.0])
@pytest.mark.parametrize("N,nrx", [(256, 1), (512, 2), (128, 1)])
def test_noise(N, nrx, snr):
    off = 11 * N + 5
    x = sim_capture(N, 400, 32, off, 75 * N * 4 + N, nrx=nrx, snr=snr, seed=9, cfo=500.0)
    r, out, _ = S.cell_search(N, x)
    c = best(out)
    assert c.pci == 400
    d = (int(c.frame_offset) - truth_offset(N, off) + 75 * N) % (150 * N) - 75 * N
    assert abs(d) <= 2
    if snr >= 20:
        assert c.detected


def test_multipath_delay():
    """chan_delay spreads each path over up to 6 samples: the timing lands inside that spread"""
    N, off = 512, 1000
    x = sim_capture(N, 55, 32, off, 75 * N * 4, nrx=2, nof_ports=2, chan_delay=6, seed=12)
    c = best(S.cell_search(N, x)[1])
    d = (int(c.frame_offset) - truth_offset(N, off) + 75 * N) % (150 * N) - 75 * N
    assert c.pci == 55 and 0 <= d <= 6, d


def test_fractional_delay():
    N, off = 256, 333
    x = sim_capture(N, 98, 22, off, 75 * N * 2 + N, seed=13, frac=True)
    c = best(S.cell_search(N, x)[1])
    d = (int(c.frame_offset) - truth_offset(N, off) + 75 * N) % (150 * N) - 75 * N
    assert c.pci == 98 and abs(d) <= 1


# ---- edge cases of the timing rules: N = 256, PSS of subframe 0 at 13 * N / 2 + 15 N * 10 k
@pytest.mark.parametrize("case", ["pss_at_0", "pss_in_last_window", "sss_before_start", "exactly_hf_plus_n", "starts_in_sf5"])
def test_edge_cases(case):
    N = 256
    HF, p0 = 75 * N, 13 * N // 2
    t0, L = 0, 2 * HF + N
    if case == "pss_at_0":
        off, L = p0, HF + N + 100   # the capture starts on the PSS of subframe 0: its SSS is before the start
    elif case == "pss_in_last_window":
        off, L = p0 - 37, HF + 37 + N   # the second PSS window ends on the last sample
    elif case == "sss_before_start":
        off = p0 - N // 2           # the first PSS window fits, its SSS does not
    elif case == "exactly_hf_plus_n":
        off, L = 1234, HF + N
    else:
        t0, off = 5, 4321           # the recording starts in subframe 5
    x = sim_capture(N, 321, 22, off, L, t0=t0, seed=21)
    r, out, _ = S.cell_search(N, x)
    c = best(out)
    assert r == 0 and c.pci == 321 and c.frame_offset == truth_offset(N, off, t0), (c.pci, c.frame_offset, truth_offset(N, off, t0))
    if case == "pss_at_0":
        assert c.nof_half_frames == 1   # only the PSS at sample 75 N has its SSS inside


def test_two_cells():
    """two cells with different N_ID_2, 6 dB apart, at different timings: each is found with its own PCI and frame timing"""
    N = 512
    a = sim_capture(N, 3 * 40 + 0, 32, 2000, 75 * N * 4, seed=31)
    b = sim_capture(N, 3 * 90 + 2, 32, 9000, 75 * N * 4, seed=32) * np.float32(10 ** (-6 / 20))
    r, out, _ = S.cell_search(N, a + b)
    got = {o.n_id_2: o for o in out}
    assert got[0].pci == 120 and got[0].frame_offset == truth_offset(N, 2000) and got[0].detected
    assert got[2].pci == 272 and got[2].frame_offset == truth_offset(N, 9000)
    assert out[0].n_id_2 == 0


def test_noise_only_never_detects():
    """200 noise-only captures over every symbol size: no detection (the false-alarm figure of DESIGN.md §2)"""
    worst_psr = worst_sss = 0.0
    for seed in range(200):
        rng = np.random.default_rng(1000 + seed)
        N, A = NS[seed % 8], 1 + (seed // 8) % 2
        L = 76 * N + int(rng.integers(0, 75 * N))
        x = ((rng.standard_normal((A, L)) + 1j * rng.standard_normal((A, L))) / np.sqrt(2)).astype(np.complex64)
        r, out, _ = S.cell_search(N, x)
        assert r == 0 and not any(o.detected for o in out)
        worst_psr = max(worst_psr, max(o.psr for o in out))
        worst_sss = max(worst_sss, max(o.sss_ratio for o in out))
    assert worst_psr < 2.0 and worst_sss < 1.75


def test_invalid_inputs():
    x = np.zeros((1, 75 * 256 + 256), np.complex64)
    assert S.cell_search(256, x[:, :-1])[0] == -2
    assert S.cell_search(192, x)[0] == -2
    assert S.cell_search(256, np.zeros((3, x.shape[1]), np.complex64))[0] == -2
    r, out, _ = S.cell_search(256, x)          # all zero: nothing found, nothing NaN
    assert r == 0 and not any(o.detected for o in out) and all(np.isfinite(o.psr) and np.isfinite(o.sss_ratio) for o in out)


@pytest.mark.parametrize("N,nrx,cfo,snr", [(128, 1, 0.0, 60.0), (256, 2, 2500.0, 10.0), (384, 1, -700.0, 30.0)])
def test_float64_reference_agrees(N, nrx, cfo, snr):
    off = 5 * N + 3
    x = sim_capture(N, 191, 32, off, 75 * N * 3 + N // 2, nrx=nrx, cfo=cfo, snr=snr, seed=41)
    r, out, t = S.cell_search(N, x)
    ref = R.search(N, x.astype(np.complex128))
    np.testing.assert_allclose(t["coarse"], ref["coarse"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(t["refined"], ref["refined"], rtol=1e-5, atol=1e-7)
    s_cfo = t["cfo"][:, 0] + 1j * t["cfo"][:, 1]
    np.testing.assert_allclose(s_cfo, ref["S"], rtol=1e-5, atol=1e-5 * np.abs(ref["S"]).max())
    scale = np.abs(ref["sss"]).max(axis=(1, 2), keepdims=True)
    np.testing.assert_allclose(t["sss"], ref["sss"], rtol=1e-5, atol=1e-5 * scale.max())
    for o in out:   # identical decisions
        u = o.n_id_2
        assert int(np.argmax(ref["coarse"][u])) == int(np.argmax(t["coarse"][u]))
        assert int(np.argmax(ref["refined"][u])) == int(np.argmax(t["refined"][u]))
        if o.n_id_1 != 0xFFFF:
            assert int(np.argmax(ref["sss"][u])) == 2 * o.n_id_1 + int(np.argmax(t["sss"][u].reshape(-1)) % 2)


def test_pbch_at_the_found_timing():
    """end to end on the CPU: at the frame timing and PCI found, after lteo_cfo_correct, lteo_pbch_decode returns the MIB the simulator sent"""
    N, cfo, off, pci = 512, 2100.0, 5555, 217
    cell = ltelib.Cell(25, 2, pci, 2, N)
    x = sim_capture(N, pci, 32, off, 75 * N * 5, nrx=2, cfo=cfo, seed=51, nof_ports=2, pbch=1, snr=30.0)
    c = best(S.cell_search(N, x)[1])
    assert c.detected and c.pci == pci
    o = ltelib.Oracle(ltelib.Cell(25, 2, c.pci, 2, N))
    fo = int(c.frame_offset)
    sf = x[:, fo:fo + 15 * N]
    # the subframe starts fo samples in: the CFO phase there is carried by the channel estimate, so the per-subframe correction suffices
    sym = o.ofdm(o.cfo_correct(c.cfo_hz, sf))
    ce, _ = o.chest(0, sym)
    found, mib, nports, q = o.pbch_decode(sym, ce)
    assert found == 1 and nports == 2
    want = np.zeros(24, np.uint8)
    sfn = (off + fo) // (150 * N)   # frame index of that subframe 0 in the recording
    sim = ltelib.sim()
    sim.lte_mib_pack.argtypes = [ltelib.C.c_uint32] * 4 + [ltelib.C.c_void_p]
    sim.lte_mib_pack(25, cell.phich_ext, cell.phich_ng, sfn, ltelib.ptr(want))
    assert np.array_equal(mib, want) and q == sfn % 4


def test_example_builds_and_refuses_to_run_without_a_gpu(tmp_path):
    import os
    import subprocess
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present: covered by the gpu test")
    except ImportError:
        pass
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run(["make", "-s", "-C", root, "examples/cell_search"], check=True)
    f = tmp_path / "x.cf32"
    f.write_bytes(b"\0" * 8 * (76 * 256))
    r = subprocess.run([os.path.join(root, "examples", "cell_search"), str(f), "256", "1"], capture_output=True, text=True)
    assert r.returncode == 1 and "ltephy_sync_create" in r.stderr, (r.returncode, r.stderr)


@pytest.mark.parametrize("N", [128, 512])
def test_ties_go_to_the_lowest_index(N):
    """an all-zero capture makes every comparison a tie: coarse bin 0, refined offset -(D - 1), N_ID_1 = 0 with q = 0, N_ID_2 in order"""
    D, HF = N // 128, 75 * N
    r, out, t = S.cell_search(N, np.zeros((2, 2 * HF + N), np.complex64))
    assert r == 0 and [o.n_id_2 for o in out] == [0, 1, 2]
    for o in out:
        assert o.n_id_1 == 0 and o.pci == o.n_id_2 and not o.detected and o.psr == 0.0 and o.sss_ratio == 0.0
        assert o.frame_offset == ((HF - (D - 1)) % HF - 13 * N // 2) % (150 * N)
