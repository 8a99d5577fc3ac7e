"""Uplink tracking on the CPU (DESIGN.md §2, "tracking", uplink): the oracle's UL cut (lteo_track_set_ul / lteo_track_push_ul) against the
downlink cut and a float64 restatement, its chunking invariance, its physics against the oracle PUSCH decode on a two-carrier capture with a
sampling-clock offset and a carrier offset, the constant uplink CFO correction, and the argument checks of the oracle and the C-ABI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ltelib
import track_lib as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "examples", "decode_recording_ul")


def _dl_capture(N=256, nsf=40, ppm=20.0, seed=6):
    return T.capture(N, 33, nsf, nrx=2, ppm=ppm, cfo=700.0, ramp=500.0, snr=12.0, lead=1234, seed=seed)[0]


def test_ul_cut_of_downlink_antenna_equals_downlink_cut():
    """cfo_ratio 1, ul_offset 0 and the uplink equal to DL antenna 0: the UL cut is DL cut antenna 0 bit for bit, and the DL records and cut equal
    those of a tracker without the uplink"""
    x = _dl_capture()
    ref = T.Oracle(256, 2, 33, 1234, cfo_hz=650.0).push(x, 0)
    got = T.Oracle(256, 2, 33, 1234, cfo_hz=650.0, ul=dict(cfo_ratio=1.0, ul_offset=0)).push_ul(x, x[0], 0)
    assert got["sf"].tobytes() == ref["sf"].tobytes() and got["hf"].tobytes() == ref["hf"].tobytes()
    assert got["iq"].tobytes() == ref["iq"].tobytes()
    assert got["ul_iq"].tobytes() == np.ascontiguousarray(ref["iq"][:, 0]).tobytes()


@pytest.mark.parametrize("rho", [1.0, 0.948, 1.05])
@pytest.mark.parametrize("off_n", [-1, 0, 1])
def test_ul_cut_equals_float64_restatement(rho, off_n):
    """UL subframe k = x_ul[start_k + ul_offset + n] exp(-j 2 pi f_ul n / (15000 N)), f_ul = cfo_hz_k rho, within 1e-5 relative; the clock offset
    cycles through 0 / +20 / -20 ppm over the cases"""
    N = 256
    ppm = [0.0, 20.0, -20.0][(int(rho * 100) + off_n) % 3]
    x = _dl_capture(N, 40, ppm, seed=7)
    rng = np.random.default_rng(off_n + 5)
    xu = (rng.standard_normal(x.shape[1]) + 1j * rng.standard_normal(x.shape[1])).astype(np.complex64)
    off = off_n * N
    r = T.Oracle(N, 2, 33, 1234, cfo_hz=650.0, ul=dict(cfo_ratio=rho, ul_offset=off)).push_ul(x, xu, 0)
    assert len(r["sf"]) >= 35
    n = np.arange(15 * N)
    for k, s in enumerate(r["sf"]):
        f = float(s["cfo_hz"]) * rho
        ref = xu[s["start"] + off:s["start"] + off + 15 * N].astype(complex) * np.exp(-2j * np.pi * f * n / (15000.0 * N))
        np.testing.assert_allclose(r["ul_iq"][k], ref, rtol=0, atol=1e-5 * np.abs(ref).max())


@pytest.mark.parametrize("off", [0, -200, 200, 1500])
@pytest.mark.parametrize("sizes_i", range(5))
def test_ul_chunking_invariance(off, sizes_i):
    """any split of the recording gives the same records and both cuts, including pieces that end between a DL window and its UL window"""
    from test_track import chunk_cases
    N = 256
    x = _dl_capture(N, 60, -20.0)
    xu = np.ascontiguousarray(x[1][::-1])
    ref = T.Oracle(N, 2, 33, 1234, cfo_hz=650.0, ul=dict(cfo_ratio=0.948, ul_offset=off)).push_ul(x, xu, 0)
    sizes = chunk_cases(N)[sizes_i] + ([15 * N + off // 2 + 1] if off else [])
    got = T.run_chunks(T.Oracle(N, 2, 33, 1234, cfo_hz=650.0, ul=dict(cfo_ratio=0.948, ul_offset=off)), x, sizes, xu=xu)
    assert got["sf"].tobytes() == ref["sf"].tobytes() and got["hf"].tobytes() == ref["hf"].tobytes()
    assert got["iq"].tobytes() == ref["iq"].tobytes() and got["ul_iq"].tobytes() == ref["ul_iq"].tobytes()


def test_tracked_ul_cut_decodes_what_the_aligned_uplink_does():
    """25 PRB, 500 ms, 20 ppm, 800 Hz DL carrier offset, rho = 0.948, the uplink 300 samples after the downlink: the tracked, rotated UL cut
    decodes every UL transport block that the oracle reads from the simulator's aligned, offset-free UL subframes.  The fixed cut at
    frame_offset + k 15 N (rotated by the constant offset) and the tracked cut without the UL rotation each lose blocks."""
    N, nsf, lead, off, rho, cfo = 384, 500, 1000, 300, 0.948, 800.0
    SF = 15 * N
    cap = T.TwoCarrier(N, 77, nsf, ppm=20.0, cfo=cfo, rho=rho, lead=lead, ul_offset=off, seed=11, mcs_max=20)
    r = T.Oracle(N, 1, 77, lead, cfo_hz=cfo - 30.0, ul=dict(cfo_ratio=rho, ul_offset=off)).push_ul(cap.x, cap.xu, 0)
    k = r["sf"]["index"]
    assert len(k) >= nsf - 3 and np.array_equal(k, np.arange(len(k)))
    ideal = T.decode_ul(cap, lambda q: cap.ul[q], k)
    assert len(ideal) >= 0.95 * len([q for q in cap.sent if q[0] in set(k.tolist())]) and len(ideal) > 300
    qm = {(q, int(g.rnti), int(g.n_prb)): int(g.qm) for q in k for g in cap.grants[q]}
    assert any(qm[t] >= 4 for t in ideal)
    tracked = T.decode_ul(cap, lambda q: r["ul_iq"][q], k)
    assert ideal <= tracked, sorted(ideal - tracked)[:10]
    n = np.arange(SF)
    fixed = T.decode_ul(cap, lambda q: cap.xu[lead + off + q * SF:lead + off + (q + 1) * SF] * np.exp(-2j * np.pi * rho * cfo * n / (15000.0 * N)), k)
    assert len(ideal - fixed) >= 1, len(fixed)
    st = r["sf"]["start"]
    unrot = T.decode_ul(cap, lambda q: cap.xu[st[q] + off:st[q] + off + SF], k)
    assert len(ideal - unrot) >= 1, len(unrot)


def test_constant_ul_cfo_correction():
    """UL subframes rotated by a constant offset, 25 PRB, 28 16QAM grants: after lteo_cfo_correct every one passes.  Without it, 600 Hz loses some
    (8 of 28 measured: the slot-to-slot interpolation of the PUSCH estimate follows part of a 108 degree turn between the DMRS symbols) and
    1000 Hz loses every one."""
    N = 384
    cap = T.TwoCarrier(N, 9, 40, lead=500, seed=21, mcs_max=24)
    ks = [k for k in range(40) if any(g.qm >= 4 for g in cap.grants[k])]
    hi = {(k, int(g.rnti), int(g.n_prb)) for k in ks for g in cap.grants[k] if g.qm >= 4}
    assert len(hi) >= 20
    n = np.arange(15 * N)
    rot = lambda f: (lambda k: cap.ul[k] * np.exp(2j * np.pi * f * n / (15000.0 * N)))
    assert hi <= T.decode_ul(cap, lambda k: cap.ul[k], ks)
    for f in (600.0, 1000.0):
        assert hi <= T.decode_ul(cap, rot(f), ks, cfo_hz=f), f
    assert len(hi - T.decode_ul(cap, rot(600.0), ks)) >= 5
    assert not (hi & T.decode_ul(cap, rot(1000.0), ks))


def test_oracle_argument_checks():
    L = T.lib()
    t = T.Oracle(256, 1, 1, 1000)
    for ratio, off in [(0.0, 0), (-1.0, 0), (2.01, 0), (float("nan"), 0), (1.0, 15 * 256), (1.0, -15 * 256), (1.0, -1001)]:
        assert L.lteo_track_set_ul(t.t, ratio, off) == -2, (ratio, off)
    assert L.lteo_track_set_ul(t.t, 2.0, -1000) == 0
    assert L.lteo_track_set_ul(t.t, 1.0, 0) == -2                  # only once
    x = np.zeros((1, 5000), np.complex64)
    nsf, nhf, nxt = C.c_uint32(), C.c_uint32(), C.c_uint64()
    sf, hf = np.zeros(10, T.SF_DTYPE), np.zeros(10, T.HF_DTYPE)
    args = (0, 5000, 10, ltelib.ptr(sf), C.byref(nsf), ltelib.ptr(hf), C.byref(nhf), None)
    assert L.lteo_track_push(t.t, ltelib.ptr(x), *args, C.byref(nxt)) == -2        # DL-only push with the uplink set
    assert L.lteo_track_push_ul(t.t, ltelib.ptr(x), ltelib.ptr(x), *args, None, C.byref(nxt)) == 0 and (nsf.value, nxt.value) == (1, 4840 - 1000)
    t2 = T.Oracle(256, 1, 1, 1000)
    assert L.lteo_track_push_ul(t2.t, ltelib.ptr(x), ltelib.ptr(x), *args, None, C.byref(nxt)) == -2   # push_ul without set_ul
    t2.push(x, 0, cut=False)
    assert L.lteo_track_set_ul(t2.t, 1.0, 0) == -2                 # after a push


def test_capi_argument_checks(phylib):
    from ltesniffer_b200 import capi
    phylib.ltephy_track_set_ul.argtypes = [C.c_void_p, C.c_void_p]
    phylib.ltephy_track_push_ul.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]
    phylib.ltephy_submit_ul_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    phylib.ltephy_set_ul_cfo.argtypes = [C.c_void_p, C.c_float]
    u = capi.TrackUlCfg(cfo_ratio=1.0, ul_offset=0)
    assert phylib.ltephy_track_set_ul(None, C.byref(u)) == -2
    assert phylib.ltephy_track_push_ul(None, None, None, 0, 0, None, None) == -2
    assert phylib.ltephy_submit_ul_device(None, None, None, 0, None, 0) == -2
    assert phylib.ltephy_set_ul_cfo(None, 1.0) == -2


def test_example_builds_and_refuses_to_run_without_a_gpu(infra, tmp_path):
    from ltesniffer_b200 import capi
    capi.load_library()
    subprocess.run(["make", "-s", "-C", ROOT, "examples/decode_recording_ul"], check=True)
    assert os.path.exists(EXE)
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present: covered by the gpu test")
    except ImportError:
        pass
    iq = tmp_path / "x.cf32"
    iq.write_bytes(b"\0" * 8 * 512 * 15 * 40)
    r = subprocess.run([EXE, str(iq), str(iq), "512", str(tmp_path / "o.pcap")], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stderr, (r.returncode, r.stderr)
