"""Integer samples on every narrowband input (pytest -m gpu; DESIGN.md §2 "integer samples"): a run on sc16 / sc8 samples equals the cf32 run on
the converted samples q * 2^-15 / q * 2^-7 bit for bit -- the decoder (phase A, the combined MIB, phase B, host and device submits), the uplink, the
cell search with its intermediates, the tracker's records and cuts (DL and UL, split into pushes anywhere, with a re-acquisition), and the
examples' pcap and DCI trace.  The integer data is the simulator's captures quantised in numpy; each device entry point refuses a pointer that is
not aligned to its sample."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ltelib
import sync_lib as S
import track_lib as T
from helpers import make_capture
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BITS = {"sc16": 15, "sc8": 7}
PEAK = 0.5  # the largest I or Q component of a capture lands at half of full scale


def quantise(x, fmt):
    """complex samples [...] -> (q: int16 / int8 [...][2], the cf32 reference q * 2^-bits, complex64 [...])"""
    b = BITS[fmt]
    v = np.ascontiguousarray(x, np.complex64).view(np.float32).reshape(np.shape(x) + (2,))
    s = PEAK * 2.0 ** b / float(np.abs(v).max())
    q = np.clip(np.rint(v.astype(np.float64) * s), -2 ** b, 2 ** b - 1).astype(np.int16 if fmt == "sc16" else np.int8)
    ref = np.ascontiguousarray(q.astype(np.float32) * np.float32(2.0 ** -b)).view(np.complex64)[..., 0]
    return q, ref


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    return t if isinstance(t, np.ndarray) else t.cpu().numpy()


# ------------------------------------------------------------------------------------------------ the decoder
DEC_CASES = [  # nof_prb, nof_rx, symbol_sz (0: the standard 2^k), cfo_hz
    (25, 1, 0, 0.0), (25, 2, 384, 350.0), (100, 2, 0, -420.0), (100, 1, 1536, 0.0),
]


def _decode(prb, nrx, sz, cfo, pci, x, tti, fmt):
    """phase A (full table and survivor form), the combined MIB, phase A again from device memory, phase B through ltephy_decode_subframes"""
    n = len(tti)
    phy = capi.LtePhy(prb, 2, pci, nrx, max_subframes=n, symbol_sz=sz, iq_format=fmt)
    if cfo:
        phy.set_cfo(cfo)
    phy.submit_iq(x, tti)
    info_c, comp = phy.get_phase_a_compact()
    info, cands = phy.get_phase_a()
    mib = phy.mib_decode_combined(search_ports=True)
    out = dict(info=bytes(info), info_c=bytes(info_c), comp=comp.tobytes(), cands=cands.tobytes(), mib=bytes(mib))
    phy.submit_iq_device(_dev(x), tti)
    info_d, cands_d = phy.get_phase_a()
    out.update(info_dev=bytes(info_d), cands_dev=cands_d.tobytes())
    srch = capi.Search(prb, 2, pci, nrx)
    info_b, dcis, tbs, payload = capi.decode_subframes(phy, srch, x, tti)
    nd = len(dcis)
    out.update(info_b=bytes(info_b), dcis=dcis.tobytes(), tbs=bytes(tbs)[:2 * nd * C.sizeof(capi.TbResult)], payload=payload.tobytes())
    out["ok"] = sum(tbs[i].crc != 0 for i in range(2 * nd))
    out["found"] = sum(m.mib.found for m in mib)
    srch.close(), phy.close()
    return out


@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
@pytest.mark.parametrize("case", range(len(DEC_CASES)))
def test_decoder_equals_cf32_of_the_converted_samples(infra, phylib, case, fmt):
    prb, nrx, sz, cfo = DEC_CASES[case]
    pci = 60 + prb + nrx
    cell = ltelib.Cell(prb, 2, pci, nrx, sz)
    _, iq, tti, _, _ = make_capture(cell, 10, seed=11 + case, pbch=1, cfo_hz=cfo, snr_db=26.0, nof_ues=5, dl_min=2, dl_max=3, tm=13, mcs_min=2,
                                    mcs_max=20)
    q, ref = quantise(iq, fmt)
    got, want = _decode(prb, nrx, sz, cfo, pci, q, tti, fmt), _decode(prb, nrx, sz, cfo, pci, ref, tti, "cf32")
    for k in want:
        assert got[k] == want[k], (k, fmt, DEC_CASES[case])
    assert want["info"] == want["info_dev"] and want["found"] >= 1
    if fmt == "sc16":
        assert want["ok"] > 0


# ------------------------------------------------------------------------------------------------ the uplink
def _ul(iq, tti, grants, A, cfo, fmt, prb, pci):
    phy = capi.LtePhy(prb, 1, pci, 1, max_subframes=len(tti), ul_nof_rx=A, iq_format=fmt)
    phy.set_ul_cfg(3, 2)
    if cfo:
        phy.set_ul_cfo(cfo)
    out = []
    for dev in (False, True):
        res, ch, pl = phy.decode_ul_device(_dev(iq), tti, grants) if dev else phy.decode_ul(iq, tti, grants)
        out.append((bytes(res), bytes(ch), pl.tobytes(), sum(r.crc != 0 for r in res)))
    phy.close()
    return out


@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
@pytest.mark.parametrize("A,cfo", [(1, 0.0), (2, 0.0), (1, 530.0), (2, -610.0)])
def test_uplink_equals_cf32_of_the_converted_samples(infra, phylib, A, cfo, fmt):
    from test_gpu_pusch_rx_diversity import _batch
    cell = ltelib.Cell(50, 1, 150 + A, 1, 0)
    iq, tti, _, grants = _batch(cell, ltelib.UlCfg(n_dmrs1=3, delta_ss=2), 3, 4)
    iq = np.ascontiguousarray(iq[:, 0] if A == 1 else iq)   # one UL antenna: [n][sf_len], as the binding takes it
    if cfo:  # the offset ltephy_set_ul_cfo removes
        n = np.arange(iq.shape[-1])
        iq = (iq * np.exp(2j * np.pi * cfo * n / (15000.0 * 1024))).astype(np.complex64)
    q, ref = quantise(iq, fmt)
    got, want = _ul(q, tti, grants, A, cfo, fmt, 50, cell.cell_id), _ul(ref, tti, grants, A, cfo, "cf32", 50, cell.cell_id)
    assert got == want
    assert want[0] == want[1]
    if fmt == "sc16":
        assert want[0][3] >= len(grants) - 2


# ------------------------------------------------------------------------------------------------ the cell search
def _search(N, nrx, x, fmt, dev):
    cs = capi.CellSearch(N, nrx, x.shape[1], iq_format=fmt)
    res = cs.search_device(_dev(x)) if dev else cs.search(x)
    out = [bytes(c) for c in res] + [cs.tap(w).tobytes() for w in (capi.SYNC_TAP_COARSE, capi.SYNC_TAP_REFINED, capi.SYNC_TAP_CFO, capi.SYNC_TAP_SSS)]
    cs.close()
    return out, res


@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
@pytest.mark.parametrize("N,nrx", [(128, 1), (128, 2), (1536, 1), (1536, 2), (2048, 1), (2048, 2)])
def test_cell_search_equals_cf32_of_the_converted_samples(infra, phylib, N, nrx, fmt):
    pci = 211 + N % 7
    x = T.capture(N, pci, 12, nrx=nrx, cfo=1300.0, snr=15.0, lead=3 * N + 5, seed=N + nrx)[0]
    q, ref = quantise(x, fmt)
    want, res = _search(N, nrx, ref, "cf32", False)
    for dev in (False, True):
        assert _search(N, nrx, q, fmt, dev)[0] == want, (N, nrx, fmt, dev)
    if fmt == "sc16":
        assert res[0].detected and res[0].pci == pci


# ------------------------------------------------------------------------------------------------ the tracker
def _same(a, b, keys):
    for k in keys:
        assert _host(a[k]).tobytes() == _host(b[k]).tobytes(), k


@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
@pytest.mark.parametrize("N,nrx", [(512, 1), (384, 2)])
def test_tracker_equals_cf32_of_the_converted_samples(infra, phylib, N, nrx, fmt):
    from test_track import chunk_cases
    x = T.capture(N, 33, 40, nrx=nrx, ppm=20.0, cfo=700.0, ramp=500.0, snr=12.0, lead=1234, seed=4)[0]
    q, ref = quantise(x, fmt)
    mk = lambda f: capi.Tracker(N, nrx, 33, 1234, cfo_hz=650.0, max_subframes=200, iq_format=f)
    want = T.run_chunks(mk("cf32"), ref, [ref.shape[1]])
    assert len(want["sf"]) >= 35
    for sizes in [[x.shape[1]]] + chunk_cases(N)[:3]:
        for dev in (False, True):
            tr = mk(fmt)
            push = (lambda a, f: tr.push_device(_dev(a), f)) if dev else tr.push
            got = T.run_chunks(tr, q, sizes, push=push)
            _same(got, want, ("sf", "hf", "iq"))
            tr.close()


@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
@pytest.mark.parametrize("A", [1, 2])
def test_tracker_uplink_equals_cf32_of_the_converted_samples(infra, phylib, A, fmt):
    N = 512
    x = T.capture(N, 33, 40, nrx=1, ppm=20.0, cfo=700.0, snr=12.0, lead=1234, seed=5)[0]
    rng = np.random.default_rng(A)
    xu = (rng.standard_normal((A, x.shape[1])) + 1j * rng.standard_normal((A, x.shape[1]))).astype(np.complex64)
    q, ref = quantise(x, fmt)
    qu, refu = quantise(xu, fmt)
    mk = lambda f: capi.Tracker(N, 1, 33, 1234, cfo_hz=650.0, max_subframes=200, ul=dict(cfo_ratio=0.948, ul_offset=-200, nof_rx=A), iq_format=f)
    want = T.run_chunks(mk("cf32"), ref, [ref.shape[1]], xu=refu)
    assert len(want["sf"]) >= 35
    for sizes in ([x.shape[1]], [7919, 3 * 15 * N + 17]):
        for dev in (False, True):
            tr = mk(fmt)
            push = (lambda a, b, f: tr.push_ul_device(_dev(a), _dev(b), f)) if dev else tr.push_ul
            got = T.run_chunks(tr, q, sizes, xu=qu, push=push)
            _same(got, want, ("sf", "hf", "iq", "ul_iq"))
            tr.close()


@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
def test_tracker_reacquire_equals_cf32_of_the_converted_samples(infra, phylib, fmt):
    from test_track_reacquire import PCI, T0, drop_capture
    N, nrx = 384, 2
    SF, FR = 15 * N, 150 * N
    x, _, _, _, lead = drop_capture(N, nrx, 20.0, "37SF+1234")
    q, ref = quantise(x, fmt)
    mk = lambda f: capi.Tracker(N, nrx, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=capi.TRACK_REACQUIRE, max_subframes=300, iq_format=f)
    want = T.run_chunks(mk("cf32"), ref, [ref.shape[1]])
    assert want["finds"] >= 1 and ((want["sf"]["flags"] & capi.TRACK_REACQUIRED) != 0).sum() == 1
    for sizes in [[x.shape[1]], [SF - 1, FR + N + 1], [7919, 3 * SF + 17, 104729]]:
        for dev in (False, True):
            tr = mk(fmt)
            push = (lambda a, f: tr.push_device(_dev(a), f)) if dev else tr.push
            got = T.run_chunks(tr, q, sizes, push=push)
            _same(got, want, ("sf", "hf", "iq"))
            assert got["finds"] == want["finds"] and got["next_sample"] == want["next_sample"]
            tr.close()


# ------------------------------------------------------------------------------------------------ misaligned device pointers
@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
def test_device_entry_points_refuse_misaligned_samples(infra, phylib, fmt):
    import torch
    L = phylib
    buf = torch.zeros(8 * 2 * 15 * 2048 * 2 + 64, dtype=torch.uint8, device="cuda")
    bad = C.c_void_p(buf.data_ptr() + 1)
    tti = np.zeros(1, np.uint32)

    def refused(rc):
        assert rc == -2 and b"aligned" in L.ltephy_last_error(), (rc, L.ltephy_last_error())

    phy = capi.LtePhy(25, 1, 1, 1, max_subframes=1, iq_format=fmt)
    phy.set_ul_cfg()
    refused(L.ltephy_submit_iq_device(phy.h, bad, capi._p(tti), 1))
    L.ltephy_submit_ul_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    refused(L.ltephy_submit_ul_device(phy.h, bad, capi._p(tti), 1, None, 0))
    srch = capi.Search(25, 1, 1, 1)
    info, cands = (capi.SfInfo * 1)(), np.zeros((1, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
    dcis, tbs, pay, nd = np.zeros(32, capi.DCI_DTYPE), (capi.TbResult * 64)(), np.zeros(1 << 16, np.uint8), C.c_uint32(0)
    refused(L.ltephy_decode_subframes_device(phy.h, srch.h, bad, capi._p(tti), 1, capi.SEQ_NONE, info, capi._p(cands), capi._p(dcis), 32, C.byref(nd),
                                             tbs, capi._p(pay), pay.nbytes))
    srch.close(), phy.close()
    cs = capi.CellSearch(512, 1, 76 * 512, iq_format=fmt)
    refused(L.ltephy_cell_search_device(cs.h, bad, 76 * 512, (capi.CellInfo * 3)()))
    cs.close()
    tr = capi.Tracker(512, 1, 1, 0, max_subframes=10, iq_format=fmt)
    refused(L.ltephy_track_push_device(tr.h, bad, 0, 1000, C.byref(capi.TrackOut())))
    tr.close()
    good = C.c_void_p(buf.data_ptr())
    for a, b in ((bad, good), (good, bad)):
        tr = capi.Tracker(512, 1, 1, 0, max_subframes=10, ul=dict(nof_rx=1), iq_format=fmt)
        u = C.c_void_p()
        refused(L.ltephy_track_push_ul_device(tr.h, a, b, 0, 1000, C.byref(capi.TrackOut()), C.byref(u)))
        tr.close()


# ------------------------------------------------------------------------------------------------ the examples end to end
def _run(args):
    r = subprocess.run(args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stdout


def _tofile(a, path):
    np.ascontiguousarray(a).tofile(str(path))
    return str(path)


def test_decode_recording_sc16_file(infra, phylib, tmp_path):
    """decode_recording fmt=sc16 on a 25 PRB 2x2 recording (20 ppm, 1.7 kHz off) writes the pcap and the DCI trace of the same example on the cf32
    file of the converted samples, byte for byte, and the transport blocks of the example on the unquantised capture"""
    from test_decode_recording import EXE, _build
    _build()
    N, pci, nsf, lead, B = 512, 262, 600, 4321, 200
    cell = ltelib.Cell(25, 2, pci, 2, N)
    s = S.sim(sync=1, cell=cell, seed=71, pbch=1, snr_db=25.0, nof_ues=6, dl_min=2, dl_max=4, tm=13, mcs_min=2, mcs_max=16)
    tx = np.concatenate([np.zeros((2, lead))] + [s.subframe(t)[0] for t in range(nsf)], axis=1)
    L = tx.shape[1] - 2 * T.TAPS
    x = (T.resample(tx, 20.0, L) * np.exp(2j * np.pi * 1700.0 * np.arange(L) / (15000 * N))).astype(np.complex64)
    q, ref = quantise(x, "sc16")
    out = {}
    for name, arr, fmt in (("sc16", q, ["fmt=sc16"]), ("ref", ref, []), ("orig", x, ["fmt=cf32"])):
        f = _tofile(arr, tmp_path / ("%s.iq" % name))
        pc, tsv = str(tmp_path / ("%s.pcap" % name)), str(tmp_path / ("%s.tsv" % name))
        stdout = _run([EXE, f, str(N), "2", pc, tsv, str(B)] + fmt)
        out[name] = (stdout, open(pc, "rb").read(), open(tsv, "rb").read())
    assert out["sc16"] == out["ref"]
    from test_decode_recording import _read_pcap
    got = _read_pcap(str(tmp_path / "sc16.pcap"))
    assert len(got) > 300 and got == _read_pcap(str(tmp_path / "orig.pcap"))


def test_decode_recording_ul_sc16_files(infra, phylib, tmp_path):
    """decode_recording_ul fmt=sc16 with two UL antennas writes the pcap of the same example on the cf32 files of the converted samples, byte for
    byte, and the transport blocks of the example on the unquantised captures"""
    from test_gpu_track_ul import EXE, LEAD_E2E, N_E2E, OFF_E2E, PCI_E2E, RHO_E2E, _read_pcap
    subprocess.run(["make", "-s", "-C", ROOT, "examples/decode_recording_ul"], check=True)
    cap = T.TwoCarrier(N_E2E, PCI_E2E, 200, ppm=20.0, cfo=800.0, rho=RHO_E2E, lead=LEAD_E2E, ul_offset=OFF_E2E, seed=73, pbch=1, nof_ports=2,
                       mcs_max=20, ul_snr=12.0, ul_nof_rx=2)
    qd, rd = quantise(cap.x[0], "sc16")
    qu, ru = quantise(cap.xu, "sc16")
    out = {}
    for name, d, u, fmt in (("sc16", qd, qu, ["fmt=sc16"]), ("ref", rd, ru, []), ("orig", cap.x[0], cap.xu, [])):
        fd, fu = _tofile(d, tmp_path / ("%s_dl.iq" % name)), _tofile(u, tmp_path / ("%s_ul.iq" % name))
        pc = str(tmp_path / ("%s.pcap" % name))
        stdout = _run([EXE, fd, fu, str(N_E2E), pc, str(RHO_E2E), str(OFF_E2E), str(T.UCFG["n_dmrs1"]), str(T.UCFG["delta_ss"]), "0", "2"] + fmt)
        out[name] = (stdout, open(pc, "rb").read())
    assert out["sc16"] == out["ref"]
    got = _read_pcap(str(tmp_path / "sc16.pcap"))
    assert sum(1 for r in got if r[0] == 0) > 50 and got == _read_pcap(str(tmp_path / "orig.pcap"))
