"""Tracker on the GPU: ltephy_track_push against the oracle lteo_track_push, every half-frame record, subframe record and cut sample bit for
bit; the host and device entry points and chunking invariance on the device; the re-measure path; invalid inputs; and cell search -> tracker ->
decode of every truth transport block of a capture whose sampling clock is 20 ppm off."""
import ctypes as C

import numpy as np
import pytest

import ltelib
import sync_lib as S
import track_lib as T

pytestmark = pytest.mark.gpu

CASES = [  # N, nrx, nsf, capture kwargs
    (128, 1, 40, dict(ppm=20.0, cfo=300.0, snr=20.0)),
    (256, 2, 60, dict(ppm=-20.0, cfo=-2000.0, ramp=400.0, snr=8.0, chan_delay=3)),
    (384, 1, 40, dict(ppm=2.0, cfo=4000.0, snr=0.0)),
    (512, 2, 80, dict(ppm=20.0, cfo=1200.0, ramp=200.0, snr=15.0, chan_delay=5)),
    (1536, 1, 25, dict(ppm=-50.0, cfo=-700.0, snr=25.0)),
    (2048, 2, 30, dict(ppm=20.0, cfo=2500.0, snr=20.0)),
]


def _same(a, b):
    assert a["sf"].tobytes() == b["sf"].tobytes(), (a["sf"][:4], b["sf"][:4])
    assert a["hf"].tobytes() == b["hf"].tobytes(), (a["hf"][:4], b["hf"][:4])
    ia = a["iq"] if isinstance(a["iq"], np.ndarray) else a["iq"].cpu().numpy()
    ib = b["iq"] if isinstance(b["iq"], np.ndarray) else b["iq"].cpu().numpy()
    assert ia.shape == ib.shape and ia.tobytes() == ib.tobytes()


@pytest.mark.parametrize("case", range(len(CASES)))
def test_bit_exact_with_the_oracle(phylib, case):
    from ltesniffer_b200 import capi
    N, nrx, nsf, kw = CASES[case]
    x, _, _ = T.capture(N, 301, nsf, nrx=nrx, lead=3 * N + 11, seed=case, t0=2, **kw)
    ref = T.Oracle(N, nrx, 301, 3 * N + 11, cfo_hz=kw["cfo"] * 0.9, first_tti=2).push(x, 0)
    tr = capi.Tracker(N, nrx, 301, 3 * N + 11, cfo_hz=kw["cfo"] * 0.9, first_tti=2)
    got = tr.push(x, 0)
    assert len(ref["sf"]) >= nsf - 2
    _same(ref, got)
    tr.close()


@pytest.mark.parametrize("sizes_i", range(5))
def test_chunking_host_and_device(phylib, sizes_i):
    """one chunk, one-subframe chunks, odd sizes and boundaries inside a PSS window, through both entry points, give the oracle's bytes"""
    import torch
    from ltesniffer_b200 import capi
    from test_track import chunk_cases
    N = 256
    x, _, _ = T.capture(N, 33, 120, nrx=2, ppm=-20.0, cfo=700.0, ramp=500.0, snr=12.0, lead=1234, seed=6)
    ref = T.Oracle(N, 2, 33, 1234, cfo_hz=650.0).push(x, 0)
    sizes = chunk_cases(N)[sizes_i]
    tr = capi.Tracker(N, 2, 33, 1234, cfo_hz=650.0, max_subframes=200)
    _same(ref, T.run_chunks(tr, x, sizes))
    tr.close()
    tr = capi.Tracker(N, 2, 33, 1234, cfo_hz=650.0, max_subframes=200)
    _same(ref, T.run_chunks(tr, x, sizes, push=lambda xx, s: tr.push_device(torch.from_numpy(np.ascontiguousarray(xx)).cuda(), s)))
    tr.close()


def test_max_subframes_splits_a_push(phylib):
    from ltesniffer_b200 import capi
    N = 128
    x, _, _ = T.capture(N, 5, 60, nrx=1, ppm=20.0, snr=20.0, lead=50, seed=2)
    ref = T.Oracle(N, 1, 5, 50).push(x, 0)
    tr = capi.Tracker(N, 1, 5, 50, max_subframes=7)
    _same(ref, T.run_chunks(tr, x, [10 ** 9]))
    tr.close()


def test_offset_beyond_max_ppm_is_measured_again(phylib):
    """a clock 200 ppm off with windows sized for 1 ppm: the tracked PSS leaves the predicted windows, those half-frames are measured again,
    and every record still equals the oracle's"""
    from ltesniffer_b200 import capi
    N = 512
    x, _, _ = T.capture(N, 8, 200, nrx=1, ppm=200.0, snr=20.0, lead=99, seed=9)
    ref = T.Oracle(N, 1, 8, 99).push(x, 0)
    tr = capi.Tracker(N, 1, 8, 99, max_ppm=1.0, max_subframes=500)
    got = tr.push(x, 0)
    assert got["remeasured"] > 0
    _same(ref, got)
    tr.close()


def test_invalid_inputs(phylib):
    from ltesniffer_b200 import capi
    tr = capi.Tracker(256, 1, 1, 1000)
    o = capi.TrackOut()
    x = np.zeros((1, 5000), np.complex64)
    assert tr.L.ltephy_track_push(tr.h, capi._p(x), 1001, 5000, C.byref(o)) == -2     # starts after the next sample needed
    assert tr.L.ltephy_track_push(tr.h, None, 0, 5000, C.byref(o)) == -2
    assert tr.L.ltephy_track_push(tr.h, capi._p(x), 0, 5000, None) == -2
    assert tr.L.ltephy_track_push(tr.h, capi._p(x), 0, 4000, C.byref(o)) == 0 and o.nof_subframes == 0 and o.next_sample == 1000
    tr.close()


def test_search_track_decode_at_20ppm(phylib, infra):
    """cell search on the first 40 ms, tracker over 500 ms with the sampling clock 20 ppm off, then the decoder on the tracked cut from device
    memory: every truth transport block decodes with the right bytes.  The fixed cut of the same capture loses blocks at the end."""
    import torch
    from ltesniffer_b200 import capi
    from helpers import to_phy_grant, truth_grants
    N, pci, nsf, lead = 512, 262, 500, 4321
    cell = ltelib.Cell(25, 2, pci, 2, N)
    s = S.sim(sync=1, cell=cell, seed=71, pbch=1, snr_db=25.0, nof_ues=6, dl_min=2, dl_max=4, tm=13, mcs_min=2, mcs_max=16)
    sub = [s.subframe(t) for t in range(nsf)]
    tx = np.concatenate([np.zeros((2, lead))] + [q[0] for q in sub], axis=1)
    L = tx.shape[1] - 2 * T.TAPS
    n = np.arange(L)
    x = (T.resample(tx, 20.0, L) * np.exp(2j * np.pi * 1700.0 * n / (15000 * N))).astype(np.complex64)
    cs = capi.CellSearch(N, 2, 40 * 15 * N)
    c = cs.search(x[:, :40 * 15 * N])[0]
    cs.close()
    assert c.detected and c.pci == pci
    fo, sfl = int(c.frame_offset), 15 * N
    tr = capi.Tracker(N, 2, c.pci, fo, cfo_hz=c.cfo_hz, first_tti=0, max_subframes=nsf)
    r = tr.push_device(torch.from_numpy(x).cuda(), 0)
    tr.close()
    m = len(r["sf"])
    assert m >= nsf - 4 and not (r["sf"]["flags"] & capi.TRACK_LOST).any()
    tti = r["sf"]["tti"].astype(np.uint32)
    k0 = int(r["sf"]["index"][0])

    def decode(iq_dev):
        phy = capi.LtePhy(25, 2, pci, 2, max_subframes=m, symbol_sz=N)
        phy._chk(phy.L.ltephy_submit_iq_device(phy.h, C.c_void_p(iq_dev.data_ptr()), capi._p(tti), m), "submit_iq_device")
        phy.n = m                                   # what LtePhy.submit_iq records: get_phase_a sizes its result arrays by it
        info, _ = phy.get_phase_a(want_cands=False)
        truths = [sub[k0 + i][1] for i in range(m)]
        tg = truth_grants(cell, truths, tti)
        # a subframe whose CFI decodes wrong loses its transport blocks: its truth grants do not fit the control region found
        bad = sum(g.tb[t].enabled for sf, d, g in tg for t in range(2) if info[sf].cfi != truths[sf].cfi)
        tg = [(sf, d, g) for sf, d, g in tg if info[sf].cfi == truths[sf].cfi]
        phy.submit_grants([to_phy_grant(sf, d.rnti, g) for sf, d, g in tg])
        res, pl = phy.get_phase_b()
        ok = 0
        for gi, (sf, d, g) in enumerate(tg):
            payload = sub[k0 + sf][2]
            for t in range(2):
                if g.tb[t].enabled:
                    rr, nb = res[2 * gi + t], g.tb[t].tbs // 8
                    good = rr.crc == 1 and bytes(pl[rr.payload_off:rr.payload_off + nb]) == bytes(payload[d.payload_off[t]:d.payload_off[t] + nb])
                    ok, bad = ok + good, bad + (not good)
        phy.close()
        return ok, bad

    ok, bad = decode(r["iq"])
    assert ok > 100 and bad == 0, (ok, bad)
    # the fixed cut of the same capture, with the constant carrier-offset correction of ltephy_set_cfo done here in float64
    fixed = np.stack([x[:, fo + i * sfl:fo + (i + 1) * sfl] for i in range(m)])
    nn = np.arange(sfl)
    fixed = (fixed * np.exp(-2j * np.pi * c.cfo_hz * nn / (15000 * N))).astype(np.complex64)
    ok2, bad2 = decode(torch.from_numpy(fixed).cuda())
    assert bad2 > 0, (ok2, bad2)
