"""The tracker's find state on the GPU (LTEPHY_TRACK_REACQUIRE): ltephy_track_push against the oracle lteo_track_push on captures whose
receiver dropped samples and on a zero-filled fade -- every record, cut sample, find count and next_sample bit for bit, through the host and
device entry points in one chunk and in odd chunkings, without measuring a window again; the uplink; and cell search -> tracker -> decoder
across a drop."""
import ctypes as C

import numpy as np
import pytest

import ltelib
import sync_lib as S
import track_lib as T
import track_reacq_lib as Q
from test_track_reacquire import PCI, T0, drop_capture

pytestmark = pytest.mark.gpu

CASES = [  # N, nrx, snr, drop
    (128, 2, 10.0, "37SF+1234"), (256, 1, 15.0, "3N+17"), (384, 2, 20.0, "37SF+1234"),
    (512, 1, 25.0, "37SF+1234"), (1536, 2, 12.0, "3N+17"), (2048, 1, 20.0, "3N+17"),
]


def _same(a, b):
    assert a["sf"].tobytes() == b["sf"].tobytes(), (a["sf"][:4], b["sf"][:4])
    assert a["hf"].tobytes() == b["hf"].tobytes(), (a["hf"][:4], b["hf"][:4])
    ia = a["iq"] if isinstance(a["iq"], np.ndarray) else a["iq"].cpu().numpy()
    ib = b["iq"] if isinstance(b["iq"], np.ndarray) else b["iq"].cpu().numpy()
    assert ia.shape == ib.shape and ia.tobytes() == ib.tobytes()
    assert a["finds"] == b["finds"] and a["next_sample"] == b["next_sample"], (a["finds"], b["finds"], a["next_sample"], b["next_sample"])


@pytest.mark.parametrize("case", range(len(CASES)))
def test_drop_bit_exact_with_the_oracle(phylib, case):
    import torch
    from ltesniffer_b200 import capi
    N, nrx, snr, drop = CASES[case]
    SF, FR = 15 * N, 150 * N
    x, _, _, _, lead = drop_capture(N, nrx, snr, drop)
    mk_o = lambda: T.Oracle(N, nrx, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE)
    mk_g = lambda: capi.Tracker(N, nrx, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=capi.TRACK_REACQUIRE, max_subframes=300)
    ref = mk_o().push(x, 0, max_sf=300)
    assert ref["finds"] == 1 and ((ref["sf"]["flags"] & capi.TRACK_REACQUIRED) != 0).sum() == 1
    tr = mk_g()
    got = tr.push(x, 0)
    assert got["remeasured"] == 0
    _same(ref, got)
    tr.close()
    for sizes in [[FR + N], [SF - 1, FR + N + 1], [7919, 3 * SF + 17, 104729]]:
        o = T.run_chunks(mk_o(), x, sizes)
        tr = mk_g()
        g = T.run_chunks(tr, x, sizes, push=lambda xx, s: tr.push_device(torch.from_numpy(np.ascontiguousarray(xx)).cuda(), s))
        _same(o, g)
        tr.close()


def test_fade_bit_exact_with_the_oracle(phylib):
    from ltesniffer_b200 import capi
    N = 256
    x, _, _ = T.capture(N, 100, 400, nrx=1, ppm=20.0, snr=20.0, lead=500, seed=4, gap=(150 * 15 * N, 100 * 15 * N))
    ref = T.Oracle(N, 1, 100, 500, flags=Q.REACQUIRE).push(x, 0, max_sf=500)
    tr = capi.Tracker(N, 1, 100, 500, flags=capi.TRACK_REACQUIRE, max_subframes=500)
    got = tr.push(x, 0)
    assert ref["finds"] >= 1
    _same(ref, got)
    tr.close()
    tr = capi.Tracker(N, 1, 100, 500, flags=capi.TRACK_REACQUIRE | capi.TRACK_NO_CFO, max_subframes=37)
    _same(T.run_chunks(T.Oracle(N, 1, 100, 500, flags=Q.REACQUIRE | T.NO_CFO), x, [15 * N * 7 + 3]), T.run_chunks(tr, x, [15 * N * 7 + 3]))
    tr.close()


@pytest.mark.parametrize("N", [128, 384, 512, 1536, 2048])
def test_short_fade_bit_exact_with_the_oracle(phylib, N):
    """60 ms of zeros 40 ms in, at the other five symbol sizes, 2 antennas: host push in one chunk and device pushes in odd chunks"""
    import torch
    from ltesniffer_b200 import capi
    SF = 15 * N
    x, _, _ = T.capture(N, 100, 160, nrx=2, ppm=20.0, snr=20.0, lead=500, seed=N, gap=(40 * SF, 60 * SF))
    ref = T.Oracle(N, 2, 100, 500, flags=Q.REACQUIRE).push(x, 0, max_sf=300)
    assert ref["finds"] >= 1 and ((ref["sf"]["flags"] & capi.TRACK_REACQUIRED) != 0).sum() == 1
    tr = capi.Tracker(N, 2, 100, 500, flags=capi.TRACK_REACQUIRE, max_subframes=300)
    _same(ref, tr.push(x, 0))
    tr.close()
    sizes = [150 * N + 7, 3 * SF + 17]
    tr = capi.Tracker(N, 2, 100, 500, flags=capi.TRACK_REACQUIRE, max_subframes=300)
    g = T.run_chunks(tr, x, sizes, push=lambda xx, s: tr.push_device(torch.from_numpy(np.ascontiguousarray(xx)).cuda(), s))
    _same(T.run_chunks(T.Oracle(N, 2, 100, 500, flags=Q.REACQUIRE), x, sizes), g)
    tr.close()


def test_uplink_equals_the_oracle(phylib):
    from ltesniffer_b200 import capi
    N, off, rho = 384, -(3 * 384 + 5), 0.95
    x, _, _, _, lead = drop_capture(N, 1, 20.0, "37SF+1234")
    xu = Q.noise(np.random.default_rng(5), 1, x.shape[1], 1.0)[0]
    o = T.Oracle(N, 1, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE, ul=dict(cfo_ratio=rho, ul_offset=off))
    ref = o.push_ul(x, xu, 0, max_sf=300)
    tr = capi.Tracker(N, 1, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=capi.TRACK_REACQUIRE, max_subframes=300, ul=dict(cfo_ratio=rho, ul_offset=off))
    got = tr.push_ul(x, xu, 0)
    assert ref["finds"] == 1
    _same(ref, got)
    assert got["ul_iq"].cpu().numpy().tobytes() == ref["ul_iq"].tobytes()
    tr.close()
    sizes = [15 * N * 150 + N + 1, 7919]
    o = T.Oracle(N, 1, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE, ul=dict(cfo_ratio=rho, ul_offset=off))
    tr = capi.Tracker(N, 1, PCI, lead, cfo_hz=900.0, first_tti=T0, flags=capi.TRACK_REACQUIRE, max_subframes=300, ul=dict(cfo_ratio=rho, ul_offset=off))
    a = T.run_chunks(o, x, sizes, xu=xu)
    b = T.run_chunks(tr, x, sizes, xu=xu)
    assert a["sf"].tobytes() == b["sf"].tobytes() and a["ul_iq"].tobytes() == b["ul_iq"].tobytes()
    tr.close()


def test_search_track_decode_across_a_drop(phylib, infra):
    """25 PRB, 2 x 2, 20 ppm, 37 SF + 1234 samples dropped 60 ms in: with the flag every truth transport block of every subframe cut after the
    re-acquisition decodes with the right bytes (the subframe numbers, and so the scrambling, are right); without it none does"""
    import torch
    from ltesniffer_b200 import capi
    from helpers import to_phy_grant, truth_grants
    N, pci, nsf, lead = 512, 262, 200, 4321
    SF = 15 * N
    cell = ltelib.Cell(25, 2, pci, 2, N)
    s = S.sim(sync=1, cell=cell, seed=71, pbch=1, snr_db=25.0, nof_ues=6, dl_min=2, dl_max=4, tm=13, mcs_min=2, mcs_max=16)
    sub = [s.subframe(t) for t in range(nsf)]
    tx = np.concatenate([np.zeros((2, lead))] + [q[0] for q in sub], axis=1)
    L = tx.shape[1] - 2 * T.TAPS
    n = np.arange(L)
    x = (T.resample(tx, 20.0, L) * np.exp(2j * np.pi * 1700.0 * n / (15000 * N))).astype(np.complex64)
    a, cnt = lead + 60 * SF + 777, 37 * SF + 1234
    x = np.ascontiguousarray(np.delete(x, np.s_[a:a + cnt], axis=1))
    truth = (lead + np.arange(nsf) * SF) / (1.0 + 20e-6)
    truth = np.where(truth >= a + cnt, truth - cnt, truth)
    cs = capi.CellSearch(N, 2, 40 * SF)
    c = cs.search(x[:, :40 * SF])[0]
    cs.close()
    assert c.detected and c.pci == pci

    def track(flags):
        tr = capi.Tracker(N, 2, c.pci, int(c.frame_offset), cfo_hz=c.cfo_hz, first_tti=0, max_subframes=nsf, flags=flags)
        r = tr.push_device(torch.from_numpy(x).cuda(), 0)
        tr.close()
        return r

    def decode(r, sel):
        """the truth blocks of the cut subframes sel, each matched to the transmit subframe whose start is nearest; (ok, bad)"""
        m = len(sel)
        iq = r["iq"][torch.as_tensor(sel, device=r["iq"].device)].contiguous()
        tti = r["sf"]["tti"][sel].astype(np.uint32)
        kt = [int(np.argmin(np.abs(truth - r["sf"]["start"][i]))) for i in sel]
        phy = capi.LtePhy(25, 2, pci, 2, max_subframes=m, symbol_sz=N)
        phy._chk(phy.L.ltephy_submit_iq_device(phy.h, C.c_void_p(iq.data_ptr()), capi._p(tti), m), "submit_iq_device")
        phy.n = m
        info, _ = phy.get_phase_a(want_cands=False)
        truths = [sub[k][1] for k in kt]
        tg = truth_grants(cell, truths, tti)
        bad = sum(g.tb[t].enabled for sf, d, g in tg for t in range(2) if info[sf].cfi != truths[sf].cfi)
        tg = [(sf, d, g) for sf, d, g in tg if info[sf].cfi == truths[sf].cfi]
        ok = 0
        if tg:
            phy.submit_grants([to_phy_grant(sf, d.rnti, g) for sf, d, g in tg])
            res, pl = phy.get_phase_b()
            for gi, (sf, d, g) in enumerate(tg):
                payload = sub[kt[sf]][2]
                for t in range(2):
                    if g.tb[t].enabled:
                        rr, nb = res[2 * gi + t], g.tb[t].tbs // 8
                        good = rr.crc == 1 and bytes(pl[rr.payload_off:rr.payload_off + nb]) == bytes(payload[d.payload_off[t]:d.payload_off[t] + nb])
                        ok, bad = ok + good, bad + (not good)
        phy.close()
        return ok, bad

    r = track(capi.TRACK_REACQUIRE)
    i = int(np.flatnonzero(r["sf"]["flags"] & capi.TRACK_REACQUIRED)[0])
    assert r["finds"] == 1 and r["remeasured"] == 0
    sel = np.arange(i, len(r["sf"]))
    assert len(sel) >= 60
    ok, bad = decode(r, sel)
    assert ok > 50 and bad == 0, (ok, bad)
    r0 = track(0)
    sel0 = np.flatnonzero(r0["sf"]["start"] >= a + 2 * SF)
    assert len(sel0) >= 60
    ok0, bad0 = decode(r0, sel0)
    assert ok0 == 0 and bad0 > 0, (ok0, bad0)
