"""Cell search on the GPU: ltephy_cell_search against the oracle's lteo_cell_search, every field of every result and every intermediate bit for
bit, over symbol sizes, antennas, CFO, noise, two cells and the edge cases of the timing rules; the host and device entry points; a long
capture over many CTAs; invalid inputs; and a decode from an unaligned, CFO-shifted recording, started from what the search found."""
import os
import subprocess
import numpy as np
import pytest

import ltelib
import sync_lib as S
from test_cell_search import sim_capture, truth_offset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _both(N, x):
    from ltesniffer_b200 import capi
    r, ref, taps = S.cell_search(N, x)
    assert r == 0
    cs = capi.CellSearch(N, x.shape[0], x.shape[1])
    got = cs.search(x)
    gtaps = {k: cs.tap(w) for k, w in (("coarse", capi.SYNC_TAP_COARSE), ("refined", capi.SYNC_TAP_REFINED), ("cfo", capi.SYNC_TAP_CFO),
                                        ("sss", capi.SYNC_TAP_SSS))}
    cs.close()
    return ref, taps, got, gtaps


def _same(ref, taps, got, gtaps):
    for k in taps:
        assert taps[k].tobytes() == gtaps[k].tobytes(), k
    for a, b in zip(ref, got):
        assert bytes(a) == bytes(b), ([(f, getattr(a, f)) for f, _ in a._fields_], [(f, getattr(b, f)) for f, _ in b._fields_])


CASES = [  # N, nrx, capture kwargs
    (128, 1, dict(pci=17, nsf=22, off=901, L=75 * 128 * 2 + 128)),
    (256, 2, dict(pci=300, nsf=32, off=5000, L=75 * 256 * 4, cfo=-3000.0)),
    (384, 1, dict(pci=11, nsf=22, off=77, L=75 * 384 * 2 + 384, snr=5.0)),
    (512, 2, dict(pci=402, nsf=32, off=12345, L=75 * 512 * 4, cfo=1200.0, snr=15.0, chan_delay=5, nof_ports=2)),
    (768, 1, dict(pci=250, nsf=22, off=3000, L=75 * 768 * 2 + 768, t0=5)),
    (1024, 2, dict(pci=503, nsf=22, off=999, L=75 * 1024 * 2 + 1024, cfo=4000.0)),
    (1536, 1, dict(pci=0, nsf=22, off=50000, L=75 * 1536 + 1536)),
    (2048, 2, dict(pci=333, nsf=22, off=2048 * 13 // 2, L=75 * 2048 + 2048 + 100, snr=20.0)),
    (256, 1, dict(pci=321, nsf=22, off=256 * 13 // 2 - 37, L=75 * 256 + 37 + 256)),      # PSS in the last window that fits
    (256, 1, dict(pci=321, nsf=22, off=256 * 13 // 2 - 128, L=2 * 75 * 256 + 256)),      # SSS before the start
]


@pytest.mark.parametrize("N,nrx,kw", CASES, ids=["%d-%d-%d" % (c[0], c[1], i) for i, c in enumerate(CASES)])
def test_bit_exact_with_oracle(phylib, infra, N, nrx, kw):
    kw = dict(kw)
    x = sim_capture(N, kw.pop("pci"), kw.pop("nsf"), kw.pop("off"), kw.pop("L"), nrx=nrx, seed=N + nrx, **kw)
    _same(*_both(N, x))


def test_bit_exact_two_cells_and_noise(phylib, infra):
    N = 512
    a = sim_capture(N, 120, 32, 2000, 75 * N * 4, seed=31)
    b = sim_capture(N, 272, 32, 9000, 75 * N * 4, seed=32) * np.float32(0.5)
    ref, taps, got, gtaps = _both(N, a + b)
    _same(ref, taps, got, gtaps)
    assert {o.pci for o in got} >= {120, 272}
    _same(*_both(512, np.zeros((2, 2 * 75 * 512 + 512), np.complex64)))   # all ties
    rng = np.random.default_rng(5)
    for N, A in ((256, 1), (1536, 2)):
        x = ((rng.standard_normal((A, 76 * N + 999)) + 1j * rng.standard_normal((A, 76 * N + 999))) / np.sqrt(2)).astype(np.complex64)
        ref, taps, got, gtaps = _both(N, x)
        _same(ref, taps, got, gtaps)
        assert not any(o.detected for o in got)


def test_all_504_pcis_at_256(phylib, infra):
    from ltesniffer_b200 import capi
    N = 256
    cs = capi.CellSearch(N, 1, 75 * N * 2 + N)
    rng = np.random.default_rng(3)
    for pci in range(504):
        off = int(rng.integers(0, 150 * N))
        x = sim_capture(N, pci, 22, off, 75 * N * 2 + N, seed=pci)
        c = cs.search(x)[0]
        assert c.detected and c.pci == pci and c.frame_offset == truth_offset(N, off), pci
        if pci % 50 == 0:
            assert bytes(S.cell_search(N, x)[1][0]) == bytes(c)
    cs.close()


def test_host_and_device_paths_agree(phylib, infra):
    import torch
    from ltesniffer_b200 import capi
    N = 1024
    x = sim_capture(N, 77, 22, 4321, 75 * N * 2 + N, nrx=2, cfo=800.0, seed=8)
    cs = capi.CellSearch(N, 2, x.shape[1])
    a = cs.search(x)
    ta = cs.tap(capi.SYNC_TAP_SSS)
    b = cs.search_device(torch.from_numpy(x).cuda())
    assert [bytes(o) for o in a] == [bytes(o) for o in b] and ta.tobytes() == cs.tap(capi.SYNC_TAP_SSS).tobytes()
    cs.close()


def test_long_capture_many_ctas(phylib, infra):
    """200 ms, 2 antennas, N = 512: 384 000 coarse offsets over 375 CTAs; the decisions equal the oracle's"""
    N = 512
    x = sim_capture(N, 188, 201, 7777, 200 * 15 * N, nrx=2, cfo=-2200.0, snr=10.0, seed=61)
    ref, taps, got, gtaps = _both(N, x)
    _same(ref, taps, got, gtaps)
    assert got[0].pci == 188 and got[0].detected and got[0].frame_offset == truth_offset(N, 7777) and got[0].nof_half_frames == 40


def test_invalid_inputs(phylib):
    import ctypes as C
    from ltesniffer_b200 import capi
    L = phylib
    h = C.c_void_p()
    for N, A, mx in ((192, 1, 10 ** 6), (4096, 1, 10 ** 6), (256, 3, 10 ** 6), (256, 0, 10 ** 6), (256, 1, 75 * 256)):
        cfg = capi.SyncCfg(symbol_sz=N, nof_rx=A, max_samples=mx)
        assert L.ltephy_sync_create(C.byref(cfg), C.byref(h)) == -2
    cs = capi.CellSearch(256, 1, 75 * 256 * 2)
    out = (capi.CellInfo * 3)()
    short = np.zeros(75 * 256 + 255, np.complex64)
    assert L.ltephy_cell_search(cs.h, short.ctypes.data_as(C.c_void_p), len(short), out) == -2
    big = np.zeros(75 * 256 * 2 + 1, np.complex64)
    assert L.ltephy_cell_search(cs.h, big.ctypes.data_as(C.c_void_p), len(big), out) == -2
    assert L.ltephy_cell_search(cs.h, None, 75 * 256 * 2, out) == -2
    cs.close()


def test_decode_from_an_unaligned_cfo_shifted_capture(phylib, infra):
    """search -> ltephy_set_cfo -> ltephy_mib_decode -> decode: the MIB the simulator broadcast, and every transport block of the
    simulator's truth decoded and equal at 25 dB"""
    from ltesniffer_b200 import capi
    from helpers import to_phy_grant, truth_grants
    N, off, cfo, pci = 512, 31337, 1700.0, 262
    cell = ltelib.Cell(25, 2, pci, 2, N)
    s = S.sim(sync=1, cell=cell, seed=71, pbch=1, snr_db=25.0, nof_ues=6, dl_min=2, dl_max=4, tm=13, mcs_min=2, mcs_max=16)
    nsf = 40
    sub = [s.subframe(t) for t in range(nsf)]
    full = np.concatenate([q[0] for q in sub], axis=1).astype(np.complex128)[:, off:]
    n = np.arange(off, off + full.shape[1])
    x = (full * np.exp(2j * np.pi * cfo * n / (15000 * N))).astype(np.complex64)
    cs = capi.CellSearch(N, 2, x.shape[1])
    c = cs.search(x)[0]
    cs.close()
    assert c.detected and c.pci == pci and c.frame_offset == truth_offset(N, off)
    fo, sfl = int(c.frame_offset), 15 * N
    k0 = (off + fo) // sfl                     # subframe index of the recording at frame_offset (a subframe 0)
    m = (x.shape[1] - fo) // sfl
    iq = np.stack([x[:, fo + i * sfl:fo + (i + 1) * sfl] for i in range(m)])
    tti = np.arange(k0, k0 + m, dtype=np.uint32)
    phy = capi.LtePhy(15, 2, c.pci, 2, max_subframes=m, symbol_sz=N)
    phy.set_cfo(c.cfo_hz)
    phy.submit_iq(iq, tti)
    mib = [mm for mm in phy.mib_decode() if mm.found]
    assert mib and mib[0].nof_prb == 25 and mib[0].nof_ports == 2 and mib[0].sfn == k0 // 10
    phy.close()
    phy = capi.LtePhy(mib[0].nof_prb, 2, c.pci, 2, max_subframes=m, symbol_sz=N, phich_resources=mib[0].phich_resources,
                      phich_length=mib[0].phich_length)
    phy.set_cfo(c.cfo_hz)
    phy.submit_iq(iq, tti)
    info, _ = phy.get_phase_a(want_cands=False)
    truths = [sub[int(t)][1] for t in tti]
    tg = truth_grants(cell, truths, tti)
    assert len(tg) > 20 and all(info[i].cfi == truths[i].cfi for i in range(m))
    phy.submit_grants([to_phy_grant(sf, d.rnti, g) for sf, d, g in tg])
    res, pl = phy.get_phase_b()
    for gi, (sf, d, g) in enumerate(tg):
        payload = sub[int(tti[sf])][2]
        for t in range(2):
            if g.tb[t].enabled:
                rr, nb = res[2 * gi + t], g.tb[t].tbs // 8
                assert rr.crc == 1, (sf, d.rnti, t)
                assert bytes(pl[rr.payload_off:rr.payload_off + nb]) == bytes(payload[d.payload_off[t]:d.payload_off[t] + nb])
    phy.close()


def test_example_matches_the_binding(phylib, infra, tmp_path):
    from ltesniffer_b200 import capi
    subprocess.run(["make", "-s", "-C", ROOT, "examples/cell_search"], check=True)
    N = 512
    cell = ltelib.Cell(25, 2, 99, 1, N)
    s = S.sim(sync=1, cell=cell, seed=81, pbch=1, snr_db=25.0, nof_ues=3)
    x = np.concatenate([s.subframe(t)[0] for t in range(30)], axis=1)[:, 4444:].astype(np.complex64)
    cs = capi.CellSearch(N, 1, x.shape[1])
    c = cs.search(x)[0]
    cs.close()
    f = tmp_path / "cap.cf32"
    x.tofile(str(f))
    r = subprocess.run([os.path.join(ROOT, "examples", "cell_search"), str(f), str(N), "1"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    w = r.stdout.split()
    assert int(w[1]) == c.pci == 99 and int(w[3]) == c.frame_offset and abs(float(w[5]) - c.cfo_hz) < 0.06
    assert int(w[7]) == 25 and int(w[9]) == 2
