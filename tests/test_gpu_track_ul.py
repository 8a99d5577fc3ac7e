"""Uplink tracking and uplink decode on the GPU: ltephy_track_push_ul / _device against the oracle lteo_track_push_ul (records, DL cut and UL
cut bit for bit, and the DL side equal to a tracker without the uplink); ltephy_submit_ul_device against ltephy_submit_ul; ltephy_set_ul_cfo
against lteo_cfo_correct + lteo_ul_ofdm; and examples/decode_recording_ul end to end on a two-carrier recording whose clock is 20 ppm off."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import ltelib
import track_lib as T
from helpers import UlModeStep, ul_records

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "examples", "decode_recording_ul")

CASES = [  # N, nrx, nsf, capture kwargs, cfo_ratio, ul_offset in units of N / 8
    (128, 1, 40, dict(ppm=20.0, cfo=300.0, snr=20.0), 1.0, 0),
    (256, 2, 40, dict(ppm=-20.0, cfo=-2000.0, ramp=400.0, snr=8.0), 0.948, -8),
    (384, 1, 30, dict(ppm=0.0, cfo=4000.0, snr=10.0), 1.05, 8),
    (512, 2, 30, dict(ppm=20.0, cfo=1200.0, ramp=200.0, snr=15.0), 0.948, 3),
    (768, 1, 25, dict(ppm=-20.0, cfo=-700.0, snr=25.0), 1.0, -5),
    (1024, 2, 20, dict(ppm=2.0, cfo=900.0, snr=20.0), 0.948, 8),
    (1536, 1, 20, dict(ppm=-20.0, cfo=-700.0, ramp=300.0, snr=25.0), 1.05, -8),
    (2048, 2, 20, dict(ppm=20.0, cfo=2500.0, snr=20.0), 0.948, 1),
]


def _host(q):
    return q if isinstance(q, np.ndarray) else q.cpu().numpy()


def _same(a, b, keys=("iq", "ul_iq")):
    assert a["sf"].tobytes() == b["sf"].tobytes(), (a["sf"][:4], b["sf"][:4])
    assert a["hf"].tobytes() == b["hf"].tobytes(), (a["hf"][:4], b["hf"][:4])
    for k in keys:
        qa, qb = _host(a[k]), _host(b[k])
        assert qa.shape == qb.shape and qa.tobytes() == qb.tobytes(), k


@pytest.mark.parametrize("case", range(len(CASES)))
def test_ul_cut_bit_exact_with_the_oracle(phylib, case):
    """one push and odd chunkings through the host and device entry points; the DL records and cut equal a tracker without the uplink"""
    import torch
    from ltesniffer_b200 import capi
    N, nrx, nsf, kw, rho, off8 = CASES[case]
    off, lead = off8 * N // 8, 3 * N + 11
    x, _, _ = T.capture(N, 301, nsf, nrx=nrx, lead=lead, seed=case, t0=2, **kw)
    rng = np.random.default_rng(case)
    xu = np.ascontiguousarray(np.roll(x[nrx - 1], off) + 0.1 * (rng.standard_normal(x.shape[1]) + 1j * rng.standard_normal(x.shape[1])), np.complex64)
    mk = lambda: dict(cfo_hz=kw["cfo"] * 0.9, first_tti=2)
    ref = T.Oracle(N, nrx, 301, lead, ul=dict(cfo_ratio=rho, ul_offset=off), **mk()).push_ul(x, xu, 0)
    assert len(ref["sf"]) >= nsf - 3
    dl = T.Oracle(N, nrx, 301, lead, **mk()).push(x, 0)
    n = len(ref["sf"])
    assert ref["sf"].tobytes() == dl["sf"][:n].tobytes() and ref["iq"].tobytes() == dl["iq"][:n].tobytes()
    tr = capi.Tracker(N, nrx, 301, lead, max_subframes=200, ul=dict(cfo_ratio=rho, ul_offset=off), **mk())
    _same(ref, tr.push_ul(x, xu, 0))
    tr.close()
    for sizes in ([15 * N + 1], [7919, 3 * 15 * N + 17, 104729], [13 * N // 2 + 3, 15 * N - 5 + abs(off) // 2]):
        tr = capi.Tracker(N, nrx, 301, lead, max_subframes=200, ul=dict(cfo_ratio=rho, ul_offset=off), **mk())
        _same(ref, T.run_chunks(tr, x, sizes, xu=xu))
        tr.close()
        tr = capi.Tracker(N, nrx, 301, lead, max_subframes=200, ul=dict(cfo_ratio=rho, ul_offset=off), **mk())
        dev = lambda a, b, s: tr.push_ul_device(torch.from_numpy(np.ascontiguousarray(a)).cuda(), torch.from_numpy(np.ascontiguousarray(b)).cuda(), s)
        _same(ref, T.run_chunks(tr, x, sizes, xu=xu, push=dev))
        tr.close()
    # the same tracker without the uplink, over the subframes both cut
    tr = capi.Tracker(N, nrx, 301, lead, **mk())
    got = tr.push(x, 0)
    tr.close()
    assert got["sf"][:n].tobytes() == ref["sf"].tobytes() and _host(got["iq"])[:n].tobytes() == ref["iq"].tobytes()


def test_ul_invalid_inputs(phylib):
    from ltesniffer_b200 import capi
    for ul in (dict(cfo_ratio=0.0), dict(cfo_ratio=-1.0), dict(cfo_ratio=2.5), dict(cfo_ratio=float("nan")), dict(ul_offset=15 * 256),
               dict(ul_offset=-15 * 256), dict(ul_offset=-1001)):
        with pytest.raises(RuntimeError):
            capi.Tracker(256, 1, 1, 1000, ul=ul)
    x = np.zeros((1, 5000), np.complex64)
    o, u = capi.TrackOut(), C.c_void_p()
    tr = capi.Tracker(256, 1, 1, 1000)
    assert tr.L.ltephy_track_push_ul(tr.h, capi._p(x), capi._p(x), 0, 5000, C.byref(o), C.byref(u)) == -2       # without set_ul
    assert tr.L.ltephy_track_push(tr.h, capi._p(x), 0, 5000, C.byref(o)) == 0
    assert tr.L.ltephy_track_set_ul(tr.h, C.byref(capi.TrackUlCfg(cfo_ratio=1.0, ul_offset=0))) == -2           # after a push
    tr.close()
    tr = capi.Tracker(256, 1, 1, 1000, ul=dict(cfo_ratio=1.0, ul_offset=-500))
    assert tr.next_sample == 500
    assert tr.L.ltephy_track_push(tr.h, capi._p(x), 0, 5000, C.byref(o)) == -2                                 # DL-only push with UL set
    assert tr.L.ltephy_track_push_ul(tr.h, capi._p(x), None, 0, 5000, C.byref(o), C.byref(u)) == -2
    assert tr.L.ltephy_track_push_ul(tr.h, capi._p(x), capi._p(x), 501, 4000, C.byref(o), C.byref(u)) == -2   # after the UL window's start
    assert tr.L.ltephy_track_push_ul(tr.h, capi._p(x), capi._p(x), 0, 5000, C.byref(o), C.byref(u)) == 0 and o.nof_subframes == 1
    assert o.next_sample == 1000 + 15 * 256 - 500
    tr.close()


def _phy_grant(k, g):
    from ltesniffer_b200 import capi
    return capi.UlGrant(sf=k, rnti=g.rnti, qm=g.qm, rv=g.rv, L_prb=g.L_prb, n_prb=g.n_prb, n_dmrs2=g.n_dmrs2, tbs=g.tbs)


def test_submit_ul_device_equals_host(phylib):
    """results, chest and payload bit for bit, for the first decode and for the iq = NULL re-decode with other grants, with and without a UL CFO"""
    import torch
    from ltesniffer_b200 import capi
    N, n = 768, 24
    cap = T.TwoCarrier(N, 40, n, lead=200, seed=5, mcs_max=24)
    grants = [_phy_grant(k, g) for k in range(n) for g in cap.grants[k]]
    assert len(grants) >= 20
    iq = np.stack(cap.ul).astype(np.complex64)
    for cfo in (0.0, 350.0):
        outs = []
        for dev in (False, True):
            phy = capi.LtePhy(50, 1, 40, 1, max_subframes=n, symbol_sz=N)
            phy.set_ul_cfg(**T.UCFG)
            phy.set_ul_cfo(cfo)
            run = (lambda a, g: phy.decode_ul_device(None if a is None else torch.from_numpy(a).cuda(), cap.tti, g)) if dev else \
                (lambda a, g: phy.decode_ul(a, cap.tti, g))
            r1 = run(iq, grants)
            sym = phy.tap(capi.TAP_UL_SYM, (n, 14, 600), np.complex64)
            r2 = run(None, grants[::2])
            outs.append((r1, r2, sym))
            phy.close()
        for (a1, a2, sa), (b1, b2, sb) in [outs]:
            assert sa.tobytes() == sb.tobytes()
            for (ra, ca, pa), (rb, cb, pb), m in ((a1, b1, len(grants)), (a2, b2, len(grants[::2]))):
                assert bytes(ra)[:m * C.sizeof(capi.TbResult)] == bytes(rb)[:m * C.sizeof(capi.TbResult)]
                assert bytes(ca)[:m * C.sizeof(capi.UlChest)] == bytes(cb)[:m * C.sizeof(capi.UlChest)]
                assert pa.tobytes() == pb.tobytes()
        if cfo == 0.0:
            assert sum(r.crc for r in outs[0][0][0][:len(grants)]) >= 0.9 * len(grants)


@pytest.mark.parametrize("N", [256, 384, 512, 768, 1024, 1536, 2048])   # ltephy_create takes 11-100 PRB: no decoder exists at N = 128 (6 PRB)
def test_ul_cfo_tap_equals_oracle(phylib, N):
    """LTEPHY_TAP_UL_SYM after ltephy_set_ul_cfo, at every symbol size the decoder accepts: equals the handle's own UL OFDM without the offset on
    samples rotated beforehand in float32 by the same table (exp(-j 2 pi f n / (15000 N)) in double, rounded to float, products as
    lteo_cfo_correct), and lteo_cfo_correct + lteo_ul_ofdm.  0 gives the outputs of a handle that never set it; the downlink offset of
    ltephy_set_cfo does not touch the uplink"""
    from ltesniffer_b200 import capi
    prb = T.PRB_OF[N]
    rng = np.random.default_rng(N)
    n = 3
    iq = ((rng.standard_normal((n, 15 * N)) + 1j * rng.standard_normal((n, 15 * N))) * 0.5).astype(np.complex64)

    def tap(x, cfo=None, dl_cfo=None):
        phy = capi.LtePhy(prb, 1, 7, 1, max_subframes=n, symbol_sz=N)
        phy.set_ul_cfg()
        if dl_cfo is not None:
            phy.set_cfo(dl_cfo)
        if cfo is not None:
            phy.set_ul_cfo(cfo)
        phy.decode_ul(x, np.arange(n, dtype=np.uint32), [])
        out = phy.tap(capi.TAP_UL_SYM, (n, 14 * 12 * prb), np.complex64)
        phy.close()
        return out

    def rotate(x, cfo):
        ph = -2.0 * np.pi * float(np.float32(cfo)) * np.arange(15 * N, dtype=np.float64) / (15000.0 * N)
        cr, ci = np.cos(ph).astype(np.float32), np.sin(ph).astype(np.float32)
        xr, xi = x.real.astype(np.float32), x.imag.astype(np.float32)
        y = np.empty_like(x)
        y.real, y.imag = xr * cr - xi * ci, xr * ci + xi * cr
        return y

    o = ltelib.Oracle(ltelib.Cell(prb, 1, 7, 1, N))
    O = ltelib.oracle()
    O.lteo_ul_ofdm.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    for cfo in (-1234.5, 600.0):
        got = tap(iq, cfo)
        assert got.tobytes() == tap(rotate(iq, cfo)).tobytes(), cfo
        ref = np.zeros((n, 14 * 12 * prb), np.complex64)
        for i in range(n):
            y = o.cfo_correct(cfo, iq[i][None, :])[0]
            O.lteo_ul_ofdm(o.h, ltelib.ptr(np.ascontiguousarray(y)), ltelib.ptr(ref[i]))
        assert got.tobytes() == ref.tobytes(), cfo
    plain = tap(iq)
    assert tap(iq, 0.0).tobytes() == plain.tobytes() and tap(iq, dl_cfo=900.0).tobytes() == plain.tobytes()


def _read_pcap(path):
    b = open(path, "rb").read()
    off, got = 24, []
    while off < len(b):
        il = struct.unpack("<I", b[off + 8:off + 12])[0]
        rec = b[off + 16:off + 16 + il]
        off += 16 + il
        sfn_sf = (rec[10] << 8) | rec[11]
        got.append((rec[1], (rec[4] << 8) | rec[5], (sfn_sf >> 4) * 10 + (sfn_sf & 15), rec[19:]))
    return got


N_E2E, PCI_E2E, LEAD_E2E, OFF_E2E, RHO_E2E, B_E2E = 384, 262, 4321, 300, 0.948, 200


def _example_and_chain(cap, tmp_path):
    """runs examples/decode_recording_ul on the capture, and the same chain through the binding: cell search, tracker push by push
    (ltephy_track_push_ul), DL decode in UL mode, RAR and DCI-0 grants with carry-over (grants that land beyond a push stay carried),
    ltephy_submit_ul_device on the UL cut.  Every grant the chain submits is also decoded, by the same decoder, on the simulator's aligned,
    offset-free UL subframe of the same tti -> dict(r: the example's CompletedProcess, got: its pcap records, expect: the chain's records,
    aligned: the UL records (0, rnti, tti, payload) the aligned subframes give under the chain's grants, done, lost, carried_beyond: the largest
    number of carried grants that fell beyond a push, carry_left: grants still carried at the end)"""
    from ltesniffer_b200 import capi
    subprocess.run(["make", "-s", "-C", ROOT, "examples/decode_recording_ul"], check=True)
    N, pci, off, rho, B, SF = N_E2E, PCI_E2E, OFF_E2E, RHO_E2E, B_E2E, 15 * N_E2E
    fd, fu = tmp_path / "dl.cf32", tmp_path / "ul.cf32"
    cap.x[0].tofile(str(fd))
    cap.xu.tofile(str(fu))
    pc = str(tmp_path / "o.pcap")
    r = subprocess.run([EXE, str(fd), str(fu), str(N), pc, str(rho), str(off), str(T.UCFG["n_dmrs1"]), str(T.UCFG["delta_ss"])],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    head = r.stdout.splitlines()[0].split()
    kv = {head[i]: head[i + 1] for i in range(0, len(head), 2)}
    x = cap.x[:1]
    cs = capi.CellSearch(N, 1, 40 * SF)
    c = cs.search(x[:, :40 * SF])[0]
    cs.close()
    assert c.detected and c.pci == pci and int(kv["frame_offset"]) == c.frame_offset
    sfn, fo = int(kv["sfn"]), int(c.frame_offset)
    assert sfn == 0
    phich = dict(phich_resources=int(kv["phich_resources"]), phich_length=int(kv["phich_length"]))
    step = UlModeStep(25, int(kv["nof_ports"]), pci, B, symbol_sz=N, **phich)
    ul_ref = capi.LtePhy(25, int(kv["nof_ports"]), pci, 1, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER, symbol_sz=N, **phich)
    ul_ref.set_ul_cfg(**T.UCFG)
    tr = capi.Tracker(N, 1, pci, fo, cfo_hz=c.cfo_hz, first_tti=10 * sfn, max_subframes=B, ul=dict(cfo_ratio=rho, ul_offset=off))
    L = cap.x.shape[1]
    expect, aligned, recv, done, lost = [], [], 0, 0, 0
    while True:
        if recv < L:
            recv = min(recv + B * SF, L)
        nxt = tr.next_sample
        if nxt >= recv:
            if recv == L:
                break
            continue
        o = tr.push_ul(x[:, nxt:recv], cap.xu[nxt:recv], nxt)
        m = len(o["sf"])
        if not m:
            if recv == L:
                break
            continue
        lost += int((o["sf"]["flags"] & capi.TRACK_LOST).sum())
        tti = o["sf"]["tti"]
        expect += step(o["iq"], tti, o["ul_iq"])
        if step.now:
            # the same grants on the simulator's own UL subframes of these ttis (no clock or carrier offset, no uplink delay)
            res, _, pl = ul_ref.decode_ul(np.stack([cap.ul[int(t)] for t in tti]).astype(np.complex64), tti, step.now)
            aligned += ul_records(step.now, res, pl, tti)
        done += m
    tr.close(), step.close(), ul_ref.close()
    return dict(r=r, got=_read_pcap(pc), expect=expect, aligned=aligned, done=done, lost=lost, carried_beyond=step.beyond,
                carry_left=len(step.carry))


def test_recording_ul_to_pcap_at_20ppm(infra, phylib, tmp_path):
    """2 s, 25 PRB, 20 ppm, 800 Hz DL offset, rho 0.948, the uplink 300 samples late: the example's pcap equals record for record the chain driven
    through the binding; it holds every UL block that the same decoder reads, under the same grants, from the simulator's aligned UL subframes,
    and every DL block that the same decoder in UL mode reads from the aligned DL subframes"""
    from ltesniffer_b200 import capi
    nsf, B = 2000, B_E2E
    cap = T.TwoCarrier(N_E2E, PCI_E2E, nsf, ppm=20.0, cfo=800.0, rho=RHO_E2E, lead=LEAD_E2E, ul_offset=OFF_E2E, seed=71, pbch=1, nof_ports=2,
                       mcs_max=20)
    e = _example_and_chain(cap, tmp_path)
    got, done = e["got"], e["done"]
    # the example writes a push's DL records, then its UL records; so does the chain
    assert got == e["expect"] and done >= nsf - 5 and e["lost"] == 0
    assert ("subframes %d " % done) in e["r"].stdout
    have_ul = {q for q in got if q[0] == 0}
    have_dl = {(rn, t, p) for d, rn, t, p in got if d == 1}
    # UL: every block the aligned subframes give under the grants the chain submitted, with its bytes, and those are the blocks the simulator sent
    aligned = set(e["aligned"])
    sent = {(k, rn, pl) for (k, rn, _), pl in cap.sent.items()}
    assert len(aligned) > 1000 and {(t, rn, p) for _, rn, t, p in aligned} <= sent
    assert aligned <= have_ul, sorted((t, rn) for _, rn, t, _ in aligned - have_ul)[:10]
    # DL: every truth block that the same decoder, in UL mode, reads from the simulator's aligned DL subframes (decode_recording's criterion)
    head = e["r"].stdout.splitlines()[0].split()
    kv = {head[i]: head[i + 1] for i in range(0, len(head), 2)}
    phich = dict(phich_resources=int(kv["phich_resources"]), phich_length=int(kv["phich_length"]))
    phy = capi.LtePhy(25, int(kv["nof_ports"]), PCI_E2E, 1, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER, symbol_sz=N_E2E, **phich)
    srch = capi.Search(25, int(kv["nof_ports"]), PCI_E2E, 1, phich_resources=phich["phich_resources"])
    phy.L.ltephy_search_set_ul_mode(srch.h, 1, 0)
    ideal_dl = set()
    for lo in range(0, done, B):
        hi = min(lo + B, done)
        tti = np.arange(lo, hi, dtype=np.uint32) % 10240
        info, dcis, tbs, payload = capi.decode_subframes(phy, srch, np.stack([cap.dl[t][0][:1] for t in range(lo, hi)]).astype(np.complex64), tti)
        for i, d in enumerate(dcis):
            for q in range(2):
                rr = tbs[2 * i + q]
                if rr.crc and rr.payload_len:
                    ideal_dl.add((int(d["rnti"]), int(tti[int(d["sf"])]), bytes(payload[rr.payload_off:rr.payload_off + rr.payload_len])))
    phy.close(), srch.close()
    truth = set()
    for t in range(done):
        tr_, pl = cap.dl[t][1], cap.dl[t][2]
        for i in range(tr_.nof_dci):
            d = tr_.dci[i]
            for q in range(2):
                if d.nof_tb > q and d.tbs[q] > 0:
                    truth.add((int(d.rnti), t % 10240, bytes(pl[d.payload_off[q]:d.payload_off[q] + d.tbs[q] // 8])))
    assert truth & ideal_dl <= have_dl, (len(truth & ideal_dl), len((truth & ideal_dl) - have_dl), len(have_dl))
    print("UL blocks: aligned under the chain's grants %d, pcap %d; DL blocks: truth read from aligned %d, pcap %d" %
          (len(aligned), len(have_ul), len(truth & ideal_dl), len(have_dl)))


def test_recording_ul_with_a_short_last_push(infra, phylib, tmp_path):
    """a recording that ends two subframes after a push boundary: the last push cuts fewer subframes than the grants carried into it reach, those
    grants stay carried (counted as beyond the recording), and the example still decodes the rest of that push and prints its summary"""
    nsf = 202   # push 1 cuts subframes 0..198 (its last UL window ends before 200 subframes' worth of samples), push 2 cuts 199 and 200
    cap = T.TwoCarrier(N_E2E, PCI_E2E, nsf, ppm=20.0, cfo=800.0, rho=RHO_E2E, lead=LEAD_E2E, ul_offset=OFF_E2E, seed=72, pbch=1, nof_ports=2,
                       mcs_max=20)
    e = _example_and_chain(cap, tmp_path)
    assert e["carried_beyond"] >= 1 and e["carry_left"] >= 1, (e["carried_beyond"], e["carry_left"])
    assert e["got"] == e["expect"] and e["lost"] == 0
    assert ("subframes %d " % e["done"]) in e["r"].stdout
    assert ("ul grants beyond the recording %d" % e["carry_left"]) in e["r"].stdout
    assert set(e["aligned"]) <= {q for q in e["got"] if q[0] == 0}
