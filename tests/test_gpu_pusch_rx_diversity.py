"""Uplink receive diversity on the GPU (pytest -m gpu; DESIGN.md §2, "uplink receive diversity"): ltephy_submit_ul with ul_nof_rx = 2 against the
two-antenna oracle lteo_pusch_decode_rx bit for bit (soft bits, chest figures, CRC, payload), the UL grid tap against lteo_ul_ofdm per antenna, the
largest batch, and the tracker's two-antenna UL cut against the oracle tracker."""
import ctypes as C

import numpy as np
import pytest

import ltelib
import pusch_rx_lib as X
import track_lib as T
from helpers import UlModeStep, describe_mismatch
from ltelib import Cell, Oracle, Sim, UlCfg
from ltesniffer_b200 import capi
from test_pusch_rx_diversity import CASES, _grants

pytestmark = pytest.mark.gpu


def _to_capi(i, g):
    return capi.UlGrant(sf=i, rnti=g.rnti, qm=g.qm, rv=g.rv, L_prb=g.L_prb, n_prb=g.n_prb, n_dmrs2=g.n_dmrs2, tbs=g.tbs,
                        n_prb_slot1=g.n_prb_slot1 if g.hop else g.n_prb, flags=capi.UL_FLAG_SLOT1, nof_ack=g.nof_ack, ri_len=g.ri_len, cqi_len=g.cqi_len,
                        I_offset_ack=g.I_offset_ack, I_offset_ri=g.I_offset_ri, I_offset_cqi=g.I_offset_cqi)


def _check(phy, o, ucfg, tti, per_sf, iq, res, ch, payload, what, cfo=0.0):
    """every grant of the batch against lteo_pusch_decode_rx on the oracle's grids (after lteo_cfo_correct with cfo != 0) -> CRC passes"""
    A = iq.shape[1]
    tot = sum((ltelib.uci_layout(g).G + 7) & ~7 for gr in per_sf for g in gr)
    llr = phy.tap(capi.TAP_PDSCH_LLR, (tot,), np.int16)
    ulsym = phy.tap(capi.TAP_UL_SYM, (len(per_sf), A, 14 * phy.nsc), np.complex64)
    O = ltelib.oracle()
    O.lteo_cfo_correct.argtypes = [C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]
    k = lo = nok = 0
    for i, gr in enumerate(per_sf):
        x = np.ascontiguousarray(iq[i])
        if cfo:
            y = np.zeros_like(x)
            for a in range(A):
                O.lteo_cfo_correct(o.h, cfo, ltelib.ptr(x[a]), ltelib.ptr(y[a]))
            x = y
        sym, ref = X.oracle_ul_rx(o, ucfg, int(tti[i]), gr, x)
        assert ulsym[i].tobytes() == sym.tobytes(), (what, i, describe_mismatch(ulsym[i], sym, "UL grid"))
        for g, (r, opl, ocrc, och, ollr, _) in zip(gr, ref):
            assert r == 0
            rr, nby, G = res[k], g.tbs // 8, ltelib.uci_layout(g).G
            assert np.array_equal(llr[lo:lo + G], ollr), (what, k, describe_mismatch(llr[lo:lo + G], ollr, "soft bits"))
            lo += (G + 7) & ~7
            assert (ch[k].noise, ch[k].rsrp, ch[k].snr_db) == (och.noise, och.rsrp, och.snr_db), (what, k)
            assert abs(ch[k].ta_us - och.ta_us) < 1e-3
            assert rr.crc == ocrc and np.array_equal(payload[rr.payload_off:rr.payload_off + nby], opl[:nby]), (what, k)
            nok += rr.crc
            k += 1
    return nok, k


def _batch(cell, ucfg, nsf, ngr, table=1, mutate=None, min_prb=3, snr=22.0, seed=5):
    s = Sim(cell=Cell(cell.nof_prb, 1, cell.cell_id, 2, cell.symbol_sz), seed=seed, snr_db=snr, nof_ues=1, chan_delay=3)
    rng = np.random.default_rng(seed)
    iq = np.zeros((nsf, 2, s.sf_len), np.complex64)
    per_sf, grants, pls = [], [], []
    for i in range(nsf):
        gr = _grants(cell, rng, ngr, table, mutate, min_prb)
        iq[i], pl, off = X.sim_ul_rx(s, 3 + i, ucfg, gr, 2)
        per_sf.append(gr)
        grants += [_to_capi(i, g) for g in gr]
    return iq, np.arange(3, 3 + nsf, dtype=np.uint32), per_sf, grants


@pytest.mark.parametrize("prb,sz,table", [(15, 0, 1), (25, 384, 2), (25, 0, 1), (75, 1536, 2), (75, 0, 1), (100, 1536, 1), (100, 0, 2)])
def test_two_antennas_equal_the_oracle(infra, phylib, prb, sz, table):
    """15 / 25 / 75 / 100 PRB at the standard symbol size and at srsRAN's 3 * 2^k one; host submit, then the same batch through the device entry
    point, then NULL re-decode with other grants"""
    import torch
    cell = Cell(prb, 1, 100 + prb, 1, sz)
    ucfg = UlCfg(n_dmrs1=3, delta_ss=2)
    iq, tti, per_sf, grants = _batch(cell, ucfg, 3, 4, table=table)
    o = Oracle(cell)
    phy = capi.LtePhy(prb, 1, cell.cell_id, 1, max_subframes=3, symbol_sz=sz, ul_nof_rx=2)
    phy.set_ul_cfg(3, 2)
    res, ch, payload = phy.decode_ul(iq, tti, grants)
    nok, k = _check(phy, o, ucfg, tti, per_sf, iq, res, ch, payload, "host")
    assert nok >= k - 1
    res, ch, payload = phy.decode_ul_device(torch.from_numpy(iq).cuda(), tti, grants)
    assert _check(phy, o, ucfg, tti, per_sf, iq, res, ch, payload, "device") == (nok, k)
    rev = [list(reversed(gr)) for gr in per_sf]
    res, ch, payload = phy.decode_ul(None, tti, [_to_capi(i, g) for i, gr in enumerate(rev) for g in gr])
    assert _check(phy, o, ucfg, tti, rev, iq, res, ch, payload, "NULL re-decode") == (nok, k)
    phy.close()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_uci_hopping_and_every_modulation(infra, phylib, case):
    cid, cell, ucfg, table, mut, ngr, min_prb = case
    iq, tti, per_sf, grants = _batch(cell, ucfg, 3, ngr, table=table, mutate=mut, min_prb=min_prb, snr=26.0, seed=13)
    phy = capi.LtePhy(cell.nof_prb, 1, cell.cell_id, 1, max_subframes=3, ul_nof_rx=2)
    phy.set_ul_cfg(ucfg.n_dmrs1, ucfg.delta_ss, ucfg.group_hopping, ucfg.seq_hopping)
    res, ch, payload = phy.decode_ul(iq, tti, grants)
    nok, k = _check(phy, Oracle(cell), ucfg, tti, per_sf, iq, res, ch, payload, cid)
    assert nok >= k - 1
    phy.close()


def test_every_dft_size_and_ul_cfo(infra, phylib):
    """all 32 allocation sizes from 3 PRB up in one batch, Qm 2 to 8, with ltephy_set_ul_cfo applied to both antennas"""
    cell = Cell(100, 1, 77, 1)
    S = ltelib.sim()
    S.lte_ul_valid_prb.argtypes = [C.c_uint32]
    S.lte_ul_dci_to_grant.argtypes = [C.POINTER(Cell), C.POINTER(ltelib.Dci), C.c_int, C.POINTER(ltelib.UlGrant)]
    sizes = [L for L in range(3, 101) if S.lte_ul_valid_prb(L)]
    assert len(sizes) == 32
    ucfg = UlCfg(n_dmrs1=5, delta_ss=3)
    s = Sim(cell=Cell(100, 1, 77, 2), seed=8, snr_db=30.0, nof_ues=1)
    rng = np.random.default_rng(8)
    iq = np.zeros((32, 2, s.sf_len), np.complex64)
    per_sf = []
    for n, L in enumerate(sizes):
        d = ltelib.Dci()
        st = int(rng.integers(0, 101 - L))
        d.format, d.rnti, d.alloc_type = 0, 0x1000 + L, 2
        d.riv = 100 * (L - 1) + st if (L - 1) <= 50 else 100 * (100 - L + 1) + (99 - st)
        d.mcs[0], d.n_dmrs = int(rng.integers(0, 27)), int(rng.integers(0, 8))
        g = ltelib.UlGrant()
        assert S.lte_ul_dci_to_grant(C.byref(cell), C.byref(d), 1 + (n & 1), C.byref(g)) == 0 and g.L_prb == L
        iq[n] = X.sim_ul_rx(s, n, ucfg, [g], 2)[0]
        per_sf.append([g])
    assert {gr[0].qm for gr in per_sf} == {2, 4, 6, 8}
    tti = np.arange(32, dtype=np.uint32)
    phy = capi.LtePhy(100, 1, 77, 1, max_subframes=32, ul_nof_rx=2)
    phy.set_ul_cfg(5, 3)
    grants = [_to_capi(i, gr[0]) for i, gr in enumerate(per_sf)]
    res, ch, payload = phy.decode_ul(iq, tti, grants)
    o = Oracle(cell)
    nok, k = _check(phy, o, ucfg, tti, per_sf, iq, res, ch, payload, "sizes")
    assert nok == k == 32
    phy.set_ul_cfo(-310.0)
    res, ch, payload = phy.decode_ul(iq, tti, grants)
    _check(phy, o, ucfg, tti, per_sf, iq, res, ch, payload, "ul cfo", cfo=-310.0)
    phy.close()


def test_one_antenna_handle_equals_the_default(infra, phylib):
    """ul_nof_rx = 1 is ul_nof_rx = 0: the same grid, soft bits, chest figures and payload"""
    cell = Cell(50, 1, 17, 1)
    ucfg = UlCfg(n_dmrs1=3, delta_ss=2)
    iq, tti, per_sf, grants = _batch(cell, ucfg, 3, 4)
    out = []
    for A in (0, 1):
        phy = capi.LtePhy(50, 1, 17, 1, max_subframes=3, ul_nof_rx=A)
        phy.set_ul_cfg(3, 2)
        res, ch, payload = phy.decode_ul(np.ascontiguousarray(iq[:, 0]), tti, grants)
        tot = sum((ltelib.uci_layout(g).G + 7) & ~7 for gr in per_sf for g in gr)
        out.append((phy.tap(capi.TAP_UL_SYM, (3, 14 * phy.nsc), np.complex64).tobytes(), phy.tap(capi.TAP_PDSCH_LLR, (tot,), np.int16).tobytes(),
                    bytes(ch), bytes(res), payload.tobytes()))
        phy.close()
    assert out[0] == out[1]


def test_largest_two_antenna_batch(infra, phylib):
    """65 535 two-antenna subframes at 25 PRB (6.0 GB of samples at 15 x 384 per subframe and antenna, 4.4 GB of symbols, past 2^32 bytes): the last subframe's grants equal a one-subframe submit"""
    import torch
    cell = Cell(25, 1, 5, 1)
    ucfg = UlCfg(n_dmrs1=3, delta_ss=2)
    iq1, tti1, per_sf, grants1 = _batch(cell, ucfg, 1, 3, snr=26.0)
    n = 65535                                                   # LTEPHY_MAX_BATCH_SUBFRAMES
    big = torch.zeros((n, 2, iq1.shape[-1]), dtype=torch.complex64, device="cuda")
    big[n - 1] = torch.from_numpy(iq1[0]).cuda()
    tti = (np.arange(n, dtype=np.uint32) + 3 - (n - 1)) % 10240
    grants = [_to_capi(n - 1, g) for g in per_sf[0]]
    phy = capi.LtePhy(25, 1, 5, 1, max_subframes=n, ul_nof_rx=2)
    phy.set_ul_cfg(3, 2)
    res, ch, payload = phy.decode_ul_device(big, tti, grants)
    del big
    one = capi.LtePhy(25, 1, 5, 1, max_subframes=1, ul_nof_rx=2)
    one.set_ul_cfg(3, 2)
    res1, ch1, payload1 = one.decode_ul(iq1, tti1, grants1)
    for k, g in enumerate(per_sf[0]):
        nby = g.tbs // 8
        assert res[k].crc == res1[k].crc == 1
        assert bytes(ch[k]) == bytes(ch1[k])
        assert np.array_equal(payload[res[k].payload_off:res[k].payload_off + nby], payload1[res1[k].payload_off:res1[k].payload_off + nby])
    phy.close(), one.close()


@pytest.mark.parametrize("N,off", [(256, -200), (512, 700)])
def test_tracker_two_antenna_ul_cut(infra, phylib, N, off):
    """the two-antenna UL cut equals lteo_track_push_ul with two UL antennas bit for bit, through host and device pushes and in several chunkings"""
    import torch
    from test_track import chunk_cases
    x = T.capture(N, 33, 40, nrx=2, ppm=20.0, cfo=700.0, ramp=500.0, snr=12.0, lead=1234, seed=4)[0]
    rng = np.random.default_rng(N)
    xu = (rng.standard_normal((2, x.shape[1])) + 1j * rng.standard_normal((2, x.shape[1]))).astype(np.complex64)
    ref = T.Oracle(N, 2, 33, 1234, cfo_hz=650.0, ul=dict(cfo_ratio=0.948, ul_offset=off, nof_rx=2)).push_ul(x, xu, 0)
    assert len(ref["sf"]) >= 35
    mk = lambda: capi.Tracker(N, 2, 33, 1234, cfo_hz=650.0, max_subframes=200, ul=dict(cfo_ratio=0.948, ul_offset=off, nof_rx=2))
    for sizes in [[x.shape[1]]] + chunk_cases(N)[:3]:
        for dev in (False, True):
            tr = mk()
            if dev:
                push = lambda a, b, f: tr.push_ul_device(torch.from_numpy(np.ascontiguousarray(a)).cuda(), torch.from_numpy(np.ascontiguousarray(b)).cuda(), f)
            else:
                push = tr.push_ul
            got = T.run_chunks(tr, x, sizes, xu=xu, push=push)
            assert got["sf"].tobytes() == ref["sf"].tobytes() and got["hf"].tobytes() == ref["hf"].tobytes()
            assert got["iq"].tobytes() == ref["iq"].tobytes() and got["ul_iq"].tobytes() == ref["ul_iq"].tobytes(), (sizes, dev)
            tr.close()
    with pytest.raises(RuntimeError):
        capi.Tracker(N, 2, 33, 1234, ul=dict(nof_rx=3))


def _recording_chain_rx(cap, kv, B):
    """the chain of examples/decode_recording_ul driven through the binding with both UL antennas: tracker push by push with ul nof_rx = 2,
    DL decode in UL mode, RAR and DCI-0 grants with carry-over, ltephy_submit_ul_device on the [k][2][15 N] UL cut of a handle with
    ul_nof_rx = 2 -> the pcap records the example must write, in its order"""
    from test_gpu_track_ul import OFF_E2E, PCI_E2E, RHO_E2E
    N, pci, SF = cap.N, PCI_E2E, cap.SF
    fo, sfn = int(kv["frame_offset"]), int(kv["sfn"])
    phich = dict(phich_resources=int(kv["phich_resources"]), phich_length=int(kv["phich_length"]))
    step = UlModeStep(25, int(kv["nof_ports"]), pci, B, ul_nof_rx=2, symbol_sz=N, **phich)
    cs = capi.CellSearch(N, 1, 40 * SF)
    c = cs.search(cap.x[:, :40 * SF])[0]
    cs.close()
    assert c.detected and c.pci == pci and c.frame_offset == fo
    tr = capi.Tracker(N, 1, pci, fo, cfo_hz=c.cfo_hz, first_tti=10 * sfn, max_subframes=B, ul=dict(cfo_ratio=RHO_E2E, ul_offset=OFF_E2E, nof_rx=2))
    expect, recv, L = [], 0, cap.x.shape[1]
    while True:
        if recv < L:
            recv = min(recv + B * SF, L)
        nxt = tr.next_sample
        if nxt >= recv:
            if recv == L:
                break
            continue
        o = tr.push_ul(cap.x[:, nxt:recv], cap.xu[:, nxt:recv], nxt)
        m = len(o["sf"])
        if not m:
            if recv == L:
                break
            continue
        assert tuple(o["ul_iq"].shape) == (m, 2, SF)
        expect += step(o["iq"], o["sf"]["tti"], o["ul_iq"])
    tr.close(), step.close()
    return expect


def test_two_antenna_recording_to_pcap(infra, phylib, tmp_path):
    """examples/decode_recording_ul with ul_rx=2 on a 300-subframe recording (25 PRB, 20 ppm, 800 Hz, rho 0.948, the uplink 300 samples late) whose
    two UL antennas see the UEs at 6 dB each: its pcap equals record for record the chain driven through the binding with ul_nof_rx = 2, and it
    holds more uplink blocks than the example with ul_rx=1 on antenna 0 of the same recording (on the aligned subframes the oracle decodes 218 of
    419 grants from antenna 0 and 337 from both)"""
    import subprocess
    from test_gpu_track_ul import EXE, LEAD_E2E, N_E2E, OFF_E2E, PCI_E2E, RHO_E2E, ROOT, _read_pcap
    subprocess.run(["make", "-s", "-C", ROOT, "examples/decode_recording_ul"], check=True)
    cap = T.TwoCarrier(N_E2E, PCI_E2E, 300, ppm=20.0, cfo=800.0, rho=RHO_E2E, lead=LEAD_E2E, ul_offset=OFF_E2E, seed=73, pbch=1, nof_ports=2,
                       mcs_max=20, ul_snr=6.0, ul_nof_rx=2)
    fd, fu2, fu1 = tmp_path / "dl.cf32", tmp_path / "ul2.cf32", tmp_path / "ul1.cf32"
    cap.x[0].tofile(str(fd))
    cap.xu.tofile(str(fu2))                                          # antenna-major: all of antenna 0, then all of antenna 1
    cap.xu[0].tofile(str(fu1))
    runs = {}
    for A, fu in ((2, fu2), (1, fu1)):
        pc = str(tmp_path / ("o%d.pcap" % A))
        r = subprocess.run([EXE, str(fd), str(fu), str(N_E2E), pc, str(RHO_E2E), str(OFF_E2E), str(T.UCFG["n_dmrs1"]), str(T.UCFG["delta_ss"]), "0",
                            str(A)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        runs[A] = (r, _read_pcap(pc))
    head = runs[2][0].stdout.splitlines()[0].split()
    kv = {head[i]: head[i + 1] for i in range(0, len(head), 2)}
    expect = _recording_chain_rx(cap, kv, 200)
    got2, got1 = runs[2][1], runs[1][1]
    assert got2 == expect
    n2, n1 = sum(1 for q in got2 if q[0] == 0), sum(1 for q in got1 if q[0] == 0)
    sent = {(k, rn, pl) for (k, rn, _), pl in cap.sent.items()}
    assert {(t, rn, p) for d, rn, t, p in got2 if d == 0} <= sent
    print("UL blocks in the pcap: %d with ul_rx=2, %d with ul_rx=1 on antenna 0" % (n2, n1))
    assert n1 > 100 and n2 >= n1 + 50, (n1, n2)
