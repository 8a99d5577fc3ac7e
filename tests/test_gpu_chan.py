"""Channeliser on the GPU: every output sample of ltephy_chan_run / _device equals the oracle lteo_chan_run bit for bit, over both symbol-size
families, decimations from 2 to 128, one and two antennas, five chunkings and calls that reach max_samples; the OFDM grid of each channelised
carrier against the carrier's own narrowband capture; channeliser -> cell search -> tracker on a three-carrier capture; invalid inputs on a
live handle."""
import ctypes as C

import numpy as np
import pytest

import chan_lib as CH
from test_chan import CHUNKINGS, _signal

pytestmark = pytest.mark.gpu

PLANS = [  # fs_in, carriers, nof_rx, samples
    (30720000, [(-7500000, 1024), (5000000, 512), (11000000, 256)], 2, 40000),
    (46080000, [(1000, 1536), (-15000000, 768), (20000000, 256)], 1, 30000),
    (245760000, [(-101377000, 256), (99999000, 128), (-60000000, 2048), (30000000, 512)], 2, 120000),
]


def _same(ref, got):
    for a, b in zip(ref, got):
        assert a["first"] == b["first"] and a["iq"].shape == b["iq"].shape, (a["first"], b["first"], a["iq"].shape, b["iq"].shape)
        assert a["iq"].tobytes() == b["iq"].tobytes()


@pytest.mark.parametrize("plan", range(len(PLANS)))
def test_bit_exact_with_the_oracle(phylib, plan):
    import torch
    from ltesniffer_b200 import capi
    fs, carriers, nrx, n = PLANS[plan]
    x = _signal(n, nrx, fs, 11 + plan)
    ref, nxt = CH.run(fs, carriers, x, 0)
    ch = capi.Channelizer(fs, carriers, nrx, n)
    got, nxt_h = ch.run(x, 0)
    assert nxt_h == nxt
    _same(ref, [dict(first=o["first"], iq=o["iq"].cpu().numpy()) for o in got])
    got, nxt_d = ch.run_device(torch.from_numpy(x).cuda(), 0)
    assert nxt_d == nxt
    _same(ref, [dict(first=o["first"], iq=o["iq"].cpu().numpy()) for o in got])
    ch.close()


@pytest.mark.parametrize("sizes", CHUNKINGS)
@pytest.mark.parametrize("device", [False, True])
def test_chunking_host_and_device(phylib, sizes, device):
    """the five chunkings of the CPU test, through both entry points, give the one-call oracle's bytes and next_sample"""
    import torch
    from ltesniffer_b200 import capi
    fs, carriers, nrx, n = PLANS[0]
    n = 9000
    x = _signal(n, nrx, fs, 5)
    ref, nxt = CH.run(fs, carriers, x, 0)
    ch = capi.Channelizer(fs, carriers, nrx, n)
    run = (lambda xx, f: ch.run_device(torch.from_numpy(np.ascontiguousarray(xx)).cuda(), f)) if device else ch.run
    got, nexts = CH.stream(run, x, sizes)
    assert nexts[-1] == nxt
    _same(ref, got)
    ch.close()


def test_calls_that_reach_max_samples(phylib):
    """a handle sized for 3000 samples, fed spans of exactly 3000 from each next_sample: the outputs equal one oracle call over the whole capture"""
    from ltesniffer_b200 import capi
    fs, carriers, nrx = 245760000, [(-101377000, 256), (-60000000, 2048)], 1
    x = _signal(40000, nrx, fs, 8)
    ref, nxt = CH.run(fs, carriers, x, 0)
    ch = capi.Channelizer(fs, carriers, nrx, 3000)
    got, start, full = [dict(first=None, iq=[]) for _ in carriers], 0, 0
    while start < x.shape[1]:
        span = x[:, start:start + 3000]
        full += span.shape[1] == 3000
        outs, n2 = ch.run(span, start)
        for g, o in zip(got, outs):
            have = (g["first"] or 0) + sum(q.shape[1] for q in g["iq"])
            if g["first"] is None:
                g["first"] = o["first"]
            if o["count"] and o["first"] + o["count"] > have:
                g["iq"].append(o["iq"].cpu().numpy()[:, have - o["first"]:])
        if start + span.shape[1] == x.shape[1]:
            break
        start = n2
    assert full >= 10 and n2 == nxt
    _same(ref, [dict(first=g["first"], iq=np.concatenate(g["iq"], axis=1)) for g in got])
    ch.close()


def test_grid_matches_the_narrowband_capture(phylib):
    """one carrier at a time, no neighbours and no noise: the OFDM grid (LTEPHY_TAP_SYM) of the channelised stream is the grid of the carrier's
    own capture within an error vector below -40 dB"""
    from ltesniffer_b200 import capi
    fs = 30720000
    for off, N, prb in [(-7500000, 1024, 50), (5000000, 512, 25), (11000000, 256, 15)]:
        spec = [dict(offset_hz=off, N=N, pci=17, cfo=0.0, lead=0, snr=80.0)]
        x, truths = CH.compose(fs, spec, 6, nrx=1, noise_db=-200.0, seed=4)
        ch = capi.Channelizer(fs, [(off, N)], 1, x.shape[1])
        outs, _ = ch.run(x, 0)
        ch.close()
        y = outs[0]["iq"].cpu().numpy()
        nb = truths[0]["narrow"]
        SF = 15 * N
        nsf = min(y.shape[1], nb.shape[1]) // SF - 1        # the last subframe may run into the unfilled end
        scale = np.vdot(nb[0, :nsf * SF], nb[0, :nsf * SF]).real / np.vdot(nb[0, :nsf * SF], y[0, :nsf * SF]).real
        grids = []
        for iq in (nb, y * scale):
            phy = capi.LtePhy(prb, 1, 17, 1, max_subframes=nsf, symbol_sz=N)
            phy.submit_iq(np.stack([iq[:, k * SF:(k + 1) * SF] for k in range(nsf)]).astype(np.complex64), np.arange(nsf, dtype=np.uint32))
            phy.get_phase_a(want_cands=False)
            grids.append(phy.tap(capi.TAP_SYM, (nsf, 1, 14, 12 * prb), np.complex64))
            phy.close()
        a, b = grids[1][1:], grids[0][1:]                     # subframe 0 holds the filter's start-up from the zero history
        evm = 10 * np.log10(np.sum(np.abs(a - b) ** 2) / np.sum(np.abs(b) ** 2))
        assert evm < -40.0, (N, evm)


def test_search_and_track_each_carrier(phylib):
    """three carriers of one 30.72 Msps capture, 20 ppm clock offset, one carrier 20 dB weaker: Channelizer -> ltephy_cell_search_device on the
    first 40 ms of each carrier stream -> Tracker.push_device.  Each search finds its PCI as close to the truth timing in carrier samples as on the
    carrier's narrowband capture, and every subframe the tracker cuts after the first 40 ms lies as close to the truth as the tracker's cut of the
    narrowband capture"""
    import torch
    from ltesniffer_b200 import capi
    fs = 30720000
    spec = [dict(offset_hz=-7500000, N=1024, pci=101, cfo=900.0, lead=3000, gain_db=0.0),
            dict(offset_hz=5000000, N=512, pci=257, cfo=-1700.0, lead=777, gain_db=-20.0),
            dict(offset_hz=11000000, N=256, pci=44, cfo=300.0, lead=2500, gain_db=0.0)]
    nsf = 120
    x, truths = CH.compose(fs, spec, nsf, nrx=2, ppm=20.0, noise_db=-35.0, seed=2)
    ch = capi.Channelizer(fs, [(c["offset_hz"], c["N"]) for c in spec], 2, x.shape[1])
    outs, _ = ch.run_device(torch.from_numpy(x).cuda(), 0)
    for c, o, tr in zip(spec, outs, truths):
        N = c["N"]
        y = o["iq"]
        assert o["first"] == 0
        cs = capi.CellSearch(N, 2, 40 * 15 * N)
        cell = cs.search_device(y[:, :40 * 15 * N].contiguous())[0]
        narrow = cs.search(tr["narrow"][:, :40 * 15 * N])[0]
        cs.close()
        assert cell.detected and cell.pci == c["pci"], (c, cell.pci)
        # the search averages its PSS over the 40 ms, which the 20 ppm clock moves by several samples: as close as on the narrowband capture
        assert abs(int(cell.frame_offset) - tr["truth"][0]) <= abs(int(narrow.frame_offset) - tr["truth"][0]) + 1.5
        errs = []
        for iq, found, push in ((y.contiguous(), cell, "push_device"), (tr["narrow"], narrow, "push")):
            trk = capi.Tracker(N, 2, found.pci, int(found.frame_offset), cfo_hz=found.cfo_hz, max_subframes=nsf)
            r = getattr(trk, push)(iq, 0)
            trk.close()
            k = r["sf"]["index"].astype(np.int64)
            assert len(k) >= nsf - 3 and not (r["sf"]["flags"] & capi.TRACK_LOST).any()
            errs.append(np.abs(r["sf"]["start"] - tr["truth"][k])[k >= 40].max())
        # over 120 ms the timing corrections still saw-tooth with the clock: as close as the tracker gets on the narrowband capture
        assert errs[0] <= errs[1] + 1.0 and errs[0] <= 4.0, errs
    ch.close()


def test_invalid_inputs(phylib):
    from ltesniffer_b200 import capi
    ch = capi.Channelizer(30720000, [(0, 1024)], 1, 5000)
    out, nxt = (capi.ChanOut * 8)(), C.c_uint64()
    x = np.zeros((1, 6000), np.complex64)
    L = ch.L
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 5001, out, C.byref(nxt)) == -2          # more than max_samples
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 0, out, C.byref(nxt)) == -2             # no samples
    assert L.ltephy_chan_run(ch.h, None, 0, 100, out, C.byref(nxt)) == -2
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 100, None, C.byref(nxt)) == -2
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 100, out, None) == -2
    assert L.ltephy_chan_run_device(ch.h, None, 0, 100, out, C.byref(nxt)) == -2
    assert L.ltephy_chan_run(None, capi._p(x), 0, 100, out, C.byref(nxt)) == -2
    # too short for a window: nothing out, and the next call must start again from 0
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 5, out, C.byref(nxt)) == 0 and out[0].count == 0 and nxt.value == 0
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 5000, out, C.byref(nxt)) == 0 and out[0].count > 0
    ch.close()


def test_full_chain_and_decode_wideband(phylib, infra, tmp_path):
    """the three-carrier capture of the CPU decode test lengthened to 400 ms: Channelizer -> ltephy_cell_search_device -> tracker from tti 0 ->
    the MIB from the subframes 0 of its cut -> ltephy_decode_subframes_device, span by span as examples/decode_wideband reads the file.  Every
    carrier decodes the truth transport blocks the same decoder reads from the simulator's own subframes, and decode_wideband's pcap of each
    carrier equals this chain's records one for one"""
    import os
    import subprocess
    import torch
    from ltesniffer_b200 import capi
    from test_decode_recording import _read_pcap
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run(["make", "-s", "-C", root, "examples/decode_wideband"], check=True)
    fs, A, B, nsf = 30720000, 2, 100, 400
    spec = [dict(offset_hz=-7500000, N=1024, pci=101, cfo=900.0, lead=3000, gain_db=0.0, decode=True),
            dict(offset_hz=5000000, N=512, pci=257, cfo=-1700.0, lead=777, gain_db=-20.0, decode=True),
            dict(offset_hz=11000000, N=256, pci=44, cfo=300.0, lead=2500, gain_db=0.0, decode=True)]
    x, truths = CH.compose(fs, spec, nsf, nrx=A, ppm=20.0, noise_db=-35.0, seed=2)
    f = tmp_path / "wide.cf32"
    x.tofile(str(f))
    prefix = str(tmp_path / "o")
    r = subprocess.run([os.path.join(root, "examples", "decode_wideband"), str(f), str(fs), str(A), prefix] +
                       ["%d:%d" % (c["offset_hz"], c["N"]) for c in spec] + [str(B)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    carriers = [(c["offset_hz"], c["N"]) for c in spec]
    L, MS = x.shape[1], fs // 1000
    ch = capi.Channelizer(fs, carriers, A, min(L, (B + 20) * MS))
    taps = [ch.taps(c) for c in range(3)]
    L0 = min(L, 40 * MS + max(t["T"] for t in taps))
    outs, _ = ch.run(x[:, :L0], 0)
    st = []
    for c, o in zip(spec, outs):
        cs = capi.CellSearch(c["N"], A, o["count"])
        cell = [q for q in cs.search_device(o["iq"]) if q.detected][0]
        cs.close()
        assert cell.pci == c["pci"]
        st.append(dict(cell=cell, tr=capi.Tracker(c["N"], A, cell.pci, int(cell.frame_offset), cfo_hz=cell.cfo_hz, max_subframes=B),
                       next=int(cell.frame_offset), mib=None, phy=None, expect=[], nsf=0))
    md = 32 * B
    recv = 0
    while True:
        recv = min(recv + B * MS, L)
        first = min(max(0, s["next"] * t["D"] - t["T"] // 2) for s, t in zip(st, taps))
        if first >= recv:
            if recv == L:
                break
            continue
        end = min(recv, first + min(L, (B + 20) * MS))
        outs, _ = ch.run(x[:, first:end], first)
        anyg = False
        for c, o, s in zip(spec, outs, st):
            if not o["count"]:
                continue
            q = s["tr"].push_device(o["iq"], o["first"])
            s["next"] = q["next_sample"]
            m = len(q["sf"])
            anyg = anyg or m > 0
            if s["mib"] is None:
                mp = capi.LtePhy(15, 2, s["cell"].pci, A, max_subframes=1, symbol_sz=c["N"])
                mp.n = 1
                for i in range(m):
                    t = q["sf"]["tti"][i:i + 1].astype(np.uint32)
                    if t[0] % 10:
                        continue
                    mp._chk(mp.L.ltephy_submit_iq_device(mp.h, C.c_void_p(q["iq"][i].data_ptr()), capi._p(t), 1), "submit_iq_device")
                    mc = mp.mib_decode_combined(search_ports=True)[0]
                    if mc.mib.found:
                        s["mib"], s["sfn"] = mc.mib, (mc.mib.sfn + 1024 - int(t[0]) // 10 % 1024) % 1024
                        break
                mp.close()
                if s["mib"] is None:
                    continue
                mib = s["mib"]
                s["phy"] = capi.LtePhy(mib.nof_prb, mib.nof_ports, s["cell"].pci, A, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER,
                                       symbol_sz=c["N"], phich_resources=mib.phich_resources, phich_length=mib.phich_length)
                s["srch"] = capi.Search(mib.nof_prb, mib.nof_ports, s["cell"].pci, A, phich_resources=mib.phich_resources)
                s["scr"] = dict(info=(capi.SfInfo * B)(), cands=np.zeros((B, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE),
                                dcis=np.zeros(md, capi.DCI_DTYPE), tbs=(capi.TbResult * (2 * md))(), payload=np.zeros(B * 64 * 1024, np.uint8))
            if not m:
                continue
            tti = np.ascontiguousarray((q["sf"]["tti"].astype(np.int64) + 10 * s["sfn"]) % 10240, np.uint32)
            sc, nd = s["scr"], C.c_uint32(0)
            rc = phylib.ltephy_decode_subframes_device(s["phy"].h, s["srch"].h, C.c_void_p(q["iq"].data_ptr()), capi._p(tti), m, capi.SEQ_NONE, sc["info"],
                                                       capi._p(sc["cands"]), capi._p(sc["dcis"]), md, C.byref(nd), sc["tbs"], capi._p(sc["payload"]),
                                                       sc["payload"].nbytes)
            assert rc == 0, phylib.ltephy_last_error()
            for i, d in enumerate(sc["dcis"][:nd.value]):
                for t in range(2):
                    rr = sc["tbs"][2 * i + t]
                    if rr.crc and rr.payload_len:
                        s["expect"].append((int(d["rnti"]), int(tti[int(d["sf"])]), bytes(sc["payload"][rr.payload_off:rr.payload_off + rr.payload_len])))
            s["nsf"] += m
        if not anyg and recv == L:
            break
    ch.close()
    for ci, (c, s, tr) in enumerate(zip(spec, st, truths)):
        s["tr"].close()
        assert s["mib"] is not None and s["sfn"] == 0 and s["nsf"] >= nsf - 5, (c, s["nsf"])
        got = _read_pcap(prefix + "_%d.pcap" % ci)
        assert got == s["expect"], (c, len(got), len(s["expect"]))
        assert ("subframes %d " % s["nsf"]) in r.stdout
        # the truth blocks the same decoder reads from the simulator's own subframes are all in the pcap
        mib = s["mib"]
        phy = capi.LtePhy(mib.nof_prb, mib.nof_ports, c["pci"], A, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER, symbol_sz=c["N"],
                          phich_resources=mib.phich_resources, phich_length=mib.phich_length)
        srch = capi.Search(mib.nof_prb, mib.nof_ports, c["pci"], A, phich_resources=mib.phich_resources)
        ideal, truth = set(), set()
        for lo in range(0, s["nsf"], B):
            hi = min(lo + B, s["nsf"])
            tti = np.arange(lo, hi, dtype=np.uint32) % 10240
            info, dcis, tbs, payload = capi.decode_subframes(phy, srch, np.stack([tr["sub"][t][0] for t in range(lo, hi)]).astype(np.complex64), tti)
            for i, d in enumerate(dcis):
                for q in range(2):
                    rr = tbs[2 * i + q]
                    if rr.crc and rr.payload_len:
                        ideal.add((int(d["rnti"]), int(tti[int(d["sf"])]), bytes(payload[rr.payload_off:rr.payload_off + rr.payload_len])))
        phy.close(), srch.close()
        for t in range(s["nsf"]):
            tru, pl = tr["sub"][t][1], tr["sub"][t][2]
            for i in range(tru.nof_dci):
                d = tru.dci[i]
                for q in range(2):
                    if d.nof_tb > q and d.tbs[q] > 0:
                        truth.add((int(d.rnti), t % 10240, bytes(pl[d.payload_off[q]:d.payload_off[q] + d.tbs[q] // 8])))
        have = set(s["expect"])
        assert len(truth) > 100 and len(truth & ideal) >= 0.95 * len(truth), (c, len(truth), len(truth & ideal))
        assert truth & ideal <= have, (c, len((truth & ideal) - have))
