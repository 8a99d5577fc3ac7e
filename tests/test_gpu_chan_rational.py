"""Rational carriers and integer samples of the channeliser on the GPU: every output of ltephy_chan_run / _device equals lteo_chan_run_poly bit for
bit (capture rates from 15.36 to 200 Msps, up- and downsampling, 1 and 2 antennas, cf32 / sc16 / sc8, host and device input, five chunkings,
calls of exactly max_samples, integer and rational carriers in one plan); the flag leaves integer plans as they were; the OFDM grid of a
resampled carrier against its narrowband capture; channeliser -> cell search -> tracker -> MIB -> decode on sc16 captures at 25 and 20 Msps, with
decode_wideband's pcaps equal to the chain's records; invalid inputs on a live rational handle."""
import ctypes as C

import numpy as np
import pytest

import chan_lib as CH
import chan_rational_lib as R
from test_chan import CHUNKINGS, _signal
from test_chan_rational import MIXED, SPEC
from test_gpu_chan import PLANS, _same

pytestmark = pytest.mark.gpu

RPLANS = [  # fs_in, carriers, nof_rx, samples
    (20000000, [(-4000000, 1024), (1000000, 1536)], 2, 30000),
    (20000000, [(0, 2048)], 1, 30000),
    (25000000, [(-6000000, 1024), (5000000, 512)], 2, 40000),
    (56000000, [(-18000000, 2048), (13000000, 1024)], 1, 60000),
    (100000000, [(-30000000, 2048), (0, 2048), (30000000, 2048)], 2, 100000),
    (200000000, [(30000000, 2048), (-60000000, 128)], 1, 150000),
    (15360000, [(1000, 1024)], 2, 20000),
    MIXED + (2, 30000),
]


def _host(outs):
    return [dict(first=o["first"], iq=o["iq"].cpu().numpy()) for o in outs]


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.parametrize("fmt", ["cf32", "sc16", "sc8"])
@pytest.mark.parametrize("plan", range(len(RPLANS)))
def test_bit_exact_with_the_oracle(phylib, plan, fmt):
    from ltesniffer_b200 import capi
    fs, carriers, nrx, n = RPLANS[plan]
    q, _ = R.to_format(_signal(n, nrx, fs, 11 + plan) / 4.0, fmt)
    ref, nxt = R.run(fs, carriers, q, 0, fmt)
    ch = capi.Channelizer(fs, carriers, nrx, n, rational=True, iq_format=fmt)
    got, nxt_h = ch.run(q, 0)
    assert nxt_h == nxt
    _same(ref, _host(got))
    got, nxt_d = ch.run_device(_dev(q), 0)
    assert nxt_d == nxt
    _same(ref, _host(got))
    ch.close()


@pytest.mark.parametrize("sizes", CHUNKINGS)
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("fmt", ["cf32", "sc16"])
def test_chunking_host_and_device(phylib, sizes, device, fmt):
    """the five chunkings, a plan of integer and rational carriers, both entry points: the one-call oracle's bytes and next_sample"""
    from ltesniffer_b200 import capi
    fs, carriers = MIXED
    x = _signal(9000, 2, fs, 5) / 4.0
    q, _ = R.to_format(x, fmt)
    ref, nxt = R.run(fs, carriers, q, 0, fmt)
    ch = capi.Channelizer(fs, carriers, 2, 9000, rational=True, iq_format=fmt)

    def run(xx, f):   # stream() cuts the complex capture x; an sc16 span is the same samples of q, two values each
        if fmt != "cf32":
            xx = np.ascontiguousarray(q[:, 2 * f:2 * (f + xx.shape[1])])
        return ch.run_device(_dev(xx), f) if device else ch.run(xx, f)
    got, nexts = CH.stream(run, q if fmt == "cf32" else x, sizes)
    assert nexts[-1] == nxt
    _same(ref, got)
    ch.close()


def test_calls_that_reach_max_samples(phylib):
    """a 200 Msps handle sized for 5000 samples, fed spans of exactly 5000 from each next_sample: one oracle call over the whole capture"""
    from ltesniffer_b200 import capi
    fs, carriers, nrx = 200000000, [(30000000, 2048), (-60000000, 128)], 1
    x = _signal(60000, nrx, fs, 8)
    ref, nxt = R.run(fs, carriers, x, 0)
    ch = capi.Channelizer(fs, carriers, nrx, 5000, rational=True)
    got, start, full = [dict(first=None, iq=[]) for _ in carriers], 0, 0
    while start < x.shape[1]:
        span = x[:, start:start + 5000]
        full += span.shape[1] == 5000
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


@pytest.mark.parametrize("plan", range(len(PLANS)))
def test_flag_leaves_integer_plans_unchanged(phylib, plan):
    """with LTEPHY_CHAN_RATIONAL every integer plan gives the outputs and next_sample of the unflagged handle"""
    from ltesniffer_b200 import capi
    fs, carriers, nrx, n = PLANS[plan]
    x = _signal(n, nrx, fs, 11 + plan)
    a = capi.Channelizer(fs, carriers, nrx, n)
    b = capi.Channelizer(fs, carriers, nrx, n, rational=True)
    ra, na = a.run(x, 0)
    rb, nb = b.run(x, 0)
    assert na == nb
    _same(_host(ra), _host(rb))
    a.close(), b.close()


@pytest.mark.parametrize("fs,off,N,prb", [(25000000, -6000000, 1024, 50), (20000000, 0, 2048, 100), (56000000, 13000000, 1024, 50)])
def test_grid_matches_the_narrowband_capture(phylib, fs, off, N, prb):
    """one resampled carrier, no neighbours and no noise: its OFDM grid (LTEPHY_TAP_SYM) is the grid of its own capture within -40 dB"""
    from ltesniffer_b200 import capi
    spec = [dict(offset_hz=off, N=N, pci=17, cfo=0.0, lead=0, snr=80.0)]
    x, truths = R.compose(fs, spec, 6, nrx=1, noise_db=-200.0, seed=4)
    ch = capi.Channelizer(fs, [(off, N)], 1, x.shape[1], rational=True)
    outs, _ = ch.run(x, 0)
    ch.close()
    y = outs[0]["iq"].cpu().numpy()
    nb = truths[0]["narrow"]
    SF = 15 * N
    nsf = min(y.shape[1], nb.shape[1]) // SF - 1
    scale = np.vdot(nb[0, :nsf * SF], nb[0, :nsf * SF]).real / np.vdot(nb[0, :nsf * SF], y[0, :nsf * SF]).real
    grids = []
    for iq in (nb, y * scale):
        phy = capi.LtePhy(prb, 1, 17, 1, max_subframes=nsf, symbol_sz=N)
        phy.submit_iq(np.stack([iq[:, k * SF:(k + 1) * SF] for k in range(nsf)]).astype(np.complex64), np.arange(nsf, dtype=np.uint32))
        phy.get_phase_a(want_cands=False)
        grids.append(phy.tap(capi.TAP_SYM, (nsf, 1, 14, 12 * prb), np.complex64))
        phy.close()
    a, b = grids[1][1:], grids[0][1:]
    evm = 10 * np.log10(np.sum(np.abs(a - b) ** 2) / np.sum(np.abs(b) ** 2))
    assert evm < -40.0, (N, evm)


def test_invalid_inputs(phylib):
    from ltesniffer_b200 import capi
    ch = capi.Channelizer(25000000, [(0, 1024)], 1, 5000, rational=True, iq_format="sc16")
    out, nxt = (capi.ChanOut * 8)(), C.c_uint64()
    x = np.zeros((1, 12000), np.int16)
    L = ch.L
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 5001, out, C.byref(nxt)) == -2
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 0, out, C.byref(nxt)) == -2
    assert L.ltephy_chan_run(ch.h, None, 0, 100, out, C.byref(nxt)) == -2
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 100, None, C.byref(nxt)) == -2
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 100, out, None) == -2
    assert L.ltephy_chan_run_device(ch.h, None, 0, 100, out, C.byref(nxt)) == -2
    import torch
    xd = torch.zeros(2 * 6000, dtype=torch.int16, device="cuda")
    assert L.ltephy_chan_run_device(ch.h, C.c_void_p(xd.data_ptr() + 2), 0, 100, out, C.byref(nxt)) == -2   # not on a 4-byte sample
    # too short for a window: nothing out, and the next call must start again from 0
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 5, out, C.byref(nxt)) == 0 and out[0].count == 0 and nxt.value == 0
    assert L.ltephy_chan_run(ch.h, capi._p(x), 0, 5000, out, C.byref(nxt)) == 0 and out[0].count > 0
    ch.close()


def _quantise(x):
    """sc16 of a capture scaled so its peak uses most of the int16 range"""
    q, _ = R.to_format(x * (0.5 / np.abs(x).max()), "sc16")
    return q


CHAINS = [
    ("25 Msps, N 1024 and N 512", 25000000, SPEC),
    ("20 Msps, one 20 MHz cell (192 / 125)", 20000000, [dict(offset_hz=0, N=2048, pci=321, cfo=-600.0, lead=1200, gain_db=0.0, decode=True)]),
]


@pytest.mark.parametrize("name,fs,spec", CHAINS, ids=[c[0] for c in CHAINS])
def test_full_chain_and_decode_wideband(phylib, infra, tmp_path, name, fs, spec):
    """400 ms of an sc16 capture: Channelizer -> ltephy_cell_search_device -> tracker from tti 0 -> the MIB from the subframes 0 of its cut ->
    ltephy_decode_subframes_device, span by span as examples/decode_wideband reads the file with fmt=sc16.  Every carrier decodes the truth
    transport blocks the same decoder reads from the simulator's own subframes, and decode_wideband's pcap of each carrier equals this chain's
    records one for one"""
    import os
    import subprocess
    from ltesniffer_b200 import capi
    from test_decode_recording import _read_pcap
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run(["make", "-s", "-C", root, "examples/decode_wideband"], check=True)
    A, B, nsf = 2, 100, 400
    x, truths = R.compose(fs, spec, nsf, nrx=A, ppm=20.0, noise_db=-35.0, seed=2)
    q = _quantise(x)
    del x
    f = tmp_path / "wide.sc16"
    q.tofile(str(f))
    prefix = str(tmp_path / "o")
    r = subprocess.run([os.path.join(root, "examples", "decode_wideband"), str(f), str(fs), str(A), prefix] +
                       ["%d:%d" % (c["offset_hz"], c["N"]) for c in spec] + [str(B), "fmt=sc16"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    carriers = [(c["offset_hz"], c["N"]) for c in spec]
    L, MS = q.shape[1] // 2, fs // 1000
    ch = capi.Channelizer(fs, carriers, A, min(L, (B + 20) * MS), rational=True, iq_format="sc16")
    geo = [ch.design(c) for c in range(len(spec))]
    L0 = min(L, 40 * MS + max(g["Kp"] for g in geo))
    outs, _ = ch.run(q[:, :2 * L0], 0)
    st = []
    for c, o in zip(spec, outs):
        cs = capi.CellSearch(c["N"], A, o["count"])
        cell = [z for z in cs.search_device(o["iq"]) if z.detected][0]
        cs.close()
        assert cell.pci == c["pci"]
        st.append(dict(cell=cell, tr=capi.Tracker(c["N"], A, cell.pci, int(cell.frame_offset), cfo_hz=cell.cfo_hz, max_subframes=B),
                       next=int(cell.frame_offset), mib=None, phy=None, expect=[], nsf=0))
    md = 32 * B
    recv = 0
    while True:
        recv = min(recv + B * MS, L)
        first = min(max(0, s["next"] * g["M"] // g["L"] - g["Ka"]) for s, g in zip(st, geo))
        if first >= recv:
            if recv == L:
                break
            continue
        end = min(recv, first + min(L, (B + 20) * MS))
        outs, _ = ch.run(q[:, 2 * first:2 * end], first)
        anyg = False
        for c, o, s in zip(spec, outs, st):
            if not o["count"]:
                continue
            z = s["tr"].push_device(o["iq"], o["first"])
            s["next"] = z["next_sample"]
            m = len(z["sf"])
            anyg = anyg or m > 0
            if s["mib"] is None:
                mp = capi.LtePhy(15, 2, s["cell"].pci, A, max_subframes=1, symbol_sz=c["N"])
                mp.n = 1
                for i in range(m):
                    t = z["sf"]["tti"][i:i + 1].astype(np.uint32)
                    if t[0] % 10:
                        continue
                    mp._chk(mp.L.ltephy_submit_iq_device(mp.h, C.c_void_p(z["iq"][i].data_ptr()), capi._p(t), 1), "submit_iq_device")
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
            tti = np.ascontiguousarray((z["sf"]["tti"].astype(np.int64) + 10 * s["sfn"]) % 10240, np.uint32)
            sc, nd = s["scr"], C.c_uint32(0)
            rc = phylib.ltephy_decode_subframes_device(s["phy"].h, s["srch"].h, C.c_void_p(z["iq"].data_ptr()), capi._p(tti), m, capi.SEQ_NONE, sc["info"],
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
                for z in range(2):
                    rr = tbs[2 * i + z]
                    if rr.crc and rr.payload_len:
                        ideal.add((int(d["rnti"]), int(tti[int(d["sf"])]), bytes(payload[rr.payload_off:rr.payload_off + rr.payload_len])))
        phy.close(), srch.close()
        for t in range(s["nsf"]):
            tru, pl = tr["sub"][t][1], tr["sub"][t][2]
            for i in range(tru.nof_dci):
                d = tru.dci[i]
                for z in range(2):
                    if d.nof_tb > z and d.tbs[z] > 0:
                        truth.add((int(d.rnti), t % 10240, bytes(pl[d.payload_off[z]:d.payload_off[z] + d.tbs[z] // 8])))
        have = set(s["expect"])
        assert len(truth) > 100 and len(truth & ideal) >= 0.95 * len(truth), (c, len(truth), len(truth & ideal))
        assert truth & ideal <= have, (c, len((truth & ideal) - have))
