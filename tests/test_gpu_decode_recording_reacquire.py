"""examples/decode_recording.cpp with reacquire = 1 on the 2 s, 25 PRB, 2x2, 20 ppm recording of test_decode_recording, with 37 subframes and
1234 samples dropped 1 s in: the tracker finds the cell again, the example reads the SFN from the MIB again before it decodes anything more, and
its pcap equals record for record a chain driven through the Python binding with the same fallback; every record after the drop has the truth
SFN.  On the recording without the drop, reacquire = 1 changes nothing but the extra summary line."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ltelib
import sync_lib as S
import track_lib as T
from test_decode_recording import EXE, _build, _read_pcap

pytestmark = pytest.mark.gpu


def _binding_chain(x, N, B, pci):
    """cell search, MIB, tracker with the find state and the MIB fallback, decoder: the example's steps through capi -> (pcap records, index of
    the first record after the fallback, subframes spent in the find and MIB states)"""
    from ltesniffer_b200 import capi
    SF, L = 15 * N, x.shape[1]
    cs = capi.CellSearch(N, 2, 40 * SF)
    c = cs.search(x[:, :40 * SF])[0]
    cs.close()
    fo = int(c.frame_offset)
    nfr = (40 * SF - fo) // (10 * SF)
    mphy = capi.LtePhy(15, 2, pci, 2, max_subframes=nfr, symbol_sz=N)
    mphy.set_cfo(c.cfo_hz)
    mphy.submit_iq(np.stack([x[:, fo + k * 10 * SF:fo + k * 10 * SF + SF] for k in range(nfr)]), np.arange(nfr, dtype=np.uint32) * 10)
    k, mib = [(k, q.mib) for k, q in enumerate(mphy.mib_decode_combined(search_ports=True)) if q.mib.found][0]
    mphy.close()
    sfn = (mib.sfn + 1024 - k % 1024) % 1024
    phy = capi.LtePhy(25, 2, pci, 2, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER, symbol_sz=N,
                      phich_resources=mib.phich_resources, phich_length=mib.phich_length)
    srch = capi.Search(25, 2, pci, 2, phich_resources=mib.phich_resources)
    mibh = capi.LtePhy(mib.nof_prb, mib.nof_ports, pci, 2, max_subframes=1, symbol_sz=N)
    tr = capi.Tracker(N, 2, pci, fo, cfo_hz=c.cfo_hz, first_tti=10 * sfn, max_subframes=B, flags=capi.TRACK_REACQUIRE)
    L_ = phy.L
    md = 32 * B
    info, cands = (capi.SfInfo * B)(), np.zeros((B, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
    dcis, tbs, payload = np.zeros(md, capi.DCI_DTYPE), (capi.TbResult * (2 * md))(), np.zeros(B * 64 * 1024, np.uint8)
    expect, recv, awaiting, corr, first_after, spent = [], 0, False, 0, None, 0
    while True:
        if recv < L:
            recv = min(recv + B * SF, L)
        nxt = tr.next_sample
        if nxt >= recv:
            if recv == L:
                break
            continue
        o = tr.push(x[:, nxt:recv], nxt)
        spent += 10 * o["finds"]
        sf, m = o["sf"], len(o["sf"])
        if not m:
            if recv == L:
                break
            continue
        i0 = 0
        while i0 < m:
            if awaiting or sf["flags"][i0] & capi.TRACK_REACQUIRED:
                if sf["flags"][i0] & capi.TRACK_REACQUIRED:
                    mibh.mib_reset()
                    awaiting = True
                spent += 1
                if sf["tti"][i0] % 10 == 0:
                    t = np.array([sf["tti"][i0]], np.uint32)
                    mibh._chk(L_.ltephy_submit_iq_device(mibh.h, C.c_void_p(o["iq"][i0].data_ptr()), capi._p(t), 1), "submit_iq_device")
                    mibh.n = 1
                    q = mibh.mib_decode_combined()[0].mib
                    if q.found:
                        corr, awaiting = (q.sfn + 1024 - int(sf["tti"][i0]) // 10 % 1024) % 1024, False
                        first_after = len(expect)
                i0 += 1
                continue
            i1 = i0 + 1
            while i1 < m and not sf["flags"][i1] & capi.TRACK_REACQUIRED:
                i1 += 1
            tti = np.ascontiguousarray((sf["tti"][i0:i1].astype(np.int64) + 10 * corr) % 10240, np.uint32)
            iq = o["iq"][i0:i1].contiguous()
            nd = C.c_uint32(0)
            rc = L_.ltephy_decode_subframes_device(phy.h, srch.h, C.c_void_p(iq.data_ptr()), capi._p(tti), i1 - i0, capi.SEQ_NONE, info, capi._p(cands),
                                                   capi._p(dcis), md, C.byref(nd), tbs, capi._p(payload), payload.nbytes)
            assert rc == 0, L_.ltephy_last_error()
            for i, d in enumerate(dcis[:nd.value]):
                for t in range(2):
                    rr = tbs[2 * i + t]
                    if rr.crc and rr.payload_len:
                        expect.append((int(d["rnti"]), int(tti[int(d["sf"])]), bytes(payload[rr.payload_off:rr.payload_off + rr.payload_len])))
            i0 = i1
    tr.close(), phy.close(), srch.close(), mibh.close()
    return expect, first_after, spent


def _run(f, tmp_path, tag, N, B, reacq):
    pc, tsv = str(tmp_path / ("%s.pcap" % tag)), str(tmp_path / ("%s.tsv" % tag))
    r = subprocess.run([EXE, str(f), str(N), "2", pc, tsv, str(B), "50", "0", str(reacq)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stdout, open(pc, "rb").read(), open(tsv, "rb").read(), pc


def test_recording_with_a_drop_reads_the_sfn_again(infra, phylib, tmp_path):
    _build()
    N, pci, nsf, lead, B, SF = 512, 262, 2000, 4321, 200, 15 * 512
    cell = ltelib.Cell(25, 2, pci, 2, N)
    s = S.sim(sync=1, cell=cell, seed=71, pbch=1, snr_db=25.0, nof_ues=6, dl_min=2, dl_max=4, tm=13, mcs_min=2, mcs_max=16)
    sub = [s.subframe(t) for t in range(nsf)]
    tx = np.concatenate([np.zeros((2, lead))] + [q[0] for q in sub], axis=1)
    L = tx.shape[1] - 2 * T.TAPS
    n = np.arange(L)
    x = np.ascontiguousarray((T.resample(tx, 20.0, L) * np.exp(2j * np.pi * 1700.0 * n / (15000 * N))).astype(np.complex64))
    a, cnt = lead + 1000 * SF + 777, 37 * SF + 1234
    xd = np.ascontiguousarray(np.delete(x, np.s_[a:a + cnt], axis=1))
    f, fd = tmp_path / "rec.cf32", tmp_path / "drop.cf32"
    x.tofile(str(f)), xd.tofile(str(fd))

    # the loss-free recording: reacquire = 1 writes the same pcap, trace and lines, plus its own
    out0, pc0, ts0, _ = _run(f, tmp_path, "a0", N, B, 0)
    out1, pc1, ts1, _ = _run(f, tmp_path, "a1", N, B, 1)
    assert pc0 == pc1 and ts0 == ts1
    assert out1.splitlines()[:-1] == out0.splitlines() and out1.splitlines()[-1] == "reacquire: finds 0 reacquired 0 awaiting_mib 0"

    # the drop
    out, _, _, pc = _run(fd, tmp_path, "d1", N, B, 1)
    kv = out.splitlines()[-1].split()
    assert kv[0] == "reacquire:" and kv[1::2] == ["finds", "reacquired", "awaiting_mib"]
    finds, reacq, awaiting = (int(v) for v in kv[2::2])
    assert finds >= 1 and reacq == 1
    got = _read_pcap(pc)
    expect, first_after, spent = _binding_chain(xd, N, B, pci)
    assert got == expect
    assert first_after is not None and spent == 10 * finds + awaiting and spent <= 60, (first_after, spent, finds, awaiting)
    # every record after the fallback carries the truth tti, SFN included: the blocks the simulator sent in that subframe
    truth = set()
    for t in range(nsf):
        tr_, pl = sub[t][1], sub[t][2]
        for i in range(tr_.nof_dci):
            d = tr_.dci[i]
            for q in range(2):
                if d.nof_tb > q and d.tbs[q] > 0:
                    truth.add((int(d.rnti), t % 10240, bytes(pl[d.payload_off[q]:d.payload_off[q] + d.tbs[q] // 8])))
    after = got[first_after:]
    assert len(after) > 500 and set(after) <= truth, (len(after), len(set(after) - truth))
    # without the fallback the records after the drop are cut in the wrong place and decode nothing
    out0, _, _, pc0 = _run(fd, tmp_path, "d0", N, B, 0)
    assert "reacquire:" not in out0
    assert len(_read_pcap(pc0)) < first_after + 10
