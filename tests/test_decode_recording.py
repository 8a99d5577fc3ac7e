"""examples/decode_recording.cpp: raw recording in, pcap out.  CPU: it builds against libltephy_b200.so and without a GPU fails loudly.  GPU: on a
2 s, 25 PRB, 2x2 recording whose sampling clock is 20 ppm off, the cell and MIB it prints are the binding's, its pcap equals record for record
what the same chain driven through the Python binding writes (cell search -> combined MIB -> capi.Tracker push by push ->
ltephy_decode_subframes_device), and that pcap holds every transport block the simulator sent that the same decoder reads from the
simulator's own, perfectly aligned subframes."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import ltelib
import sync_lib as S
import track_lib as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "examples", "decode_recording")


def _build():
    from ltesniffer_b200 import capi
    capi.load_library()
    subprocess.run(["make", "-s", "-C", ROOT, "examples/decode_recording"], check=True)
    assert os.path.exists(EXE)


def _read_pcap(path):
    b = open(path, "rb").read()
    off, got = 24, []
    while off < len(b):
        ts, tu, il, ol = struct.unpack("<IIII", b[off:off + 16])
        rec = b[off + 16:off + 16 + il]
        off += 16 + il
        sfn_sf = (rec[10] << 8) | rec[11]
        got.append(((rec[4] << 8) | rec[5], (sfn_sf >> 4) * 10 + (sfn_sf & 15), rec[19:]))
    return got


def test_example_builds_and_refuses_to_run_without_a_gpu(infra, tmp_path):
    _build()
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a GPU is present: covered by the gpu test")
    except ImportError:
        pass
    iq = tmp_path / "x.cf32"
    iq.write_bytes(b"\0" * 8 * 512 * 15 * 40)
    r = subprocess.run([EXE, str(iq), "512", "1", str(tmp_path / "o.pcap"), str(tmp_path / "o.tsv")], capture_output=True, text=True)
    assert r.returncode == 1 and "no CUDA device" in r.stderr, (r.returncode, r.stderr)


@pytest.mark.gpu
def test_recording_to_pcap_at_20ppm(infra, phylib, tmp_path):
    import torch
    from ltesniffer_b200 import capi
    _build()
    N, pci, nsf, lead, B, SF = 512, 262, 2000, 4321, 200, 15 * 512
    cell = ltelib.Cell(25, 2, pci, 2, N)
    s = S.sim(sync=1, cell=cell, seed=71, pbch=1, snr_db=25.0, nof_ues=6, dl_min=2, dl_max=4, tm=13, mcs_min=2, mcs_max=16)
    sub = [s.subframe(t) for t in range(nsf)]
    tx = np.concatenate([np.zeros((2, lead))] + [q[0] for q in sub], axis=1)
    L = tx.shape[1] - 2 * T.TAPS
    n = np.arange(L)
    x = np.ascontiguousarray((T.resample(tx, 20.0, L) * np.exp(2j * np.pi * 1700.0 * n / (15000 * N))).astype(np.complex64))
    f = tmp_path / "rec.cf32"
    x.tofile(str(f))                                    # antenna-major
    pc, tsv = str(tmp_path / "o.pcap"), str(tmp_path / "o.tsv")
    r = subprocess.run([EXE, str(f), str(N), "2", pc, tsv, str(B)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    head = r.stdout.splitlines()[0].split()
    kv = {head[i]: head[i + 1] for i in range(0, len(head), 2)}
    # the binding-driven chain
    cs = capi.CellSearch(N, 2, 40 * SF)
    c = cs.search(x[:, :40 * SF])[0]
    cs.close()
    assert c.detected and c.pci == pci and int(kv["pci"]) == pci and int(kv["frame_offset"]) == c.frame_offset
    assert np.float32(float(kv["cfo_hz"])) == np.float32(c.cfo_hz)
    fo = int(c.frame_offset)
    nfr = (40 * SF - fo) // (10 * SF)
    sf0 = np.stack([x[:, fo + k * 10 * SF:fo + k * 10 * SF + SF] for k in range(nfr)])
    mphy = capi.LtePhy(15, 2, pci, 2, max_subframes=nfr, symbol_sz=N)
    mphy.set_cfo(c.cfo_hz)
    mphy.submit_iq(sf0, np.arange(nfr, dtype=np.uint32) * 10)
    mm = [(k, q.mib) for k, q in enumerate(mphy.mib_decode_combined(search_ports=True)) if q.mib.found]
    mphy.close()
    assert mm
    k, mib = mm[0]
    sfn = (mib.sfn + 1024 - k % 1024) % 1024
    assert (mib.nof_prb, mib.nof_ports, sfn) == (25, 2, 0)
    assert [int(kv[q]) for q in ("nof_prb", "nof_ports", "phich_resources", "phich_length", "sfn")] == \
        [mib.nof_prb, mib.nof_ports, mib.phich_resources, mib.phich_length, sfn]
    phy = capi.LtePhy(25, 2, pci, 2, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER, symbol_sz=N,
                      phich_resources=mib.phich_resources, phich_length=mib.phich_length)
    srch = capi.Search(25, 2, pci, 2, phich_resources=mib.phich_resources)
    tr = capi.Tracker(N, 2, pci, fo, cfo_hz=c.cfo_hz, first_tti=10 * sfn, max_subframes=B)
    L_ = phy.L
    md = 32 * B
    scratch = dict(info=(capi.SfInfo * B)(), cands=np.zeros((B, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE), dcis=np.zeros(md, capi.DCI_DTYPE),
                   tbs=(capi.TbResult * (2 * md))(), payload=np.zeros(B * 64 * 1024, np.uint8))
    expect, recv, nsf_done, lost = [], 0, 0, 0
    while True:
        if recv < L:
            recv = min(recv + B * SF, L)
        nxt = tr.next_sample
        if nxt >= recv:
            if recv == L:
                break
            continue
        o = tr.push(x[:, nxt:recv], nxt)
        m = len(o["sf"])
        if not m:
            if recv == L:
                break
            continue
        lost += int((o["sf"]["flags"] & capi.TRACK_LOST).sum())
        tti = np.ascontiguousarray(o["sf"]["tti"], np.uint32)
        nd = C.c_uint32(0)
        rc = L_.ltephy_decode_subframes_device(phy.h, srch.h, C.c_void_p(o["iq"].data_ptr()), capi._p(tti), m, capi.SEQ_NONE, scratch["info"],
                                               capi._p(scratch["cands"]), capi._p(scratch["dcis"]), md, C.byref(nd), scratch["tbs"],
                                               capi._p(scratch["payload"]), scratch["payload"].nbytes)
        assert rc == 0, L_.ltephy_last_error()
        for i, d in enumerate(scratch["dcis"][:nd.value]):
            for t in range(2):
                rr = scratch["tbs"][2 * i + t]
                if rr.crc and rr.payload_len:
                    expect.append((int(d["rnti"]), int(tti[int(d["sf"])]), bytes(scratch["payload"][rr.payload_off:rr.payload_off + rr.payload_len])))
        nsf_done += m
    tr.close(), phy.close(), srch.close()
    got = _read_pcap(pc)
    assert got == expect and nsf_done >= nsf - 5 and lost == 0
    assert ("subframes %d " % nsf_done) in r.stdout and "lost 0 " in r.stdout
    # every transport block the simulator sent in the subframes decoded is in the pcap, with its bytes
    have = set(got)
    truth = set()
    for t in range(nsf_done):
        tr_, pl = sub[t][1], sub[t][2]
        for i in range(tr_.nof_dci):
            d = tr_.dci[i]
            for q in range(2):
                if d.nof_tb > q and d.tbs[q] > 0:
                    truth.add((int(d.rnti), t % 10240, bytes(pl[d.payload_off[q]:d.payload_off[q] + d.tbs[q] // 8])))
    # the DCI search only accepts an RNTI once its history has seen it (rnti_histogram_threshold 5), so a few blocks of a UE's first subframes
    # are not reported even from a perfect cut: the yardstick is the same decoder on the simulator's own subframes (no clock or carrier offset)
    phy = capi.LtePhy(25, 2, pci, 2, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER, symbol_sz=N,
                      phich_resources=mib.phich_resources, phich_length=mib.phich_length)
    srch = capi.Search(25, 2, pci, 2, phich_resources=mib.phich_resources)
    ideal = set()
    for lo in range(0, nsf_done, B):
        hi = min(lo + B, nsf_done)
        tti = np.arange(lo, hi, dtype=np.uint32) % 10240
        info, dcis, tbs, payload = capi.decode_subframes(phy, srch, np.stack([sub[t][0] for t in range(lo, hi)]).astype(np.complex64), tti)
        for i, d in enumerate(dcis):
            for q in range(2):
                rr = tbs[2 * i + q]
                if rr.crc and rr.payload_len:
                    ideal.add((int(d["rnti"]), int(tti[int(d["sf"])]), bytes(payload[rr.payload_off:rr.payload_off + rr.payload_len])))
    phy.close(), srch.close()
    assert len(truth) > 1000 and len(truth & ideal) >= 0.99 * len(truth), (len(truth), len(truth & ideal))
    assert truth & ideal <= have, len((truth & ideal) - have)
