"""examples/offline_ul end to end on the GPU: the UL mode on a downlink and an uplink capture written subframe after subframe (the simulator's
aligned subframes, no clock or carrier offset).  Its pcap equals record for record the same chain driven through the binding: DL decode in UL
mode, RAR and DCI-0 grants carried across batches (a grant that lands past a short last batch stays carried), the uplink decode."""
import os
import struct
import subprocess

import numpy as np
import pytest

import track_lib as T
from helpers import UlModeStep

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "examples", "offline_ul")
N, PRB, PCI, PORTS, B = 512, 25, 262, 2, 200   # offline_ul takes no symbol size: 25 PRB reads subframes of 15 * 512 samples


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


def _example_and_chain(cap, tmp_path):
    """runs examples/offline_ul on the capture in batches of B, and the same chain through the binding -> dict(r: the example's
    CompletedProcess, got: its pcap records, expect: the chain's records, carried_beyond: the largest number of carried grants that fell
    beyond a batch, carry_left: grants still carried at the end)"""
    import torch
    subprocess.run(["make", "-s", "-C", ROOT, "examples/offline_ul"], check=True)
    n = cap.nsf
    dl = np.ascontiguousarray(np.stack([cap.dl[t][0][:1] for t in range(n)]), np.complex64)
    ul_iq = np.ascontiguousarray(np.stack(cap.ul), np.complex64)
    assert dl.shape == (n, 1, 15 * N) and ul_iq.shape == (n, 15 * N)
    fd, fu, pc = tmp_path / "dl.cf32", tmp_path / "ul.cf32", str(tmp_path / "o.pcap")
    dl.tofile(str(fd))
    ul_iq.tofile(str(fu))
    r = subprocess.run([EXE, str(fd), str(fu), str(PRB), str(PORTS), str(PCI), pc, str(B), "0", str(T.UCFG["n_dmrs1"]), str(T.UCFG["delta_ss"])],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    step = UlModeStep(PRB, PORTS, PCI, B)
    expect = []
    for lo in range(0, n, B):
        m = min(B, n - lo)
        expect += step(torch.from_numpy(dl[lo:lo + m]).cuda(), np.arange(lo, lo + m) % 10240, torch.from_numpy(ul_iq[lo:lo + m]).cuda())
    step.close()
    return dict(r=r, got=_read_pcap(pc), expect=expect, carried_beyond=step.beyond, carry_left=len(step.carry))


def _check(cap, e):
    """the example's pcap is the chain's, its summary counts that pcap, and every UL block in it is one the simulator sent"""
    got = e["got"]
    assert got == e["expect"]
    n_ul = sum(q[0] == 0 for q in got)
    assert ("subframes %d  dl blocks %d  dci0 " % (cap.nsf, len(got) - n_ul)) in e["r"].stdout, e["r"].stdout
    assert ("ul blocks %d\n" % n_ul) in e["r"].stdout, e["r"].stdout
    sent = {(k, rn, pl) for (k, rn, _), pl in cap.sent.items()}
    assert {(t, rn, p) for d, rn, t, p in got if d == 0} <= sent
    return n_ul


def test_offline_ul_to_pcap(infra, phylib, tmp_path):
    """1000 subframes in five full batches: grants carried across every batch boundary"""
    cap = T.TwoCarrier(N, PCI, 1000, seed=81, nof_ports=PORTS, mcs_max=20)
    e = _example_and_chain(cap, tmp_path)
    assert e["carried_beyond"] == 0
    assert _check(cap, e) > 500


def test_offline_ul_with_a_short_last_batch(infra, phylib, tmp_path):
    """202 subframes: the last batch holds 2 subframes, fewer than the grants carried into it reach; those stay carried, and the example still
    decodes the rest of that batch and prints its summary"""
    cap = T.TwoCarrier(N, PCI, 202, seed=82, nof_ports=PORTS, mcs_max=20)
    e = _example_and_chain(cap, tmp_path)
    assert e["carried_beyond"] >= 1 and e["carry_left"] >= 1, (e["carried_beyond"], e["carry_left"])
    assert _check(cap, e) > 50
