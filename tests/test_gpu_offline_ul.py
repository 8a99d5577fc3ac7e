"""examples/offline_ul end to end on the GPU: the UL mode on a downlink and an uplink capture written subframe after subframe (the simulator's
aligned subframes, no clock or carrier offset).  Its pcap equals record for record the same chain driven through the binding: DL decode in UL
mode, RAR and DCI-0 grants carried across batches (a grant that lands past a short last batch stays carried), ltephy_submit_ul on the uplink."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import track_ul_lib as U

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
    from ltesniffer_b200 import capi
    subprocess.run(["make", "-s", "-C", ROOT, "examples/offline_ul"], check=True)
    n = cap.nsf
    dl = np.ascontiguousarray(np.stack([cap.dl[t][0][:1] for t in range(n)]), np.complex64)
    ul_iq = np.ascontiguousarray(np.stack(cap.ul), np.complex64)
    assert dl.shape == (n, 1, 15 * N) and ul_iq.shape == (n, 15 * N)
    fd, fu, pc = tmp_path / "dl.cf32", tmp_path / "ul.cf32", str(tmp_path / "o.pcap")
    dl.tofile(str(fd))
    ul_iq.tofile(str(fu))
    r = subprocess.run([EXE, str(fd), str(fu), str(PRB), str(PORTS), str(PCI), pc, str(B), "0", str(U.UCFG["n_dmrs1"]), str(U.UCFG["delta_ss"])],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    mk = lambda: capi.LtePhy(PRB, PORTS, PCI, 1, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
    phy, ul = mk(), mk()
    ul.set_ul_cfg(**U.UCFG)
    srch = capi.Search(PRB, PORTS, PCI, 1)
    L_ = phy.L
    L_.ltephy_search_set_ul_mode(srch.h, 1, 0)
    L_.ltephy_search_set_ul_hopping(srch.h, 0)
    L_.ltephy_search_activate.argtypes = [C.c_void_p, C.c_uint16, C.c_uint32, C.c_int]
    md = 32 * B
    sc = dict(info=(capi.SfInfo * B)(), cands=np.zeros((B, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE), dcis=np.zeros(md, capi.DCI_DTYPE),
              tbs=(capi.TbResult * (2 * md))(), payload=np.zeros(B * 64 * 1024, np.uint8))

    def kept(now, res, pl, tti):
        """the UL records of one submit: the first attempt of a DCI-0 that passed (PUSCH_Decoder::decode stops there), as the example writes them"""
        out, passed = [], False
        for k, g in enumerate(now):
            if k == 0 or now[k - 1].rnti != g.rnti or now[k - 1].sf != g.sf:
                passed = False
            ok = res[k].crc and not passed
            passed = passed or res[k].crc != 0
            if ok and res[k].payload_len:
                out.append((0, int(g.rnti), int(tti[g.sf]), bytes(pl[res[k].payload_off:res[k].payload_off + res[k].payload_len])))
        return out

    expect, carry, beyond = [], [], 0
    for lo in range(0, n, B):
        m = min(B, n - lo)
        tti = np.arange(lo, lo + m, dtype=np.uint32) % 10240
        nd = C.c_uint32(0)
        assert L_.ltephy_decode_subframes(phy.h, srch.h, capi._p(dl[lo:lo + m]), capi._p(tti), m, capi.SEQ_NONE, sc["info"], capi._p(sc["cands"]),
                                          capi._p(sc["dcis"]), md, C.byref(nd), sc["tbs"], capi._p(sc["payload"]), sc["payload"].nbytes) == 0
        dcis = sc["dcis"][:nd.value].copy()
        now = [g for g in carry if g.sf < m]
        carry = [g for g in carry if g.sf >= m]
        beyond = max(beyond, len(carry))
        for i, d in enumerate(dcis):
            for t in range(2):
                rr = sc["tbs"][2 * i + t]
                if rr.crc and rr.payload_len:
                    expect.append((1, int(d["rnti"]), int(tti[int(d["sf"])]), bytes(sc["payload"][rr.payload_off:rr.payload_off + rr.payload_len])))
        for i, d in enumerate(dcis):
            rr = sc["tbs"][2 * i]
            if not (1 <= int(d["rnti"]) <= 10 and rr.crc and rr.payload_len):
                continue
            rc, rars, _ = capi.rar_unpack(srch, bytes(sc["payload"][rr.payload_off:rr.payload_off + rr.payload_len]))
            if rc != 0:
                continue
            for a in rars:
                L_.ltephy_search_activate(srch.h, a.t_crnti, 0, 2)
                if a.valid:
                    g = capi.UlGrant.from_buffer_copy(a.grant)
                    g.sf = int(d["sf"]) + 6
                    (now if g.sf < m else carry).append(g)
        for _, _, g in capi.ul_grants_from_dcis(srch, sc["info"], dcis):
            (now if g.sf < m else carry).append(g)
        for g in carry:
            g.sf -= m
        if now:
            res, _, pl = ul.decode_ul(ul_iq[lo:lo + m], tti, now)
            expect += kept(now, res, pl, tti)
    phy.close(), ul.close(), srch.close()
    return dict(r=r, got=_read_pcap(pc), expect=expect, carried_beyond=beyond, carry_left=len(carry))


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
    cap = U.TwoCarrier(N, PCI, 1000, seed=81, nof_ports=PORTS, mcs_max=20)
    e = _example_and_chain(cap, tmp_path)
    assert e["carried_beyond"] == 0
    assert _check(cap, e) > 500


def test_offline_ul_with_a_short_last_batch(infra, phylib, tmp_path):
    """202 subframes: the last batch holds 2 subframes, fewer than the grants carried into it reach; those stay carried, and the example still
    decodes the rest of that batch and prints its summary"""
    cap = U.TwoCarrier(N, PCI, 202, seed=82, nof_ports=PORTS, mcs_max=20)
    e = _example_and_chain(cap, tmp_path)
    assert e["carried_beyond"] >= 1 and e["carry_left"] >= 1, (e["carried_beyond"], e["carry_left"])
    assert _check(cap, e) > 50
