"""Tier-2 shim (libltephy_srsran_compat.so) on the GPU, driven the way the reference drives srsRAN, against tier 1 and the CPU oracle (pytest -m gpu).

examples/compat_check.cpp (downlink) and examples/compat_ul_check.cpp (uplink) call the srsRAN names; everything they get back must equal what
the tier-1 C-ABI returns for the same input, bit for bit, and decoded payloads must equal what the simulator sent:
  A. HARQ soft combining through srsran_softbuffer_rx_t, with the reference's buffer protocol (DL_Sniffer_PDSCH.cc:955-990), against the oracle's
     HARQ walk and tier 1 with explicit harq_op / harq_slot;
  B. the downlink across transmission schemes, bandwidths, symbol-size families, PHICH configurations and a second srsran_ue_dl_set_cell;
  C. the uplink (srsran_enb_ul_fft, srsran_chest_ul_estimate_pusch, srsran_pusch_decode) across DMRS configurations, modulations, UCI and
     hopping, including a decode whose configuration differs from the one just estimated;
  D. the soft-buffer lifecycle: reset, reuse, free / init, two TBs, no buffer, and a store with fewer slots than buffers."""
import ctypes as C
import os
import struct
import subprocess
import numpy as np
import pytest
import ltelib
from ltelib import Cell, Sim, Oracle, UlCfg
from helpers import make_capture, to_phy_grant, truth_grants, oracle_frontend
from test_harq import HARQ_CELL, HARQ_KW, harq_walk, oracle_harq_decoder
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DL_EXE = os.path.join(ROOT, "examples", "compat_check")
UL_EXE = os.path.join(ROOT, "examples", "compat_ul_check")
# soft-buffer operation of one TB in the downlink driver (enum SbOp of examples/compat_check.cpp)
SB_NULL, SB_SCRATCH, SB_NEW, SB_RETX, SB_DECODED, SB_RESET, SB_REINIT = range(7)
DMRS2 = [0, 6, 3, 4, 2, 8, 10, 9]          # 36.211 Table 5.5.2.1.1-1: DCI-0 cyclic-shift field -> n_DMRS^(2)
LIBM = C.CDLL("libm.so.6")
LIBM.log10f.argtypes, LIBM.log10f.restype = [C.c_float], C.c_float
LIBM.powf.argtypes, LIBM.powf.restype = [C.c_float, C.c_float], C.c_float


@pytest.fixture(scope="module")
def drivers(phylib):
    capi.load_library()
    subprocess.run(["make", "-s", "-C", ROOT, "examples/compat_check", "examples/compat_ul_check"], check=True)


def fnv(b):
    h = 1469598103934665603
    for x in np.frombuffer(b, np.uint8).tolist():
        h = ((h ^ x) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


# ------------------------------------------------------------------------------------------------------------------ downlink
class Step:
    """one srsran_ue_dl_decode_pdsch call: grant of subframe sf, the driver's soft-buffer operation and buffer per TB, and the tier-1 harq_op and
    harq_slot per TB that must give the same result (slot: the buffer number unless given)"""

    def __init__(self, sf, rnti, pg, sb=(SB_NULL, SB_NULL), buf=(0, 0), op=(capi.HARQ_NONE, capi.HARQ_NONE), slot=None):
        self.sf, self.rnti, self.pg, self.sb, self.buf, self.op = sf, rnti, pg, tuple(sb), tuple(buf), tuple(op)
        self.slot = tuple(buf) if slot is None else tuple(slot)


def run_dl_shim(tmp_path, cell, iq, tti, steps, sizes, opts=()):
    """-> (per-subframe records, per-step [(crc, payload bytes)] * 2)"""
    f = tmp_path / "cap.cf32"
    iq.astype(np.complex64).tofile(str(f))
    harq = "--harq" in opts
    with open(tmp_path / "grants.bin", "wb") as gf:
        for s in steps:
            gf.write(struct.pack("<II", s.sf, s.rnti) + bytes(s.pg))
            if harq:
                gf.write(struct.pack("<BBHH", s.sb[0], s.sb[1], s.buf[0], s.buf[1]))
    out = tmp_path / "out.bin"
    opts = ["--phich=%d,%d" % (cell.phich_ng, cell.phich_ext)] + list(opts)
    r = subprocess.run([DL_EXE] + opts + [str(f), str(cell.nof_prb), str(cell.nof_ports), str(cell.cell_id), str(cell.nof_rx), str(len(tti)),
                       str(int(tti[0])), str(tmp_path / "grants.bin"), str(out)] + [str(s) for s in sizes], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    b = out.read_bytes()
    off, sfs, tbs = 0, [], []
    for i in range(len(tti)):
        cfi, snr, noise, cfo, hs, hc, ncce = struct.unpack_from("<IfffQQI", b, off)
        off += struct.calcsize("<IfffQQI")
        llr = np.frombuffer(b, np.float32, 72 * ncce, off)
        off += 4 * 72 * ncce
        lim = min(ncce, 84)
        nloc = sum(lim >> L for L in range(4))
        dci = []
        for _ in range(nloc * len(sizes)):
            dci.append(struct.unpack_from("<HQ", b, off))
            off += 10
        sfs.append(dict(cfi=cfi, snr=snr, noise=noise, cfo=cfo, hs=hs, hc=hc, ncce=ncce, llr=llr, dci=dci))
        for s in steps:
            if s.sf != i:
                continue
            tb = []
            for t in range(2):
                crc, nby = struct.unpack_from("<BI", b, off)
                off += 5
                tb.append((crc, b[off:off + nby]))
                off += nby
            tbs.append(tb)
    assert off == len(b)
    return sfs, tbs


def tier1_replay(cell, iq, tti, steps, nslots=0):
    """tier 1 decoding the steps one grant at a time, each subframe's phase A first, with the steps' harq_op and harq_slot"""
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=1, turbo_max_iter=8, symbol_sz=cell.symbol_sz,
                      phich_resources=cell.phich_ng, phich_length=cell.phich_ext)
    if nslots:
        phy.harq_reserve(nslots)
    out, cur = [], -1
    for s in steps:
        if s.sf != cur:
            phy.submit_iq(iq[s.sf:s.sf + 1], tti[s.sf:s.sf + 1])
            phy.get_phase_a()
            cur = s.sf
        pg = capi.Grant.from_buffer_copy(s.pg)
        pg.sf = 0
        for t in range(2):
            if s.sb[t] == SB_DECODED:
                pg.tb[t].enabled = 0
            pg.tb[t].harq_op, pg.tb[t].harq_slot = (s.op[t], s.slot[t]) if pg.tb[t].enabled else (capi.HARQ_NONE, 0)
        if not (pg.tb[0].enabled or pg.tb[1].enabled):
            out.append([(0, b""), (0, b"")])
            continue
        phy.submit_grants([pg])
        res, pl = phy.get_phase_b()
        out.append([(int(res[t].crc != 0), bytes(pl[res[t].payload_off:res[t].payload_off + res[t].payload_len])) for t in range(2)])
    phy.close()
    return out


def distinct_sizes(phy):
    sizes, _ = phy.sizes()
    out = []
    for s in sizes:
        if s not in out:
            out.append(s)
    return out


def check_dl_matrix(tmp_path, cell, n, kw, opts=(), alt=0, extra=None):
    """shim == one tier-1 batch for sf_symbols, ce, PDCCH LLRs, every (location, size) decode, every TB; decoded payloads == what was sent.
    extra(sf, cfi) -> [(rnti, DlGrant)]: grants added to the simulator's (their payloads are not known)"""
    sim, iq, tti, truths, payloads = make_capture(cell, n, **kw)
    tg = truth_grants(cell, truths, tti, alt)
    items = [(sf, d.rnti, g, d) for sf, d, g in tg]
    if extra:
        for sf in range(n):
            items += [(sf, rnti, g, None) for rnti, g in extra(sf, truths[sf].cfi)]
    items.sort(key=lambda x: x[0])
    steps = [Step(sf, rnti, to_phy_grant(sf, rnti, g)) for sf, rnti, g, _ in items]
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8, symbol_sz=cell.symbol_sz,
                      phich_resources=cell.phich_ng, phich_length=cell.phich_ext)
    phy.submit_iq(iq, tti)
    info, cands = phy.get_phase_a()
    g = 14 * 12 * cell.nof_prb
    sym = phy.tap(capi.TAP_SYM, (n, cell.nof_rx, g), np.complex64)
    ce = phy.tap(capi.TAP_CE, (n, cell.nof_ports, cell.nof_rx, g), np.complex64)
    llr = phy.tap(capi.TAP_LLR, (n, capi.LLR_STRIDE), np.float32)
    phy.submit_grants([s.pg for s in steps])
    res, pl = phy.get_phase_b()
    sizes = distinct_sizes(phy)
    sfs, tbs = run_dl_shim(tmp_path, cell, iq, tti, steps, sizes, opts)
    for i, r in enumerate(sfs):
        assert r["cfi"] == info[i].cfi and np.float32(r["snr"]) == np.float32(info[i].snr_db) and np.float32(r["noise"]) == np.float32(info[i].noise_avg)
        assert np.float32(r["cfo"]) == np.float32(info[i].cfo)
        es = 0
        for a in range(cell.nof_rx):
            es ^= (fnv(sym[i, a].tobytes()) * (a + 1)) & 0xFFFFFFFFFFFFFFFF
        ec = 0
        for p in range(cell.nof_ports):
            for a in range(cell.nof_rx):
                ec ^= (fnv(ce[i, p, a].tobytes()) * (p * 2 + a + 1)) & 0xFFFFFFFFFFFFFFFF
        assert r["hs"] == es and r["hc"] == ec, "sf %d: sf_symbols / ce handed out by the shim differ from the device buffers" % i
        assert r["ncce"] == phy.nof_cce(r["cfi"])
        assert np.array_equal(r["llr"].view(np.uint32), llr[i, :72 * r["ncce"]].view(np.uint32))
        nc, Ls = phy.locations(r["cfi"])
        assert len(r["dci"]) == len(nc) * len(sizes)
        for li in range(len(nc)):
            for si in range(len(sizes)):
                c = cands[i, li, si]
                assert r["dci"][li * len(sizes) + si] == ((int(c["rnti"]), int(c["bits"])) if c["valid"] else (0, 0)), (i, li, sizes[si])
    nok = 0
    for k, ((sf, rnti, gg, d), tb) in enumerate(zip(items, tbs)):
        for t in range(2):
            rr = res[2 * k + t]
            crc, data = tb[t]
            assert len(data) == rr.payload_len and bool(crc) == bool(rr.crc), (sf, hex(rnti), t)
            assert data == bytes(pl[rr.payload_off:rr.payload_off + rr.payload_len]), (sf, hex(rnti), t)
            if crc and d is not None:
                assert data == bytes(payloads[sf][d.payload_off[t]:d.payload_off[t] + d.tbs[t] // 8]), (sf, hex(rnti), t)
                nok += 1
    phy.close()
    return items, tbs, nok


def _items_of(items, pred):
    return [(sf, rnti, g) for sf, rnti, g, d in items if pred(g)]


def test_port0_one_antenna_50prb(infra, drivers, tmp_path):
    items, tbs, nok = check_dl_matrix(tmp_path, Cell(50, 1, 71, 1), 3, dict(seed=21, cfi=2, nof_ues=5, dl_min=2, dl_max=4, tm=1, mcs_min=2, mcs_max=20,
                                                                             snr_db=28.0, si_period=2))
    assert nok >= sum(1 for *_, d in items for t in range(2) if d is not None and d.tbs[t] > 0) - 1


def test_sfbc_2x2_15prb_noguru(infra, drivers, tmp_path):
    """transmit diversity; odd subframes enter through srsran_ue_dl_decode_fft_estimate_noguru from other buffers"""
    items, tbs, nok = check_dl_matrix(tmp_path, Cell(15, 2, 33, 2), 4, dict(seed=22, cfi=3, nof_ues=4, dl_min=1, dl_max=2, tm=1, mcs_min=2, mcs_max=18,
                                                                             snr_db=26.0), opts=["--noguru"])
    assert all(g.tx_scheme == capi.TX_DIVERSITY for *_, g, d in items) and nok >= len(items) - 1


def test_tm3_two_codewords_swapped_pdsch_decode(infra, drivers, tmp_path):
    """CDD with both TBs, the DCI 2A swap flag set at random; through srsran_pdsch_decode"""
    items, tbs, nok = check_dl_matrix(tmp_path, Cell(25, 2, 150, 2), 6, dict(seed=23, cfi=2, nof_ues=5, dl_min=2, dl_max=3, tm=3, mcs_min=4, mcs_max=20,
                                                                              snr_db=30.0, tb_swap=1), opts=["--pdsch-decode"])
    assert any(g.cw_swap and g.nof_tb == 2 for *_, g, d in items) and nok >= 4


def test_tm4_256qam_100prb(infra, drivers, tmp_path):
    """closed-loop spatial multiplexing with 1 and 2 layers, 256QAM table: the largest two-TB payloads of one grant"""
    items, tbs, nok = check_dl_matrix(tmp_path, Cell(100, 2, 35, 2), 3, dict(seed=24, cfi=1, nof_ues=2, dl_min=1, dl_max=2, tm=4, mcs_min=24, mcs_max=27,
                                                                              snr_db=38.0, alt_table=1, full_band=1), alt=1)
    assert {g.nof_tb for *_, g, d in items} == {1, 2}, "the capture must hold 1- and 2-layer grants"
    assert max(len(tb[0][1]) + len(tb[1][1]) for tb in tbs) > 16000 and nok >= 2


@pytest.mark.parametrize("prb,N", [(100, 1536), (50, 768)])
def test_rate34_symbol_size(infra, drivers, tmp_path, prb, N):
    """srsRAN's default 3/4-rate sampling: srsran_use_standard_symbol_size is never called"""
    items, tbs, nok = check_dl_matrix(tmp_path, Cell(prb, 2, 36 + prb, 2, N), 3, dict(seed=25, cfi=2, nof_ues=5, dl_min=2, dl_max=3, tm=13, mcs_min=2,
                                                                                       mcs_max=18, snr_db=27.0), opts=["--rate34"])
    assert nok >= len(items) - 1


def _format1c_si_grant(cell, sf_idx, cfi, seed):
    """a format-1C SI-RNTI grant with distributed VRBs: slot 1's PRBs differ from slot 0's"""
    S = ltelib.sim()
    nb = S.lte_dci_sizeof(C.byref(cell), 4)
    rng = np.random.default_rng(seed)
    for _ in range(2000):
        bits = rng.integers(0, 2, nb).astype(np.uint8)
        r, dd, g = ltelib.unpack_and_grant(cell, 4, 0xFFFF, bits, sf_idx, cfi, 0)
        if r == 0 and g.nof_tb and any(g.prb_mask[0][p] != g.prb_mask[1][p] for p in range(cell.nof_prb)):
            return g
    raise AssertionError("no distributed format-1C grant found")


def test_ng2_extended_phich_with_format1c(infra, drivers, tmp_path):
    """Ng = 2, extended PHICH duration (CFI 3), and a format-1C SI grant per subframe: its two slots use different PRBs"""
    cell = Cell(50, 2, 38, 2, 0, 3, 1)
    extra = lambda sf, cfi: [(0xFFFF, _format1c_si_grant(cell, (4 + sf) % 10, cfi, 90 + sf))]
    items, tbs, nok = check_dl_matrix(tmp_path, cell, 3, dict(seed=26, cfi=3, nof_ues=4, dl_min=1, dl_max=2, tm=13, mcs_min=2, mcs_max=16, snr_db=27.0,
                                                                tti0=4), extra=extra)
    assert sum(1 for *_, d in items if d is None) == 3 and nok >= 3


def test_second_set_cell_on_the_same_object(infra, drivers, tmp_path):
    """srsran_ue_dl_set_cell with another cell (50 PRB, 1 port, PCI 12) and one subframe through it, then the cell of the capture"""
    items, tbs, nok = check_dl_matrix(tmp_path, Cell(25, 2, 39, 2), 3, dict(seed=27, cfi=2, nof_ues=4, dl_min=1, dl_max=3, tm=13, mcs_min=2, mcs_max=16,
                                                                             snr_db=27.0), opts=["--pre-cell=50,1,12"])
    assert nok >= len(items) - 1


# ------------------------------------------------------------------------------------------------------------------ HARQ (A, D)
def _harq_capture():
    cell = Cell(*HARQ_CELL)
    sim, iq, tti, truths, payloads = make_capture(cell, 16, **HARQ_KW)
    return cell, iq, tti, truths, payloads


def test_harq_through_soft_buffers(infra, drivers, tmp_path):
    """the reference's HARQ mode through the shim: getHARQBuffer + reset_tbs for a new transmission, getHARQBuffer alone for a retransmission, the TB
    disabled once decoded (DL_Sniffer_PDSCH.cc:955-990).  Every TB equals the oracle's HARQ walk and tier 1 with explicit harq_op / harq_slot."""
    cell, iq, tti, truths, payloads = _harq_capture()
    o = ltelib.Oracle(cell)
    fe = oracle_frontend(o, iq, tti)
    odec = oracle_harq_decoder(o, fe, tti, {})
    steps = []

    def decode(sf, d, dd, g, ops, slots):
        sb = [{capi.HARQ_NEW: SB_NEW, capi.HARQ_RETX: SB_RETX, -1: SB_DECODED}.get(ops[t], SB_NULL) if g.tb[t].enabled else SB_NULL for t in range(2)]
        steps.append(Step(sf, d.rnti, to_phy_grant(sf, d.rnti, g), sb, slots, [max(op, 0) for op in ops]))
        return odec(sf, d, dd, g, ops, slots)
    ref = harq_walk(cell, iq, tti, truths, decode)
    sfs, got = run_dl_shim(tmp_path, cell, iq, tti, steps, distinct_sizes(capi.LtePhy(*HARQ_CELL, max_subframes=1)), ["--harq"])
    t1 = tier1_replay(cell, iq, tti, steps, nslots=150 * 16)
    ncomb = 0
    for s, (sf, rnti, ops, crc), tb, tt in zip(steps, ref, got, t1):
        assert (s.sf, s.rnti) == (sf, rnti)
        if ops[0] == -1:
            assert tb[0] == (0, b"") == tt[0]              # already decoded: not decoded again
            continue
        assert tb[0] == tt[0], ("shim != tier 1", sf, hex(rnti), ops, tb[0][0], tt[0][0])
        assert tb[0][0] == crc[0], ("shim != oracle HARQ walk", sf, hex(rnti), ops, tb[0][0], crc[0])
        if crc[0]:
            assert tb[0][1] == bytes(odec.payloads[(sf, rnti)][0][:len(tb[0][1])])
            d = [x for x in truths[sf].dci[:truths[sf].nof_dci] if x.rnti == rnti][0]
            assert tb[0][1] == bytes(payloads[sf][d.payload_off[0]:d.payload_off[0] + d.tbs[0] // 8])
        ncomb += ops[0] == capi.HARQ_RETX and crc[0]
    assert ncomb >= 15


def _first_and_retx(truths, tti, cell):
    """[(sf, rnti, DlGrant of the first transmission, DlGrant of its retransmission 8 ms later)] of the HARQ capture"""
    tg = truth_grants(cell, truths, tti)
    first = {(sf, d.rnti): g for sf, d, g in tg if sf < 8}
    return [(sf - 8, d.rnti, first[(sf - 8, d.rnti)], g) for sf, d, g in tg if sf >= 8 and (sf - 8, d.rnti) in first]


def _check_lifecycle(tmp_path, cell, iq, tti, steps, opts, nslots):
    sfs, got = run_dl_shim(tmp_path, cell, iq, tti, steps, distinct_sizes(capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx,
                                                                                      max_subframes=1)), ["--harq"] + list(opts))
    t1 = tier1_replay(cell, iq, tti, steps, nslots=nslots)
    bad = ["step %d (sf %d, rnti %s, buffer ops %s, buffers %s, expected harq ops %s): shim crc %s, tier 1 crc %s" %
           (k, s.sf, hex(s.rnti), s.sb, s.buf, s.op, [x[0] for x in tb], [x[0] for x in tt]) for k, (s, tb, tt) in enumerate(zip(steps, got, t1)) if tb != tt]
    assert len(got) == len(t1) == len(steps) and not bad, "\n".join(bad)
    return got


def test_soft_buffer_lifecycle(infra, drivers, tmp_path):
    """a reset buffer, a buffer reset for another RNTI / TBS, a buffer freed and initialised again at the same address and a decode without a buffer
    all equal a decode on its own; a buffer used again without a reset combines"""
    cell, iq, tti, truths, payloads = _harq_capture()
    pairs = _first_and_retx(truths, tti, cell)
    assert len(pairs) >= 6
    N, R, X = capi.HARQ_NONE, capi.HARQ_RETX, capi.HARQ_NEW
    plan = [  # (retransmission's soft-buffer op, buffer of the retransmission, tier-1 op of the retransmission)
        (SB_RETX, 0, R),        # combines: the control
        (SB_RESET, 1, X),       # srsran_softbuffer_rx_reset: empty
        (SB_NEW, 0, X),         # buffer 0, which pair 0 just combined in, reset_tbs for this RNTI / TBS: nothing of pair 0 left in it
        (SB_REINIT, 3, X),      # freed and initialised again at the same address: empty
        (SB_NULL, 0, N),        # no soft buffer
        (SB_SCRATCH, 0, X),     # the scratch buffer with reset_tbs
    ]
    first, second = [], []
    for k, (sf, rnti, g1, g2) in enumerate(pairs[:len(plan)]):
        first.append(Step(sf, rnti, to_phy_grant(sf, rnti, g1), (SB_NEW, SB_NULL), (k, 0), (X, N)))
        op, b, t1op = plan[k]
        second.append(Step(sf + 8, rnti, to_phy_grant(sf + 8, rnti, g2), (op, SB_NULL), (b, 0), (t1op, N)))
    # tier 1 decodes these two into slots of their own (an overwrite, so any slot would do); the driver reuses its buffer 0 and its scratch buffer
    second[2].slot = (10, 0)
    second[5].slot = (11, 0)
    steps = sorted(first, key=lambda s: s.sf) + sorted(second, key=lambda s: s.sf)
    # pair 0 combines in buffer 0 before pair 2 takes it over: a shim that keyed slots on the buffer's address alone would combine pair 2 with it
    assert steps.index(second[0]) < steps.index(second[2]) and pairs[0][1] != pairs[2][1]
    got = _check_lifecycle(tmp_path, cell, iq, tti, steps, [], 16)
    assert got[len(first)][0][0] == 1, "the combined retransmission must pass"
    assert sum(tb[0][0] for tb in got[len(first) + 1:]) <= 2, "the retransmissions decoded on their own mostly fail at this SNR"


def test_harq_slots_run_out(infra, drivers, tmp_path):
    """ltephy_compat_harq_slots(2) and three buffers: the buffer decoded least recently loses its slot and starts empty at its next decode"""
    cell, iq, tti, truths, payloads = _harq_capture()
    pairs = _first_and_retx(truths, tti, cell)
    by_sf = {}
    for p in pairs:
        by_sf.setdefault(p[0], []).append(p)
    sf3 = [v for v in by_sf.values() if len(v) >= 3][0][:3]
    N, R, X = capi.HARQ_NONE, capi.HARQ_RETX, capi.HARQ_NEW
    a, b, c = sf3
    steps = [Step(a[0], p[1], to_phy_grant(a[0], p[1], p[2]), (SB_NEW, SB_NULL), (k, 0), (X, N)) for k, p in enumerate(sf3)]   # c evicts a
    sf = a[0] + 8
    steps += [Step(sf, c[1], to_phy_grant(sf, c[1], c[3]), (SB_RETX, SB_NULL), (2, 0), (R, N)),       # kept its slot: combines
              Step(sf, a[1], to_phy_grant(sf, a[1], a[3]), (SB_RETX, SB_NULL), (0, 0), (X, N)),       # lost its slot: on its own (evicts b)
              Step(sf, b[1], to_phy_grant(sf, b[1], b[3]), (SB_RETX, SB_NULL), (1, 0), (X, N))]       # lost its slot too
    steps.sort(key=lambda s: s.sf)
    _check_lifecycle(tmp_path, cell, iq, tti, steps, ["--harq-slots=2"], 4)


def test_two_tbs_of_one_grant_use_two_slots(infra, drivers, tmp_path):
    """TM3 retransmissions of both TBs: each TB combines with its own earlier transmission"""
    cell = Cell(25, 2, 150, 2)
    sim, iq, tti, truths, payloads = make_capture(cell, 16, seed=12, cfi=2, nof_ues=3, dl_min=2, dl_max=3, tm=3, mcs_min=14, mcs_max=16, snr_db=9.0,
                                                  full_band=1, harq_retx=1)
    pairs = [p for p in _first_and_retx(truths, tti, cell) if p[2].nof_tb == 2]
    assert len(pairs) >= 3
    R, X = capi.HARQ_RETX, capi.HARQ_NEW
    steps = []
    for k, (sf, rnti, g1, g2) in enumerate(pairs):
        steps.append(Step(sf, rnti, to_phy_grant(sf, rnti, g1), (SB_NEW, SB_NEW), (2 * k, 2 * k + 1), (X, X)))
        steps.append(Step(sf + 8, rnti, to_phy_grant(sf + 8, rnti, g2), (SB_RETX, SB_RETX), (2 * k, 2 * k + 1), (R, R)))
    steps.sort(key=lambda s: s.sf)
    got = _check_lifecycle(tmp_path, cell, iq, tti, steps, [], 2 * len(pairs))
    assert sum(tb[t][0] for s, tb in zip(steps, got) if s.sf >= 8 for t in range(2)) >= 2


# ------------------------------------------------------------------------------------------------------------------ uplink (C)
class UlRec:
    """one grant as the uplink driver hands it to the shim: mode 0 estimate + decode, 1 estimate only, 2 decode only"""

    def __init__(self, g, mode=0, cqi=(0, 0, 0, 0, 0), sent=True):
        self.g, self.mode, self.cqi, self.sent = g, mode, cqi, sent      # cqi: (data_enable, type, N, L, rank_is_not_one)

    def pack(self, sf):
        g = self.g
        return struct.pack("<20I", sf, self.mode, g.rnti, g.qm, g.rv, g.L_prb, g.n_prb, g.n_prb_slot1 if g.hop else g.n_prb, DMRS2.index(g.n_dmrs2),
                           g.tbs, g.nof_ack, g.ri_len, *self.cqi, g.I_offset_ack, g.I_offset_cqi, g.I_offset_ri)


def cqi_size(cqi):
    """36.212 5.2.2.6.1-3: CQI bits on PUSCH of each report type (the srsRAN type numbering of uci_cfg.h)"""
    en, typ, N, L, rank = cqi
    if not en:
        return 0
    return {0: 4, 3: 4 + (4 if rank else 0) + 2 * N * (2 if rank else 1), 1: 4 + 2 + L}.get(typ, 7)


def ul_grant(cell, rnti, L, start, mcs, n_dmrs, table=2):
    S = ltelib.sim()
    S.lte_ul_dci_to_grant.argtypes = [C.POINTER(Cell), C.POINTER(ltelib.Dci), C.c_int, C.POINTER(ltelib.UlGrant)]
    N = cell.nof_prb
    d = ltelib.Dci()
    d.format, d.rnti, d.alloc_type = 0, rnti, 2
    d.riv = N * (L - 1) + start if (L - 1) <= N // 2 else N * (N - L + 1) + (N - 1 - start)
    d.mcs[0], d.n_dmrs = mcs, n_dmrs
    g = ltelib.UlGrant()
    assert S.lte_ul_dci_to_grant(C.byref(cell), C.byref(d), table, C.byref(g)) == 0
    assert (g.L_prb, g.n_prb, g.n_dmrs2) == (L, start, DMRS2[n_dmrs])
    return g


def check_ul(tmp_path, cell, ucfg, subframes, snr=32.0, seed=5, rate34=False, tier1=None):
    """subframes: per subframe a list of UlRec; the sent ones are transmitted by the simulator.  The shim's estimate and decode of every record equal
    tier 1 (ltephy_submit_ul / ltephy_get_ul) and the oracle (lteo_pusch_decode) for that record's configuration; sent blocks that pass equal the truth.
    Returns the number of sent blocks that passed; tier1 (a list) receives tier 1's (crc, payload) of every record, estimate-only ones included."""
    s = Sim(cell=cell, seed=seed, snr_db=snr, nof_ues=1)
    n = len(subframes)
    tti = np.arange(6, 6 + n, dtype=np.uint32)
    iq = np.zeros((n, s.sf_len), np.complex64)
    sent_pl = []
    for i, recs in enumerate(subframes):
        for r in recs:
            r.g.cqi_len = cqi_size(r.cqi)
        sent = [r.g for r in recs if r.sent]
        x, pl, off = ltelib.sim_ul_subframe(s, int(tti[i]), ucfg, sent)
        iq[i] = x
        sent_pl.append({id(g): pl[o:o + g.tbs // 8] for g, o in zip(sent, off)})
    f = tmp_path / "ul.cf32"
    iq.tofile(str(f))
    with open(tmp_path / "ulgrants.bin", "wb") as gf:
        for i, recs in enumerate(subframes):
            for r in recs:
                gf.write(r.pack(i))
    out = tmp_path / "ulout.bin"
    cmd = [UL_EXE] + (["--rate34"] if rate34 else []) + [str(f), str(cell.nof_prb), str(cell.cell_id), str(n), str(int(tti[0])), str(ucfg.n_dmrs1),
                                                         str(ucfg.delta_ss), str(ucfg.group_hopping), str(ucfg.seq_hopping), str(tmp_path / "ulgrants.bin"), str(out)]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    # tier 1 and the oracle: every record's configuration, one grant list per subframe
    phy = capi.LtePhy(cell.nof_prb, 1, cell.cell_id, 1, max_subframes=n, symbol_sz=cell.symbol_sz)
    phy.set_ul_cfg(ucfg.n_dmrs1, ucfg.delta_ss, ucfg.group_hopping, ucfg.seq_hopping)
    gp = [capi.UlGrant(sf=i, rnti=r.g.rnti, qm=r.g.qm, rv=r.g.rv, L_prb=r.g.L_prb, n_prb=r.g.n_prb, n_dmrs2=r.g.n_dmrs2, tbs=r.g.tbs,
                       n_prb_slot1=r.g.n_prb_slot1 if r.g.hop else r.g.n_prb, flags=capi.UL_FLAG_SLOT1, nof_ack=r.g.nof_ack, ri_len=r.g.ri_len,
                       cqi_len=r.g.cqi_len, I_offset_ack=r.g.I_offset_ack, I_offset_ri=r.g.I_offset_ri, I_offset_cqi=r.g.I_offset_cqi)
          for i, recs in enumerate(subframes) for r in recs]
    res, ch, payload = phy.decode_ul(iq, tti, gp)
    phy.close()
    if tier1 is not None:
        tier1 += [(res[k].crc, bytes(payload[res[k].payload_off:res[k].payload_off + res[k].payload_len])) for k in range(len(gp))]
    o = Oracle(cell)
    b = out.read_bytes()
    off = k = nok = 0
    for i, recs in enumerate(subframes):
        _, oref = ltelib.oracle_ul(o, ucfg, int(tti[i]), [r.g for r in recs], iq[i])
        for r, (orc, opl, ocrc, och, _) in zip(recs, oref):
            assert orc == 0
            (cqi_len,) = struct.unpack_from("<I", b, off)
            off += 4
            assert cqi_len == r.g.cqi_len, ("srsran_cqi_size", r.cqi, cqi_len, r.g.cqi_len)
            what = (i, hex(r.g.rnti), r.mode)
            if r.mode != 2:
                noise, dbm, rsrp, snr_db, snr_lin, ta = struct.unpack_from("<6f", b, off)
                off += 24
                assert (noise, rsrp, snr_db) == (ch[k].noise, ch[k].rsrp, ch[k].snr_db) == (och.noise, och.rsrp, och.snr_db), what
                assert dbm == np.float32(LIBM.log10f(ch[k].noise) * np.float32(10.0) + np.float32(30.0)), (what, dbm, ch[k].noise)
                assert snr_lin == LIBM.powf(10.0, np.float32(ch[k].snr_db) / np.float32(10.0)) and ta == ch[k].ta_us, what
            if r.mode != 1:
                crc, nby = struct.unpack_from("<BI", b, off)
                off += 5
                data = b[off:off + nby]
                off += nby
                rr = res[k]
                assert nby == rr.payload_len == r.g.tbs // 8
                assert (crc, data) == (rr.crc, bytes(payload[rr.payload_off:rr.payload_off + nby])), ("shim != tier 1", what, crc, rr.crc)
                assert (crc, data) == (ocrc, bytes(opl[:nby])), ("shim != oracle", what, crc, ocrc)
                if crc and r.sent:
                    assert data == bytes(sent_pl[i][id(r.g)]), what
                    nok += 1
            k += 1
    assert off == len(b)
    return nok


@pytest.mark.parametrize("cs", range(8))
def test_ul_every_cyclic_shift_and_dmrs_field(infra, drivers, tmp_path, cs):
    """SIB2 cyclicShift cs; two grants whose DCI cyclic-shift fields, over the eight cases, take every value 0..7"""
    cell = Cell(25, 1, 40 + cs, 1)
    recs = [UlRec(ul_grant(cell, 0x100 + cs, 6, 0, 8, (2 * cs) % 8)), UlRec(ul_grant(cell, 0x200 + cs, 10, 8, 3, (2 * cs + 1) % 8))]
    assert check_ul(tmp_path, cell, UlCfg(n_dmrs1=cs, delta_ss=(3 * cs) % 30), [recs], seed=30 + cs) == 2


@pytest.mark.parametrize("gh,sh", [(1, 0), (0, 1)])
def test_ul_group_and_sequence_hopping_type1_hopping(infra, drivers, tmp_path, gh, sh):
    """DMRS group / sequence hopping (sequence hopping from 6 PRB on), and type-1 PUSCH hopping: slot 1 elsewhere"""
    cell = Cell(50, 1, 301, 1)
    subframes = []
    for i in range(2):
        g0, g1 = ul_grant(cell, 0x300 + i, 8, 2, 10, 3), ul_grant(cell, 0x400 + i, 12, 20, 5, 6)
        g0.hop, g0.n_prb_slot1 = 1, 36
        subframes.append([UlRec(g0), UlRec(g1)])
    assert check_ul(tmp_path, cell, UlCfg(n_dmrs1=2, delta_ss=11, group_hopping=gh, seq_hopping=sh), subframes, seed=60 + gh) == 4


@pytest.mark.parametrize("prb,N", [(100, 0), (50, 768)])
def test_ul_modulations_and_uci(infra, drivers, tmp_path, prb, N):
    """four grants per subframe with Qm 2, 4, 6 and 8 (36.213 Table 8.6.1-3); ACK, RI and CQI multiplexed, with the CQI size of each report type;
    standard and 3/4-rate symbol sizes"""
    cell = Cell(prb, 1, 77, 1, N)
    uci = [dict(nof_ack=1, I_offset_ack=9), dict(nof_ack=2, I_offset_ack=10, ri_len=1, I_offset_ri=8), dict(I_offset_cqi=8), dict(I_offset_cqi=6, ri_len=1,
                                                                                                                              I_offset_ri=5, nof_ack=2, I_offset_ack=5)]
    cqis = [(0, 0, 0, 0, 0), (1, 0, 0, 0, 0), (1, 3, 13 if prb == 100 else 9, 0, 1), (1, 1, 0, 5, 0)]
    subframes = []
    for i in range(3):
        recs = []
        for j, (mcs, L, start) in enumerate([(3, 5, 0), (8, 9, 5), (16, 12, 14), (24, 15, 26)]):
            g = ul_grant(cell, 0x500 + 16 * i + j, L, start, mcs, (i + j) % 8)
            g.I_offset_cqi = 7
            for kk, v in uci[(i + j) % 4].items():
                setattr(g, kk, v)
            recs.append(UlRec(g, cqi=cqis[(i + 2 * j) % 4]))
        subframes.append(recs)
    assert {r.g.qm for r in subframes[0]} == {2, 4, 6, 8}
    assert {cqi_size(r.cqi) for recs in subframes for r in recs} >= {0, 4, 11}
    assert check_ul(tmp_path, cell, UlCfg(n_dmrs1=4, delta_ss=7), subframes, snr=36.0, seed=80 + prb, rate34=N != 0) >= 11


@pytest.mark.parametrize("field", ["rv", "n_dmrs", "I_offset_ack", "I_offset_ri", "I_offset_cqi", "cqi_len"])
def test_ul_decode_after_estimating_another_configuration(infra, drivers, tmp_path, field):
    """srsran_chest_ul_estimate_pusch with one configuration (A), then srsran_pusch_decode with one that differs only in field (B): the decode is that of
    B, not the cached result of A.  Tier 1 must decode A and B differently, or the case could not tell the two apart.  For rv, n_dmrs, I_offset_cqi
    and cqi_len, A is the block on the air (it passes) and B fails.  A larger I_offset_ack only punctures more data REs and a larger I_offset_ri only
    shortens the data's rate-matching output, so a block on the air would still pass under B; there A and B are addressed to another RNTI, both fail,
    and the bytes of the failed decodes differ because the soft bits in front of the turbo decoder do."""
    cell = Cell(25, 1, 9, 1)
    sent = ul_grant(cell, 0x777, 8, 4, 8, 1)
    sent.nof_ack, sent.I_offset_ack, sent.ri_len, sent.I_offset_ri, sent.I_offset_cqi = 2, 0, 1, 0, 2
    cqi_a = (1, 3, 7, 0, 0)
    ga = ltelib.UlGrant.from_buffer_copy(sent)
    if field in ("I_offset_ack", "I_offset_ri"):
        ga.rnti = 0x778
    gb = ltelib.UlGrant.from_buffer_copy(ga)
    cqi_b = cqi_a
    if field == "rv":
        gb.rv = 2
    elif field == "n_dmrs":
        gb.n_dmrs2 = DMRS2[5]
    elif field == "cqi_len":
        cqi_b = (1, 3, 5, 0, 0)
    else:
        setattr(gb, field, {"I_offset_ack": 14, "I_offset_ri": 12, "I_offset_cqi": 15}[field])
    recs = [UlRec(ga, mode=1, cqi=cqi_a, sent=False), UlRec(gb, mode=2, cqi=cqi_b, sent=False), UlRec(sent, mode=0, cqi=cqi_a)]
    assert cqi_size(cqi_a) != cqi_size(cqi_b) or field != "cqi_len"
    t1 = []
    assert check_ul(tmp_path, cell, UlCfg(n_dmrs1=1, delta_ss=4), [recs], seed=99, tier1=t1) == 1
    assert t1[0] != t1[1], "tier 1 decodes A and B alike: this case cannot detect a stale result"
    assert t1[0][0] == (field not in ("I_offset_ack", "I_offset_ri")) and t1[1][0] == 0
