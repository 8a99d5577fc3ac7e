"""Several PHY handles driven at once from host threads, all sharing one search object, the way bench.py runs the library (pytest -m gpu).

Thread t decodes batches t, t + T, ... with seq = batch index; the walk must still run in batch order, so every batch has to equal one handle
decoding the same batches one after the other with LTEPHY_SEQ_NONE, bit for bit: SfInfo, every DCI field, crc, avg_iters, nof_cb and the payload
bytes.  The serial decode is itself checked against the CPU oracle pipeline and the transmitter's truth.  Also covered: batches that arrive out of
order, the full-table re-fetch inside a turn, one handle reused across different batch sizes / loads / IQ sources, two cells at once, and batches
the library refuses -- which must neither hang the other pipelines nor change what they decode.

Worker threads are daemons joined with a timeout: a turn that is never passed fails the test instead of hanging it (the stuck threads wait on a
host condition variable with no kernel outstanding)."""
import ctypes as C
import functools
import threading
import time

import numpy as np
import pytest

import ltelib
from ltelib import Cell
from helpers import make_capture
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu

# the captures of test_gpu_pipeline.py that have golden walk records
CAPTURES = {
    "cfg2_like_150ue_tm3": (Cell(100, 2, 7, 2), 40, dict(seed=2, cfi=3, nof_ues=150, dl_min=8, dl_max=12, tm=3, mcs_min=17, mcs_max=26, snr_db=28.0, full_band=1)),
    "mixed_10MHz": (Cell(50, 2, 301, 2), 40, dict(seed=3, cfi=3, nof_ues=10, dl_min=3, dl_max=5, ul_min=1, ul_max=2, tm=13, mcs_min=2, mcs_max=18, snr_db=25.0,
                                                  chan_delay=5)),
}
EVEN = (5,) * 8                       # batches of 5 subframes: the RNTI history carries across batches
UNEVEN = (12, 4, 5, 6, 3, 5, 5)       # batch 0 the largest
JOIN_S = 60.0
INVALID_INPUTS = -2                   # LTEPHY_ERROR_INVALID_INPUTS
DCI_FIELDS = ("sf", "rnti", "format", "L", "ncce", "nof_bits", "bits", "histogram_value")


@functools.lru_cache(None)
def capture(name):
    cell, n, kw = CAPTURES[name]
    sim, iq, tti, truths, payloads = make_capture(cell, n, **kw)
    return cell, sim, iq, tti, truths, payloads


def bounds(sizes):
    e = np.cumsum((0,) + tuple(sizes))
    return [(int(e[k]), int(e[k + 1])) for k in range(len(sizes))]


def new_phy(cell, nmax):
    return capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=nmax, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)


def new_search(cell, rar=None):
    s = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    if rar is not None:
        s.L.ltephy_search_activate(s.h, rar, 0, 2)      # ActivationReason RAR: the walk needs the full candidate table
    return s


class Scratch:
    """caller-owned outputs of one pipeline, reused across its batches as bench.py does"""

    def __init__(self, nmax):
        self.max_dcis = 32 * nmax
        self.info = (capi.SfInfo * nmax)()
        self.cands = np.zeros((nmax, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
        self.dcis = np.zeros(self.max_dcis, capi.DCI_DTYPE)
        self.tbs = (capi.TbResult * (2 * self.max_dcis))()
        self.payload = np.zeros(self.max_dcis * 2 * 2048 + nmax * 40000, np.uint8)
        self.nd = C.c_uint32(0)


def iq_ptr(src, lo):
    """pointer to subframe lo of a numpy array or a (pinned host / device) torch tensor [n][rx][sf_len] complex64"""
    if isinstance(src, np.ndarray):
        return C.c_void_p(src[lo:].ctypes.data)
    return C.c_void_p(src[lo:].data_ptr())


def decode(phy, srch, src, tti, lo, hi, seq, S, tbs_null=False, n_override=None):
    L = phy.L
    capi._bind_search(L)
    on_device = not isinstance(src, np.ndarray) and src.is_cuda
    fn = L.ltephy_decode_subframes_device if on_device else L.ltephy_decode_subframes
    t = np.ascontiguousarray(tti[lo:], np.uint32)
    return fn(phy.h, srch.h, iq_ptr(src, lo), t.ctypes.data_as(C.c_void_p), n_override or hi - lo, seq, S.info, S.cands.ctypes.data_as(C.c_void_p),
              S.dcis.ctypes.data_as(C.c_void_p), S.max_dcis, C.byref(S.nd), None if tbs_null else S.tbs, S.payload.ctypes.data_as(C.c_void_p),
              S.payload.nbytes)


def snapshot(S, n):
    """what one batch returned: SfInfo bytes, every DCI field, (crc, avg_iters, nof_cb, payload_len, payload bytes) per result slot"""
    nd = S.nd.value
    info = [bytes(S.info[i]) for i in range(n)]
    dcis = [tuple(int(d[k]) for k in DCI_FIELDS) for d in S.dcis[:nd]]
    tbs = []
    for j in range(2 * nd):
        r = S.tbs[j]
        tbs.append((int(r.crc), int(r.avg_iters), int(r.nof_cb), int(r.payload_len), S.payload[r.payload_off:r.payload_off + r.payload_len].tobytes()))
    return info, dcis, tbs


def decode_ok(phy, srch, src, tti, lo, hi, seq, S):
    r = decode(phy, srch, src, tti, lo, hi, seq, S)
    assert r == 0, (r, phy.L.ltephy_last_error().decode())
    return snapshot(S, hi - lo)


def serial_run(name, sizes, rar=None, order=None, skip=()):
    """one handle, LTEPHY_SEQ_NONE, fresh outputs per batch, batches in `order` (default: batch order) -> {batch: snapshot}"""
    cell, sim, iq, tti, _, _ = capture(name)
    b = bounds(sizes)
    phy = new_phy(cell, max(sizes))
    srch = new_search(cell, rar)
    out = {}
    for k in (order if order is not None else range(len(b))):
        if k in skip:
            continue
        out[k] = decode_ok(phy, srch, iq, tti, *b[k], capi.SEQ_NONE, Scratch(max(sizes)))
    phy.close()
    return out


@functools.lru_cache(None)
def serial(name, sizes, rar=False):
    cell, sim = capture(name)[:2]
    return serial_run(name, sizes, int(sim.rntis()[0]) if rar else None)


_KEPT = []   # handles and searches that stuck threads still wait in: destroying a search under a waiting thread would be undefined


def run_threads(jobs, start_last=None, settle_s=1.0, keep=()):
    """jobs[t] = callable run by thread t; start_last: a thread started only after the others have had settle_s to block in their turn waits.
    Fails if a thread is still running after JOIN_S (keeping `keep` alive for it), else re-raises the first exception of a thread."""
    errs = [None] * len(jobs)

    def body(t):
        try:
            jobs[t]()
        except BaseException as e:  # noqa: B902 -- handed to the main thread
            errs[t] = e

    th = [threading.Thread(target=body, args=(t,), daemon=True) for t in range(len(jobs))]
    for t, x in enumerate(th):
        if t != start_last:
            x.start()
    if start_last is not None:
        time.sleep(settle_s)
        assert all(x.is_alive() for t, x in enumerate(th) if t != start_last and jobs[t] is not None), "a later batch did not wait for batch 0"
        th[start_last].start()
    deadline = time.time() + JOIN_S
    for x in th:
        x.join(max(0.0, deadline - time.time()))
    stuck = [t for t, x in enumerate(th) if x.is_alive()]
    if stuck:
        _KEPT.append(keep)
    assert not stuck, "threads %s never finished: a walk turn was not passed on" % stuck
    for e in errs:
        if e is not None:
            raise e


def concurrent(name, sizes, T, src, rar=None, start_last=None, refuse=None):
    """T pipelines on one search; thread t takes batches t, t + T, ... with seq = batch index -> ({batch: snapshot}, {batch: return code})"""
    cell, sim, iq, tti, _, _ = capture(name)
    b = bounds(sizes)
    nmax = max(sizes)
    phys = [new_phy(cell, nmax) for _ in range(T)]
    srch = new_search(cell, rar)
    out, rets = {}, {}

    def job(t):
        def run():
            S = Scratch(nmax)
            for k in range(t, len(b), T):
                lo, hi = b[k]
                if refuse and k == refuse[0]:
                    rets[k] = refuse[1](phys[t], srch, src, tti, lo, hi, k, S)
                    continue
                r = decode(phys[t], srch, src, tti, lo, hi, k, S)
                assert r == 0, (k, r, phys[t].L.ltephy_last_error().decode())
                out[k] = snapshot(S, hi - lo)
                if refuse and refuse[0] == ("stale", k):      # after batch k has had its turn, its seq again: refused, no turn consumed
                    rets["stale"] = decode(phys[t], srch, src, tti, lo, hi, k, S)
        return run

    run_threads([job(t) for t in range(T)], start_last=start_last, keep=(phys, srch))
    for p in phys:
        p.close()
    return out, rets


def merged(snaps, sizes):
    """{batch: snapshot} in batch order -> per-subframe info bytes, DCIs with global sf, result slots"""
    info, dcis, tbs = [], [], []
    for k, (lo, hi) in enumerate(bounds(sizes)):
        i, d, t = snaps[k]
        info += i
        dcis += [(x[0] + lo,) + x[1:] for x in d]
        tbs += t
    return info, dcis, tbs


@functools.lru_cache(None)
def oracle_ref(name):
    cell, sim, iq, tti, truths, payloads = capture(name)
    return ltelib.oracle_pipeline(cell, iq, tti, walk=ltelib.OracleWalk(cell, golden="oraclewalk_" + name))


def check_against_oracle_and_truth(name, snaps, sizes):
    """the assertions of test_gpu_pipeline.py::test_decode_subframes_matches_oracle_pipeline on a batched decode"""
    cell, sim, iq, tti, truths, payloads = capture(name)
    ref = oracle_ref(name)
    info, dcis, tbs = merged(snaps, sizes)
    k = ntb_ok = 0
    for sf in range(len(tti)):
        rd, rt, snr, cfi = ref[sf]
        si = capi.SfInfo.from_buffer_copy(info[sf])
        assert si.cfi == cfi and si.snr_db == snr
        mine = [d for d in dcis if d[0] == sf]
        assert len(mine) == len(rd), (name, sf, len(mine), len(rd))
        for a, b, t in zip(mine, rd, rt):
            assert (a[1], a[2], a[3], a[4], a[7]) == (b.rnti, b.format, b.L, b.ncce, b.histval)
            assert np.array_equal(capi.cand_bits(a[6], b.nof_bits), np.frombuffer(bytes(b.bits), np.uint8)[:b.nof_bits])
            for tb in range(2):
                crc, _, _, plen, pl = tbs[2 * k + tb]
                if t is None or not t[0].tb[tb].enabled:
                    assert plen == 0
                    continue
                gr, opl, ok = t
                nby = gr.tb[tb].tbs // 8
                assert plen == nby and crc == ok[tb], (name, sf, hex(b.rnti), tb, crc, ok[tb])
                assert np.array_equal(np.frombuffer(pl, np.uint8), opl[tb][:nby])
                ntb_ok += crc
            k += 1
    assert k == len(dcis)
    sent = {}
    for sf, tr in enumerate(truths):
        for i in range(tr.nof_dci):
            d = tr.dci[i]
            for tb in range(2):
                if d.tbs[tb] > 0:
                    sent[(sf, d.rnti, tb)] = payloads[sf][d.payload_off[tb]:d.payload_off[tb] + d.tbs[tb] // 8]
    hits = 0
    for i, d in enumerate(dcis):
        for tb in range(2):
            crc, _, _, _, pl = tbs[2 * i + tb]
            if crc and (d[0], d[1], tb) in sent:
                assert np.array_equal(np.frombuffer(pl, np.uint8), sent[(d[0], d[1], tb)])
                hits += 1
    assert hits >= 1 and ntb_ok >= 1


def iq_source(name, kind):
    import torch
    iq = capture(name)[2]
    if kind == "numpy":
        return iq
    t = torch.from_numpy(iq)
    return t.pin_memory() if kind == "pinned" else t.cuda()


# ------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CAPTURES))
def test_serial_batches_equal_the_oracle_pipeline_and_order_matters(infra, phylib, name):
    """the reference of every test below, checked once against the oracle and the truth; decoding the same batches in another order on a fresh
    search gives other DCIs, so equality with it does say something about the order the walk ran in"""
    check_against_oracle_and_truth(name, serial(name, EVEN), EVEN)
    order = [3, 0, 5, 1, 7, 2, 6, 4]
    permuted = serial_run(name, EVEN, order=order)
    assert merged(permuted, EVEN)[1] != merged(serial(name, EVEN), EVEN)[1], "the batch order should change what the walk reports"


@pytest.mark.parametrize("src", ["numpy", "pinned", "device"])
@pytest.mark.parametrize("T", [1, 2, 6])
@pytest.mark.parametrize("name", list(CAPTURES))
def test_concurrent_pipelines_equal_serial_decode(infra, phylib, name, T, src):
    out, _ = concurrent(name, EVEN, T, iq_source(name, src))
    ref = serial(name, EVEN)
    for k in range(len(EVEN)):
        assert out[k] == ref[k], (name, T, src, k)
    check_against_oracle_and_truth(name, out, EVEN)


@pytest.mark.parametrize("name", list(CAPTURES))
def test_batch_zero_arriving_last(infra, phylib, name):
    """the other pipelines finish phase A and wait in their turn; batch 0, the largest, starts only then"""
    out, _ = concurrent(name, UNEVEN, 6, iq_source(name, "pinned"), start_last=0)
    ref = serial(name, UNEVEN)
    for k in range(len(UNEVEN)):
        assert out[k] == ref[k], (name, k)


def test_full_table_fallback_inside_the_turn(infra, phylib):
    """a RAR-activated RNTI makes every batch re-fetch the full candidate table while it holds its turn"""
    name = "mixed_10MHz"
    rar = int(capture(name)[1].rntis()[0])
    out, _ = concurrent(name, EVEN, 3, iq_source(name, "device"), rar=rar)
    ref = serial(name, EVEN, rar=True)
    for k in range(len(EVEN)):
        assert out[k] == ref[k], k
    assert merged(ref, EVEN)[1] != merged(serial(name, EVEN), EVEN)[1], "the RAR activation should change what the walk reports"


def test_handle_reuse_equals_fresh_handles(infra, phylib):
    """one handle and one set of outputs through batches of 8, 1, 7, 8 and 3 subframes: busy, noise only, busy; host and device IQ alternating;
    the fourth batch after a RAR activation (full-table re-fetch) -- against a fresh handle and fresh outputs per batch on the same search
    progression.  Later batches hold DCIs without a transport block in result slots that carried one before, so stale entries would show."""
    import torch
    name = "mixed_10MHz"
    cell, sim, iq, tti, _, _ = capture(name)
    rng = np.random.default_rng(5)
    noise = (rng.standard_normal((7,) + iq.shape[1:]) + 1j * rng.standard_normal((7,) + iq.shape[1:])).astype(np.complex64) * np.float32(0.02)
    # (iq, tti) of each batch; tti keeps counting through the noise-only batch
    plan = [(iq[0:8], tti[0:8]), (iq[8:9], tti[8:9]), (noise, np.arange(9, 16, dtype=np.uint32)), (iq[16:24], tti[16:24]), (iq[24:27], tti[24:27])]
    on_dev = [False, True, False, True, False]
    rar = int(sim.rntis()[0])
    phy = new_phy(cell, 8)
    S = Scratch(8)
    s_reuse, s_fresh = new_search(cell), new_search(cell)
    got, want = [], []
    for k, ((x, t), dev) in enumerate(zip(plan, on_dev)):
        if k == 3:
            for s in (s_reuse, s_fresh):
                s.L.ltephy_search_activate(s.h, rar, 0, 2)
        x = np.ascontiguousarray(x)
        src = torch.from_numpy(x).cuda() if dev else x
        got.append(decode_ok(phy, s_reuse, src, t, 0, len(t), capi.SEQ_NONE, S))
        fresh = new_phy(cell, len(t))
        want.append(decode_ok(fresh, s_fresh, x, t, 0, len(t), capi.SEQ_NONE, Scratch(len(t))))
        fresh.close()
    phy.close()
    for k in range(len(plan)):
        assert got[k] == want[k], k
    assert len(want[0][1]) > 0 and len(want[3][1]) > 0
    # evidence that the test can see stale slots: a slot without a transport block that an earlier batch filled
    last = {}
    stale_visible = 0
    for _, dcis, tbs in want:
        for j, slot in enumerate(tbs):
            if slot[3] == 0 and last.get(j, 0) > 0:
                stale_visible += 1
            if slot[3] > 0:
                last[j] = slot[3]
    assert stale_visible > 0


def test_two_cells_at_once(infra, phylib):
    """two handles of different cells, each with its own search, decode host IQ at the same time (both through the host-to-device copy chain)"""
    names = list(CAPTURES)
    out = {}

    def job(name):
        def run():
            cell, sim, iq, tti, _, _ = capture(name)
            phy = new_phy(cell, max(EVEN))
            srch = new_search(cell)
            S = Scratch(max(EVEN))
            out[name] = {k: decode_ok(phy, srch, iq, tti, lo, hi, capi.SEQ_NONE, S) for k, (lo, hi) in enumerate(bounds(EVEN))}
            phy.close()
        return run

    for n in names:
        capture(n)
    run_threads([job(n) for n in names])
    for n in names:
        ref = serial(n, EVEN)
        for k in range(len(EVEN)):
            assert out[n][k] == ref[k], (n, k)


def _too_many_subframes(phy, srch, src, tti, lo, hi, seq, S):
    return decode(phy, srch, src, tti, 0, 0, seq, S, n_override=phy.cfg.max_subframes + 1)


def _null_tbs(phy, srch, src, tti, lo, hi, seq, S):
    return decode(phy, srch, src, tti, lo, hi, seq, S, tbs_null=True)


@pytest.mark.parametrize("mode", ["too_many_subframes", "null_tbs", "stale_seq"])
def test_refused_batch_in_a_sequence(infra, phylib, mode):
    """three pipelines; one call is refused with LTEPHY_ERROR_INVALID_INPUTS: more subframes than the handle holds, or a NULL tbs (both give their
    turn on), or a seq whose turn is over (consumes none).  The other batches finish and equal the serial decode without the refused batch."""
    name = "mixed_10MHz"
    src = iq_source(name, "numpy")
    if mode == "stale_seq":
        out, rets = concurrent(name, EVEN, 3, src, refuse=(("stale", 4), None))
        ref, key = serial(name, EVEN), "stale"
        assert set(out) == set(range(len(EVEN)))
    else:
        out, rets = concurrent(name, EVEN, 3, src, refuse=(4, _too_many_subframes if mode == "too_many_subframes" else _null_tbs))
        ref, key = serial_run(name, EVEN, skip=(4,)), 4
        assert set(out) == set(range(len(EVEN))) - {4}
    assert rets[key] == INVALID_INPUTS, rets
    for k in out:
        assert out[k] == ref[k], (mode, k)
