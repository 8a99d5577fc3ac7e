"""Sharded operation on the GPU (pytest -m gpu): the pack kernel against its host restatement, ltephy_decode_subframes_sharded
with one rank against ltephy_decode_subframes, and -- when the box has two GPUs -- two ranks (one process per GPU, NCCL)
against one GPU decoding the whole capture: rank 0 must end up with the same DCIs, CRC flags and transport-block bytes."""
import ctypes as C
import os
import sys
import threading
import time
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

CELL = (50, 2, 301, 2)
SIM_KW = dict(seed=3, cfi=3, nof_ues=10, dl_min=3, dl_max=5, ul_min=1, ul_max=2, tm=13, mcs_min=2, mcs_max=18, snr_db=25.0, chan_delay=5)
N_TOTAL = 24


def _key(d):
    return (int(d["sf"]), int(d["rnti"]), int(d["format"]), int(d["L"]), int(d["ncce"]), int(d["bits"]), int(d["histogram_value"]))


def _tb_table(dcis, tbs, payload):
    out = []
    for i in range(len(dcis)):
        for t in range(2):
            r = tbs[2 * i + t]
            out.append((r.crc, r.payload_len, r.nof_cb, bytes(payload[r.payload_off:r.payload_off + r.payload_len]) if r.payload_len else b""))
    return out


def _sharded_call(capi, shard, phy, srch, iq, tti, seq, max_dcis, world, tbs_null=False):
    """-> (return code, last error of this thread, info, dcis, tbs, payload, stats)"""
    L = phy.L
    capi._bind_search(L)
    n = len(tti)
    iq = np.ascontiguousarray(iq, np.complex64)
    tti = np.ascontiguousarray(tti, np.uint32)
    info = (capi.SfInfo * n)()
    dcis = np.zeros(max_dcis, capi.DCI_DTYPE)
    tbs = (capi.TbResult * (2 * max_dcis))()
    payload = np.zeros(n * world * 40000 + 65536, np.uint8)
    nd = C.c_uint32(0)
    st = capi.ShardStats()
    r = L.ltephy_decode_subframes_sharded(shard.h, phy.h, srch.h, iq.ctypes.data_as(C.c_void_p), 0, tti.ctypes.data_as(C.c_void_p), n, seq, info,
                                          dcis.ctypes.data_as(C.c_void_p), max_dcis, C.byref(nd), None if tbs_null else tbs,
                                          payload.ctypes.data_as(C.c_void_p), payload.nbytes, C.byref(st))
    return r, L.ltephy_last_error().decode(), info, dcis[:nd.value], tbs, payload, st


def _sharded_decode(capi, shard, phy, srch, iq, tti, seq, max_dcis, world):
    r, err, info, dcis, tbs, payload, st = _sharded_call(capi, shard, phy, srch, iq, tti, seq, max_dcis, world)
    assert r == 0, err
    return info, dcis, tbs, payload, st


def _join_all(threads, timeout_s=60.0):
    """daemon threads joined with one deadline: a turn never given back fails the test instead of hanging it"""
    deadline = time.time() + timeout_s
    for t in threads:
        t.join(max(0.0, deadline - time.time()))
    assert not any(t.is_alive() for t in threads), "a pipeline never finished: an ordered section was not given back"


def _three_pipelines_on_one_shard(capi, cell, sh, srch, iq, tti, ref_dcis, ref_table, T):
    """T host threads, one handle each, on one Shard of world size 1 (thread t takes batches t, t + T, ... with seq = batch index), against the
    unsharded serial decode.  Then a batch refused for a NULL argument: it takes and gives back every turn and marks the rank failed, so the
    batches after it return at once with the rank-failed error."""
    sizes = [3, 3, 3, 3, 2, 2]
    lo = np.cumsum([0] + sizes)
    phys = [capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=max(sizes), turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
            for _ in range(T)]
    out, errs = {}, []

    def worker(t, seqs, **kw):
        try:
            for k in seqs:
                a, b = (int(lo[k]), int(lo[k + 1])) if k < len(sizes) else (0, sizes[0])
                out[k] = _sharded_call(capi, sh, phys[t], srch, iq[a:b], tti[a:b], k, 32 * 16, 1, **kw)
        except BaseException as e:  # noqa: B902 -- handed to the main thread
            errs.append(e)

    th = [threading.Thread(target=worker, args=(t, range(t, len(sizes), T)), daemon=True) for t in range(T)]
    for x in th:
        x.start()
    _join_all(th)
    assert not errs, errs
    got, table = [], []
    for k in range(len(sizes)):
        r, err, info, dcis, tbs, pl, st = out[k]
        assert r == 0, (k, err)
        got += [(d[0] + int(lo[k]),) + d[1:] for d in (_key(d) for d in dcis)]
        table += _tb_table(dcis, tbs, pl)
    assert got == [_key(d) for d in ref_dcis]
    assert table == ref_table
    # the refused batch (seq 6), then two more from two threads
    k = len(sizes)
    th = [threading.Thread(target=worker, args=(0, [k]), kwargs=dict(tbs_null=True), daemon=True)]
    th[0].start()
    _join_all(th)
    assert out[k][0] == -2, out[k][:2]                                       # LTEPHY_ERROR_INVALID_INPUTS
    th = [threading.Thread(target=worker, args=(t, [k + t]), daemon=True) for t in (1, 2)]
    t0 = time.time()
    for x in th:
        x.start()
    _join_all(th)
    assert not errs, errs
    for j in (k + 1, k + 2):
        assert out[j][0] == -1 and "an earlier batch failed on this rank" in out[j][1], out[j][:2]   # LTEPHY_ERROR
    assert time.time() - t0 < 10.0
    for p in phys:
        p.close()


def test_pack_kernel_matches_host_restatement(infra, phylib):
    import ltelib
    from helpers import make_capture
    from ltesniffer_b200 import capi
    cell = ltelib.Cell(*CELL)
    sim, iq, tti, truths, payloads = make_capture(cell, 12, **SIM_KW)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=12, flags=capi.FLAG_SKIP_LOW_POWER)
    srch = capi.Search(*CELL)
    phy.submit_iq(iq, tti)
    info, comp = phy.get_phase_a_compact()
    rec_gpu, offs_gpu = capi.pack_phase_a(phy)
    rec_host, offs_host = capi.pack_subframes(srch, info, comp)
    assert np.array_equal(offs_gpu, offs_host)
    assert np.array_equal(rec_gpu, rec_host)
    assert len(rec_gpu) < 12 * capi.PACK_MAX_BYTES // 2      # packed to the used length
    hd = rec_gpu[:64].view(capi.PACKED_HDR_DTYPE)[0]
    assert hd["tti"] == tti[0] and hd["cfi"] == info[0].cfi and hd["count"] == comp[0]["count"]
    phy.close()


def _one_rank_setup(n):
    """a capture of n subframes, its unsharded serial decode, a Shard of world size 1 and a fresh search"""
    import ltelib
    from helpers import make_capture
    from ltesniffer_b200 import capi
    cell = ltelib.Cell(*CELL)
    sim, iq, tti, truths, payloads = make_capture(cell, n, **SIM_KW)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
    ref_info, ref_dcis, ref_tbs, ref_pl = capi.decode_subframes(phy, capi.Search(*CELL), iq, tti)
    sh = capi.Shard(capi.Shard.unique_id(), 0, 1, 0)
    return capi, cell, iq, tti, phy, ref_info, ref_dcis, _tb_table(ref_dcis, ref_tbs, ref_pl), sh, capi.Search(*CELL)


def test_sharded_one_rank_equals_single_gpu_pipeline(infra, phylib):
    n = 16
    capi, cell, iq, tti, phy, ref_info, ref_dcis, ref_table, sh, srch = _one_rank_setup(n)
    # two consecutive batches through the ordered sections (seq 0, 1): the second continues the RNTI history of the first
    info, dcis, tbs, pl, st = _sharded_decode(capi, sh, phy, srch, iq[:8], tti[:8], 0, 32 * n, 1)
    info2, dcis2, tbs2, pl2, st2 = _sharded_decode(capi, sh, phy, srch, iq[8:], tti[8:], 1, 32 * n, 1)
    got = [_key(d) for d in dcis] + [(k[0] + 8,) + k[1:] for k in (_key(d) for d in dcis2)]
    assert got == [_key(d) for d in ref_dcis] and len(got) >= n
    assert _tb_table(dcis, tbs, pl) + _tb_table(dcis2, tbs2, pl2) == ref_table
    assert sum(t[0] for t in ref_table) >= 4
    assert [info[i].snr_db for i in range(8)] == [ref_info[i].snr_db for i in range(8)]
    assert st.exchanged_bytes > 0 and st.used_full_table == 0
    sh.close()
    phy.close()


def test_sharded_one_rank_three_threads_and_a_refused_batch(infra, phylib):
    capi, cell, iq, tti, phy, ref_info, ref_dcis, ref_table, sh, srch = _one_rank_setup(16)
    _three_pipelines_on_one_shard(capi, cell, sh, srch, iq, tti, ref_dcis, ref_table, 3)
    sh.close()
    phy.close()


def test_sharded_one_rank_refuses_a_seq_whose_turn_is_over(infra, phylib):
    """batch 0, then batch 0 again: the second call returns LTEPHY_ERROR_INVALID_INPUTS at once instead of waiting for a turn that has
    passed, and consumes nothing -- batch 1 then decodes as the unsharded pipeline does"""
    n = 16
    capi, cell, iq, tti, phy, ref_info, ref_dcis, ref_table, sh, srch = _one_rank_setup(n)
    info, dcis, tbs, pl, st = _sharded_decode(capi, sh, phy, srch, iq[:8], tti[:8], 0, 32 * n, 1)
    out = []
    th = threading.Thread(target=lambda: out.append(_sharded_call(capi, sh, phy, srch, iq[:8], tti[:8], 0, 32 * n, 1)), daemon=True)
    th.start()
    _join_all([th], 30.0)
    assert out[0][0] == -2, out[0][:2]                                       # LTEPHY_ERROR_INVALID_INPUTS
    info2, dcis2, tbs2, pl2, st2 = _sharded_decode(capi, sh, phy, srch, iq[8:], tti[8:], 1, 32 * n, 1)
    got = [_key(d) for d in dcis] + [(k[0] + 8,) + k[1:] for k in (_key(d) for d in dcis2)]
    assert got == [_key(d) for d in ref_dcis]
    assert _tb_table(dcis, tbs, pl) + _tb_table(dcis2, tbs2, pl2) == ref_table
    sh.close()
    phy.close()


def _rank_main(rank, world, uid, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ltelib
    from helpers import make_capture
    from ltesniffer_b200 import capi
    cell = ltelib.Cell(*CELL)
    sim, iq, tti, truths, payloads = make_capture(cell, N_TOTAL, **SIM_KW)
    mine = np.arange(rank, N_TOTAL, world)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=N_TOTAL, turbo_max_iter=8, device=rank, flags=capi.FLAG_SKIP_LOW_POWER)
    sh = capi.Shard(uid, rank, world, rank)
    srch = capi.Search(*CELL)
    half = len(mine) // 2
    out = []
    for seq, sel in enumerate((mine[:half], mine[half:])):   # two batches: global subframes 0..N/2-1, then N/2..N-1
        info, dcis, tbs, pl, st = _sharded_decode(capi, sh, phy, srch, iq[sel], tti[sel], seq, 32 * N_TOTAL, world)
        out.append(([_key(d) for d in dcis], _tb_table(dcis, tbs, pl), st.exchanged_bytes, st.n_grants))
    if rank == 0:
        phy1 = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=N_TOTAL, turbo_max_iter=8, device=0, flags=capi.FLAG_SKIP_LOW_POWER)
        ri, rd, rt, rp = capi.decode_subframes(phy1, capi.Search(*CELL), iq, tti)
        q.put(("ref", [_key(d) for d in rd], _tb_table(rd, rt, rp)))
        phy1.close()
    q.put((rank, out))
    sh.close()
    phy.close()


def test_two_ranks_equal_one_gpu(infra, phylib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    from ltesniffer_b200 import capi
    uid = capi.Shard.unique_id()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_main, args=(r, 2, uid, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(3):
        m = q.get(timeout=900)
        got[m[0]] = m[1:]
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    ref_keys, ref_table = got["ref"]
    half = N_TOTAL // 2
    for rank in (0, 1):
        (k0, t0, x0, g0), (k1, t1, x1, g1) = got[rank][0]
        keys = k0 + [(k[0] + half,) + k[1:] for k in k1]
        assert keys == ref_keys                                   # every rank replays the same walk
        assert x0 > 0 and g0 > 0
        if rank == 0:
            assert t0 + t1 == ref_table                           # rank 0 holds every transport block of both ranks, byte for byte
        else:
            mine = [t for t in t0 + t1 if t[1]]
            assert 0 < len(mine) < len([t for t in ref_table if t[1]])   # the other rank keeps only its own
    assert sum(t[0] for t in ref_table) >= 6
