"""End-to-end GPU parity (pytest -m gpu): ltephy_decode_subframes (host IQ -> accepted DCIs + transport
blocks through the C-ABI) against the whole CPU oracle pipeline (oracle receiver + the walk that runs on
the reference's own RNTIManager) and against the transmitter's ground truth.  Where oracle/_ref cannot be built, the walk's answers come
from tests/golden/oraclewalk_*.npz (ltelib.WalkRecord); the oracle receiver runs either way."""
import numpy as np
import pytest
import ltelib
from ltelib import Cell
from helpers import make_capture
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,cell,n,kw", [
    ("cfg1_10sf_1rnti_tm1_qpsk", Cell(100, 1, 1, 1), 10, dict(seed=1, cfi=2, nof_ues=1, tm=1, mcs_min=5, mcs_max=5, snr_db=30.0, fixed_L=2, si_period=5)),
    ("cfg2_like_150ue_tm3", Cell(100, 2, 7, 2), 40, dict(seed=2, cfi=3, nof_ues=150, dl_min=8, dl_max=12, tm=3, mcs_min=17, mcs_max=26, snr_db=28.0, full_band=1)),
    ("mixed_10MHz", Cell(50, 2, 301, 2), 40, dict(seed=3, cfi=3, nof_ues=10, dl_min=3, dl_max=5, ul_min=1, ul_max=2, tm=13, mcs_min=2, mcs_max=18, snr_db=25.0, chan_delay=5)),
    # Cell(nof_prb, ports, cell id, antennas, symbol size, phich-Resource Ng (3: Ng = 2), phich-Duration extended)
    ("mixed_3MHz", Cell(15, 2, 33, 2), 20, dict(seed=5, cfi=3, nof_ues=6, dl_min=1, dl_max=3, ul_min=1, ul_max=1, tm=13, mcs_min=2, mcs_max=18, snr_db=26.0, si_period=4)),
    ("mixed_15MHz_1536", Cell(75, 2, 34, 2, 1536), 20, dict(seed=6, cfi=2, nof_ues=10, dl_min=2, dl_max=5, ul_min=1, ul_max=2, tm=13, mcs_min=2, mcs_max=22, snr_db=26.0,
                                                            chan_delay=4)),
    ("tm3_20MHz_ng2_ext", Cell(100, 2, 35, 2, 0, 3, 1), 20, dict(seed=7, cfi=3, nof_ues=12, dl_min=3, dl_max=6, tm=3, mcs_min=4, mcs_max=22, snr_db=27.0)),
])
def test_decode_subframes_matches_oracle_pipeline(infra, phylib, name, cell, n, kw):
    sim, iq, tti, truths, payloads = make_capture(cell, n, **kw)
    walk = ltelib.OracleWalk(cell, golden="oraclewalk_" + name)
    ref = ltelib.oracle_pipeline(cell, iq, tti, walk=walk)
    walk.save_record()
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER,
                      symbol_sz=cell.symbol_sz, phich_resources=cell.phich_ng, phich_length=cell.phich_ext)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, phich_resources=cell.phich_ng | (cell.phich_ext << 8))
    info, dcis, tbs, payload = capi.decode_subframes(phy, srch, iq, tti)
    k = 0
    ntb_ok = 0
    for sf in range(n):
        rd, rt, snr, cfi = ref[sf]
        assert info[sf].cfi == cfi and info[sf].snr_db == snr
        mine = [d for d in dcis if d["sf"] == sf]
        assert len(mine) == len(rd), (name, sf, len(mine), len(rd))
        for a, b, t in zip(mine, rd, rt):
            assert (int(a["rnti"]), int(a["format"]), int(a["L"]), int(a["ncce"]), int(a["histogram_value"])) == (b.rnti, b.format, b.L, b.ncce, b.histval)
            assert np.array_equal(capi.cand_bits(a["bits"], b.nof_bits), np.frombuffer(bytes(b.bits), np.uint8)[:b.nof_bits])
            for tb in range(2):
                r = tbs[2 * k + tb]
                if t is None or not t[0].tb[tb].enabled:
                    assert r.payload_len == 0
                    continue
                gr, pl, ok = t
                nby = gr.tb[tb].tbs // 8
                assert r.payload_len == nby and r.crc == ok[tb], (name, sf, hex(b.rnti), tb, r.crc, ok[tb])
                assert np.array_equal(payload[r.payload_off:r.payload_off + nby], pl[tb][:nby])
                ntb_ok += r.crc
            k += 1
    assert k == len(dcis)
    # ground truth: transport blocks with CRC ok carry the transmitted bytes
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
            r = tbs[2 * i + tb]
            if r.crc and (int(d["sf"]), int(d["rnti"]), tb) in sent:
                assert np.array_equal(payload[r.payload_off:r.payload_off + r.payload_len], sent[(int(d["sf"]), int(d["rnti"]), tb)])
                hits += 1
    assert hits >= 1 and ntb_ok >= 1
    phy.close()


def test_decode_subframes_falls_back_to_full_table_for_rar_rntis(infra, phylib):
    """A RAR-activated RNTI makes the walk look at every format-0 candidate (temp_dci0, DCISearch.cc:150-161), which the
    survivor form cannot serve: ltephy_decode_subframes must fetch the full table and give what a walk over the full table gives."""
    import ctypes as C
    cell = Cell(50, 2, 301, 2)
    n = 24
    sim, iq, tti, truths, payloads = make_capture(cell, n, seed=9, cfi=3, nof_ues=5, dl_min=2, dl_max=3, ul_min=1, ul_max=2, tm=13, mcs_min=2, mcs_max=14, snr_db=26.0)
    rar = int(sim.rntis()[0])
    L = capi.load_library()
    capi._bind_search(L)
    out = []
    for mode in ("pipeline", "full_table_walk", "no_rar"):
        phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
        srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
        if mode != "no_rar":
            L.ltephy_search_activate(srch.h, rar, 0, 2)      # ActivationReason RAR
        if mode == "full_table_walk":
            phy.submit_iq(iq, tti)
            info, cands = phy.get_phase_a()
            dcis = np.zeros(64 * n, capi.DCI_DTYPE)
            nd = C.c_uint32(0)
            assert L.ltephy_search_batch(srch.h, info, cands.ctypes.data_as(C.c_void_p), n, dcis.ctypes.data_as(C.c_void_p), len(dcis), C.byref(nd)) == 0
            dcis = dcis[:nd.value]
        else:
            info, dcis, tbs, payload = capi.decode_subframes(phy, srch, iq, tti)
        out.append([tuple(int(d[k]) for k in ("sf", "rnti", "format", "L", "ncce", "nof_bits", "bits", "histogram_value")) for d in dcis])
        phy.close()
    assert out[0] == out[1] and len(out[0]) > n
    assert out[0] != out[2], "the RAR activation should change what the walk reports (otherwise this test exercises nothing)"


def test_device_side_exchange_equals_host_fetch(infra, phylib):
    """shard.gather_tables_device (device -> NCCL all-gather -> host, records finalised after the exchange) must hand the walk
    exactly what ltephy_get_phase_a_compact hands it (world size 1 here; the interleaving is covered by the gloo test)."""
    import os
    import torch
    import torch.distributed as dist
    from ltesniffer_b200 import shard
    cell = Cell(50, 2, 301, 2)
    n = 6
    sim, iq, tti, truths, payloads = make_capture(cell, n, seed=4, cfi=3, nof_ues=5, dl_min=2, dl_max=3, tm=13, mcs_min=2, mcs_max=14, snr_db=26.0)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, flags=capi.FLAG_SKIP_LOW_POWER)
    phy.submit_iq(iq, tti)
    info, comp = phy.get_phase_a_compact()
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method="tcp://127.0.0.1:%d" % (29600 + os.getpid() % 300), rank=0, world_size=1)
    try:
        info_all, comp_all = shard.gather_tables_device(phy.L, phy.h, n, 1, cell.nof_ports, cell.nof_rx)
        assert bytes(info_all) == bytes(info)
        got = comp_all.numpy().view(capi.COMPACT_DTYPE).reshape(n)
        for i in range(n):
            k = int(comp[i]["count"])
            assert int(got[i]["count"]) == k and got[i]["loc"].tobytes() == comp[i]["loc"].tobytes()
            assert got[i]["list"][:k].tobytes() == comp[i]["list"][:k].tobytes()
    finally:
        dist.destroy_process_group()
    phy.close()


@pytest.mark.parametrize("alt", [1, 0])
def test_speculative_mcs_table(infra, phylib, alt):
    """UEs configured with the 256QAM MCS table (alt = 1) or the normal one (alt = 0), receiver not told which:
    ltephy_search_speculate_256qam makes the pipeline decode both readings of every C-RNTI DCI in the same batch and report the
    one whose CRC passes (crc = 1: Table 7.1.7.1-1, crc = 2: Table 7.1.7.1-1A), DL_Sniffer_PDSCH.cc:1089-1210."""
    cell = Cell(50, 2, 11, 2)
    n = 30
    kw = dict(seed=15 + alt, cfi=2, nof_ues=5, dl_min=2, dl_max=3, tm=4 if alt else 3, mcs_min=5, mcs_max=20, snr_db=33.0, alt_table=alt)
    sim, iq, tti, truths, payloads = make_capture(cell, n, **kw)
    sent = {}
    for sf, tr in enumerate(truths):
        for i in range(tr.nof_dci):
            d = tr.dci[i]
            for tb in range(2):
                if d.tbs[tb] > 0:
                    sent[(sf, d.rnti, tb)] = payloads[sf][d.payload_off[tb]:d.payload_off[tb] + d.tbs[tb] // 8]
    L = capi.load_library()
    capi._bind_search(L)
    hits = {}
    for spec in (1, 0):
        phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
        srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
        L.ltephy_search_speculate_256qam(srch.h, spec)
        info, dcis, tbs, payload = capi.decode_subframes(phy, srch, iq, tti)
        ok = {}
        for i, d in enumerate(dcis):
            for tb in range(2):
                r = tbs[2 * i + tb]
                key = (int(d["sf"]), int(d["rnti"]), tb)
                if r.crc and key in sent:
                    assert r.payload_len == len(sent[key]) and np.array_equal(payload[r.payload_off:r.payload_off + r.payload_len], sent[key])
                    ok[key] = int(r.crc)
        hits[spec] = ok
        phy.close()
    late = [k for k in sent if k[0] >= n // 2]
    got = [k for k in late if k in hits[1]]
    assert len(got) >= 0.8 * len(late), (alt, len(got), len(late))
    assert set(hits[1].values()) == ({2} if alt else {1}), (alt, set(hits[1].values()))
    if alt:
        assert len(hits[0]) < 0.2 * max(1, len(hits[1]))      # without speculation the 256QAM-table UEs are (almost) never decoded
    else:
        assert hits[0] == hits[1]                             # speculation does not change what is reported for normal UEs
