"""The product against the REFERENCE'S OWN code, compiled unmodified from /root/reference by oracle/build_ref.sh against the
srsRAN-compatible header tree compat/srsran (oracle/_ref/libfalcon_ref.so, wrapper oracle/ref_walk.cc):
  * DCISearch::search / recursive_blind_dci_search / inspect_dci_location_recursively (src/src/DCISearch.cc) on the reference's
    RNTIManager and DCIMetaFormats -- vs ltephy_search_batch (full table) and the survivor-form walk, on identical tables;
  * dl_sniffer_ra_dl_dci_to_grant + dl_sniffer_config_mimo (lib/src/phy/falcon_phch/dl_sniffer_pdsch.c) and the two UL conversions
    (srsran_ra_ul_dci_to_grant path / ulsniffer_ra_ul_dci_to_grant_256, ul_sniffer_pusch.c) -- vs ltephy_dci_to_grant /
    ltephy_ul_dci_to_grant for every accepted DCI;
  * srsran_pdcch_validate_location (falcon_pdcch.c:223-250), srsran_pdcch_ue_locations_all_map (:321-356),
    srsran_pdcch_cce_avg_llr_power (:595-620) -- vs the product's O(1) validation, location list and per-CCE power rule.
The candidate tables come from the CPU oracle here (no GPU needed); tests/test_gpu_reference_code.py repeats the walk comparison
on the tables the GPU produced."""
import ctypes as C
import os
import numpy as np
import pytest
import ltelib
from ltelib import Cell, Sim, Oracle
from ltesniffer_b200 import capi
from test_host_search import oracle_table, host_geometry, locations

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libfalcon_ref.so")


class RefDci(C.Structure):
    _fields_ = [("rnti", C.c_uint16), ("format", C.c_uint8), ("L", C.c_uint8), ("ncce", C.c_uint16), ("nof_bits", C.c_uint16), ("histval", C.c_uint32),
                ("bits", C.c_uint8 * 64), ("grant_ret", C.c_int32 * 2), ("nof_prb", C.c_uint32), ("nof_re", C.c_uint32 * 2), ("nof_tb", C.c_uint32 * 2),
                ("tx_scheme", C.c_uint32 * 2), ("pmi", C.c_uint32 * 2), ("nof_layers", C.c_uint32 * 2), ("tbs", (C.c_int32 * 2) * 2),
                ("qm", (C.c_uint8 * 2) * 2), ("rv", (C.c_uint8 * 2) * 2), ("tb_en", (C.c_uint8 * 2) * 2), ("cw_idx", (C.c_uint8 * 2) * 2),
                ("prb_mask", (C.c_uint8 * 110) * 2), ("ul_L_prb", C.c_uint32), ("ul_n_prb", C.c_uint32 * 2), ("ul_n_dmrs", C.c_uint32),
                ("ul_tbs", C.c_int32 * 2), ("ul_qm", C.c_uint8 * 2)]


class RefStats(C.Structure):
    _fields_ = [("nof_decoded_locations", C.c_uint32), ("nof_cce", C.c_uint32), ("nof_missed_cce", C.c_uint32), ("nof_subframes", C.c_uint32),
                ("nof_locations", C.c_uint32)]


def reflib():
    if not os.path.exists(REF_SO):
        if os.path.isdir("/root/reference"):
            import subprocess
            capi.load_library()
            subprocess.run(["bash", os.path.join(ROOT, "oracle", "build_ref.sh")], check=True)
    if not os.path.exists(REF_SO):
        pytest.skip("oracle/_ref/libfalcon_ref.so not built (needs /root/reference)")
    L = C.CDLL(REF_SO)
    P = C.c_void_p
    L.refwalk_create.argtypes = [C.c_uint32] * 5
    L.refwalk_create.restype = P
    L.refwalk_destroy.argtypes = [P]
    L.refwalk_config.argtypes = [P, C.c_int, C.c_int, C.c_uint32]
    L.refwalk_activate.argtypes = [P, C.c_uint16, C.c_uint32, C.c_int]
    L.refwalk_subframe.argtypes = [P, P, P, P, P, C.c_uint32, P]
    L.refwalk_get_stats.argtypes = [P, P]
    L.refwalk_validate_location.argtypes = [C.c_uint32] * 4 + [C.c_uint16]
    L.refwalk_validate_location.restype = C.c_uint32
    L.refwalk_locations.argtypes = [P, C.c_uint32, P, P, P, P, P]
    L.refwalk_locations.restype = C.c_uint32
    return L


class RefWalk:
    """the reference's DCISearch behind oracle/ref_walk.cc.  golden: name of a ltelib.WalkRecord that stands in for it where
    oracle/_ref/libfalcon_ref.so cannot be built"""
    rec = None

    def __init__(self, cell, threshold=5, golden=None):
        self.rec = None
        if golden and not _ref_so_buildable():
            self.L, self.h, self.rec = None, None, ltelib.WalkRecord(golden, RefDci, RefStats, live=False)
            return
        self.L = reflib()
        self.h = self.L.refwalk_create(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, threshold)
        assert self.h
        if ltelib.WalkRecord.wanted(golden):
            self.rec = ltelib.WalkRecord(golden, RefDci, RefStats, live=True)

    def config(self, shortcut, skip_secondary, update_interval):
        if self.L is not None:
            self.L.refwalk_config(self.h, shortcut, skip_secondary, update_interval)

    def subframe(self, info, table, llr):
        if self.L is None:
            return self.rec.get()
        out = (RefDci * 64)()
        n = C.c_uint32(0)
        table = np.ascontiguousarray(table)
        llr = np.ascontiguousarray(llr, np.float32)
        assert self.L.refwalk_subframe(self.h, C.byref(info), table.ctypes.data_as(C.c_void_p), llr.ctypes.data_as(C.c_void_p), out, 64, C.byref(n)) == 0
        res = [out[i] for i in range(n.value)]
        return self.rec.put(res) if self.rec else res

    def stats(self):
        if self.L is None:
            return self.rec.stats()
        st = RefStats()
        self.L.refwalk_get_stats(self.h, C.byref(st))
        return self.rec.stats(st) if self.rec else st

    def close(self):
        if self.h:
            if self.rec:
                self.stats()
                self.rec.save()
            self.L.refwalk_destroy(self.h)
            self.h = None


def _ref_so_buildable():
    if not os.path.exists(REF_SO):
        ltelib.build_ref()
    return os.path.exists(REF_SO)


def phase_a_oracle(s, o, geo, tti):
    iq, tr, pl = s.subframe(tti)
    sym = o.ofdm(iq)
    ce, res = o.chest(tti % 10, sym)
    cfi, corr = o.pcfich(tti % 10, sym, ce)
    llr = o.pdcch_llr(tti % 10, cfi, sym, ce)
    ncce = len(llr) // 72
    info = capi.SfInfo()
    info.tti, info.cfi, info.nof_cce, info.snr_db = tti, cfi, ncce, res.snr_db
    info.noise_avg, info.rsrp_avg = res.noise_avg, res.rsrp_avg
    for p in range(2):
        for a in range(2):
            info.noise[p][a], info.rsrp[p][a] = res.noise[p][a], res.rsrp[p][a]
    pw = np.zeros(ncce, np.float32)
    ltelib.oracle().lteo_cce_power(ltelib.ptr(llr), ncce, ltelib.ptr(pw))
    for i in range(ncce):
        info.cce_power[i] = pw[i]
    nc, Ls = locations(ncce)
    T = oracle_table(o, geo, nc, Ls, llr) if res.snr_db > 6.0 else np.zeros((capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
    return info, T, llr, tr


def compare_grants(srch, cell, info, d, r):
    """product DCI -> grant conversions of accepted DCI d against what the reference's own conversion made of r"""
    if d["format"] == 0:
        for table in (0, 1):      # reference: Table 8.6.1-1 (64QAM reading), Table 8.6.1-3; product: enable_64qam 1 / 2
            rc, g = capi.ul_dci_to_grant(srch, d, 1 if table == 0 else 2)
            if r.grant_ret[0] != 0:
                continue
            L = r.ul_L_prb
            decodable = L >= 3 and all(L % p for p in ()) and _dft_size(L) and r.ul_n_prb[0] == r.ul_n_prb[1]
            ref_tbs = r.ul_tbs[table]
            if decodable and ref_tbs > 0 and int(d_mcs(d, cell)) <= 28:
                assert rc == 0, (hex(r.rnti), table, L, ref_tbs)
                assert (g.L_prb, g.n_prb, g.tbs, g.qm) == (L, r.ul_n_prb[0], ref_tbs, r.ul_qm[table]), (hex(r.rnti), table)
        return
    for table in (0, 1):
        rc, g, f = srch.dci_to_grant(d, info.tti % 10, info.cfi, table)
        assert (rc == 0) == (r.grant_ret[table] == 0), (hex(r.rnti), capi.NOF_FORMATS, d["format"], table, rc, r.grant_ret[table])
        if rc != 0:
            continue
        assert (g.nof_re, g.nof_tb, g.tx_scheme) == (r.nof_re[table], r.nof_tb[table], r.tx_scheme[table]), (hex(r.rnti), table)
        if g.tx_scheme == capi.TX_SPATIALMUX:
            assert g.pmi == r.pmi[table]
        for t in range(2):
            assert bool(g.tb[t].enabled) == bool(r.tb_en[table][t])
            if g.tb[t].enabled:
                assert (g.tb[t].tbs, g.tb[t].qm, g.tb[t].rv) == (r.tbs[table][t], r.qm[table][t], r.rv[table][t]), (hex(r.rnti), table, t)
                if g.nof_tb == 2:
                    assert g.tb[t].cw_idx == r.cw_idx[table][t]
        if table == 0:
            for sl in range(2):
                for prb in range(cell.nof_prb):
                    assert ((g.prb_mask[sl][prb >> 5] >> (prb & 31)) & 1) == r.prb_mask[sl][prb], (hex(r.rnti), sl, prb)


def _dft_size(L):
    for p in (2, 3, 5):
        while L % p == 0:
            L //= p
    return L == 1


def d_mcs(d, cell):
    N = cell.nof_prb
    rivb = int(np.ceil(np.log2(N * (N + 1) / 2)))
    return (int(d["bits"]) >> (63 - (2 + rivb + 4))) & 31


needs_ref = pytest.mark.skipif(not (os.path.exists(REF_SO) or os.path.isdir("/root/reference")), reason="reference sources not available")


@needs_ref
@pytest.mark.parametrize("name,cell,n,kw", [
    ("tm1_shortcut", Cell(100, 1, 1, 1), 30, dict(seed=1, cfi=2, nof_ues=2, dl_min=1, dl_max=2, tm=1, mcs_min=5, mcs_max=5, snr_db=30.0, fixed_L=2, si_period=5)),
    ("busy_mix_ul", Cell(50, 2, 7, 2), 60, dict(seed=2, cfi=3, nof_ues=12, dl_min=3, dl_max=5, ul_min=1, ul_max=2, tm=13, mcs_min=3, mcs_max=12, snr_db=26.0)),
    ("tm4_swap_256qam", Cell(50, 2, 11, 2), 40, dict(seed=6, cfi=2, nof_ues=8, dl_min=2, dl_max=4, tm=4, mcs_min=4, mcs_max=22, snr_db=33.0, alt_table=1, tb_swap=1)),
    ("cfg2_like_20MHz", Cell(100, 2, 7, 2), 24, dict(seed=2, cfi=3, nof_ues=150, dl_min=8, dl_max=12, tm=3, mcs_min=17, mcs_max=26, snr_db=28.0, full_band=1)),
    ("low_snr_gate", Cell(25, 1, 9, 1), 6, dict(seed=3, cfi=2, nof_ues=2, dl_min=1, dl_max=1, tm=1, mcs_min=2, mcs_max=2, snr_db=3.0)),
])
def test_product_walk_and_grants_equal_the_reference_code(infra, name, cell, n, kw):
    s, o = Sim(cell=cell, **kw), Oracle(cell)
    geo = host_geometry(cell)
    ref = RefWalk(cell)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    srch_c = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    ref.L.refwalk_config(ref.h, 1, 0, 10)
    srch.config(1, 0, 10)
    srch_c.config(1, 0, 10)
    # the reference's own DCI trace file (DCIToFile::printDCICollection, src/src/SubframeInfoConsumer.cc:66-138) against ltephy_dci_trace_line
    import tempfile
    trace_path = os.path.join(tempfile.mkdtemp(), "dci_trace.tsv")
    ref.L.refwalk_set_trace.argtypes = [C.c_void_p, C.c_char_p]
    assert ref.L.refwalk_set_trace(ref.h, trace_path.encode()) == 0
    PL = capi.load_library()
    PL.ltephy_dci_trace_line.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, C.c_char_p, C.c_size_t]
    own_lines, ntrace = [], 0
    total = nul = 0
    for tti in range(n):
        info, T, llr, tr = phase_a_oracle(s, o, geo, tti)
        want = ref.subframe(info, T, llr)
        got = srch.subframe(info, T)
        buf = C.create_string_buffer(512)
        for is_ul in (False, True):          # the reference prints the downlink container first, then the uplink one
            for d in got:
                if (d["format"] == 0) != is_ul:
                    continue
                row = np.array([d])
                nb = PL.ltephy_dci_trace_line(srch.h, row.ctypes.data_as(C.c_void_p), info.tti, info.cfi, 0, 0, 0, buf, 512)
                own_lines.append(buf.value.decode() if nb > 0 else None)
        got_c = srch_c.subframe_compact(info, srch_c.compact_from_table(info, T))
        assert got_c is not None and len(got_c) == len(got) and all(np.array_equal(got_c[k], got[k]) for k in got.dtype.names)
        # the reference keeps DL and UL DCIs in separate containers (each in acceptance order): compare per direction
        for is_ul in (False, True):
            a = [d for d in got if (d["format"] == 0) == is_ul]
            b = [r for r in want if (r.format == 0) == is_ul]
            assert len(a) == len(b), (name, tti, is_ul, len(a), len(b))
            for d, r in zip(a, b):
                assert (int(d["rnti"]), int(d["format"]), int(d["L"]), int(d["ncce"]), int(d["nof_bits"]), int(d["histogram_value"])) == \
                       (r.rnti, r.format, r.L, r.ncce, r.nof_bits, r.histval), (name, tti, is_ul)
                assert np.array_equal(capi.cand_bits(d["bits"], r.nof_bits), np.frombuffer(bytes(r.bits), np.uint8)[:r.nof_bits])
                compare_grants(srch, cell, info, d, r)
                nul += is_ul
        total += len(got)
    rs, ps = ref.stats(), srch.stats()
    assert (rs.nof_decoded_locations, rs.nof_cce, rs.nof_missed_cce, rs.nof_subframes, rs.nof_locations) == \
           (ps.nof_decoded_locations, ps.nof_cce, ps.nof_missed_cce, ps.nof_subframes, ps.nof_locations)
    ref.L.refwalk_set_trace(ref.h, None)
    ref_lines = open(trace_path).read().splitlines(keepends=True)
    own = [l for l in own_lines if l is not None]
    assert len(ref_lines) == len(own), (name, len(ref_lines), len(own), len(own_lines))
    for a, b in zip(ref_lines, own):         # everything but the wall-clock timestamp of the first column
        assert a.split("\t", 1)[1] == b.split("\t", 1)[1], (name, a, b)
        ntrace += 1
    if name != "low_snr_gate":
        assert ntrace >= n // 2
    if name == "low_snr_gate":
        assert total == 0
    else:
        assert total >= n // 2
    if kw.get("ul_min"):
        assert nul >= 5
    ref.close()


@needs_ref
def test_validate_location_equals_reference(infra):
    R, L = reflib(), capi.load_library()
    capi._bind_search(L)
    rng = np.random.default_rng(1)
    for nof_cce in (20, 25, 54, 87, 41, 8, 3):
        for _ in range(3000):
            rnti = int(rng.choice([rng.integers(0, 65536), rng.integers(0, 12), rng.integers(0xFFF0, 0x10000)]))
            l = int(rng.integers(0, 4))
            ncce = int(rng.integers(0, max(1, nof_cce))) // (1 << l) * (1 << l)
            sf = int(rng.integers(0, 10))
            assert L.ltephy_search_validate_location(nof_cce, ncce, l, sf, rnti) == R.refwalk_validate_location(nof_cce, ncce, l, sf, rnti), (nof_cce, ncce, l, sf, rnti)


@needs_ref
def test_locations_and_cce_power_equal_reference(infra):
    """srsran_pdcch_ue_locations_all_map order and the sufficient-power rule over srsran_pdcch_cce_avg_llr_power, reference code vs product"""
    cell = Cell(100, 2, 7, 2)
    ref = RefWalk(cell)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    rng = np.random.default_rng(3)
    ncce_of = {1: 20, 2: 54, 3: 87}
    for cfi in (1, 2, 3):
        ncce = ncce_of[cfi]
        llr = rng.standard_normal(72 * ncce).astype(np.float32)
        for c in rng.choice(ncce, 6, replace=False):
            llr[72 * c:72 * c + 72] *= 0.3          # some CCEs below the 0.7 threshold
        nc = np.zeros(160, np.uint16)
        Ls = np.zeros(160, np.uint8)
        sp = np.zeros(160, np.uint8)
        pw = np.zeros(88, np.float32)
        n = ref.L.refwalk_locations(ref.h, cfi, llr.ctypes.data_as(C.c_void_p), nc.ctypes.data_as(C.c_void_p), Ls.ctypes.data_as(C.c_void_p),
                                    sp.ctypes.data_as(C.c_void_p), pw.ctypes.data_as(C.c_void_p))
        enc, eL = locations(ncce)
        assert n == len(enc) and np.array_equal(nc[:n], enc) and np.array_equal(Ls[:n], eL)
        opw = np.zeros(ncce, np.float32)
        ltelib.oracle().lteo_cce_power(ltelib.ptr(llr), ncce, ltelib.ptr(opw))
        lim = min(ncce, 84)
        assert np.array_equal(pw[:lim], opw[:lim])                       # double-accumulated mean |LLR| (falcon_pdcch.c:595-620)
        # product: survivor form lists nothing for a location without sufficient power
        info = capi.SfInfo()
        info.tti, info.cfi, info.nof_cce, info.snr_db = 0, cfi, ncce, 20.0
        for i in range(ncce):
            info.cce_power[i] = opw[i]
        T = np.zeros((capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
        T["valid"] = 1
        comp = srch.compact_from_table(info, T)[0]
        for i in range(n):
            assert (comp["loc"][i]["mask"] != 0) == bool(sp[i]), (cfi, i)
    ref.close()


def test_harq_bookkeeping_equals_the_reference_class(infra):
    """ltephy_harq_classify / _update against the reference's own HARQ class (src/src/HARQ.cc compiled unmodified into oracle/_ref/libfalcon_ref.so) on a
    random traffic pattern: 40 RNTIs, 8 processes, 2 TBs, retransmissions 8 ms apart with and without NDI toggles / TBS changes, tti wrapping at 10240;
    same status every time, and "same slot" exactly when the reference hands out the same soft buffer"""
    from ltesniffer_b200 import capi
    R = reflib()
    R.refharq_create.restype = C.c_void_p
    R.refharq_destroy.argtypes = [C.c_void_p]
    R.refharq_size.argtypes = [C.c_void_p]
    R.refharq_is_retransmission.argtypes = [C.c_void_p, C.c_uint16, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint32, C.POINTER(C.c_void_p)]
    R.refharq_update.argtypes = [C.c_void_p, C.c_uint16, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_int]
    R.refharq_last_tbs.argtypes = [C.c_void_p, C.c_uint16, C.c_int, C.c_int]
    ref = R.refharq_create()
    q = capi.Harq(max_rnti=R.refharq_size(ref))
    rng = np.random.default_rng(12)
    rntis = [int(x) for x in rng.integers(0x100, 0xFFF0, 40)]
    pending = {}                     # (rnti, pid, tb) -> (ndi, tbs, tti of the last transmission)
    buf_of_slot, seen = {}, {0: 0, 1: 0, 3: 0}
    tti = 10200
    for step in range(6000):
        tti = (tti + int(rng.integers(0, 3))) % 10240
        rnti, pid, tb = rntis[int(rng.integers(0, 40))], int(rng.integers(0, 8)), int(rng.integers(0, 2))
        key = (rnti, pid, tb)
        if key in pending and rng.random() < 0.6:     # a repetition: usually 8 ms later, same NDI and size
            ndi, tbs, last = pending[key]
            t = (last + (8 if rng.random() < 0.8 else int(rng.integers(1, 20)))) % 10240
            if rng.random() < 0.15:
                ndi ^= 1
            if rng.random() < 0.1:
                tbs += 8
        else:
            ndi, tbs, t = int(rng.integers(0, 2)), int(rng.integers(2, 2000)) * 8, tti
        rv = int(rng.integers(0, 4))
        b = C.c_void_p()
        s_ref = R.refharq_is_retransmission(ref, rnti, pid, tb, ndi, rv, tbs, t, C.byref(b))
        assert q.last_tbs(rnti, pid, tb) == R.refharq_last_tbs(ref, rnti, pid, tb)     # HARQ::getlastTbs: what a reserved-MCS block is sized with
        s_own, slot = q.classify(rnti, pid, tb, ndi, tbs, t)
        assert s_own == s_ref, (step, hex(rnti), pid, tb, s_own, s_ref)
        seen[s_ref] = seen.get(s_ref, 0) + 1
        if s_ref in (capi.HARQ_NEW_TX, capi.HARQ_RE_TX):
            assert buf_of_slot.setdefault(slot, b.value) == b.value          # one slot <-> one reference buffer
            decoded = bool(rng.random() < 0.4)
            R.refharq_update(ref, rnti, pid, tb, ndi, rv, tbs, t, int(decoded))
            q.update(rnti, pid, tb, ndi, rv, tbs, t, decoded)
        pending[key] = (ndi, tbs, t)
    assert len(set(buf_of_slot.values())) == len(buf_of_slot)               # and different slots <-> different buffers
    assert seen[0] > 1000 and seen[1] > 300 and seen[3] > 100              # new / retransmission / already decoded all exercised
    R.refharq_destroy(ref)
    q.close()


def test_rb_power_equals_reference(infra):
    """per-PRB power (K10): the oracle's mean |y|^2 per PRB, which the CUDA kernel reproduces bit for bit, in dB == SubframePower::computePower
    (src/src/SubframePower.cc:18-47, called at DCISearch.cc:565) on the same symbols, up to float rounding of the different summation order"""
    from helpers import make_capture, oracle_frontend
    R = reflib()
    R.refwalk_rb_power.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p]
    cell = Cell(50, 2, 9, 2)
    sim, iq, tti, truths, payloads = make_capture(cell, 3, seed=2, cfi=2, nof_ues=4, dl_min=2, dl_max=4, tm=13, snr_db=20.0)
    o = Oracle(cell)
    for fe in oracle_frontend(o, iq, tti):
        sym0 = np.ascontiguousarray(fe["sym"][0], np.complex64)
        ref = np.zeros(cell.nof_prb, np.float32)
        R.refwalk_rb_power(cell.nof_prb, sym0.ctypes.data_as(C.c_void_p), ref.ctypes.data_as(C.c_void_p))
        own = 10.0 * np.log10(np.asarray(fe["rb_power"], np.float64))
        assert np.abs(own - ref).max() < 1e-3, np.abs(own - ref).max()


@needs_ref
@pytest.mark.parametrize("cellp", [(100, 2, 7, 2), (75, 2, 3, 2), (50, 2, 301, 2), (25, 1, 5, 1), (15, 1, 4, 1), (15, 2, 9, 2)])
def test_random_dcis_grants_equal_reference(infra, cellp):
    """2 500 random payloads per cell over the downlink formats LTESniffer decodes (1, 1A, 1C, 2, 2A), C-RNTIs and the SI / P / RA-RNTIs, every CFI
    and subframe index: ltephy_dci_to_grant against the reference's own dl_sniffer_ra_dl_dci_to_grant + dl_sniffer_config_mimo
    (lib/src/phy/falcon_phch/dl_sniffer_pdsch.c:95-132,255-276) for both MCS tables -- return code, PRB masks, TBS, Qm, rv, codeword mapping, tx scheme, PMI"""
    cell = Cell(*cellp)
    R = reflib()
    R.refgrant_dl.argtypes = [C.c_void_p, C.c_uint32, C.c_uint16, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(RefDci)]
    ref = RefWalk(cell)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    S = infra.sim()
    rng = np.random.default_rng(cell.nof_prb)
    nok = nfail = 0
    for it in range(2500):
        f = int(rng.choice([1, 2, 4, 6, 7]))
        nb = S.lte_dci_sizeof(C.byref(cell), f)
        bits = rng.integers(0, 2, nb).astype(np.uint8)
        if f == 2:
            bits[0] = 1                                   # format 0 / 1A flag
        if rng.random() < 0.3:                            # plausible MCS / RV fields more often than pure noise gives
            bits[rng.integers(0, nb, 6)] = 0
        rnti = int(rng.choice([int(rng.integers(11, 0xFFF3)), 0xFFFF, 0xFFFE, int(rng.integers(1, 11))], p=[0.7, 0.1, 0.1, 0.1]))
        tti, cfi = int(rng.integers(0, 10240)), int(rng.integers(1, 4))
        r = RefDci()
        ru = R.refgrant_dl(ref.h, f, rnti, bits.ctypes.data_as(C.c_void_p), nb, tti, cfi, C.byref(r))
        v = 0
        for i, b in enumerate(bits):
            v |= int(b) << (63 - i)
        row = np.zeros(1, capi.DCI_DTYPE)
        row["rnti"], row["format"], row["nof_bits"], row["bits"], row["ncce"], row["L"] = rnti, f, nb, v, 0, 2
        info = capi.SfInfo()
        info.tti, info.cfi = tti, cfi
        if ru != 0:
            for table in (0, 1):
                assert srch.dci_to_grant(row[0], tti % 10, cfi, table)[0] != 0
            nfail += 1
            continue
        compare_grants(srch, cell, info, row[0], r)
        nok += (r.grant_ret[0] == 0)
    assert nok > 500, (nok, nfail)
    ref.close()


@needs_ref
@pytest.mark.parametrize("cellp,n_rb_ho", [((100, 2, 7, 2), 0), ((100, 2, 7, 2), 5), ((75, 2, 3, 2), 2), ((50, 2, 301, 2), 8), ((25, 1, 5, 1), 0), ((25, 1, 5, 1), 3),
                                           ((15, 2, 9, 2), 0), ((15, 1, 4, 1), 2)])
def test_random_format0_grants_equal_reference(infra, cellp, n_rb_ho):
    """3 000 random format-0 payloads per cell and pusch-HoppingOffset (half of them with the hopping flag set, i.e. all four hop kinds of 36.213
    Tables 8.4-1/2): ltephy_ul_dci_to_grant against the reference's own ul_sniffer_ra_ul_dci_to_grant / ulsniffer_ra_ul_dci_to_grant_256 over
    ul_sniffer_ra_ul_grant_to_grant_prb_allocation (lib/src/phy/falcon_phch/ul_sniffer_pusch.c:20-245) -- L_prb, both slots' first PRB, TBS and Qm
    of Tables 8.6.1-1 and 8.6.1-3, the cyclic-shift field.  The product refuses what PUSCH_Decoder never decodes (L_prb that is no DFT size or < 3,
    valid_prb_ul at src/src/UL_Sniffer_PUSCH.cc:3-10; retransmission MCS 29-31; no TBS); everything else must agree, refusals included."""
    cell = Cell(*cellp)
    R = reflib()
    R.refgrant_ul.argtypes = [C.c_void_p, C.c_uint16, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(RefDci)]
    ref = RefWalk(cell)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    srch.L.ltephy_search_set_ul_hopping(srch.h, n_rb_ho)
    S = infra.sim()
    nb = S.lte_dci_sizeof(C.byref(cell), 0)
    rng = np.random.default_rng(cell.nof_prb * 16 + n_rb_ho)
    dmrs2 = (0, 6, 3, 4, 2, 8, 10, 9)
    nok = nhop = 0
    for it in range(3000):
        bits = rng.integers(0, 2, nb).astype(np.uint8)
        bits[0] = 0
        bits[1] = it & 1
        rnti = int(rng.integers(11, 0xFFF3))
        r = RefDci()
        assert R.refgrant_ul(ref.h, rnti, bits.ctypes.data_as(C.c_void_p), nb, int(rng.integers(0, 10240)), n_rb_ho, C.byref(r)) == 0
        v = 0
        for i, b in enumerate(bits):
            v |= int(b) << (63 - i)
        row = np.zeros(1, capi.DCI_DTYPE)
        row["rnti"], row["format"], row["nof_bits"], row["bits"], row["L"] = rnti, 0, nb, v, 2
        mcs = d_mcs(row[0], cell)
        for table in (0, 1):
            rc, g = capi.ul_dci_to_grant(srch, row[0], 1 if table == 0 else 2)
            L = r.ul_L_prb
            expect = r.grant_ret[table] == 0 and L >= 3 and _dft_size(L) and mcs <= 28 and r.ul_tbs[table] > 0
            assert (rc == 0) == expect, (it, table, rc, r.grant_ret[table], L, mcs, r.ul_tbs[table])
            if rc == 0:
                assert (g.L_prb, g.n_prb, g.n_prb_slot1, g.tbs, g.qm) == (L, r.ul_n_prb[0], r.ul_n_prb[1], r.ul_tbs[table], r.ul_qm[table]), (it, table)
                assert g.n_dmrs2 == dmrs2[r.ul_n_dmrs] and g.rv == r.rv[table][0] == 0
                nok += 1
                nhop += r.ul_n_prb[0] != r.ul_n_prb[1]
    assert nok > 300 and nhop > 20, (nok, nhop)
    ref.close()


@needs_ref
@pytest.mark.parametrize("cellp,n_rb_ho", [((100, 2, 7, 2), 0), ((100, 2, 7, 2), 6), ((50, 2, 301, 2), 0), ((25, 1, 5, 1), 2),
                                           ((15, 2, 9, 2), 0), ((15, 1, 4, 1), 1)])
def test_random_rar_grants_equal_reference(infra, cellp, n_rb_ho):
    """4 000 random 20-bit RAR grants per cell (inside random MAC RAR PDUs of 1-3 RARs): ltephy_rar_unpack against the reference's own
    ul_sniffer_dci_rar_unpack + ul_sniffer_dci_rar_to_ul_dci + ul_sniffer_ra_ul_dci_to_grant (falcon_dci.c:648-684, ul_sniffer_pusch.c:205-245, called at
    DL_Sniffer_PDSCH.cc:646-658) -- L_prb, both slots' first PRB (a set hopping flag is read as hop value 1), TBS, Qm.  valid = 0 exactly where the
    reference's conversion fails or yields what PUSCH_Decoder cannot decode (L_prb no DFT size or < 3)."""
    cell = Cell(*cellp)
    R = reflib()
    R.refgrant_rar.argtypes = [C.c_void_p, C.c_void_p, C.c_uint16, C.c_uint32, C.c_uint32, C.POINTER(RefDci)]
    ref = RefWalk(cell)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    srch.L.ltephy_search_set_ul_hopping(srch.h, n_rb_ho)
    rng = np.random.default_rng(cell.nof_prb + n_rb_ho)
    nvalid = nhop = 0
    for it in range(1600):
        k = int(rng.integers(1, 4))
        grants = [int(rng.integers(0, 1 << 20)) for _ in range(k)]
        if it % 3 == 0:                                   # small allocations and MCS are what msg 3 really uses
            grants = [(g & ~(0x3FF << 9)) | (int(rng.integers(0, 6 * cell.nof_prb)) & 0x3FF) << 9 for g in grants]
        rntis = [int(rng.integers(1, 0xFFF0)) for _ in range(k)]
        tas = [int(rng.integers(0, 2048)) for _ in range(k)]
        pdu = bytes([(0x80 if j < k - 1 else 0) | 0x40 | int(rng.integers(0, 64)) for j in range(k)])
        for g, rn, ta in zip(grants, rntis, tas):
            pdu += bytes([ta >> 4, ((ta & 15) << 4) | (g >> 16), (g >> 8) & 255, g & 255, rn >> 8, rn & 255])
        rc, rars, _ = capi.rar_unpack(srch, pdu + bytes(int(rng.integers(0, 3))))
        assert rc == 0 and [(x.t_crnti, x.ta) for x in rars] == list(zip(rntis, tas))
        for x, g, rn in zip(rars, grants, rntis):
            bits = np.array([(g >> (19 - i)) & 1 for i in range(20)], np.uint8)
            r = RefDci()
            R.refgrant_rar(ref.h, bits.ctypes.data_as(C.c_void_p), rn, 100, n_rb_ho, C.byref(r))
            L = r.ul_L_prb
            expect = r.grant_ret[0] == 0 and L >= 3 and _dft_size(L) and r.ul_tbs[0] > 0
            assert bool(x.valid) == expect, (hex(g), r.grant_ret[0], L, r.ul_tbs[0])
            assert (x.hopping_flag, x.tpc, x.ul_delay, x.cqi_request) == (g >> 19, (g >> 2) & 7, (g >> 1) & 1, g & 1)
            if x.valid:
                assert (x.grant.rnti, x.grant.L_prb, x.grant.n_prb, x.grant.n_prb_slot1, x.grant.tbs, x.grant.qm, x.grant.rv, x.grant.n_dmrs2) == \
                    (rn, L, r.ul_n_prb[0], r.ul_n_prb[1], r.ul_tbs[0], r.ul_qm[0], r.rv[0][0], 0), hex(g)
                nvalid += 1
                nhop += r.ul_n_prb[0] != r.ul_n_prb[1]
    assert nvalid > 200 and nhop > 20, (nvalid, nhop)
    ref.close()


@needs_ref
def test_cqi_subband_count_equals_reference(infra):
    """ltephy_ul_cqi_len's subband count == the reference's ul_sniffer_cqi_hl_get_no_subbands (lib/src/phy/falcon_phch/dl_sniffer_pdsch.c:277-302), 7..110 PRB"""
    R = reflib()
    L = capi.load_library()
    capi._bind_search(L)
    for n in range(7, 111):
        assert L.ltephy_ul_cqi_len(n, 3) == 4 + 2 * R.refcqi_no_subbands(n), n


@needs_ref
@pytest.mark.parametrize("cellp", [(100, 2, 7, 2), (50, 2, 301, 2), (25, 1, 5, 1), (15, 2, 9, 2)])
def test_edge_case_dcis_grants_equal_reference(infra, cellp):
    """Structured companion of the random-payload test: random payloads are unpacked, their fields pushed to the edges (MCS 0 / 9 / 10 / 27 / 28 / 29 / 31,
    disabled blocks in every combination, every precoding value, empty / full / single-RBG bitmaps, RIVs at 0, at the last valid value, one past it and all
    ones, both gaps, the N_PRB^1A bit) and packed again; product and the reference's conversion must agree on every one of them, refusals included."""
    cell = Cell(*cellp)
    R = reflib()
    R.refgrant_dl.argtypes = [C.c_void_p, C.c_uint32, C.c_uint16, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(RefDci)]
    ref = RefWalk(cell)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    S = infra.sim()
    S.lte_dci_unpack.argtypes = [C.c_void_p, C.c_int, C.c_uint16, C.c_void_p, C.c_uint32, C.c_void_p]
    S.lte_dci_pack.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(1000 + cell.nof_prb)
    N = cell.nof_prb
    P = 1 if N <= 10 else 2 if N <= 26 else 3 if N <= 63 else 4
    nrbg = (N + P - 1) // P
    seen = {"ok": 0, "ref_fail": 0, "two_off": 0, "mimo_err": 0}
    for it in range(3000):
        f = int(rng.choice([1, 2, 4, 6, 7]))
        nb = S.lte_dci_sizeof(C.byref(cell), f)
        bits = rng.integers(0, 2, nb).astype(np.uint8)
        if f == 2:
            bits[0] = 1
        rnti = int(rng.choice([int(rng.integers(11, 0xFFF3)), 0xFFFF, 0xFFFE, int(rng.integers(1, 11))], p=[0.7, 0.1, 0.1, 0.1]))
        d = ltelib.Dci()
        if S.lte_dci_unpack(C.byref(cell), f, rnti, bits.ctypes.data_as(C.c_void_p), nb, C.byref(d)) != 0:
            continue
        for t in range(2):
            if rng.random() < 0.5:
                d.mcs[t] = int(rng.choice([0, 9, 10, 16, 17, 27, 28, 29, 31]))
            if rng.random() < 0.3:
                d.rv[t] = int(rng.choice([0, 1]))
            d.tb_en[t] = 0 if (rng.random() < 0.25 and f >= 6) else 1
        if rng.random() < 0.5:
            d.pinfo = int(rng.integers(0, 8))
        if rng.random() < 0.4:
            if d.alloc_type == 0:
                d.rbg_bitmask = int(rng.choice([0, (1 << nrbg) - 1, 1, 1 << (nrbg - 1), 1 << int(rng.integers(0, nrbg))]))
            elif d.alloc_type == 1:
                d.t1_vrb_bitmask = int(rng.choice([0, 1, 0xFFFFFFFF & ((1 << 20) - 1)]))
            else:
                lim = N * (N + 1) // 2
                d.riv = int(rng.choice([0, N - 1, lim - 1, lim, (1 << 13) - 1, int(rng.integers(0, lim))]))
                d.t2_ngap2 = int(rng.integers(0, 2))
                d.n_prb1a = int(rng.choice([2, 3]))
        out = np.zeros(64, np.uint8)
        nbo = C.c_uint32(0)
        if S.lte_dci_pack(C.byref(cell), C.byref(d), out.ctypes.data_as(C.c_void_p), C.byref(nbo)) != 0:
            continue
        assert nbo.value == nb
        bits = out[:nb].copy()
        tti, cfi = int(rng.integers(0, 10240)), int(rng.integers(1, 4))
        r = RefDci()
        ru = R.refgrant_dl(ref.h, f, rnti, bits.ctypes.data_as(C.c_void_p), nb, tti, cfi, C.byref(r))
        v = 0
        for i, b in enumerate(bits):
            v |= int(b) << (63 - i)
        row = np.zeros(1, capi.DCI_DTYPE)
        row["rnti"], row["format"], row["nof_bits"], row["bits"], row["L"] = rnti, f, nb, v, 2
        info = capi.SfInfo()
        info.tti, info.cfi = tti, cfi
        if ru != 0:
            for table in (0, 1):
                assert srch.dci_to_grant(row[0], tti % 10, cfi, table)[0] != 0
            seen["ref_fail"] += 1
            continue
        compare_grants(srch, cell, info, row[0], r)
        seen["ok"] += r.grant_ret[0] == 0
        seen["mimo_err"] += r.grant_ret[0] in (-1, -2, -3) and f >= 6
        seen["two_off"] += f >= 6 and d.tb_en[0] == 0 and d.tb_en[1] == 0
    assert seen["ok"] > 800 and seen["two_off"] > 20 and seen["mimo_err"] > 50, seen
    ref.close()


@needs_ref
@pytest.mark.parametrize("cellp,seed,shortcut,skip2,thr", [((100, 2, 7, 2), 1, 1, 0, 5), ((50, 1, 3, 1), 2, 1, 0, 5), ((25, 2, 11, 2), 3, 1, 0, 5), ((75, 2, 200, 1), 4, 1, 0, 5),
                                                           ((50, 2, 3, 2), 5, 0, 0, 5), ((50, 2, 3, 2), 6, 1, 1, 5), ((100, 2, 7, 2), 7, 1, 0, 2), ((25, 1, 4, 1), 8, 0, 1, 9)])
def test_product_walk_equals_reference_code_on_adversarial_tables(infra, cellp, seed, shortcut, skip2, thr):
    """The walk against the reference's own DCISearch.cc on candidate tables no transmitter produces (the generator of tests/test_survivor_fuzz.py): RNTIs
    from a small pool so that histograms cross the threshold, the same RNTI in a location and its first children (shortcut, disambiguation), RNTI 0,
    undecoded entries, RA / paging / SI / reserved RNTIs at random places, low-power CCEs, all CFIs, subframes under the 6 dB gate, meta-format re-splits every
    7 subframes, and from subframe 200 on a RAR-activated RNTI (the temp_dci0 rule); also with shortcut discovery off, secondary formats skipped and other
    histogram thresholds.  Same DCIs in the same order, same histogram values, same statistics."""
    from test_survivor_fuzz import _random_table
    L = capi.load_library()
    capi._bind_search(L)
    rng = np.random.default_rng(seed)
    cell = Cell(*cellp)
    ref = RefWalk(cell, threshold=thr)
    srch = capi.Search(*cellp, threshold=thr)
    ref.L.refwalk_config(ref.h, shortcut, skip2, 7)
    srch.config(shortcut, skip2, 7)
    S = infra.sim()
    sizes_n = len({S.lte_dci_sizeof(C.byref(cell), f) for f in range(9)})
    o = ltelib.Oracle(cell)
    pool = rng.integers(0x100, 0xFFF0, 12)
    ndci = nul = 0
    for sf in range(int(os.environ.get("WALK_FUZZ_SF", "260"))):
        cfi = int(rng.integers(1, 4))
        nof_cce = int(infra.oracle().lteo_nof_cce(o.h, cfi))
        info = capi.SfInfo()
        info.tti, info.cfi, info.nof_cce = sf, cfi, nof_cce
        info.snr_db = 20.0 if rng.random() > 0.03 else 3.0
        amp = np.where(rng.random(nof_cce) < 0.15, 0.3, 1.2).astype(np.float32)
        llr = (np.repeat(amp, 72) * rng.choice([-1.0, 1.0], 72 * nof_cce)).astype(np.float32)
        pw = np.zeros(nof_cce, np.float32)
        ltelib.oracle().lteo_cce_power(ltelib.ptr(llr), nof_cce, ltelib.ptr(pw))
        for c in range(nof_cce):
            info.cce_power[c] = pw[c]
        if sf == 200:
            rar = 0x7A7A
            L.ltephy_search_activate(srch.h, rar, 0, 2)
            ref.L.refwalk_activate(ref.h, rar, 0, 2)
            pool = np.append(pool, rar)
        T = _random_table(rng, L, nof_cce, sf % 10, pool, sizes_n)
        want = ref.subframe(info, T, llr)
        got = srch.subframe(info, T, max_out=256)
        for is_ul in (False, True):
            a = [d for d in got if (d["format"] == 0) == is_ul]
            b = [r for r in want if (r.format == 0) == is_ul]
            assert len(a) == len(b), (cellp, sf, is_ul, len(a), len(b))
            for d, r in zip(a, b):
                assert (int(d["rnti"]), int(d["format"]), int(d["L"]), int(d["ncce"]), int(d["nof_bits"]), int(d["histogram_value"])) == \
                       (r.rnti, r.format, r.L, r.ncce, r.nof_bits, r.histval), (cellp, sf, is_ul)
                assert np.array_equal(capi.cand_bits(d["bits"], r.nof_bits), np.frombuffer(bytes(r.bits), np.uint8)[:r.nof_bits])
                nul += is_ul
        ndci += len(got)
    rs, ps = ref.stats(), srch.stats()
    assert (rs.nof_decoded_locations, rs.nof_cce, rs.nof_missed_cce, rs.nof_subframes, rs.nof_locations) == \
           (ps.nof_decoded_locations, ps.nof_cce, ps.nof_missed_cce, ps.nof_subframes, ps.nof_locations)
    assert ndci > 200 and (nul > 10 or skip2), (ndci, nul)
    ref.close()
