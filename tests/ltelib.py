"""ctypes bindings for the TEST infrastructure: sim/libltesim.so (synthetic eNB) and
oracle/liblteoracle.so (CPU oracle).  Imported only by tests/, bench.py's cpu_baseline /
--impl reference legs and __graft_entry__.smoke()."""
import ctypes as C
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MAX_PRB = 110
DCI_MAX_BITS = 64
SIM_MAX_DCI = 32


class Cell(C.Structure):
    _fields_ = [("nof_prb", C.c_uint32), ("nof_ports", C.c_uint32), ("cell_id", C.c_uint32), ("nof_rx", C.c_uint32), ("symbol_sz", C.c_uint32),
                ("phich_ng", C.c_uint32), ("phich_ext", C.c_uint32)]

    def fft(self):
        """symbol size: symbol_sz, or the standard LTE size when it is 0"""
        return self.symbol_sz or (128 if self.nof_prb <= 6 else 256 if self.nof_prb <= 15 else 512 if self.nof_prb <= 25 else 1024 if self.nof_prb <= 50 else 2048)


class SimCfg(C.Structure):
    _fields_ = [("cell", Cell), ("seed", C.c_uint64), ("cfi", C.c_uint32), ("nof_ues", C.c_uint32),
                ("dl_min", C.c_uint32), ("dl_max", C.c_uint32), ("ul_min", C.c_uint32), ("ul_max", C.c_uint32),
                ("tm", C.c_uint32), ("mcs_min", C.c_uint32), ("mcs_max", C.c_uint32), ("si_period", C.c_uint32),
                ("snr_db", C.c_float), ("chan_delay", C.c_uint32), ("fixed_L", C.c_uint32), ("full_band", C.c_uint32),
                ("alt_table", C.c_uint32), ("ul_pusch", C.c_uint32), ("tb_swap", C.c_uint32), ("harq_retx", C.c_uint32), ("pbch", C.c_uint32), ("cfo_hz", C.c_float), ("reserved", C.c_uint32 * 2)]


class DciTruth(C.Structure):
    _fields_ = [("rnti", C.c_uint16), ("format", C.c_uint8), ("L", C.c_uint8), ("ncce", C.c_uint16), ("nbits", C.c_uint16),
                ("bits", C.c_uint8 * DCI_MAX_BITS), ("nof_tb", C.c_uint8), ("tx_scheme", C.c_uint8),
                ("qm", C.c_uint8 * 2), ("rv", C.c_uint8 * 2), ("mcs", C.c_uint8 * 2), ("tbs", C.c_int32 * 2),
                ("payload_off", C.c_uint32 * 2), ("nof_prb", C.c_uint32), ("nof_re", C.c_uint32)]


class SimTruth(C.Structure):
    _fields_ = [("tti", C.c_uint32), ("cfi", C.c_uint32), ("nof_dci", C.c_uint32), ("dci", DciTruth * SIM_MAX_DCI),
                ("payload_len", C.c_uint32)]


class Dci(C.Structure):
    _fields_ = [("rnti", C.c_uint16), ("format", C.c_uint8), ("alloc_type", C.c_uint8), ("rbg_bitmask", C.c_uint32),
                ("t1_vrb_bitmask", C.c_uint32), ("t1_subset", C.c_uint32), ("t1_shift", C.c_uint32), ("riv", C.c_uint32),
                ("t2_dist", C.c_uint8), ("t2_ngap2", C.c_uint8), ("n_prb1a", C.c_uint8),
                ("mcs", C.c_uint8 * 2), ("rv", C.c_uint8 * 2), ("ndi", C.c_uint8 * 2), ("tb_en", C.c_uint8 * 2),
                ("tb_cw_swap", C.c_uint8), ("pinfo", C.c_uint8), ("pid", C.c_uint8), ("tpc", C.c_uint8),
                ("hop", C.c_uint8), ("n_dmrs", C.c_uint8), ("cqi_req", C.c_uint8)]


class GrantTb(C.Structure):
    _fields_ = [("enabled", C.c_uint8), ("qm", C.c_uint8), ("rv", C.c_uint8), ("mcs", C.c_uint8), ("tbs", C.c_int32),
                ("nof_bits", C.c_uint32)]


class DlGrant(C.Structure):
    _fields_ = [("prb_mask", (C.c_uint8 * MAX_PRB) * 2), ("nof_prb", C.c_uint32), ("nof_tb", C.c_uint32), ("tb", GrantTb * 2),
                ("nof_re", C.c_uint32), ("tx_scheme", C.c_uint8), ("nof_layers", C.c_uint8), ("pmi", C.c_uint8), ("cw_swap", C.c_uint8)]


class ChestRes(C.Structure):
    _fields_ = [("noise", (C.c_float * 2) * 2), ("rsrp", (C.c_float * 2) * 2), ("noise_avg", C.c_float), ("rsrp_avg", C.c_float),
                ("cfo_re", C.c_float), ("cfo_im", C.c_float), ("snr_db", C.c_float), ("cfo", C.c_float)]


HARQ_CB_STRIDE = 18448
FORMATS = ["0", "1", "1A", "1B", "1C", "1D", "2", "2A", "2B"]
_built = False


def build_infra():
    """make sim/libltesim.so and oracle/liblteoracle.so if missing or stale."""
    global _built
    if _built:
        return
    subprocess.run(["make", "-s", "-C", ROOT, "all"], check=True)
    _built = True


_sim = None
_ora = None


def sim():
    global _sim
    if _sim is None:
        build_infra()
        L = C.CDLL(os.path.join(ROOT, "sim", "libltesim.so"))
        L.lte_sim_create.restype = C.c_void_p
        L.lte_sim_create.argtypes = [C.POINTER(SimCfg)]
        L.lte_sim_destroy.argtypes = [C.c_void_p]
        L.lte_sim_subframe.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(SimTruth), C.c_void_p, C.c_uint32]
        L.lte_sim_rntis.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.lte_sim_pdcch_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_uint16, C.c_uint32, C.c_void_p]
        L.lte_sim_dlsch_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
        L.lte_dci_sizeof.argtypes = [C.POINTER(Cell), C.c_int]
        L.lte_dci_sizeof.restype = C.c_uint32
        L.lte_dci_unpack.argtypes = [C.POINTER(Cell), C.c_int, C.c_uint16, C.c_void_p, C.c_uint32, C.POINTER(Dci)]
        L.lte_dci_pack.argtypes = [C.POINTER(Cell), C.POINTER(Dci), C.c_void_p, C.POINTER(C.c_uint32)]
        L.lte_dl_dci_to_grant.argtypes = [C.POINTER(Cell), C.c_uint32, C.c_uint32, C.c_int, C.POINTER(Dci), C.POINTER(DlGrant)]
        L.lte_ul_dci_to_grant.argtypes = [C.POINTER(Cell), C.POINTER(Dci), C.c_int, C.POINTER(UlGrant)]
        L.lte_sim_ul_subframe_rx.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(UlCfg), C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_uint32]
        L.lte_pdcch_validate_location.argtypes = [C.c_uint32] * 4 + [C.c_uint16]
        L.lte_pdcch_validate_location.restype = C.c_uint32
        L.lte_sf_len.argtypes = [C.c_uint32]
        L.lte_sf_len.restype = C.c_uint32
        L.lte_gold_bits.argtypes = [C.c_uint32, C.c_void_p, C.c_uint32]
        L.lte_crc.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32]
        L.lte_crc.restype = C.c_uint32
        L.lte_tbs_from_idx.argtypes = [C.c_int, C.c_uint32]
        L.lte_rm_turbo_E.argtypes = [C.c_uint32] * 5
        L.lte_rm_turbo_E.restype = C.c_uint32
        _sim = L
    return _sim


def oracle():
    global _ora
    if _ora is None:
        build_infra()
        L = C.CDLL(os.path.join(ROOT, "oracle", "liblteoracle.so"))
        P = C.c_void_p
        L.lteo_create.restype = P
        L.lteo_create.argtypes = [C.POINTER(Cell)]
        L.lteo_destroy.argtypes = [P]
        L.lteo_nof_cce.argtypes = [P, C.c_uint32]
        L.lteo_nof_cce.restype = C.c_uint32
        L.lteo_det_sum.argtypes = [P, C.c_uint32]
        L.lteo_det_sum.restype = C.c_float
        L.lteo_ofdm_rx.argtypes = [P, P, P]
        L.lteo_chest.argtypes = [P, C.c_uint32, P, P, C.POINTER(ChestRes)]
        L.lteo_rb_power.argtypes = [P, P, P]
        L.lteo_pcfich_decode.argtypes = [P, C.c_uint32, P, P, P]
        L.lteo_pcfich_decode.restype = C.c_uint32
        L.lteo_pdcch_extract_llr.argtypes = [P, C.c_uint32, C.c_uint32, P, P, P]
        L.lteo_pdcch_extract_llr.restype = C.c_uint32
        L.lteo_cce_power.argtypes = [P, C.c_uint32, P]
        L.lteo_dci_decode.argtypes = [P, C.c_uint32, C.c_uint32, P, P]
        L.lteo_pdsch_llr.argtypes = [P, C.c_uint32, C.c_uint32, C.c_uint16, C.POINTER(DlGrant), P, P, P, P]
        L.lteo_dlsch_decode.argtypes = [P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, P, P]
        L.lteo_rm_turbo_rx.argtypes = [P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, P]
        L.lteo_turbo_decode.argtypes = [P, C.c_uint32, C.c_uint32, C.c_int, P, P]
        L.lteo_turbo_decode.restype = C.c_uint32
        L.lteo_pdsch_decode.argtypes = [P, C.c_uint32, C.c_uint32, C.c_uint16, C.POINTER(DlGrant), P, P, C.c_uint32, P, P]
        _ora = L
    return _ora


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def ptr_array(arrs):
    """void*[] from a list of numpy arrays."""
    t = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    return t


class Sim:
    def __init__(self, **kw):
        cell = kw.pop("cell")
        cfg = SimCfg()
        cfg.cell = cell
        d = dict(seed=1, cfi=2, nof_ues=1, dl_min=1, dl_max=1, ul_min=0, ul_max=0, tm=1, mcs_min=5, mcs_max=5, si_period=0,
                 snr_db=30.0, chan_delay=0, fixed_L=0xFF, full_band=0, alt_table=0, ul_pusch=0)
        d.update(kw)
        for k, v in d.items():
            setattr(cfg, k, v)
        self.cfg = cfg
        self.cell = cell
        self.h = sim().lte_sim_create(C.byref(cfg))
        assert self.h, "lte_sim_create failed"
        self.sf_len = 15 * cell.fft()

    def rntis(self):
        out = np.zeros(self.cfg.nof_ues, np.uint16)
        sim().lte_sim_rntis(self.h, ptr(out), len(out))
        return out

    def subframe(self, tti):
        iq = np.zeros((self.cell.nof_rx, self.sf_len), np.complex64)
        tr = SimTruth()
        pl = np.zeros(1 << 17, np.uint8)
        r = sim().lte_sim_subframe(self.h, tti, ptr(iq), C.byref(tr), ptr(pl), len(pl))
        assert r == 0, r
        return iq, tr, pl[:tr.payload_len].copy()

    def __del__(self):
        try:
            sim().lte_sim_destroy(self.h)
        except Exception:
            pass


class Oracle:
    """Thin OO wrapper over the oracle stages for one cell."""

    def __init__(self, cell):
        self.cell = cell
        self.L = oracle()
        self.h = self.L.lteo_create(C.byref(cell))
        assert self.h
        self.nsc = 12 * cell.nof_prb

    def __del__(self):
        try:
            self.L.lteo_destroy(self.h)
        except Exception:
            pass

    def ofdm(self, iq):
        """iq [ant][sf_len] -> sym [ant][14*nsc]"""
        sym = np.zeros((self.cell.nof_rx, 14 * self.nsc), np.complex64)
        for a in range(self.cell.nof_rx):
            self.L.lteo_ofdm_rx(self.h, ptr(np.ascontiguousarray(iq[a])), ptr(sym[a]))
        return sym

    def chest(self, sf_idx, sym):
        npa = self.cell.nof_ports * self.cell.nof_rx
        ce = np.zeros((npa, 14 * self.nsc), np.complex64)
        res = ChestRes()
        self.L.lteo_chest(self.h, sf_idx, ptr_array([sym[a] for a in range(self.cell.nof_rx)]),
                          ptr_array([ce[i] for i in range(npa)]), C.byref(res))
        return ce, res

    def _pp(self, sym, ce):
        return (ptr_array([sym[a] for a in range(sym.shape[0])]), ptr_array([ce[i] for i in range(ce.shape[0])]))

    def pcfich(self, sf_idx, sym, ce):
        corr = np.zeros(3, np.float32)
        s, c = self._pp(sym, ce)
        cfi = self.L.lteo_pcfich_decode(self.h, sf_idx, s, c, ptr(corr))
        return cfi, corr

    def pdcch_llr(self, sf_idx, cfi, sym, ce):
        n = self.L.lteo_nof_cce(self.h, cfi)
        llr = np.zeros(n * 72, np.float32)
        s, c = self._pp(sym, ce)
        self.L.lteo_pdcch_extract_llr(self.h, sf_idx, cfi, s, c, ptr(llr))
        return llr

    def rb_power(self, sym0):
        p = np.zeros(self.cell.nof_prb, np.float32)
        self.L.lteo_rb_power(self.h, ptr(np.ascontiguousarray(sym0)), ptr(p))
        return p

    def dci_decode(self, e, nof_bits):
        e = np.ascontiguousarray(e, np.float32)
        bits = np.zeros(DCI_MAX_BITS, np.uint8)
        crc = C.c_uint16(0)
        r = self.L.lteo_dci_decode(ptr(e), len(e), nof_bits, ptr(bits), C.byref(crc))
        return r, bits[:nof_bits].copy(), crc.value

    def pdsch_llr(self, sf_idx, cfi, rnti, grant, sym, ce):
        n = grant.nof_re
        llr = [np.zeros(n * 8 + 16, np.int16) for _ in range(2)]
        eq = [np.zeros(n + 2, np.complex64) for _ in range(2)]
        s, c = self._pp(sym, ce)
        r = self.L.lteo_pdsch_llr(self.h, sf_idx, cfi, rnti, C.byref(grant), s, c, ptr_array(llr), ptr_array(eq))
        return r, llr, eq

    def pbch_decode(self, sym, ce):
        """-> (found, mib bits[24], nof_ports, frame position q = SFN mod 4)"""
        s, c = self._pp(sym, ce)
        mib = np.zeros(24, np.uint8)
        npo, fq = C.c_uint32(0), C.c_uint32(0)
        self.L.lteo_pbch_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        r = self.L.lteo_pbch_decode(self.h, s, c, ptr(mib), C.byref(npo), C.byref(fq))
        return r, mib, npo.value, fq.value

    def cfo_correct(self, cfo_hz, iq):
        out = np.zeros_like(iq)
        self.L.lteo_cfo_correct.argtypes = [C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]
        for a in range(iq.shape[0]):
            self.L.lteo_cfo_correct(self.h, cfo_hz, ptr(np.ascontiguousarray(iq[a])), ptr(out[a]))
        return out

    def pdsch_decode_harq(self, sf_idx, cfi, rnti, grant, sym, ce, soft, combine, max_iter=8):
        """soft: [int16 array (16 * HARQ_CB_STRIDE) or None] per TB, combine: [0/1] per TB"""
        pl = [np.zeros(16000, np.uint8) for _ in range(2)]
        ok = (C.c_int * 2)(0, 0)
        s, c = self._pp(sym, ce)
        sp = (C.c_void_p * 2)(*[None if a is None else a.ctypes.data for a in soft])
        cb = (C.c_int * 2)(*combine)
        self.L.lteo_pdsch_decode_harq.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint16, C.POINTER(DlGrant), C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.c_void_p]
        r = self.L.lteo_pdsch_decode_harq(self.h, sf_idx, cfi, rnti, C.byref(grant), s, c, max_iter, ptr_array(pl), ok, sp, cb)
        return r, pl, [ok[0], ok[1]]

    def pdsch_decode(self, sf_idx, cfi, rnti, grant, sym, ce, max_iter=8):
        pl = [np.zeros(16000, np.uint8) for _ in range(2)]
        ok = (C.c_int * 2)(0, 0)
        s, c = self._pp(sym, ce)
        r = self.L.lteo_pdsch_decode(self.h, sf_idx, cfi, rnti, C.byref(grant), s, c, max_iter, ptr_array(pl), ok)
        return r, pl, [ok[0], ok[1]]


def unpack_and_grant(cell, fmt, rnti, bits, sf_idx, cfi, alt=0):
    d = Dci()
    b = np.ascontiguousarray(bits, np.uint8)
    r = sim().lte_dci_unpack(C.byref(cell), fmt, rnti, ptr(b), len(b), C.byref(d))
    if r:
        return r, d, None
    g = DlGrant()
    r = sim().lte_dl_dci_to_grant(C.byref(cell), sf_idx, cfi, alt, C.byref(d), C.byref(g))
    return r, d, g


# ------------------------------------------------------------------------------------------------
# oracle/_ref: the reference's own RNTIManager + the oracle walk that uses it
class WalkDci(C.Structure):
    _fields_ = [("rnti", C.c_uint16), ("format", C.c_uint8), ("L", C.c_uint8), ("ncce", C.c_uint16), ("nof_bits", C.c_uint16),
                ("bits", C.c_uint8 * DCI_MAX_BITS), ("histval", C.c_uint32)]


class WalkStats(C.Structure):
    _fields_ = [("nof_decoded_locations", C.c_uint32), ("nof_cce", C.c_uint32), ("nof_missed_cce", C.c_uint32), ("nof_subframes", C.c_uint32),
                ("nof_locations", C.c_uint32)]


_walk = None
_rm = None


def build_ref():
    if os.path.isdir("/root/reference"):
        subprocess.run(["bash", os.path.join(ROOT, "oracle", "build_ref.sh")], check=True, stdout=subprocess.DEVNULL)


def ref_available():
    return os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libfalcon_walk.so"))


def ref_buildable():
    """oracle/_ref is built, or has just been built from the reference sources"""
    build_ref()
    return ref_available()


def walklib():
    global _walk
    if _walk is None:
        build_infra()
        build_ref()
        C.CDLL(os.path.join(ROOT, "oracle", "liblteoracle.so"), mode=C.RTLD_GLOBAL)
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libfalcon_walk.so"))
        P = C.c_void_p
        L.lteo_walk_create.argtypes = [C.POINTER(Cell), C.c_uint32]
        L.lteo_walk_create.restype = P
        L.lteo_walk_destroy.argtypes = [P]
        L.lteo_walk_config.argtypes = [P, C.c_int, C.c_int, C.c_uint32]
        L.lteo_walk_subframe.argtypes = [P, C.c_uint32, C.c_uint32, C.c_uint32, P, C.c_float, P, C.c_uint32, P]
        L.lteo_walk_stats.argtypes = [P, P]
        L.lteo_walk_activate.argtypes = [P, C.c_uint16, C.c_uint32, C.c_int]
        _walk = L
    return _walk


def rntimgr_ref():
    """the reference's RNTIManager through its own C wrappers (lib/include/falcon/util/rnti_manager_c.h)"""
    global _rm
    if _rm is None:
        build_ref()
        L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "librntimgr_ref.so"))
        P = C.c_void_p
        L.rnti_manager_create.argtypes = [C.c_uint32] * 3
        L.rnti_manager_create.restype = P
        L.rnti_manager_free.argtypes = [P]
        for f in ("rnti_manager_add_evergreen", "rnti_manager_add_forbidden"):
            getattr(L, f).argtypes = [P, C.c_uint16, C.c_uint16, C.c_uint32]
        L.rnti_manager_add_candidate.argtypes = [P, C.c_uint16, C.c_uint32]
        for f in ("rnti_manager_validate_and_refresh", "rnti_manager_is_evergreen", "rnti_manager_is_forbidden"):
            getattr(L, f).argtypes = [P, C.c_uint16, C.c_uint32]
        L.rnti_manager_activate_and_refresh.argtypes = [P, C.c_uint16, C.c_uint32, C.c_int]
        L.rnti_manager_step_time.argtypes = [P]
        L.rnti_manager_getFrequency.argtypes = [P, C.c_uint16, C.c_uint32]
        L.rnti_manager_getFrequency.restype = C.c_uint32
        L.rnti_manager_get_associated_format_idx.argtypes = [P, C.c_uint16]
        L.rnti_manager_get_associated_format_idx.restype = C.c_uint32
        L.rnti_manager_get_activation_reason.argtypes = [P, C.c_uint16]
        _rm = L
    return _rm


class WalkRecord:
    """What a walk over the reference's code (oracle/_ref) answered, call by call, kept as tests/golden/<name>.npz: subframe() records of
    every call and the final statistics.  A test replays it where oracle/_ref cannot be built, so that its comparison with the reference
    still runs; with LTEPHY_RECORD_GOLDEN=<dir> in the environment a live walk writes its record to <dir>/<name>.npz instead."""

    def __init__(self, name, rec_type, stats_type, live):
        self.name, self.rec_type, self.stats_type = name, rec_type, stats_type
        self.counts, self.records, self.stats_raw, self.i = [], [], b"", 0
        if not live:
            z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
            self.counts, self.stats_raw = [int(c) for c in z["counts"]], z["stats"].tobytes()
            self.records = [r.tobytes() for r in z["records"]]
            self.off = np.concatenate([[0], np.cumsum(self.counts)]).astype(int)

    @staticmethod
    def wanted(name):
        return bool(name) and bool(os.environ.get("LTEPHY_RECORD_GOLDEN"))

    def put(self, out):
        self.counts.append(len(out))
        self.records += [bytes(d) for d in out]
        return out

    def get(self):
        k = self.i
        assert k < len(self.counts), "%s: more subframes than were recorded" % self.name
        self.i += 1
        return [self.rec_type.from_buffer_copy(self.records[j]) for j in range(self.off[k], self.off[k + 1])]

    def stats(self, st=None):
        if st is not None:
            self.stats_raw = bytes(st)
            return st
        return self.stats_type.from_buffer_copy(self.stats_raw)

    def save(self):
        out = os.environ["LTEPHY_RECORD_GOLDEN"]
        os.makedirs(out, exist_ok=True)
        recs = np.frombuffer(b"".join(self.records), np.uint8).reshape(-1, C.sizeof(self.rec_type))
        np.savez_compressed(os.path.join(out, self.name + ".npz"), counts=np.array(self.counts, np.uint32), records=recs,
                            stats=np.frombuffer(self.stats_raw, np.uint8))


class OracleWalk:
    """The oracle's walk on the reference's RNTIManager (oracle/_ref/libfalcon_walk.so).  golden: name of a WalkRecord that stands in for it
    where oracle/_ref cannot be built."""
    rec = None

    def __init__(self, cell, threshold=5, golden=None):
        self.rec = None
        if golden and not ref_buildable():
            self.L, self.rec = None, WalkRecord(golden, WalkDci, WalkStats, live=False)
            return
        self.L = walklib()
        self.h = self.L.lteo_walk_create(C.byref(cell), threshold)
        if WalkRecord.wanted(golden):
            self.rec = WalkRecord(golden, WalkDci, WalkStats, live=True)

    def config(self, shortcut=1, skip_secondary=0, update_interval=500):
        if self.L is not None:
            self.L.lteo_walk_config(self.h, shortcut, skip_secondary, update_interval)

    def subframe(self, sf_idx, cfi, nof_cce, llr, snr_db):
        if self.L is None:
            return self.rec.get()
        out = (WalkDci * 64)()
        n = C.c_uint32(0)
        llr = np.ascontiguousarray(llr, np.float32)
        self.L.lteo_walk_subframe(self.h, sf_idx, cfi, nof_cce, ptr(llr), snr_db, out, 64, C.byref(n))
        res = [out[i] for i in range(n.value)]
        return self.rec.put(res) if self.rec else res

    def stats(self):
        if self.L is None:
            return self.rec.stats()
        s = WalkStats()
        self.L.lteo_walk_stats(self.h, C.byref(s))
        return self.rec.stats(s) if self.rec else s

    def save_record(self):
        if self.L is not None and self.rec:
            self.stats()
            self.rec.save()

    def __del__(self):
        try:
            if self.L is not None:
                self.L.lteo_walk_destroy(self.h)
        except Exception:
            pass


def oracle_pipeline(cell, iq, tti, walk=None, max_iter=8, want_tb=True):
    """The whole reference-shaped CPU path on a capture: phase A, FALCON walk (reference RNTIManager),
    DCI->grant (64QAM table), PDSCH decode.  Returns per-subframe list of (walk dcis, [(grant, payloads, crc)])."""
    O = oracle()
    O.lteo_phase_a.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(ChestRes), C.POINTER(C.c_uint32)]
    o = Oracle(cell)
    walk = walk or OracleWalk(cell)
    g = 14 * 12 * cell.nof_prb
    out = []
    for i in range(len(tti)):
        sym = np.zeros((cell.nof_rx, g), np.complex64)
        ce = np.zeros((cell.nof_ports * cell.nof_rx, g), np.complex64)
        llr = np.zeros(88 * 72, np.float32)
        res = ChestRes()
        cfi = C.c_uint32(0)
        sf_idx = int(tti[i]) % 10
        ncce = O.lteo_phase_a(o.h, ptr(np.ascontiguousarray(iq[i])), sf_idx, ptr(sym), ptr(ce), ptr(llr), C.byref(res), C.byref(cfi))
        dcis = walk.subframe(sf_idx, cfi.value, ncce, llr[:72 * ncce], res.snr_db)
        tbs = []
        if want_tb:
            for d in dcis:
                if d.format == 0 or d.rnti == 0:
                    tbs.append(None)
                    continue
                bits = np.frombuffer(bytes(d.bits), np.uint8)[:d.nof_bits]
                r, dd, gr = unpack_and_grant(cell, d.format, d.rnti, bits, sf_idx, cfi.value, 0)
                if r != 0 or not (gr.tb[0].tbs > 0 and not (cell.nof_rx == 1 and gr.nof_tb == 2)) or gr.tx_scheme == 3:
                    tbs.append(None)
                    continue
                r, pl, ok = o.pdsch_decode(sf_idx, cfi.value, d.rnti, gr, sym, ce, max_iter)
                tbs.append((gr, pl, ok))
        out.append((dcis, tbs, res.snr_db, cfi.value))
    return out


# ------------------------------------------------------------------------------------------------ uplink
class UlCfg(C.Structure):
    _fields_ = [("n_dmrs1", C.c_uint32), ("delta_ss", C.c_uint32), ("group_hopping", C.c_uint32), ("seq_hopping", C.c_uint32), ("n_rb_ho", C.c_uint32)]


class UlGrant(C.Structure):
    _fields_ = [("rnti", C.c_uint16), ("L_prb", C.c_uint32), ("n_prb", C.c_uint32), ("mcs", C.c_uint32), ("qm", C.c_uint32), ("rv", C.c_uint32),
                ("tbs", C.c_int32), ("n_dmrs2", C.c_uint32), ("nof_re", C.c_uint32), ("nof_bits", C.c_uint32),
                ("hop", C.c_uint32), ("n_prb_slot1", C.c_uint32), ("nof_ack", C.c_uint32), ("ri_len", C.c_uint32), ("cqi_len", C.c_uint32),
                ("I_offset_ack", C.c_uint32), ("I_offset_ri", C.c_uint32), ("I_offset_cqi", C.c_uint32), ("ta_us", C.c_float)]


class UciLayout(C.Structure):
    _fields_ = [("Qp_ack", C.c_uint32), ("Qp_ri", C.c_uint32), ("Qp_cqi", C.c_uint32), ("G", C.c_uint32)]


def uci_layout(g):
    """Q' of ACK / RI / CQI and the UL-SCH bit count G of a grant (36.212 5.2.2.6)"""
    S = sim()
    S.lte_uci_layout.argtypes = [C.POINTER(UlGrant), C.POINTER(UciLayout)]
    L = UciLayout()
    S.lte_uci_layout(C.byref(g), C.byref(L))
    return L


class UlChest(C.Structure):
    _fields_ = [("noise", C.c_float), ("rsrp", C.c_float), ("snr_db", C.c_float), ("ta_us", C.c_float)]


def make_ul_grants(cell, rng, n, table=1, min_prb=3):
    """n random non-overlapping valid UL grants (DCI format 0 fields -> lte_ul_dci_to_grant)"""
    S = sim()
    S.lte_ul_valid_prb.argtypes = [C.c_uint32]
    out, start = [], 0
    N = cell.nof_prb
    for i in range(n):
        cand = [L for L in range(min_prb, max(min_prb + 1, (N - start) // max(1, (n - i)) + 1)) if S.lte_ul_valid_prb(L)]
        if not cand or start + cand[0] > N:
            break
        L = int(rng.choice(cand))
        d = Dci()
        d.format, d.rnti, d.alloc_type = 0, int(rng.integers(0x100, 0xFFF0)), 2
        d.riv = N * (L - 1) + start if (L - 1) <= N // 2 else N * (N - L + 1) + (N - 1 - start)
        d.mcs[0] = int(rng.integers(2, 27))
        d.n_dmrs = int(rng.integers(0, 8))
        g = UlGrant()
        r = S.lte_ul_dci_to_grant(C.byref(cell), C.byref(d), table, C.byref(g))
        assert r == 0, r
        out.append(g)
        start += L
    return out


def sim_ul_subframe(simobj, tti, ucfg, grants):
    S = sim()
    S.lte_sim_ul_subframe.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(UlCfg), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    iq = np.zeros(simobj.sf_len, np.complex64)
    pl = np.zeros(1 << 16, np.uint8)
    off = np.zeros(max(1, len(grants)), np.uint32)
    arr = (UlGrant * max(1, len(grants)))(*grants)
    r = S.lte_sim_ul_subframe(simobj.h, tti, C.byref(ucfg), arr, len(grants), ptr(iq), ptr(pl), ptr(off), len(pl))
    assert r == 0, r
    return iq, pl, off


def oracle_ul(o, ucfg, tti, grants, iq, max_iter=8, want_llr=False):
    O = oracle()
    O.lteo_ul_ofdm.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    O.lteo_pusch_decode.argtypes = [C.c_void_p, C.POINTER(UlCfg), C.c_uint32, C.POINTER(UlGrant), C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_int),
                                    C.POINTER(UlChest), C.c_void_p]
    sym = np.zeros(14 * o.nsc, np.complex64)
    O.lteo_ul_ofdm(o.h, ptr(np.ascontiguousarray(iq)), ptr(sym))
    res = []
    for g in grants:
        pl = np.zeros(16000, np.uint8)
        ok = C.c_int(0)
        ch = UlChest()
        llr = np.zeros(uci_layout(g).G + 16, np.int16) if want_llr else None
        r = O.lteo_pusch_decode(o.h, C.byref(ucfg), tti % 10, C.byref(g), ptr(sym), max_iter, ptr(pl), C.byref(ok), C.byref(ch), ptr(llr) if want_llr else None)
        res.append((r, pl, ok.value, ch, llr))
    return sym, res
