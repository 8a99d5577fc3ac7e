"""ctypes binding of include/ltephy_b200.h (the tier-1 C-ABI).  Host arrays in, host arrays out;
all compute happens in the CUDA library.  Fails loudly if the library is missing or unusable."""
import ctypes as C
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libltephy_b200.so")

MAX_PRB, MAX_CCE, MAX_LOC, MAX_SIZES, NOF_FORMATS = 110, 88, 160, 8, 9
LLR_STRIDE = 72 * MAX_CCE
TX_PORT0, TX_DIVERSITY, TX_CDD, TX_SPATIALMUX = 0, 1, 2, 3
TAP_SYM, TAP_CE, TAP_LLR, TAP_PDSCH_LLR, TAP_TURBO_IN = 0, 1, 2, 3, 4
FLAG_SKIP_LOW_POWER = 1
# sample formats of every input (LTEPHY_IQ_*): complex64, or int16 / int8 interleaved I/Q (value * 2^-15 / value * 2^-7)
IQ_FORMATS = {"cf32": 0, "sc16": 1, "sc8": 2}
_IQ_DTYPES = {"cf32": np.complex64, "sc16": np.int16, "sc8": np.int8}


class Cfg(C.Structure):
    _fields_ = [("nof_prb", C.c_uint32), ("nof_ports", C.c_uint32), ("cell_id", C.c_uint32), ("nof_rx", C.c_uint32),
                ("max_subframes", C.c_uint32), ("max_grants", C.c_uint32), ("turbo_max_iter", C.c_uint32), ("device", C.c_int32),
                ("flags", C.c_uint32), ("symbol_sz", C.c_uint32), ("phich_resources", C.c_uint32), ("phich_length", C.c_uint32),
                ("ul_nof_rx", C.c_uint32), ("iq_format", C.c_uint32), ("reserved", C.c_uint32 * 2)]


class SfInfo(C.Structure):
    _fields_ = [("tti", C.c_uint32), ("cfi", C.c_uint32), ("nof_cce", C.c_uint32), ("nof_locations", C.c_uint32),
                ("pcfich_corr", C.c_float * 3), ("noise", (C.c_float * 2) * 2), ("rsrp", (C.c_float * 2) * 2),
                ("noise_avg", C.c_float), ("rsrp_avg", C.c_float), ("cfo_re", C.c_float), ("cfo_im", C.c_float),
                ("snr_db", C.c_float), ("cfo", C.c_float), ("rb_power", C.c_float * MAX_PRB), ("cce_power", C.c_float * MAX_CCE)]


class Cand(C.Structure):
    _fields_ = [("bits", C.c_uint64), ("rnti", C.c_uint16), ("valid", C.c_uint8), ("pad", C.c_uint8 * 5)]


class GrantTb(C.Structure):
    _fields_ = [("tbs", C.c_int32), ("qm", C.c_uint8), ("rv", C.c_uint8), ("enabled", C.c_uint8), ("cw_idx", C.c_uint8),
                ("harq_op", C.c_uint8), ("pad", C.c_uint8 * 3), ("harq_slot", C.c_uint32)]


class Grant(C.Structure):
    _fields_ = [("sf", C.c_uint32), ("rnti", C.c_uint16), ("tx_scheme", C.c_uint8), ("nof_tb", C.c_uint8),
                ("prb_mask", (C.c_uint32 * 4) * 2), ("nof_re", C.c_uint32), ("pmi", C.c_uint32), ("tb", GrantTb * 2)]


class TbResult(C.Structure):
    _fields_ = [("crc", C.c_uint8), ("avg_iters", C.c_uint8), ("nof_cb", C.c_uint16), ("payload_off", C.c_uint32), ("payload_len", C.c_uint32)]


class UlCfg(C.Structure):
    _fields_ = [("n_dmrs1", C.c_uint32), ("delta_ss", C.c_uint32), ("group_hopping", C.c_uint32), ("seq_hopping", C.c_uint32)]


class UlGrant(C.Structure):
    _fields_ = [("sf", C.c_uint32), ("rnti", C.c_uint16), ("qm", C.c_uint8), ("rv", C.c_uint8), ("L_prb", C.c_uint32), ("n_prb", C.c_uint32),
                ("n_dmrs2", C.c_uint32), ("tbs", C.c_int32), ("n_prb_slot1", C.c_uint32), ("nof_ack", C.c_uint8), ("ri_len", C.c_uint8),
                ("cqi_len", C.c_uint16), ("I_offset_ack", C.c_uint8), ("I_offset_cqi", C.c_uint8), ("I_offset_ri", C.c_uint8), ("flags", C.c_uint8)]


class UlUeCfg(C.Structure):
    _fields_ = [("rnti", C.c_uint16), ("mcs_mod", C.c_uint8), ("I_offset_ack", C.c_uint8), ("I_offset_cqi", C.c_uint8), ("I_offset_ri", C.c_uint8),
                ("cqi_len", C.c_uint16)]


class Rar(C.Structure):
    _fields_ = [("t_crnti", C.c_uint16), ("ta", C.c_uint16), ("rapid", C.c_uint8), ("hopping_flag", C.c_uint8), ("tpc", C.c_uint8), ("ul_delay", C.c_uint8),
                ("cqi_request", C.c_uint8), ("valid", C.c_uint8), ("grant", UlGrant)]


class Mib(C.Structure):
    _fields_ = [("found", C.c_uint8), ("nof_ports", C.c_uint8), ("sfn_offset", C.c_uint8), ("phich_length", C.c_uint8), ("phich_resources", C.c_uint8),
                ("bch_payload", C.c_uint8 * 3), ("nof_prb", C.c_uint32), ("sfn", C.c_uint32)]


class MibComb(C.Structure):
    """ltephy_mib_comb_t: one result of ltephy_mib_decode_combined"""
    _fields_ = [("mib", Mib), ("nof_frames", C.c_uint8), ("src", C.c_uint8), ("dst", C.c_uint8), ("window", C.c_uint8)]


MIB_SEARCH_PORTS = 1


class UlChest(C.Structure):
    _fields_ = [("noise", C.c_float), ("rsrp", C.c_float), ("snr_db", C.c_float), ("ta_us", C.c_float)]


TAP_UL_SYM = 5
TAP_PBCH_LLR = 6                                      # f32 [frames][2][480]: PBCH soft bits of the last MIB decode, row [port count - 1]
HARQ_NONE, HARQ_NEW, HARQ_RETX = 0, 1, 2            # grant.tb[t].harq_op
HARQ_NEW_TX, HARQ_RE_TX, HARQ_FULL_BUFFER, HARQ_DECODED = 0, 1, 2, 3   # ltephy_harq_classify
HARQ_SLOT_BYTES = 16 * 18448 * 2
UL_FLAG_SLOT1 = 1
CAND_DTYPE = np.dtype([("bits", "<u8"), ("rnti", "<u2"), ("valid", "u1"), ("pad", "u1", 5)])
assert CAND_DTYPE.itemsize == C.sizeof(Cand) == 16
COMPACT_CAP = 248
NEED_FULL_TABLE = -3
COMPACT_DTYPE = np.dtype([("count", "<u4"), ("reserved", "<u4"), ("loc", [("off", "<u2"), ("mask", "u1"), ("pad", "u1")], MAX_LOC), ("pad", "u1", 8),
                          ("list", CAND_DTYPE, COMPACT_CAP)])   # ltephy_compact_t
assert COMPACT_DTYPE.itemsize == 4624

_lib = None


def load_library(build_if_missing=True):
    """Loads libltephy_b200.so; there is no fallback implementation."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing:
        from . import build as _b
        _b.build()
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libltephy_b200.so is missing: build it with __graft_entry__.build(); there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    P = C.c_void_p
    L.ltephy_create.argtypes = [C.POINTER(Cfg), C.POINTER(P)]
    L.ltephy_destroy.argtypes = [P]
    L.ltephy_last_error.restype = C.c_char_p
    for f in ("ltephy_sf_len", "ltephy_nof_sizes"):
        getattr(L, f).argtypes = [P]
        getattr(L, f).restype = C.c_uint32
    for f in ("ltephy_nof_cce", "ltephy_dci_size", "ltephy_size_index"):
        getattr(L, f).argtypes = [P, C.c_uint32]
        getattr(L, f).restype = C.c_uint32
    L.ltephy_locations.argtypes = [P, C.c_uint32, P, P, C.c_uint32]
    L.ltephy_locations.restype = C.c_uint32
    L.ltephy_submit_iq.argtypes = [P, P, P, C.c_uint32]
    L.ltephy_submit_iq_device.argtypes = [P, P, P, C.c_uint32]
    L.ltephy_get_phase_a.argtypes = [P, P, P]
    L.ltephy_get_phase_a_compact.argtypes = [P, P, P]
    L.ltephy_phase_a_compact_buffer.argtypes = [P]
    L.ltephy_phase_a_compact_buffer.restype = P
    L.ltephy_copy_phase_a_device.argtypes = [P, P, P]
    L.ltephy_finalize_info.argtypes = [P, C.c_uint32, C.c_uint32, C.c_uint32]
    L.ltephy_finalize_info.restype = None
    L.ltephy_submit_grants.argtypes = [P, P, C.c_uint32]
    L.ltephy_get_phase_b.argtypes = [P, P, P, C.c_size_t]
    L.ltephy_copy_phase_b_device.argtypes = [P, P, C.c_size_t, P]
    L.ltephy_dci_sweep.argtypes = [P, P, P, C.c_uint32, P]
    L.ltephy_turbo_batch.argtypes = [P, P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, P, P, P]
    L.ltephy_tap.argtypes = [P, C.c_int, P, C.c_size_t]
    L.ltephy_last_timing.argtypes = [P, P]
    L.ltephy_set_ul_cfg.argtypes = [P, C.POINTER(UlCfg)]
    L.ltephy_submit_ul.argtypes = [P, P, P, C.c_uint32, P, C.c_uint32]
    L.ltephy_get_ul.argtypes = [P, P, P, P, C.c_size_t]
    L.ltephy_mark.argtypes = [P, C.c_int]
    L.ltephy_mark_elapsed_ms.argtypes = [P]
    L.ltephy_mark_elapsed_ms.restype = C.c_float
    L.ltephy_last_turbo_work.argtypes = [P, P, P, P]
    L.ltephy_launch_count.argtypes = [P]
    L.ltephy_launch_count.restype = C.c_uint64
    _lib = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _host_iq(iq, fmt):
    """-> (iq as a contiguous host array of the format's type, its shape in complex samples).  cf32: complex64; sc16 / sc8: int16 / int8 with a
    last axis of 2 (I, Q)"""
    iq = np.ascontiguousarray(iq, _IQ_DTYPES[fmt])
    if fmt == "cf32":
        return iq, iq.shape
    assert iq.ndim >= 1 and iq.shape[-1] == 2, iq.shape
    return iq, iq.shape[:-1]


def _dev_shape(t, fmt):
    """shape in complex samples of a contiguous device tensor of the format: complex64, or int16 / int8 with a last axis of 2"""
    assert t.is_cuda and t.is_contiguous(), "a contiguous CUDA tensor"
    if fmt == "cf32":
        return tuple(t.shape)
    import torch
    want = {"sc16": torch.int16, "sc8": torch.int8}[fmt]
    assert t.dtype == want and t.shape[-1] == 2, (t.dtype, tuple(t.shape), fmt)
    return tuple(t.shape[:-1])


class LtePhy:
    """One PHY context (cell + batch capacity) on one GPU."""

    def __init__(self, nof_prb, nof_ports, cell_id, nof_rx, max_subframes=16, turbo_max_iter=8, device=0, flags=0, symbol_sz=0, phich_resources=0, phich_length=0,
                 ul_nof_rx=1, iq_format="cf32"):
        """ul_nof_rx: receive antennas of the uplink carrier (1 or 2): decode_ul / decode_ul_device then take [n][ul_nof_rx][sf_len].
        iq_format "cf32" takes complex64 samples, "sc16" / "sc8" int16 / int8 ones with a last axis of 2 (I, Q), DL and UL alike."""
        self.L = load_library()
        self.iq_format = iq_format
        cfg = Cfg(nof_prb=nof_prb, nof_ports=nof_ports, cell_id=cell_id, nof_rx=nof_rx, max_subframes=max_subframes,
                  turbo_max_iter=turbo_max_iter, device=device, flags=flags, symbol_sz=symbol_sz, phich_resources=phich_resources, phich_length=phich_length,
                  ul_nof_rx=ul_nof_rx, iq_format=IQ_FORMATS[iq_format])
        self.cfg = cfg
        self.h = C.c_void_p()
        r = self.L.ltephy_create(C.byref(cfg), C.byref(self.h))
        if r != 0:
            raise RuntimeError("ltephy_create failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))
        self.sf_len = self.L.ltephy_sf_len(self.h)
        self.nsc = 12 * nof_prb
        self.ul_nof_rx = max(1, ul_nof_rx)
        self.n = 0

    def close(self):
        if self.h:
            self.L.ltephy_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, r, what):
        if r != 0:
            raise RuntimeError("%s failed (%d): %s" % (what, r, self.L.ltephy_last_error().decode()))

    # ---- geometry
    def nof_cce(self, cfi):
        return self.L.ltephy_nof_cce(self.h, cfi)

    def sizes(self):
        return [self.L.ltephy_dci_size(self.h, f) for f in range(NOF_FORMATS)], [self.L.ltephy_size_index(self.h, f) for f in range(NOF_FORMATS)]

    def locations(self, cfi):
        nc = np.zeros(MAX_LOC, np.uint16)
        L = np.zeros(MAX_LOC, np.uint8)
        n = self.L.ltephy_locations(self.h, cfi, _p(nc), _p(L), MAX_LOC)
        return nc[:n].copy(), L[:n].copy()

    # ---- phase A
    def submit_iq(self, iq, tti):
        """iq: complex64 [n][nof_rx][sf_len] (int16 / int8 [n][nof_rx][sf_len][2] for sc16 / sc8)"""
        iq, shape = _host_iq(iq, self.iq_format)
        tti = np.ascontiguousarray(tti, np.uint32)
        n = len(tti)
        assert shape == (n, self.cfg.nof_rx, self.sf_len), iq.shape
        self._keep = (iq, tti)
        self._chk(self.L.ltephy_submit_iq(self.h, _p(iq), _p(tti), n), "submit_iq")
        self.n = n

    def submit_iq_device(self, iq_dev, tti):
        """ltephy_submit_iq_device: iq_dev a torch tensor [n][nof_rx][sf_len] (of the handle's format, as submit_iq), contiguous, on this handle's
        device, read in place until phase A is fetched"""
        tti = np.ascontiguousarray(tti, np.uint32)
        n = len(tti)
        assert _dev_shape(iq_dev, self.iq_format) == (n, self.cfg.nof_rx, self.sf_len), tuple(iq_dev.shape)
        self._keep = (iq_dev, tti)
        self._chk(self.L.ltephy_submit_iq_device(self.h, C.c_void_p(iq_dev.data_ptr()), _p(tti), n), "submit_iq_device")
        self.n = n

    def get_phase_a(self, want_cands=True):
        info = (SfInfo * self.n)()
        cands = np.zeros((self.n, MAX_LOC, MAX_SIZES), CAND_DTYPE) if want_cands else None
        self._chk(self.L.ltephy_get_phase_a(self.h, info, _p(cands) if want_cands else None), "get_phase_a")
        return info, cands

    def get_phase_a_compact(self):
        """-> (info, survivor forms as a COMPACT_DTYPE array [n])"""
        info = (SfInfo * self.n)()
        comp = np.zeros(self.n, COMPACT_DTYPE)
        self._chk(self.L.ltephy_get_phase_a_compact(self.h, info, _p(comp)), "get_phase_a_compact")
        return info, comp

    def set_cfo(self, cfo_hz):
        self.L.ltephy_set_cfo.argtypes = [C.c_void_p, C.c_float]
        self._chk(self.L.ltephy_set_cfo(self.h, cfo_hz), "set_cfo")

    def mib_decode(self):
        out = (Mib * self.n)()
        self.L.ltephy_mib_decode.argtypes = [C.c_void_p, C.c_void_p]
        self._chk(self.L.ltephy_mib_decode(self.h, out), "mib_decode")
        return out

    def mib_decode_combined(self, search_ports=False):
        """ltephy_mib_decode_combined over the subframes of the last submit: [MibComb] * n; the combining state persists across calls"""
        out = (MibComb * self.n)()
        self.L.ltephy_mib_decode_combined.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        self._chk(self.L.ltephy_mib_decode_combined(self.h, MIB_SEARCH_PORTS if search_ports else 0, out), "mib_decode_combined")
        return out

    def mib_reset(self):
        """ltephy_mib_reset: empty the combining buffer"""
        self.L.ltephy_mib_reset.argtypes = [C.c_void_p]
        self._chk(self.L.ltephy_mib_reset(self.h), "mib_reset")

    def harq_reserve(self, nslots):
        self.L.ltephy_harq_reserve.argtypes = [C.c_void_p, C.c_uint32]
        self._chk(self.L.ltephy_harq_reserve(self.h, nslots), "harq_reserve")

    def tap(self, what, shape, dtype):
        out = np.zeros(shape, dtype)
        self._chk(self.L.ltephy_tap(self.h, what, _p(out), out.nbytes), "tap")
        return out

    # ---- phase B
    def submit_grants(self, grants):
        arr = (Grant * max(1, len(grants)))(*grants)
        self._grants = arr
        self._ng = len(grants)
        self._chk(self.L.ltephy_submit_grants(self.h, arr, len(grants)), "submit_grants")

    def get_phase_b(self, payload_cap=None):
        res = (TbResult * max(1, 2 * self._ng))()
        cap = payload_cap or (self._ng * 2 * 13000 + 64)
        pl = np.zeros(cap, np.uint8)
        self._chk(self.L.ltephy_get_phase_b(self.h, res, _p(pl), cap), "get_phase_b")
        return res, pl

    # ---- uplink
    def set_ul_cfg(self, n_dmrs1=0, delta_ss=0, group_hopping=0, seq_hopping=0):
        cfg = UlCfg(n_dmrs1=n_dmrs1, delta_ss=delta_ss, group_hopping=group_hopping, seq_hopping=seq_hopping)
        self._chk(self.L.ltephy_set_ul_cfg(self.h, C.byref(cfg)), "set_ul_cfg")

    def decode_ul(self, iq_ul, tti, grants):
        """iq_ul complex64 [n][sf_len] with one UL antenna, [n][ul_nof_rx][sf_len] with two (int16 / int8 with a last axis of 2 for sc16 / sc8;
        None: decode the subframes of the previous call again); grants: list of UlGrant -> (results, chest, payload)"""
        shape = None
        if iq_ul is not None:
            iq_ul, shape = _host_iq(iq_ul, self.iq_format)
        tti = np.ascontiguousarray(tti, np.uint32)
        assert iq_ul is None or int(np.prod(shape)) == len(tti) * self.ul_nof_rx * self.sf_len, (iq_ul.shape, self.ul_nof_rx)
        arr = (UlGrant * max(1, len(grants)))(*grants)
        self._chk(self.L.ltephy_submit_ul(self.h, None if iq_ul is None else _p(iq_ul), _p(tti), len(tti), arr, len(grants)), "submit_ul")
        res = (TbResult * max(1, len(grants)))()
        ch = (UlChest * max(1, len(grants)))()
        pl = np.zeros(len(grants) * 10000 + 64, np.uint8)
        self._chk(self.L.ltephy_get_ul(self.h, res, ch, _p(pl), pl.nbytes), "get_ul")
        self.n_ul = len(tti)
        return res, ch, pl

    def decode_ul_device(self, iq_dev, tti, grants):
        """ltephy_submit_ul_device: iq_dev a torch complex64 tensor [n][sf_len] ([n][ul_nof_rx][sf_len] with two UL antennas; int16 / int8 with a
        last axis of 2 for sc16 / sc8), contiguous, on this handle's device (None: decode the subframes of the previous call again), read in place ->
        (results, chest, payload) as decode_ul"""
        self.L.ltephy_submit_ul_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
        tti = np.ascontiguousarray(tti, np.uint32)
        if iq_dev is not None:
            want = (len(tti), self.sf_len) if self.ul_nof_rx == 1 else (len(tti), self.ul_nof_rx, self.sf_len)
            assert _dev_shape(iq_dev, self.iq_format) == want, tuple(iq_dev.shape)
        arr = (UlGrant * max(1, len(grants)))(*grants)
        ptr = None if iq_dev is None else C.c_void_p(iq_dev.data_ptr())
        self._chk(self.L.ltephy_submit_ul_device(self.h, ptr, _p(tti), len(tti), arr, len(grants)), "submit_ul_device")
        res = (TbResult * max(1, len(grants)))()
        ch = (UlChest * max(1, len(grants)))()
        pl = np.zeros(len(grants) * 10000 + 64, np.uint8)
        self._chk(self.L.ltephy_get_ul(self.h, res, ch, _p(pl), pl.nbytes), "get_ul")
        self.n_ul = len(tti)
        return res, ch, pl

    def set_ul_cfo(self, cfo_hz):
        """ltephy_set_ul_cfo: constant carrier-offset correction of the uplink subframes (0 switches it off)"""
        self.L.ltephy_set_ul_cfo.argtypes = [C.c_void_p, C.c_float]
        self._chk(self.L.ltephy_set_ul_cfo(self.h, cfo_hz), "set_ul_cfo")

    # ---- stand-alone kernels
    def dci_sweep(self, llr, cfi):
        llr = np.ascontiguousarray(llr, np.float32)
        cfi = np.ascontiguousarray(cfi, np.uint32)
        n = len(cfi)
        assert llr.shape == (n, LLR_STRIDE)
        cands = np.zeros((n, MAX_LOC, MAX_SIZES), CAND_DTYPE)
        self._chk(self.L.ltephy_dci_sweep(self.h, _p(llr), _p(cfi), n, _p(cands)), "dci_sweep")
        return cands

    def turbo_batch(self, d, K, max_iter, crc_type):
        d = np.ascontiguousarray(d, np.int16)
        ncb = d.shape[0]
        assert d.shape == (ncb, 3 * (K + 4))
        bits = np.zeros((ncb, K), np.uint8)
        iters = np.zeros(ncb, np.uint8)
        ok = np.zeros(ncb, np.uint8)
        self._chk(self.L.ltephy_turbo_batch(self.h, _p(d), K, ncb, max_iter, crc_type, _p(bits), _p(iters), _p(ok)), "turbo_batch")
        return bits, iters, ok

    def timing(self):
        t = (C.c_float * 4)()
        self.L.ltephy_last_timing(self.h, t)
        return list(t)

    def mark(self, slot):
        self._chk(self.L.ltephy_mark(self.h, slot), "mark")

    def mark_elapsed_ms(self):
        return float(self.L.ltephy_mark_elapsed_ms(self.h))

    def turbo_work(self):
        b, c, i = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self.L.ltephy_last_turbo_work(self.h, C.byref(b), C.byref(c), C.byref(i))
        return b.value, c.value, i.value

    def launch_count(self):
        return int(self.L.ltephy_launch_count(self.h))


def cand_bits(c, nbits):
    """uint64 payload -> array of nbits bits (bit i at position 63-i)."""
    v = int(c)
    return np.array([(v >> (63 - i)) & 1 for i in range(nbits)], np.uint8)


# ------------------------------------------------------------------------------------------------
# host search / grant conversion / one-call pipeline (include/ltephy_search.h)
class DciOut(C.Structure):
    _fields_ = [("sf", C.c_uint32), ("rnti", C.c_uint16), ("format", C.c_uint8), ("L", C.c_uint8), ("ncce", C.c_uint16),
                ("nof_bits", C.c_uint16), ("bits", C.c_uint64), ("histogram_value", C.c_uint32)]


class SearchStats(C.Structure):
    _fields_ = [("nof_decoded_locations", C.c_uint32), ("nof_cce", C.c_uint32), ("nof_missed_cce", C.c_uint32), ("nof_subframes", C.c_uint32),
                ("nof_subframe_collisions_dw", C.c_uint32), ("nof_subframe_collisions_up", C.c_uint32), ("nof_locations", C.c_uint32)]


class DciFields(C.Structure):
    _fields_ = [("rnti", C.c_uint16), ("format", C.c_uint8), ("alloc_type", C.c_uint8), ("mcs", C.c_uint8 * 2), ("rv", C.c_uint8 * 2),
                ("ndi", C.c_uint8 * 2), ("harq_pid", C.c_uint8), ("tpc", C.c_uint8), ("tb_cw_swap", C.c_uint8), ("pinfo", C.c_uint8),
                ("nof_prb", C.c_uint32)]


DCI_DTYPE = np.dtype({"names": ["sf", "rnti", "format", "L", "ncce", "nof_bits", "bits", "histogram_value"],
                      "formats": ["<u4", "<u2", "u1", "u1", "<u2", "<u2", "<u8", "<u4"],
                      "offsets": [DciOut.sf.offset, DciOut.rnti.offset, DciOut.format.offset, DciOut.L.offset, DciOut.ncce.offset,
                                  DciOut.nof_bits.offset, DciOut.bits.offset, DciOut.histogram_value.offset],
                      "itemsize": C.sizeof(DciOut)})
assert DCI_DTYPE.itemsize == C.sizeof(DciOut)
SEQ_NONE = (1 << 64) - 1


def _bind_search(L):
    if getattr(L, "_search_bound", False):
        return
    P = C.c_void_p
    L.ltephy_search_create.argtypes = [P, C.c_uint32]
    L.ltephy_search_create.restype = P
    L.ltephy_search_create_cell.argtypes = [C.c_uint32] * 5
    L.ltephy_search_create_cell.restype = P
    L.ltephy_search_create_cell_ng.argtypes = [C.c_uint32] * 6
    L.ltephy_search_create_cell_ng.restype = P
    L.ltephy_ctrl_region_map.argtypes = [C.c_uint32] * 5 + [P, C.c_uint32, P, P]
    L.ltephy_search_destroy.argtypes = [P]
    L.ltephy_search_config.argtypes = [P, C.c_int, C.c_int, C.c_uint32]
    L.ltephy_search_speculate_256qam.argtypes = [P, C.c_int]
    L.ltephy_search_keep_reserved_mcs.argtypes = [P, C.c_int]
    L.ltephy_search_set_ul_mode.argtypes = [P, C.c_int, C.c_uint16]
    L.ltephy_search_set_ul_hopping.argtypes = [P, C.c_uint32]
    L.ltephy_shard_set_gather_capacity.argtypes = [P, C.c_uint32]
    L.ltephy_search_add_evergreen.argtypes = [P, C.c_uint16, C.c_uint16, C.c_uint32]
    L.ltephy_search_add_forbidden.argtypes = [P, C.c_uint16, C.c_uint16, C.c_uint32]
    L.ltephy_search_activate.argtypes = [P, C.c_uint16, C.c_uint32, C.c_int]
    L.ltephy_search_subframe.argtypes = [P, P, P, C.c_uint32, P, C.c_uint32, P]
    L.ltephy_search_subframe_compact.argtypes = [P, P, P, C.c_uint32, P, C.c_uint32, P]
    L.ltephy_compact_from_table.argtypes = [P, P, P, P]
    L.ltephy_search_batch_compact.argtypes = [P, P, P, P, C.c_uint32, P, C.c_uint32, P]
    L.ltephy_search_needs_full_table.argtypes = [P, P, C.c_uint32]
    L.ltephy_search_get_stats.argtypes = [P, P]
    L.ltephy_search_validate_location.argtypes = [C.c_uint32] * 4 + [C.c_uint16]
    L.ltephy_search_validate_location.restype = C.c_uint32
    L.ltephy_search_rnti_validate_and_refresh.argtypes = [P, C.c_uint16, C.c_uint32]
    L.ltephy_search_rnti_add_candidate.argtypes = [P, C.c_uint16, C.c_uint32]
    L.ltephy_search_rnti_step_time.argtypes = [P]
    for f in ("ltephy_search_rnti_frequency", "ltephy_search_rnti_is_forbidden", "ltephy_search_rnti_is_evergreen"):
        getattr(L, f).argtypes = [P, C.c_uint16, C.c_uint32]
        getattr(L, f).restype = C.c_uint32
    L.ltephy_search_rnti_assoc_format.argtypes = [P, C.c_uint16]
    L.ltephy_search_rnti_assoc_format.restype = C.c_uint32
    L.ltephy_search_rnti_reason.argtypes = [P, C.c_uint16]
    L.ltephy_dci_to_grant.argtypes = [P, P, C.c_uint32, C.c_uint32, C.c_int, P, P]
    L.ltephy_ul_dci_to_grant.argtypes = [P, P, C.c_int, P]
    L.ltephy_ul_decode_plan.argtypes = [P, P, C.c_int, P, P]
    L.ltephy_rar_unpack.argtypes = [P, P, C.c_uint32, P, C.c_uint32, P, P]
    L.ltephy_ul_cqi_len.argtypes = [C.c_uint32, C.c_int]
    L.ltephy_ul_uci_layout.argtypes = [P, P, P, P, P]
    L.ltephy_ul_grants_from_dcis.argtypes = [P, P, P, C.c_uint32, P, C.c_uint32, P, P, P, C.c_uint32, P]
    L.ltephy_decode_subframes.argtypes = [P, P, P, P, C.c_uint32, C.c_uint64, P, P, P, C.c_uint32, P, P, P, C.c_size_t]
    L.ltephy_decode_subframes_device.argtypes = [P, P, P, P, C.c_uint32, C.c_uint64, P, P, P, C.c_uint32, P, P, P, C.c_size_t]
    L.ltephy_search_batch.argtypes = [P, P, P, C.c_uint32, P, C.c_uint32, P]
    L.ltephy_grants_from_dcis.argtypes = [P, P, P, C.c_uint32, C.c_uint32, C.c_uint32, P, P, C.c_uint32, P]
    # sharded operation (include/ltephy_shard.h)
    L.ltephy_packed_size.argtypes = [C.c_uint32, C.c_uint32]
    L.ltephy_packed_size.restype = C.c_size_t
    L.ltephy_pack_subframes.argtypes = [P, P, P, C.c_uint32, P, C.c_size_t, P]
    L.ltephy_search_batch_packed.argtypes = [P, P, P, P, C.c_uint32, C.c_uint32, P, C.c_uint32, P, P]
    L.ltephy_packed_needs_full_table.argtypes = [P, P, P, C.c_uint32, C.c_uint32]
    L.ltephy_grants_from_dcis_tc.argtypes = [P, P, P, C.c_uint32, C.c_uint32, C.c_uint32, P, P, C.c_uint32, P]
    L.ltephy_shard_unique_id.argtypes = [P]
    L.ltephy_shard_create.argtypes = [P, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(P)]
    L.ltephy_shard_destroy.argtypes = [P]
    L.ltephy_decode_subframes_sharded.argtypes = [P, P, P, P, C.c_int, P, C.c_uint32, C.c_uint64, P, P, C.c_uint32, P, P, P, C.c_size_t, P]
    L.ltephy_pack_phase_a.argtypes = [P, P, C.c_size_t, P]
    L._search_bound = True


class Search:
    """FALCON acceptance walk + RNTI history (host only; usable without a GPU)."""

    def __init__(self, nof_prb, nof_ports, cell_id, nof_rx, threshold=5, phich_resources=0):
        self.L = load_library()
        _bind_search(self.L)
        self.h = self.L.ltephy_search_create_cell_ng(nof_prb, nof_ports, cell_id, nof_rx, phich_resources, threshold)
        if not self.h:
            raise RuntimeError("ltephy_search_create_cell failed")

    def close(self):
        if self.h:
            self.L.ltephy_search_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def config(self, shortcut=1, skip_secondary=0, update_interval=500):
        self.L.ltephy_search_config(self.h, shortcut, skip_secondary, update_interval)

    def subframe(self, info, cands, sf_in_batch=0, max_out=64):
        """info: SfInfo, cands: CAND_DTYPE array [MAX_LOC][MAX_SIZES] -> accepted DCIs (structured array)"""
        out = np.zeros(max_out, DCI_DTYPE)
        n = C.c_uint32(0)
        cands = np.ascontiguousarray(cands)
        r = self.L.ltephy_search_subframe(self.h, C.byref(info), _p(cands), sf_in_batch, _p(out), max_out, C.byref(n))
        if r < 0:
            raise RuntimeError("ltephy_search_subframe failed (%d)" % r)
        return out[:n.value].copy()

    def compact_from_table(self, info, cands):
        """host restatement of the GPU's survivor selection for one subframe -> COMPACT_DTYPE scalar array [1]"""
        out = np.zeros(1, COMPACT_DTYPE)
        cands = np.ascontiguousarray(cands)
        r = self.L.ltephy_compact_from_table(self.h, C.byref(info), _p(cands), _p(out))
        if r < 0:
            raise RuntimeError("ltephy_compact_from_table failed (%d)" % r)
        return out

    def subframe_compact(self, info, comp, sf_in_batch=0, max_out=64):
        """walk over the survivor form; returns None when the full table is needed (nothing consumed)"""
        out = np.zeros(max_out, DCI_DTYPE)
        n = C.c_uint32(0)
        comp = np.ascontiguousarray(comp)
        r = self.L.ltephy_search_subframe_compact(self.h, C.byref(info), _p(comp), sf_in_batch, _p(out), max_out, C.byref(n))
        if r == NEED_FULL_TABLE:
            return None
        if r < 0:
            raise RuntimeError("ltephy_search_subframe_compact failed (%d)" % r)
        return out[:n.value].copy()

    def stats(self):
        st = SearchStats()
        self.L.ltephy_search_get_stats(self.h, C.byref(st))
        return st

    def dci_to_grant(self, dci_row, sf_idx, cfi, use_256qam=0):
        d = DciOut(sf=int(dci_row["sf"]), rnti=int(dci_row["rnti"]), format=int(dci_row["format"]), L=int(dci_row["L"]), ncce=int(dci_row["ncce"]),
                   nof_bits=int(dci_row["nof_bits"]), bits=int(dci_row["bits"]), histogram_value=int(dci_row["histogram_value"]))
        g = Grant()
        f = DciFields()
        r = self.L.ltephy_dci_to_grant(self.h, C.byref(d), sf_idx, cfi, use_256qam, C.byref(g), C.byref(f))
        return r, g, f


def ul_dci_to_grant(search, dci_row, enable_64qam=1):
    """accepted format-0 DCI -> (return code, UlGrant) via ltephy_ul_dci_to_grant"""
    d = DciOut(sf=int(dci_row["sf"]), rnti=int(dci_row["rnti"]), format=int(dci_row["format"]), L=int(dci_row["L"]), ncce=int(dci_row["ncce"]),
               nof_bits=int(dci_row["nof_bits"]), bits=int(dci_row["bits"]), histogram_value=int(dci_row["histogram_value"]))
    g = UlGrant()
    r = search.L.ltephy_ul_dci_to_grant(search.h, C.byref(d), enable_64qam, C.byref(g))
    return r, g


def ul_decode_plan(search, dci_row, mcs_mod):
    """the decode attempts PUSCH_Decoder::decode makes for this DCI: [(reading, UlGrant)] via ltephy_ul_decode_plan"""
    d = DciOut(sf=int(dci_row["sf"]), rnti=int(dci_row["rnti"]), format=int(dci_row["format"]), L=int(dci_row["L"]), ncce=int(dci_row["ncce"]),
               nof_bits=int(dci_row["nof_bits"]), bits=int(dci_row["bits"]), histogram_value=int(dci_row["histogram_value"]))
    g = (UlGrant * 3)()
    rd = (C.c_uint8 * 3)()
    n = search.L.ltephy_ul_decode_plan(search.h, C.byref(d), mcs_mod, g, rd)
    if n < 0:
        raise ValueError("ltephy_ul_decode_plan: %d" % n)
    return [(int(rd[k]), UlGrant.from_buffer_copy(g[k])) for k in range(n)]


def rar_unpack(search, pdu, max_out=16):
    """MAC RAR PDU -> (return code, [Rar], backoff indicator or -1) via ltephy_rar_unpack"""
    out = (Rar * max_out)()
    n = C.c_uint32(0)
    bo = C.c_int(-1)
    buf = (C.c_uint8 * max(1, len(pdu))).from_buffer_copy(bytes(pdu) if len(pdu) else b"\0")
    r = search.L.ltephy_rar_unpack(search.h, buf, len(pdu), out, max_out, C.byref(n), C.byref(bo))
    return r, [Rar.from_buffer_copy(out[k]) for k in range(n.value)], bo.value


def ul_grants_from_dcis(search, info, dcis, ue_cfgs=()):
    """accepted DCIs of a downlink batch -> [(dci index, reading, UlGrant)] via ltephy_ul_grants_from_dcis (grant.sf = dci.sf + 4)"""
    nd = len(dcis)
    cap = 3 * nd + 1
    g = (UlGrant * cap)()
    gd = np.zeros(cap, np.uint32)
    rd = np.zeros(cap, np.uint8)
    ng = C.c_uint32(0)
    ue = (UlUeCfg * max(1, len(ue_cfgs)))(*ue_cfgs)
    r = search.L.ltephy_ul_grants_from_dcis(search.h, info, dcis.ctypes.data_as(C.c_void_p), nd, ue, len(ue_cfgs), g, gd.ctypes.data_as(C.c_void_p),
                                            rd.ctypes.data_as(C.c_void_p), cap, C.byref(ng))
    if r != 0:
        raise ValueError("ltephy_ul_grants_from_dcis: %d" % r)
    return [(int(gd[k]), int(rd[k]), UlGrant.from_buffer_copy(g[k])) for k in range(ng.value)]


def decode_subframes(phy, search, iq, tti, seq=SEQ_NONE, max_dcis=None, scratch=None):
    """One call through the reference-facing pipeline: host IQ in phy's iq_format -> (info, dcis, tb results, payload)."""
    L = phy.L
    _bind_search(L)
    iq, _ = _host_iq(iq, phy.iq_format)
    tti = np.ascontiguousarray(tti, np.uint32)
    n = len(tti)
    max_dcis = max_dcis or 32 * n
    if scratch is None:
        scratch = dict(info=(SfInfo * n)(), cands=np.zeros((n, MAX_LOC, MAX_SIZES), CAND_DTYPE), dcis=np.zeros(max_dcis, DCI_DTYPE),
                       tbs=(TbResult * (2 * max_dcis))(), payload=np.zeros(max_dcis * 2 * 2048 + n * 40000, np.uint8))
    nd = C.c_uint32(0)
    r = L.ltephy_decode_subframes(phy.h, search.h, _p(iq), _p(tti), n, seq, scratch["info"], _p(scratch["cands"]), _p(scratch["dcis"]), max_dcis,
                                  C.byref(nd), scratch["tbs"], _p(scratch["payload"]), scratch["payload"].nbytes)
    if r != 0:
        raise RuntimeError("ltephy_decode_subframes failed (%d): %s" % (r, L.ltephy_last_error().decode()))
    phy.n = n
    return scratch["info"], scratch["dcis"][:nd.value], scratch["tbs"], scratch["payload"]


# ------------------------------------------------------------------------------------------------
# sharded operation (include/ltephy_shard.h)
SHARD_ID_BYTES = 384
PACK_MAX_BYTES = 64 + 4 * MAX_LOC + 16 * COMPACT_CAP
PACKED_HDR_DTYPE = np.dtype([("count", "<u4"), ("tti", "<u4"), ("cfi", "<u4"), ("nloc", "<u4"), ("noise", "<f4", (2, 2)), ("rsrp", "<f4", (2, 2)),
                             ("low", "<u8", 2)])
assert PACKED_HDR_DTYPE.itemsize == 64


class ShardStats(C.Structure):
    _fields_ = [("host_ms", C.c_double * 8), ("exchanged_bytes", C.c_uint64), ("n_grants", C.c_uint32), ("used_full_table", C.c_uint32)]


SHARD_HOST_MS = ["submit_a", "wait_a", "exchange_turn", "walk_wait", "walk", "grants", "phase_b", "gather_turn"]


def pack_subframes(search, info, comp):
    """host restatement of the GPU pack kernel: (SfInfo * n), COMPACT_DTYPE[n] -> (uint8 records, uint32 offsets[n + 1])"""
    n = len(comp)
    out = np.zeros(n * PACK_MAX_BYTES, np.uint8)
    offs = np.zeros(n + 1, np.uint32)
    comp = np.ascontiguousarray(comp)
    r = search.L.ltephy_pack_subframes(search.h, info, _p(comp), n, _p(out), out.nbytes, _p(offs))
    if r != 0:
        raise RuntimeError("ltephy_pack_subframes failed (%d)" % r)
    return out[:offs[n]].copy(), offs


def search_batch_packed(search, bufs, offs, n, max_dcis, full=None):
    """walk turn of a sharded batch: bufs[r] uint8 records / offs[r] uint32[n + 1] of every rank ->
    (dcis (sf = global index), tti_cfi uint32 [n * world][2]); None when the full tables are needed and were not given"""
    world = len(bufs)
    bp = (C.c_void_p * world)(*[b.ctypes.data for b in bufs])
    op = (C.c_void_p * world)(*[o.ctypes.data for o in offs])
    fp = (C.c_void_p * world)(*[f.ctypes.data for f in full]) if full is not None else None
    dcis = np.zeros(max_dcis, DCI_DTYPE)
    tc = np.zeros((n * world, 2), np.uint32)
    nd = C.c_uint32(0)
    r = search.L.ltephy_search_batch_packed(search.h, bp, op, fp, world, n, _p(dcis), max_dcis, C.byref(nd), _p(tc))
    if r == NEED_FULL_TABLE:
        return None
    if r != 0:
        raise RuntimeError("ltephy_search_batch_packed failed (%d)" % r)
    return dcis[:nd.value].copy(), tc


class Harq:
    """host bookkeeping of the HARQ mode (ltephy_harq_*, include/ltephy_search.h): slot numbers and NEW_TX / RE_TX / DECODED decisions"""

    def __init__(self, max_rnti=150):
        self.L = load_library()
        L = self.L
        L.ltephy_harq_create.restype = C.c_void_p
        L.ltephy_harq_create.argtypes = [C.c_uint32]
        L.ltephy_harq_destroy.argtypes = [C.c_void_p]
        L.ltephy_harq_classify.argtypes = [C.c_void_p, C.c_uint16, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.c_uint32, C.POINTER(C.c_uint32)]
        L.ltephy_harq_update.argtypes = [C.c_void_p, C.c_uint16, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.c_uint32, C.c_int]
        L.ltephy_harq_last_tbs.restype = C.c_int32
        L.ltephy_harq_last_tbs.argtypes = [C.c_void_p, C.c_uint16, C.c_uint32, C.c_uint32]
        self.h = L.ltephy_harq_create(max_rnti)
        assert self.h

    def classify(self, rnti, pid, tb, ndi, tbs, tti):
        slot = C.c_uint32(0)
        r = self.L.ltephy_harq_classify(self.h, rnti, pid, tb, ndi, tbs, tti, C.byref(slot))
        return r, slot.value

    def last_tbs(self, rnti, pid, tb):
        return self.L.ltephy_harq_last_tbs(self.h, rnti, pid, tb)

    def update(self, rnti, pid, tb, ndi, rv, tbs, tti, decoded):
        self.L.ltephy_harq_update(self.h, rnti, pid, tb, ndi, rv, tbs, tti, 1 if decoded else 0)

    def close(self):
        if self.h:
            self.L.ltephy_harq_destroy(self.h)
            self.h = None


def _prefer_torch_nccl():
    """libltephy_b200 binds NCCL with dlopen("libnccl.so.2").  In a Python process that will also import torch, torch's bundled NCCL has to be the
    copy the process holds (an older system libnccl loaded first makes `import torch` fail on missing symbols), so point LTEPHY_NCCL_LIB at it."""
    if os.environ.get("LTEPHY_NCCL_LIB"):
        return
    try:
        import importlib.util
        spec = importlib.util.find_spec("nvidia.nccl")
        for base in (list(spec.submodule_search_locations) if spec and spec.submodule_search_locations else []):
            cand = os.path.join(base, "lib", "libnccl.so.2")
            if os.path.exists(cand):
                os.environ["LTEPHY_NCCL_LIB"] = cand
                return
    except Exception:
        pass


class Shard:
    """NCCL communicators + ordered sections of the sharded pipeline (one per process / GPU)."""

    @staticmethod
    def unique_id():
        _prefer_torch_nccl()
        L = load_library()
        _bind_search(L)
        buf = (C.c_uint8 * SHARD_ID_BYTES)()
        if L.ltephy_shard_unique_id(buf) != 0:
            raise RuntimeError("ltephy_shard_unique_id failed: %s" % L.ltephy_last_error().decode())
        return bytes(buf)

    def __init__(self, uid, rank, world, device):
        _prefer_torch_nccl()
        self.L = load_library()
        _bind_search(self.L)
        self.h = C.c_void_p()
        buf = (C.c_uint8 * SHARD_ID_BYTES).from_buffer_copy(uid)
        r = self.L.ltephy_shard_create(buf, rank, world, device, C.byref(self.h))
        if r != 0:
            raise RuntimeError("ltephy_shard_create failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))
        self.rank, self.world = rank, world

    def close(self):
        if self.h:
            self.L.ltephy_shard_destroy(self.h)
            self.h = None


def pack_phase_a(phy):
    """GPU pack kernel over the current batch of phy -> (uint8 records, uint32 offsets[n + 1])"""
    n = phy.n
    out = np.zeros(n * PACK_MAX_BYTES, np.uint8)
    offs = np.zeros(n + 1, np.uint32)
    _bind_search(phy.L)
    phy._chk(phy.L.ltephy_pack_phase_a(phy.h, _p(out), out.nbytes, _p(offs)), "pack_phase_a")
    return out[:offs[n]].copy(), offs


# ------------------------------------------------------------------------------------------------
# cell search (ltephy_sync_*, include/ltephy_b200.h)
SYNC_TAP_COARSE, SYNC_TAP_REFINED, SYNC_TAP_CFO, SYNC_TAP_SSS = 0, 1, 2, 3
SYNC_BINS = 9600


class SyncCfg(C.Structure):
    _fields_ = [("symbol_sz", C.c_uint32), ("nof_rx", C.c_uint32), ("max_samples", C.c_uint64), ("device", C.c_int32), ("iq_format", C.c_uint32),
                ("reserved", C.c_uint32 * 3)]


class CellInfo(C.Structure):
    """ltephy_cell_t"""
    _fields_ = [("detected", C.c_uint8), ("n_id_2", C.c_uint8), ("pad", C.c_uint8 * 2), ("n_id_1", C.c_uint16), ("pci", C.c_uint16),
                ("frame_offset", C.c_uint64), ("nof_half_frames", C.c_uint32), ("pss_peak", C.c_float), ("psr", C.c_float), ("sss_peak", C.c_float),
                ("sss_ratio", C.c_float), ("cfo_hz", C.c_float), ("cfo_re", C.c_float), ("cfo_im", C.c_float)]


assert C.sizeof(CellInfo) == 48


class CellSearch:
    """PSS / SSS cell search of continuous recordings of symbol_sz samples per symbol and nof_rx antennas, up to max_samples per antenna.
    iq_format "cf32" takes complex64 [nof_rx][n], "sc16" / "sc8" int16 / int8 [nof_rx][n][2]."""

    def __init__(self, symbol_sz, nof_rx, max_samples, device=0, iq_format="cf32"):
        self.L = load_library()
        L = self.L
        L.ltephy_sync_create.argtypes = [C.POINTER(SyncCfg), C.POINTER(C.c_void_p)]
        L.ltephy_sync_destroy.argtypes = [C.c_void_p]
        L.ltephy_cell_search.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        L.ltephy_cell_search_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        L.ltephy_sync_tap.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
        self.iq_format = iq_format
        self.cfg = SyncCfg(symbol_sz=symbol_sz, nof_rx=nof_rx, max_samples=max_samples, device=device, iq_format=IQ_FORMATS[iq_format])
        self.h = C.c_void_p()
        r = L.ltephy_sync_create(C.byref(self.cfg), C.byref(self.h))
        if r != 0:
            self.h = None
            raise RuntimeError("ltephy_sync_create failed (%d): %s" % (r, L.ltephy_last_error().decode()))

    def close(self):
        if self.h:
            self.L.ltephy_sync_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _done(self, r, out):
        if r != 0:
            raise RuntimeError("ltephy_cell_search failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))
        return [CellInfo.from_buffer_copy(out[i]) for i in range(3)]

    def search(self, iq):
        """iq: complex64 [nof_rx][nof_samples] (host; int16 / int8 [nof_rx][nof_samples][2] for sc16 / sc8) -> three CellInfo, by pss_peak
        descending"""
        iq, shape = _host_iq(iq, self.iq_format)
        assert len(shape) == 2 and shape[0] == self.cfg.nof_rx, iq.shape
        out = (CellInfo * 3)()
        return self._done(self.L.ltephy_cell_search(self.h, _p(iq), shape[1], out), out)

    def search_device(self, iq):
        """iq: torch complex64 tensor [nof_rx][nof_samples] (int16 / int8 [nof_rx][nof_samples][2]), contiguous, on this handle's device"""
        shape = _dev_shape(iq, self.iq_format)
        assert len(shape) == 2 and shape[0] == self.cfg.nof_rx
        out = (CellInfo * 3)()
        return self._done(self.L.ltephy_cell_search_device(self.h, C.c_void_p(iq.data_ptr()), shape[1], out), out)

    def tap(self, what):
        """intermediate of the last search as float32: coarse [3][9600], refined [3][2D-1], cfo [3][2], sss [3][168][2]"""
        D = self.cfg.symbol_sz // 128
        shape = {SYNC_TAP_COARSE: (3, SYNC_BINS), SYNC_TAP_REFINED: (3, 2 * D - 1), SYNC_TAP_CFO: (3, 2), SYNC_TAP_SSS: (3, 168, 2)}[what]
        out = np.zeros(shape, np.float32)
        r = self.L.ltephy_sync_tap(self.h, what, _p(out), out.nbytes)
        if r != 0:
            raise RuntimeError("ltephy_sync_tap failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))
        return out


# ------------------------------------------------------------------------------------------------
# tracking after acquisition (ltephy_track_*, include/ltephy_b200.h)
TRACK_NO_CFO, TRACK_REACQUIRE = 1, 2
TRACK_LOCKED, TRACK_LOST, TRACK_REACQUIRED = 1, 2, 4


class TrackCfg(C.Structure):
    _fields_ = [("symbol_sz", C.c_uint32), ("nof_rx", C.c_uint32), ("pci", C.c_uint32), ("first_tti", C.c_uint32), ("frame_offset", C.c_uint64),
                ("cfo_hz", C.c_float), ("max_ppm", C.c_float), ("max_subframes", C.c_uint32), ("flags", C.c_uint32), ("device", C.c_int32),
                ("iq_format", C.c_uint32), ("reserved", C.c_uint32 * 4)]


TRACK_SF_DTYPE = np.dtype([("start", "<i8"), ("tti", "<u4"), ("cfo_hz", "<f4"), ("flags", "<u4"), ("index", "<u4")])
TRACK_HF_DTYPE = np.dtype([("tau", "<i8"), ("index", "<u4"), ("delta", "<i4"), ("peak", "<f4"), ("s_re", "<f4"), ("s_im", "<f4"), ("f_meas", "<f4"),
                           ("flags", "<u4"), ("pad", "<u4")])


class TrackOut(C.Structure):
    _fields_ = [("nof_subframes", C.c_uint32), ("nof_half_frames", C.c_uint32), ("sf", C.c_void_p), ("hf", C.c_void_p), ("iq_dev", C.c_void_p),
                ("next_sample", C.c_uint64), ("remeasured", C.c_uint32), ("finds", C.c_uint32)]


class TrackUlCfg(C.Structure):
    _fields_ = [("cfo_ratio", C.c_double), ("ul_offset", C.c_int32), ("nof_rx", C.c_uint32), ("reserved", C.c_uint32 * 4)]


assert C.sizeof(TrackCfg) == 64 and C.sizeof(TrackOut) == 48 and TRACK_SF_DTYPE.itemsize == 24 and TRACK_HF_DTYPE.itemsize == 40
assert C.sizeof(TrackUlCfg) == 32


class Tracker:
    """PSS tracking and subframe cutting of a recording after the cell search: push the recording part by part (antenna-major complex64
    [nof_rx][n] with its absolute first sample); each push returns the subframes that now lie wholly inside what was fed.  With ul=dict(cfo_ratio=..., ul_offset=...) the tracker also cuts the
    uplink carrier of the same radio (ltephy_track_set_ul); push both carriers with push_ul / push_ul_device.  ul=dict(..., nof_rx=2) cuts two UL
    antennas: push_ul then takes iq_ul [2][n] and ul_iq is [k][2][15 N] (one antenna: [n] and [k][15 N]).  With flags=TRACK_REACQUIRE a
    lost cell is searched again frame by frame; the first subframe cut after it is found carries TRACK_REACQUIRED.  iq_format "sc16" / "sc8" takes
    int16 / int8 pushes with a last axis of 2 (I, Q), DL and UL alike; the cuts stay complex64."""

    def __init__(self, symbol_sz, nof_rx, pci, frame_offset, cfo_hz=0.0, first_tti=0, max_subframes=1000, max_ppm=50.0, flags=0, device=0, ul=None,
                 iq_format="cf32"):
        self.L = load_library()
        L = self.L
        L.ltephy_track_create.argtypes = [C.POINTER(TrackCfg), C.POINTER(C.c_void_p)]
        L.ltephy_track_destroy.argtypes = [C.c_void_p]
        L.ltephy_track_push.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(TrackOut)]
        L.ltephy_track_push_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(TrackOut)]
        L.ltephy_track_set_ul.argtypes = [C.c_void_p, C.POINTER(TrackUlCfg)]
        L.ltephy_track_push_ul.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(TrackOut), C.POINTER(C.c_void_p)]
        L.ltephy_track_push_ul_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(TrackOut), C.POINTER(C.c_void_p)]
        self.cfg = TrackCfg(symbol_sz=symbol_sz, nof_rx=nof_rx, pci=pci, first_tti=first_tti, frame_offset=frame_offset, cfo_hz=cfo_hz,
                            max_ppm=max_ppm, max_subframes=max_subframes, flags=flags, device=device, iq_format=IQ_FORMATS[iq_format])
        self.iq_format = iq_format
        self.h = C.c_void_p()
        r = L.ltephy_track_create(C.byref(self.cfg), C.byref(self.h))
        if r != 0:
            self.h = None
            raise RuntimeError("ltephy_track_create failed (%d): %s" % (r, L.ltephy_last_error().decode()))
        self.next_sample = frame_offset
        self.ul = None
        if ul is not None:
            u = TrackUlCfg(cfo_ratio=float(ul.get("cfo_ratio", 1.0)), ul_offset=int(ul.get("ul_offset", 0)), nof_rx=int(ul.get("nof_rx", 1)))
            r = L.ltephy_track_set_ul(self.h, C.byref(u))
            if r != 0:
                self.close()
                raise RuntimeError("ltephy_track_set_ul failed (%d): %s" % (r, L.ltephy_last_error().decode()))
            self.ul = u
            self.next_sample = min(frame_offset, frame_offset + u.ul_offset)

    def close(self):
        if self.h:
            self.L.ltephy_track_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _view(self, ptr, shape):
        """a torch copy of the tracker's device buffer at ptr (valid until the next push)"""
        import torch
        if shape[0]:
            view = type("_Cut", (), {"__cuda_array_interface__": dict(shape=shape, typestr="<c8", data=(ptr, False), version=2)})()
            with torch.cuda.device(self.cfg.device):
                return torch.as_tensor(view, device="cuda:%d" % self.cfg.device).clone()
        return torch.empty(shape, dtype=torch.complex64, device="cuda:%d" % self.cfg.device)

    def _done(self, r, o, ul_ptr=None):
        if r != 0:
            raise RuntimeError("ltephy_track_push failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))
        sf = np.ctypeslib.as_array((C.c_uint8 * (o.nof_subframes * 24)).from_address(o.sf)).view(TRACK_SF_DTYPE).copy() if o.nof_subframes else \
            np.zeros(0, TRACK_SF_DTYPE)
        hf = np.ctypeslib.as_array((C.c_uint8 * (o.nof_half_frames * 40)).from_address(o.hf)).view(TRACK_HF_DTYPE).copy() if o.nof_half_frames else \
            np.zeros(0, TRACK_HF_DTYPE)
        iq = self._view(o.iq_dev, (o.nof_subframes, self.cfg.nof_rx, 15 * self.cfg.symbol_sz))
        self.next_sample = o.next_sample
        out = dict(sf=sf, hf=hf, iq=iq, next_sample=o.next_sample, remeasured=o.remeasured, finds=o.finds)
        if ul_ptr is not None:
            A = max(1, self.ul.nof_rx)
            out["ul_iq"] = self._view(ul_ptr.value, (o.nof_subframes, 15 * self.cfg.symbol_sz) if A == 1 else (o.nof_subframes, A, 15 * self.cfg.symbol_sz))
        return out

    def _push(self, dev, first_sample, *iqs):
        """every push: iqs = (iq,) or (iq, iq_ul), host arrays or, with dev, contiguous tensors on this handle's device"""
        if dev:
            shapes, ptrs = [_dev_shape(q, self.iq_format) for q in iqs], [C.c_void_p(q.data_ptr()) for q in iqs]
        else:
            iqs = [_host_iq(q, self.iq_format) for q in iqs]
            shapes, ptrs = [s for _, s in iqs], [_p(q) for q, _ in iqs]
        ul = len(iqs) == 2
        assert len(shapes[0]) == 2 and shapes[0][0] == self.cfg.nof_rx, shapes
        assert not ul or int(np.prod(shapes[1])) == max(1, self.ul.nof_rx) * shapes[0][1], shapes
        o, u = TrackOut(), C.c_void_p()
        push = getattr(self.L, "ltephy_track_push" + "_ul" * ul + "_device" * dev)
        r = push(self.h, *ptrs, first_sample, shapes[0][1], C.byref(o), *([C.byref(u)] if ul else []))
        return self._done(r, o, u if ul else None)

    def push(self, iq, first_sample):
        """iq: complex64 [nof_rx][n] (host) of absolute samples first_sample ... -> dict(sf, hf: record arrays, iq: torch complex64
        [k][nof_rx][15 N] on the device (a copy of the tracker's cut), next_sample, remeasured, finds)"""
        return self._push(False, first_sample, iq)

    def push_device(self, iq, first_sample):
        """iq: torch complex64 tensor [nof_rx][n] (int16 / int8 [nof_rx][n][2]), contiguous, on this handle's device"""
        return self._push(True, first_sample, iq)

    def push_ul(self, iq, iq_ul, first_sample):
        """iq as push, iq_ul: complex64 [n] of the uplink antenna ([A][n] with A = 2 UL antennas), the same absolute samples -> push's dict plus
        ul_iq: torch complex64 [k][15 N] ([k][A][15 N]) on the device (a copy of the tracker's UL cut)"""
        return self._push(False, first_sample, iq, iq_ul)

    def push_ul_device(self, iq, iq_ul, first_sample):
        """iq: torch complex64 [nof_rx][n], iq_ul: torch complex64 [n] ([A][n] with A = 2 UL antennas), both contiguous on this handle's device"""
        return self._push(True, first_sample, iq, iq_ul)


# ------------------------------------------------------------------------------------------------
# channeliser (ltephy_chan_*, include/ltephy_b200.h)
CHAN_MAX_CARRIERS = 8
CHAN_RATIONAL = 1


class ChanCarrier(C.Structure):
    _fields_ = [("offset_hz", C.c_int32), ("symbol_sz", C.c_uint32)]


class ChanCfg(C.Structure):
    _fields_ = [("fs_in", C.c_uint32), ("nof_rx", C.c_uint32), ("nof_carriers", C.c_uint32), ("pad", C.c_uint32),
                ("carrier", ChanCarrier * CHAN_MAX_CARRIERS), ("max_samples", C.c_uint64), ("device", C.c_int32), ("flags", C.c_uint32), ("iq_format", C.c_uint32),
                ("reserved", C.c_uint32 * 3)]


class ChanOut(C.Structure):
    _fields_ = [("first", C.c_uint64), ("count", C.c_uint64), ("iq_dev", C.c_void_p)]


class ChanPoly(C.Structure):
    _fields_ = [(k, C.c_uint32) for k in ("L", "M", "Tp", "Kp", "Ka", "Kb", "P")]


assert C.sizeof(ChanCfg) == 112 and C.sizeof(ChanOut) == 24


def _bind_chan(L):
    L.ltephy_chan_create.argtypes = [C.POINTER(ChanCfg), C.POINTER(C.c_void_p)]
    L.ltephy_chan_destroy.argtypes = [C.c_void_p]
    L.ltephy_chan_run.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64)]
    L.ltephy_chan_run_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64)]
    L.ltephy_chan_taps.argtypes = [C.POINTER(ChanCfg), C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                   C.POINTER(C.c_uint32)]
    L.ltephy_chan_design.argtypes = [C.POINTER(ChanCfg), C.c_uint32, C.POINTER(ChanPoly), C.c_void_p, C.c_void_p, C.c_void_p]


def chan_cfg(fs_in, carriers, nof_rx=1, max_samples=1, device=0, flags=0, iq_format=0):
    """ChanCfg from carriers = [(offset_hz, symbol_sz), ...]"""
    cfg = ChanCfg(fs_in=fs_in, nof_rx=nof_rx, nof_carriers=len(carriers), max_samples=max_samples, device=device, flags=flags, iq_format=iq_format)
    for i, (off, n) in enumerate(carriers[:CHAN_MAX_CARRIERS]):
        cfg.carrier[i] = ChanCarrier(off, n)
    return cfg


def chan_taps(fs_in, carriers, c):
    """host-only tables of carrier c -> dict(h float32 [T], g complex64 [T], rot complex64 [P], T, D, P); RuntimeError when refused"""
    L = load_library()
    _bind_chan(L)
    cfg = chan_cfg(fs_in, carriers)
    T, D, P = C.c_uint32(), C.c_uint32(), C.c_uint32()
    r = L.ltephy_chan_taps(C.byref(cfg), c, None, None, None, C.byref(T), C.byref(D), C.byref(P))
    if r != 0:
        raise RuntimeError("ltephy_chan_taps failed (%d): %s" % (r, L.ltephy_last_error().decode()))
    h, g, rot = np.zeros(T.value, np.float32), np.zeros(T.value, np.complex64), np.zeros(P.value, np.complex64)
    L.ltephy_chan_taps(C.byref(cfg), c, _p(h), _p(g), _p(rot), C.byref(T), C.byref(D), C.byref(P))
    return dict(h=h, g=g, rot=rot, T=T.value, D=D.value, P=P.value)


def chan_design(fs_in, carriers, c, rational=True):
    """host-only geometry and tables of carrier c under the plan's flags -> dict(L, M, Tp, Kp, Ka, Kb, P, hp float32 [Tp], g complex64 [L][Kp],
    rot complex64 [P]); RuntimeError when refused"""
    L = load_library()
    _bind_chan(L)
    cfg = chan_cfg(fs_in, carriers, flags=CHAN_RATIONAL if rational else 0)
    q = ChanPoly()
    r = L.ltephy_chan_design(C.byref(cfg), c, C.byref(q), None, None, None)
    if r != 0:
        raise RuntimeError("ltephy_chan_design failed (%d): %s" % (r, L.ltephy_last_error().decode()))
    hp, g, rot = np.zeros(q.Tp, np.float32), np.zeros((q.L, q.Kp), np.complex64), np.zeros(q.P, np.complex64)
    L.ltephy_chan_design(C.byref(cfg), c, C.byref(q), _p(hp), _p(g), _p(rot))
    d = {k: getattr(q, k) for k, _ in ChanPoly._fields_}
    d.update(hp=hp, g=g, rot=rot)
    return d


class Channelizer:
    """Shift, filter and resample the carriers [(offset_hz, symbol_sz), ...] of a capture at fs_in out of antenna-major [nof_rx][n] spans of up
    to max_samples; each run returns every carrier's outputs that the span completes, and next_sample, the lowest capture sample the next run must
    still include.  rational=True sets LTEPHY_CHAN_RATIONAL (any ratio the rational rule accepts); iq_format "cf32" takes complex64 [nof_rx][n],
    "sc16" / "sc8" take interleaved int16 / int8 [nof_rx][2n]."""

    def __init__(self, fs_in, carriers, nof_rx, max_samples, device=0, rational=False, iq_format="cf32"):
        self.L = load_library()
        _bind_chan(self.L)
        self.carriers = list(carriers)
        self.rational, self.iq_format = rational, iq_format
        self.cfg = chan_cfg(fs_in, self.carriers, nof_rx, max_samples, device, CHAN_RATIONAL if rational else 0, IQ_FORMATS[iq_format])
        self.h = C.c_void_p()
        r = self.L.ltephy_chan_create(C.byref(self.cfg), C.byref(self.h))
        if r != 0:
            self.h = None
            raise RuntimeError("ltephy_chan_create failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))
        self.next_sample = 0

    def close(self):
        if self.h:
            self.L.ltephy_chan_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def taps(self, c):
        return chan_taps(self.cfg.fs_in, self.carriers, c)

    def design(self, c):
        return chan_design(self.cfg.fs_in, self.carriers, c, self.rational)

    def _samples(self, iq):
        """the number of complex samples per antenna of iq in the handle's format"""
        assert iq.ndim == 2 and iq.shape[0] == self.cfg.nof_rx, iq.shape
        if self.iq_format == "cf32":
            return iq.shape[1]
        assert iq.shape[1] % 2 == 0, iq.shape
        return iq.shape[1] // 2

    def _done(self, r, out, nxt, copy):
        if r != 0:
            raise RuntimeError("ltephy_chan_run failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))
        import torch
        res = []
        for c in range(len(self.carriers)):
            o = out[c]
            shape = (self.cfg.nof_rx, o.count)
            if o.count:
                view = type("_Chan", (), {"__cuda_array_interface__": dict(shape=shape, typestr="<c8", data=(o.iq_dev, False), version=2)})()
                with torch.cuda.device(self.cfg.device):
                    iq = torch.as_tensor(view, device="cuda:%d" % self.cfg.device)
                    iq = iq.clone() if copy else iq
            else:
                iq = torch.empty(shape, dtype=torch.complex64, device="cuda:%d" % self.cfg.device)
            res.append(dict(first=o.first, count=o.count, iq=iq))
        self.next_sample = nxt.value
        return res, nxt.value

    def run(self, iq, first_sample, copy=True):
        """iq: complex64 [nof_rx][n] (host; int16 / int8 [nof_rx][2n] for sc16 / sc8) of capture samples first_sample ... -> ([dict(first,
        count, iq: torch complex64 [nof_rx][count] on the device)] per carrier, next_sample).  With copy=False iq views the handle's buffer, valid
        until the next run."""
        iq = np.ascontiguousarray(iq, _IQ_DTYPES[self.iq_format])
        n = self._samples(iq)
        out, nxt = (ChanOut * CHAN_MAX_CARRIERS)(), C.c_uint64()
        return self._done(self.L.ltephy_chan_run(self.h, _p(iq), first_sample, n, out, C.byref(nxt)), out, nxt, copy)

    def run_device(self, iq, first_sample, copy=True):
        """iq: torch complex64 [nof_rx][n] (int16 / int8 [nof_rx][2n] for sc16 / sc8), contiguous, on this handle's device"""
        import torch
        want = {"cf32": torch.complex64, "sc16": torch.int16, "sc8": torch.int8}[self.iq_format]
        assert iq.is_cuda and iq.is_contiguous() and iq.dim() == 2 and iq.dtype == want, (iq.dtype, want)
        n = self._samples(iq)
        out, nxt = (ChanOut * CHAN_MAX_CARRIERS)(), C.c_uint64()
        return self._done(self.L.ltephy_chan_run_device(self.h, C.c_void_p(iq.data_ptr()), first_sample, n, out, C.byref(nxt)), out, nxt, copy)


# ------------------------------------------------------------------------------------------------
# raster scan (ltephy_scan_*, include/ltephy_b200.h)
class ScanCfg(C.Structure):
    _fields_ = [("fs_in", C.c_uint32), ("nof_rx", C.c_uint32), ("iq_format", C.c_uint32), ("max_points_per_pass", C.c_uint32), ("center_hz", C.c_uint64),
                ("lo_hz", C.c_int32), ("hi_hz", C.c_int32), ("max_samples", C.c_uint64), ("device", C.c_int32), ("reserved", C.c_uint32 * 5)]


class ScanCell(C.Structure):
    """ltephy_scan_cell_t: a raster point's offset and its detected cell (timing in N = 128 stream samples)"""
    _fields_ = [("offset_hz", C.c_int32), ("pad", C.c_uint32), ("cell", CellInfo)]


assert C.sizeof(ScanCfg) == 64 and C.sizeof(ScanCell) == 56


def _bind_scan(L):
    L.ltephy_scan_create.argtypes = [C.POINTER(ScanCfg), C.POINTER(C.c_void_p)]
    L.ltephy_scan_destroy.argtypes = [C.c_void_p]
    L.ltephy_scan_run.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    L.ltephy_scan_run_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
    L.ltephy_scan_points.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    L.ltephy_scan_plan.argtypes = [C.POINTER(ScanCfg), C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]


def scan_cfg(fs_in, nof_rx, center_hz, max_samples, lo_hz=0, hi_hz=0, iq_format="cf32", max_points_per_pass=0, device=0):
    return ScanCfg(fs_in=fs_in, nof_rx=nof_rx, iq_format=IQ_FORMATS[iq_format], max_points_per_pass=max_points_per_pass, center_hz=center_hz, lo_hz=lo_hz,
                   hi_hz=hi_hz, max_samples=max_samples, device=device)


def scan_plan(cfg):
    """host only: the raster offsets of a ScanCfg, ascending (np.int32); RuntimeError when refused"""
    L = load_library()
    _bind_scan(L)
    n = C.c_uint32()
    r = L.ltephy_scan_plan(C.byref(cfg), None, 0, C.byref(n))
    if r != 0:
        raise RuntimeError("ltephy_scan_plan failed (%d): %s" % (r, L.ltephy_last_error().decode()))
    off = np.zeros(n.value, np.int32)
    L.ltephy_scan_plan(C.byref(cfg), _p(off), n.value, C.byref(n))
    return off


class Scanner:
    """Cell search at every 100 kHz raster point of a capture at fs_in centred on center_hz (a multiple of 1 kHz), in [lo_hz, hi_hz] (both 0: every
    offset), of up to max_samples per antenna.  iq_format "cf32" takes complex64 [nof_rx][n], "sc16" / "sc8" interleaved int16 / int8 [nof_rx][2n],
    as Channelizer does.  run / run_device -> [(offset_hz, CellInfo)] of every detected cell, by offset, then pss_peak descending."""

    def __init__(self, fs_in, nof_rx, center_hz, max_samples, lo_hz=0, hi_hz=0, iq_format="cf32", max_points_per_pass=0, device=0):
        self.L = load_library()
        _bind_scan(self.L)
        self.iq_format = iq_format
        self.cfg = scan_cfg(fs_in, nof_rx, center_hz, max_samples, lo_hz, hi_hz, iq_format, max_points_per_pass, device)
        self.offsets = scan_plan(self.cfg)
        self.h = C.c_void_p()
        r = self.L.ltephy_scan_create(C.byref(self.cfg), C.byref(self.h))
        if r != 0:
            self.h = None
            raise RuntimeError("ltephy_scan_create failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))

    def close(self):
        if self.h:
            self.L.ltephy_scan_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def plan(self):
        return self.offsets.copy()

    def _samples(self, shape):
        assert len(shape) == 2 and shape[0] == self.cfg.nof_rx, shape
        if self.iq_format == "cf32":
            return shape[1]
        assert shape[1] % 2 == 0, shape
        return shape[1] // 2

    def _done(self, r, out, n):
        if r != 0:
            raise RuntimeError("ltephy_scan_run failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))
        return [(out[i].offset_hz, CellInfo.from_buffer_copy(out[i].cell)) for i in range(min(n.value, len(out)))]

    def run(self, iq, cap=1024):
        """iq: capture samples 0 .. n - 1 on the host"""
        iq = np.ascontiguousarray(iq, _IQ_DTYPES[self.iq_format])
        out, n = (ScanCell * cap)(), C.c_uint32()
        r = self.L.ltephy_scan_run(self.h, _p(iq), self._samples(iq.shape), out, cap, C.byref(n))
        return self._done(r, out, n)

    def run_device(self, iq, cap=1024):
        """iq: torch complex64 [nof_rx][n] (int16 / int8 [nof_rx][2n] for sc16 / sc8), contiguous, on this handle's device"""
        import torch
        want = {"cf32": torch.complex64, "sc16": torch.int16, "sc8": torch.int8}[self.iq_format]
        assert iq.is_cuda and iq.is_contiguous() and iq.dtype == want, (iq.dtype, want)
        out, n = (ScanCell * cap)(), C.c_uint32()
        r = self.L.ltephy_scan_run_device(self.h, C.c_void_p(iq.data_ptr()), self._samples(tuple(iq.shape)), out, cap, C.byref(n))
        return self._done(r, out, n)

    def points(self):
        """the three CellInfo of every point of the last run: [points][3], each point's by pss_peak descending"""
        P = len(self.offsets)
        out = (CellInfo * (3 * P))()
        r = self.L.ltephy_scan_points(self.h, out, P)
        if r != 0:
            raise RuntimeError("ltephy_scan_points failed (%d): %s" % (r, self.L.ltephy_last_error().decode()))
        return [[CellInfo.from_buffer_copy(out[3 * p + i]) for i in range(3)] for p in range(P)]
