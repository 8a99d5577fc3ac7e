"""ctypes bindings for the cell search test infrastructure: the simulator's sync signals and oracle/liblteosync.so (lteo_cell_search,
oracle/lte_sync_oracle.h).  Imported only by tests/."""
import ctypes as C
import os

import numpy as np

import ltelib

SYNC_BINS = 9600


def sim(sync=1, **kw):
    """ltelib.Sim with lte_sim_cfg_t.sync set: that word is the first of the two ltelib.SimCfg calls `reserved` (the struct kept its size)"""
    return ltelib.Sim(reserved=(C.c_uint32 * 2)(sync, 0), **kw)


class CellOut(C.Structure):
    """lteo_cell_t / ltephy_cell_t: one cell-search result per N_ID_2"""
    _fields_ = [("detected", C.c_uint8), ("n_id_2", C.c_uint8), ("pad", C.c_uint8 * 2), ("n_id_1", C.c_uint16), ("pci", C.c_uint16),
                ("frame_offset", C.c_uint64), ("nof_half_frames", C.c_uint32), ("pss_peak", C.c_float), ("psr", C.c_float), ("sss_peak", C.c_float),
                ("sss_ratio", C.c_float), ("cfo_hz", C.c_float), ("cfo_re", C.c_float), ("cfo_im", C.c_float)]


class SyncTaps(C.Structure):
    _fields_ = [("coarse", C.c_void_p), ("refined", C.c_void_p), ("cfo", C.c_void_p), ("sss", C.c_void_p)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        ltelib.build_infra()
        L = C.CDLL(os.path.join(ltelib.ROOT, "oracle", "liblteosync.so"))
        L.lteo_cell_search.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(SyncTaps)]
        _lib = L
    return _lib


def cell_search(N, x):
    """lteo_cell_search on x complex64 [nof_rx][L] -> (return code, [CellOut] * 3, dict of the intermediates)"""
    x = np.ascontiguousarray(x, np.complex64)
    D = N // 128
    taps = dict(coarse=np.zeros((3, SYNC_BINS), np.float32), refined=np.zeros((3, max(1, 2 * D - 1)), np.float32),
                cfo=np.zeros((3, 2), np.float32), sss=np.zeros((3, 168, 2), np.float32))
    t = SyncTaps(*[ltelib.ptr(taps[k]) for k in ("coarse", "refined", "cfo", "sss")])
    out = (CellOut * 3)()
    r = lib().lteo_cell_search(N, x.shape[0], ltelib.ptr(x), x.shape[1], out, C.byref(t))
    return r, [out[i] for i in range(3)], taps
