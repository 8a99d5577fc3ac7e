"""Test infrastructure for the MIB decode across the 40 ms PBCH period: ctypes bindings of oracle/liblteomib.so (lteo_pbch_llr and the
combiner lteo_mib_*, oracle/lte_mib_oracle.h), an independent Python statement of srsRAN's combining loop over lteo_dci_decode, and a
generator of simulated subframes 0.  Imported only by tests/."""
import ctypes as C
import os

import numpy as np

import ltelib
from helpers import oracle_frontend
from ref64 import gold

MASK = {1: 0x0000, 2: 0xFFFF}
BW = {0: 6, 1: 15, 2: 25, 3: 50, 4: 75, 5: 100}


class MibRes(C.Structure):
    _fields_ = [("found", C.c_uint8), ("nof_ports", C.c_uint8), ("sfn_offset", C.c_uint8), ("nof_frames", C.c_uint8), ("src", C.c_uint8),
                ("dst", C.c_uint8), ("window", C.c_uint8), ("mib", C.c_uint8 * 24), ("sfn", C.c_uint32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        ltelib.build_infra()
        L = C.CDLL(os.path.join(ltelib.ROOT, "oracle", "liblteomib.so"))
        P = C.c_void_p
        L.lteo_pbch_llr.argtypes = [C.POINTER(ltelib.Cell), P, P, C.c_uint32, P]
        L.lteo_mib_create.restype = P
        L.lteo_mib_create.argtypes = [C.POINTER(ltelib.Cell)]
        L.lteo_mib_destroy.argtypes = [P]
        L.lteo_mib_reset.argtypes = [P]
        L.lteo_mib_decode.argtypes = [P, C.c_uint32, P, P, C.c_int, C.POINTER(MibRes)]
        _lib = L
    return _lib


def _pp(fe):
    return ltelib.ptr_array(list(fe["sym"])), ltelib.ptr_array(list(fe["ce"]))


def pbch_llr(cell, fe, nant):
    llr = np.zeros(480, np.float32)
    s, c = _pp(fe)
    assert lib().lteo_pbch_llr(C.byref(cell), s, c, nant, ltelib.ptr(llr)) == 0
    return llr


def res_tuple(found, nof_ports=0, sfn_offset=0, nof_frames=0, src=0, dst=0, window=0, mib=None, sfn=0):
    """the comparable form of one result: None when nothing passed"""
    if not found:
        return None
    return (nof_ports, sfn_offset, nof_frames, src, dst, window, tuple(int(b) for b in mib), sfn)


class OracleCombiner:
    """lteo_mib_* on frames given as oracle front-end dicts"""

    def __init__(self, cell):
        self.cell = cell
        self.h = lib().lteo_mib_create(C.byref(cell))
        assert self.h

    def __del__(self):
        try:
            lib().lteo_mib_destroy(self.h)
        except Exception:
            pass

    def reset(self):
        lib().lteo_mib_reset(self.h)

    def decode(self, tti, fe, search_ports=False):
        r = MibRes()
        s, c = _pp(fe)
        lib().lteo_mib_decode(self.h, tti, s, c, int(search_ports), C.byref(r))
        return res_tuple(r.found, r.nof_ports, r.sfn_offset, r.nof_frames, r.src, r.dst, r.window, list(r.mib), r.sfn)


class PyCombiner:
    """srsRAN 21.10's PBCH combiner stated again, from DESIGN.md §2, over lteo_dci_decode: a list of held frames per port count"""

    def __init__(self, cell, oracle):
        self.cell, self.o = cell, oracle
        self.scr = gold(cell.cell_id, 1920).astype(bool)
        self.reset()

    def reset(self):
        self.held = {p: [] for p in range(1, self.cell.nof_ports + 1)}
        self.last = None

    def decode(self, tti, fe, search_ports=False):
        sfn = (tti // 10) % 1024
        if self.last is not None and sfn != (self.last + 1) % 1024:
            self.held = {p: [] for p in self.held}
        self.last = sfn
        for p in self.held:
            self.held[p].append(pbch_llr(self.cell, fe, p))
        w = len(self.held[1])
        for nant in (range(1, self.cell.nof_ports + 1) if search_ports else [self.cell.nof_ports]):
            for nb in range(w):
                for dst in range(4 - nb):
                    for src in range(w - nb):
                        e = np.zeros(1920, np.float32)
                        for j in range(nb + 1):
                            sl = slice(480 * (dst + j), 480 * (dst + j + 1))
                            e[sl] = np.where(self.scr[sl], -self.held[nant][src + j], self.held[nant][src + j])
                        r, bits, rem = self.o.dci_decode(e, 24)
                        if r != 0 or rem != MASK[nant]:
                            continue
                        off = dst - src + w - 1
                        msb = int("".join(str(int(b)) for b in bits[6:14]), 2)
                        self.held = {p: [] for p in self.held}
                        return (nant, off, nb + 1, src, dst, w, tuple(int(b) for b in bits), ((msb << 2) + off) % 1024)
        if w == 4:
            for p in self.held:
                self.held[p].pop(0)
        return None


def frames(cell, sfns, snr_db, seed=5, o=None):
    """simulated subframes 0 of the frames sfns (PBCH on): -> (iq [len][nof_rx][sf_len], tti, oracle front-end dicts)"""
    s = ltelib.Sim(cell=cell, seed=seed, cfi=3 if cell.phich_ext else 2, nof_ues=1, dl_min=1, dl_max=1, tm=1, snr_db=snr_db, pbch=1)
    tti = np.array([10 * (f % 1024) for f in sfns], np.uint32)
    iq = np.zeros((len(sfns), cell.nof_rx, s.sf_len), np.complex64)
    for i, t in enumerate(tti):
        iq[i] = s.subframe(int(t))[0]
    o = o or ltelib.Oracle(cell)
    return iq, tti, oracle_frontend(o, iq, tti)


def broadcast(cell, sfn):
    """the MIB bits the simulated eNB sends in frame sfn"""
    S = ltelib.sim()
    bits = np.zeros(24, np.uint8)
    S.lte_mib_pack.argtypes = [C.c_uint32] * 4 + [C.c_void_p]
    S.lte_mib_pack(cell.nof_prb, cell.phich_ext, cell.phich_ng, sfn, ltelib.ptr(bits))
    return tuple(int(b) for b in bits)
