"""Captures and oracle bindings for the tracker's find state (LTEPHY_TRACK_REACQUIRE, DESIGN.md §2 "tracking"): a receiver that drops samples,
the oracle with its count of find windows, and chunked pushes that sum it.  Imported only by tests/."""
import ctypes as C

import numpy as np

import track_lib as T
import track_ul_lib as U

REACQUIRE, REACQUIRED = 2, 4


def _lib():
    L = T.lib()
    L.lteo_track_finds.restype = C.c_uint32
    L.lteo_track_finds.argtypes = [C.c_void_p]
    return L


def capture(N, pci, nsf, drop=None, **kw):
    """track_lib.capture, then `drop` = (first, count): count receiver samples removed at first (after resampling and the carrier offset), as a
    receiver that overflows loses them.  -> (x, truth starts, truth carrier offsets, transmit subframe number since t0 of each truth start); the
    subframes that started inside the drop are removed, the later ones move count samples earlier."""
    x, truth, ft = T.capture(N, pci, nsf, **kw)
    num = np.arange(nsf)
    if drop:
        a, c = drop
        x = np.delete(x, np.s_[a:a + c], axis=1)
        keep = (truth < a) | (truth >= a + c)
        truth = np.where(truth >= a + c, truth - c, truth)[keep]
        ft, num = ft[keep], num[keep]
    return x, truth, ft, num


def _counted(cls):
    class Counted(cls):
        """the oracle binding with `finds`: the find windows its push searched, as ltephy_track_out_t.finds"""

        def _count(self, fn, *a, **kw):
            n0 = _lib().lteo_track_finds(self.t)
            o = fn(*a, **kw)
            o["finds"] = _lib().lteo_track_finds(self.t) - n0
            return o

        def push(self, *a, **kw):
            return self._count(super().push, *a, **kw)

        def push_ul(self, *a, **kw):
            return self._count(super().push_ul, *a, **kw)
    return Counted


Oracle = _counted(T.Oracle)
OracleUl = _counted(U.OracleUl)


def run_chunks(tr, x, sizes, push=None):
    """track_lib.run_chunks, with the finds of every push summed and the tracker's last next_sample"""
    push = push or tr.push
    finds = []

    def counted(xx, s):
        o = push(xx, s)
        finds.append(o["finds"])
        return o
    r = T.run_chunks(tr, x, sizes, push=counted)
    r["finds"], r["next_sample"] = sum(finds), tr.next_sample
    return r


def drop_cases(N):
    """the drops of the tests: beyond the tracker's +-9 N / 128 window, and across 37 subframes and a part of one"""
    SF = 15 * N
    return {"3N+17": 3 * N + 17, "37SF+1234": 37 * SF + 1234}


def noise(rng, nrx, L, rms):
    return ((rng.standard_normal((nrx, L)) + 1j * rng.standard_normal((nrx, L))) * rms * np.sqrt(0.5)).astype(np.complex64)
