"""Captures for the tracker's find state (LTEPHY_TRACK_REACQUIRE, DESIGN.md §2 "tracking"): a receiver that drops samples, the drops of the tests
and noise.  Imported only by tests/."""
import numpy as np

import track_lib as T

REACQUIRE, REACQUIRED = 2, 4


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


def drop_cases(N):
    """the drops of the tests: beyond the tracker's +-9 N / 128 window, and across 37 subframes and a part of one"""
    SF = 15 * N
    return {"3N+17": 3 * N + 17, "37SF+1234": 37 * SF + 1234}


def noise(rng, nrx, L, rms):
    return ((rng.standard_normal((nrx, L)) + 1j * rng.standard_normal((nrx, L))) * rms * np.sqrt(0.5)).astype(np.complex64)
