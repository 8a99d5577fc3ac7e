"""The raster scan's rule (DESIGN.md §2 "raster scan") in Python: the raster points of a capture, each point's three results from the oracles
(lteo_chan_run_poly for the point's N = 128 stream, then lteo_cell_search), and the cells the scan reports.  Imported only by tests/."""
import numpy as np

import chan_rational_lib as CR
import sync_lib as S

RASTER = 100000      # E-UTRA channel raster (36.101 5.7.2)
F_PASS = 540000      # the channeliser's band of an N = 128 carrier: 90 kHz x 6 PRB
HALF_FRAME = 75 * 128 + 128


def plan(fs_in, center_hz, lo_hz=0, hi_hz=0):
    """offsets o = 100 kHz k - center_hz with |o| + 540 kHz <= fs_in / 2 and, unless lo_hz = hi_hz = 0, lo_hz <= o <= hi_hz; ascending"""
    k0, k1 = (center_hz - fs_in) // RASTER - 1, (center_hz + fs_in) // RASTER + 1
    out = []
    for k in range(k0, k1 + 1):
        o = RASTER * k - center_hz
        if 2 * (abs(o) + F_PASS) <= fs_in and (lo_hz == 0 and hi_hz == 0 or lo_hz <= o <= hi_hz):
            out.append(o)
    return out


def point(fs_in, offset_hz, x, fmt="cf32"):
    """the three lteo_cell_search results of the N = 128 stream of capture samples [0, n) at offset_hz"""
    res, _ = CR.run(fs_in, [(offset_hz, 128)], x, 0, fmt)
    r, cells, _ = S.cell_search(128, res[0]["iq"])
    assert r == 0, r
    return cells


def points(fs_in, offsets, x, fmt="cf32"):
    return [point(fs_in, o, x, fmt) for o in offsets]


def reported(offsets, pts):
    """every detected result, by offset ascending, then by pss_peak descending (each point's three come that way from the search)"""
    return [(o, c) for o, cs in zip(offsets, pts) for c in cs if c.detected]
