"""The raster scan without a GPU: ltephy_scan_plan against a Python statement of the raster and the band check, every refusal before a device
is looked for, and the rule (tests/scan_lib.py: lteo_chan_run_poly then lteo_cell_search at every point) on composed wideband captures: three
cells of different bandwidths, PCIs, carrier offsets and gains are each reported once at their offsets, noise reports nothing, and two co-channel
cells of different N_ID_2 at one offset are both reported."""
import ctypes as C

import numpy as np
import pytest

import chan_lib as CH
import scan_lib as SC
from ltesniffer_b200 import capi

FS = 15360000
CENTER = 1842500000
CELLS = [dict(offset_hz=-3500000, N=512, pci=101, cfo=3000.0, gain_db=0.0), dict(offset_hz=1000000, N=256, pci=202, cfo=-4000.0, gain_db=-10.0),
         dict(offset_hz=4400000, N=128, pci=303, cfo=2500.0, gain_db=-20.0)]


def _plan(fs_in, center_hz, lo=0, hi=0, max_samples=1 << 20):
    return [int(o) for o in capi.scan_plan(capi.scan_cfg(fs_in, 1, center_hz, max_samples, lo, hi))]


@pytest.mark.parametrize("fs_in", [1920000 * 2, 7680000, 15360000, 23040000, 30720000, 61440000, 100000000, 122880000, 245760000])
@pytest.mark.parametrize("center_hz", [1842500000, 2140037000, 2139980000, 751000])
@pytest.mark.parametrize("rng", [(0, 0), (-3000000, 2500000), (500000, 500000), (-100000000, -1000), (7000, 9000)])
def test_plan_is_the_raster(fs_in, center_hz, rng):
    want = SC.plan(fs_in, center_hz, *rng)
    assert _plan(fs_in, center_hz, *rng, max_samples=max(fs_in // 100, 1 << 16)) == want


def test_plan_band_edges():
    # 30.72 Msps reaches 15.36 - 0.54 = 14.82 MHz: a point exactly there is in, 100 kHz further is out
    p = _plan(30720000, 2139980000)
    assert 14820000 in p and 14920000 not in p and -14780000 in p and -14880000 not in p
    assert _plan(30720000, 2139980000, 14820000, 14820000) == [14820000]
    assert _plan(30720000, 2139980000, 14821000, 20000000) == []
    assert len(_plan(100000000, 1850000000)) == 989
    assert p == sorted(p) and all((o + 2139980000) % 100000 == 0 for o in p)


REFUSED = [
    dict(center_hz=1842500500),                    # off the 1 kHz grid
    dict(fs_in=0), dict(fs_in=245760001),          # outside 1 .. 245.76 Msps
    dict(fs_in=1920001),                           # 1.92 MHz / fs_in has L above 1024
    dict(fs_in=1000000),                           # no transition band at N = 128
    dict(lo_hz=1000, hi_hz=-1000),                 # lo > hi
    dict(max_samples=60000),                       # 7 500 N = 128 samples: below a half-frame plus a symbol
    dict(max_samples=0), dict(max_samples=(1 << 31) + 1),
    dict(nof_rx=3), dict(iq_format=7),
]


@pytest.mark.parametrize("bad", REFUSED, ids=lambda d: ",".join("%s=%s" % kv for kv in d.items()))
def test_refusals_need_no_device(phylib, bad):
    kw = dict(fs_in=FS, nof_rx=1, center_hz=CENTER, max_samples=200000)
    kw.update(bad)
    cfg = capi.scan_cfg(**{k: v for k, v in kw.items() if k != "iq_format"})
    if "iq_format" in bad:
        cfg.iq_format = bad["iq_format"]
    capi._bind_scan(phylib)
    n, h = C.c_uint32(), C.c_void_p()
    assert phylib.ltephy_scan_plan(C.byref(cfg), None, 0, C.byref(n)) == -2
    assert phylib.ltephy_scan_create(C.byref(cfg), C.byref(h)) == -2   # INVALID_INPUTS, not the missing device
    assert not h.value


def test_no_point_is_refused_by_create(phylib):
    cfg = capi.scan_cfg(FS, 1, CENTER, 200000, 7200000, 7300000)   # beyond the band check (7.14 MHz)
    capi._bind_scan(phylib)
    n, h = C.c_uint32(), C.c_void_p()
    assert phylib.ltephy_scan_plan(C.byref(cfg), None, 0, C.byref(n)) == 0 and n.value == 0
    assert phylib.ltephy_scan_create(C.byref(cfg), C.byref(h)) == -2


def shortest_capture(fs_in):
    """the fewest capture samples whose N = 128 stream holds a half-frame plus a symbol, from the rational geometry"""
    q = capi.chan_design(fs_in, [(0, 128)], 0)
    # output m needs capture samples up to floor(m M / L) + Kb: the last of HALF_FRAME outputs, m = HALF_FRAME - 1, sets the length
    return (SC.HALF_FRAME - 1) * q["M"] // q["L"] + q["Kb"] + 1


@pytest.mark.parametrize("fs_in", [FS, 23040000, 100000000])
def test_shortest_capture(phylib, fs_in):
    n = shortest_capture(fs_in)
    capi.scan_plan(capi.scan_cfg(fs_in, 1, CENTER, n))
    with pytest.raises(RuntimeError, match="half-frame"):
        capi.scan_plan(capi.scan_cfg(fs_in, 1, CENTER, n - 1))


def three_cells(nrx=1, nsf=11):
    x, _ = CH.compose(FS, CELLS, nsf, nrx=nrx, noise_db=-40.0, seed=3)
    return x


def test_three_cells_each_reported_once():
    x = three_cells()
    offs = SC.plan(FS, CENTER)
    got = SC.reported(offs, SC.points(FS, offs, x))
    assert [(o, c.pci) for o, c in got] == [(c["offset_hz"], c["pci"]) for c in CELLS], [(o, c.pci, c.psr, c.sss_ratio) for o, c in got]
    for (o, c), want in zip(got, CELLS):
        assert abs(c.cfo_hz - want["cfo"]) < 300, (o, c.cfo_hz)


def test_noise_reports_nothing():
    rng = np.random.default_rng(9)
    x = ((rng.standard_normal((1, 170000)) + 1j * rng.standard_normal((1, 170000))) * 0.3).astype(np.complex64)
    offs = SC.plan(FS, CENTER, -1000000, 1000000)
    pts = SC.points(FS, offs, x)
    assert SC.reported(offs, pts) == []


def test_co_channel_cells_both_reported():
    cells = [dict(offset_hz=2000000, N=256, pci=10, cfo=1000.0, gain_db=0.0), dict(offset_hz=2000000, N=256, pci=33, cfo=-2000.0, gain_db=-1.0, lead=5000)]
    x, _ = CH.compose(FS, cells, 12, noise_db=-40.0, seed=5)
    offs = SC.plan(FS, CENTER, 1800000, 2200000)
    got = SC.reported(offs, SC.points(FS, offs, x))
    assert sorted((o, c.pci) for o, c in got) == [(2000000, 10), (2000000, 33)], [(o, c.pci, c.psr, c.sss_ratio) for o, c in got]
