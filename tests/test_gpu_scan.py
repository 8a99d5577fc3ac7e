"""The raster scan on the GPU: every point's three results equal the oracle's (lteo_chan_run_poly then lteo_cell_search) on a subset of points and
the per-point composition through the public API (ltephy_chan_run_device with the one carrier, then ltephy_cell_search_device) on every point,
bit for bit; the reported cells are the rule applied to them; and nothing changes with max_points_per_pass, host or device input, sc16 / sc8
against cf32 of the same values, or the antenna count (each against its own composition)."""
import numpy as np
import pytest

import chan_rational_lib as CR
import scan_lib as SC
from ltesniffer_b200 import capi
from test_scan import CELLS, CENTER, FS, three_cells

pytestmark = pytest.mark.gpu


def _b(c):
    return bytes(c)


def composition(fs_in, offsets, x, fmt="cf32"):
    """per point: the channeliser's one-carrier stream, then the cell search of it, through the public API"""
    import torch
    nrx = x.shape[0]
    n = x.shape[1] if fmt == "cf32" else x.shape[1] // 2
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    out = []
    for o in offsets:
        ch = capi.Channelizer(fs_in, [(int(o), 128)], nrx, n, rational=True, iq_format=fmt)
        res, _ = ch.run_device(xd, 0, copy=False)
        cs = capi.CellSearch(128, nrx, res[0]["count"])
        out.append(cs.search_device(res[0]["iq"]))
        cs.close()
        ch.close()
    return out


@pytest.fixture(scope="module")
def capture():
    x = three_cells(nrx=2)
    sc = capi.Scanner(FS, 2, CENTER, x.shape[1])
    got = sc.run(x)
    return x, sc, got, sc.points()


def test_points_equal_the_composition_and_the_oracle(capture):
    x, sc, got, pts = capture
    offs = sc.plan()
    assert list(offs) == SC.plan(FS, CENTER)
    comp = composition(FS, offs, x)
    for o, a, b in zip(offs, pts, comp):
        assert [_b(c) for c in a] == [_b(c) for c in b], o
    subset = sorted(set([c["offset_hz"] for c in CELLS] + [int(o) for o in offs[::25]] + [int(offs[-1])]))
    for o in subset:
        p = list(offs).index(o)
        assert [_b(c) for c in pts[p]] == [_b(c) for c in SC.point(FS, o, x)], o


def test_reported_is_the_rule(capture):
    x, sc, got, pts = capture
    want = SC.reported(list(sc.plan()), pts)
    assert [(o, _b(c)) for o, c in got] == [(o, _b(c)) for o, c in want]
    assert [(o, c.pci) for o, c in got] == [(c["offset_hz"], c["pci"]) for c in CELLS]


@pytest.mark.parametrize("per_pass", [1, 7, 0])
def test_points_per_pass_and_device_input(capture, per_pass):
    import torch
    x, sc, got, pts = capture
    s2 = capi.Scanner(FS, 2, CENTER, x.shape[1], max_points_per_pass=per_pass)
    g2 = s2.run_device(torch.from_numpy(x).cuda())
    assert [(o, _b(c)) for o, c in g2] == [(o, _b(c)) for o, c in got]
    assert [[_b(c) for c in p] for p in s2.points()] == [[_b(c) for c in p] for p in pts]
    s2.close()


@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
def test_integer_samples_equal_cf32_of_their_values(capture, fmt):
    x = capture[0]
    q, exact = CR.to_format(x / (2.5 * np.abs(x).max()), fmt)
    si = capi.Scanner(FS, 2, CENTER, x.shape[1], iq_format=fmt, max_points_per_pass=40)
    sf = capi.Scanner(FS, 2, CENTER, x.shape[1])
    gi, gf = si.run(q), sf.run(exact)
    assert [(o, _b(c)) for o, c in gi] == [(o, _b(c)) for o, c in gf]
    assert [[_b(c) for c in p] for p in si.points()] == [[_b(c) for c in p] for p in sf.points()]
    assert [(o, c.pci) for o, c in gi] == [(c["offset_hz"], c["pci"]) for c in CELLS]


def test_one_antenna(capture):
    x = np.ascontiguousarray(capture[0][:1])
    lo, hi = 800000, 4600000
    sc = capi.Scanner(FS, 1, CENTER, x.shape[1], lo_hz=lo, hi_hz=hi)
    got = sc.run(x)
    offs = sc.plan()
    assert list(offs) == SC.plan(FS, CENTER, lo, hi)
    pts = sc.points()
    for o, a, b in zip(offs, pts, composition(FS, offs, x)):
        assert [_b(c) for c in a] == [_b(c) for c in b], o
    assert [(o, c.pci) for o, c in got] == [(c["offset_hz"], c["pci"]) for c in CELLS[1:]]


def test_rational_rate():
    """20 Msps (1.92 MHz / 20 MHz = 12 / 125, a rational carrier at every point): the scan equals the per-point composition at every point and
    finds the cell"""
    import scipy.signal as ss
    import chan_lib as CH
    fs = 20000000
    x15, _ = CH.compose(FS, [dict(offset_hz=-2000000, N=256, pci=77, cfo=1500.0, gain_db=0.0)], 11, nrx=1, noise_db=-40.0, seed=4)
    x = ss.resample_poly(x15.astype(np.complex128), 125, 96, axis=1).astype(np.complex64)
    sc = capi.Scanner(fs, 1, CENTER, x.shape[1], lo_hz=-2500000, hi_hz=-1500000)
    got = sc.run(x)
    offs = sc.plan()
    for o, a, b in zip(offs, sc.points(), composition(fs, offs, x)):
        assert [_b(c) for c in a] == [_b(c) for c in b], o
    assert [(o, c.pci) for o, c in got] == [(-2000000, 77)]


def test_short_capture_is_refused_on_a_live_handle(capture):
    x, sc = capture[0], capture[1]
    with pytest.raises(RuntimeError, match="half-frame"):
        sc.run(x[:, :20000])


def test_integer_rate_with_large_decimation():
    """245.76 Msps: D = 128 and T = 1 265 at every point, the taps in shared memory.  A short capture with one cell, scanned over an offset range
    around it: the scan equals the per-point composition at every point and finds the cell"""
    import chan_lib as CH
    fs = 245760000
    x, _ = CH.compose(fs, [dict(offset_hz=-30000000, N=256, pci=150, cfo=-2500.0, gain_db=0.0)], 11, nrx=2, noise_db=-40.0, seed=6)
    sc = capi.Scanner(fs, 2, CENTER, x.shape[1], lo_hz=-30400000, hi_hz=-29600000, max_points_per_pass=4)
    got = sc.run(x)
    offs = sc.plan()
    assert list(offs) == SC.plan(fs, CENTER, -30400000, -29600000)
    for o, a, b in zip(offs, sc.points(), composition(fs, offs, x)):
        assert [_b(c) for c in a] == [_b(c) for c in b], o
    assert [(o, c.pci) for o, c in got] == [(-30000000, 150)]


def test_decode_wideband_scan_mode(phylib, infra, tmp_path):
    """decode_wideband scan=<center_hz> on a capture of a 25-PRB and a 15-PRB cell with a MIB and a 6-PRB cell without one: one scan line per
    cell, the 6-PRB cell listed and not decoded, the others decoded at the smallest N that covers their PRB count (384 and 256), and each
    carrier's pcap and DCI trace byte-identical to those of the carrier-list invocation with the same carriers"""
    import os
    import subprocess
    import chan_lib as CH
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run(["make", "-s", "-C", root, "examples/decode_wideband"], check=True)
    fs, A, B, nsf, center = 30720000, 2, 100, 120, 2140000000
    spec = [dict(offset_hz=-7500000, N=512, pci=101, cfo=900.0, lead=3000, gain_db=0.0, decode=True),
            dict(offset_hz=3000000, N=256, pci=257, cfo=-1700.0, lead=777, gain_db=-10.0, decode=True),
            dict(offset_hz=11000000, N=128, pci=44, cfo=300.0, lead=2500, gain_db=0.0)]
    x, _ = CH.compose(fs, spec, nsf, nrx=A, noise_db=-35.0, seed=2)
    f = tmp_path / "wide.cf32"
    x.tofile(str(f))
    exe = os.path.join(root, "examples", "decode_wideband")
    rs = subprocess.run([exe, str(f), str(fs), str(A), str(tmp_path / "s"), "scan=%d" % center, str(B)], capture_output=True, text=True)
    assert rs.returncode == 0, rs.stdout + rs.stderr
    lines = [ln.split() for ln in rs.stdout.splitlines() if ln.startswith("scan ")]
    assert [(int(ln[2]), int(ln[4])) for ln in lines] == [(c["offset_hz"], c["pci"]) for c in spec], rs.stdout
    assert lines[0][-4:] == ["carrier", "0", "symbol_sz", "384"] and lines[1][-4:] == ["carrier", "1", "symbol_sz", "256"], rs.stdout
    assert "not decoded" in " ".join(lines[2]), rs.stdout
    rl = subprocess.run([exe, str(f), str(fs), str(A), str(tmp_path / "l"), "-7500000:384", "3000000:256", str(B)], capture_output=True, text=True)
    assert rl.returncode == 0, rl.stdout + rl.stderr
    assert [ln for ln in rs.stdout.splitlines() if not ln.startswith("scan ")] == rl.stdout.splitlines()
    for c in range(2):
        for ext in ("pcap", "tsv"):
            a, b = (tmp_path / ("s_%d.%s" % (c, ext))).read_bytes(), (tmp_path / ("l_%d.%s" % (c, ext))).read_bytes()
            assert a == b, (c, ext)
        assert len((tmp_path / ("s_%d.pcap" % c)).read_bytes()) > 1000, c
