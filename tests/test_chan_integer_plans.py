"""Every integer carrier the channeliser accepts, on the CPU (DESIGN.md §2 "channeliser"): for each symbol size N, each decimation D = 2..128 with
15 kHz · N · D <= 245.76 MHz and offsets across the band, ltephy_chan_taps and ltephy_chan_design (with and without LTEPHY_CHAN_RATIONAL) equal
lteo_chan_design bit for bit, and ltephy_chan_design describes the carrier as L = 1, M = D, Kp = Tp = T, Ka = Kb = H.  The rotation table pins
the integer rule's reduction of the angle over fs_in, which differs from a reduction over fs_out in the last bit whenever D is not a power of 2."""
import numpy as np
import pytest

import chan_lib as CH

MAX_FS = 245760000


def _offsets(fs, N):
    """offsets on the 1 kHz grid from 0 to the band edge, both signs"""
    amax = (fs // 2 - 90000 * CH.MAX_PRB[N]) // 1000 * 1000
    return sorted({o for o in (0, 1000, -7000, 5000000, amax // 3000 * 1000, -amax // 7000 * 3000, -amax, amax) if abs(o) <= amax})


@pytest.mark.parametrize("N", CH.SYMBOL_SIZES)
def test_integer_plans_equal_the_oracle(phylib, N):
    from ltesniffer_b200 import capi
    plans = 0
    for D in range(2, 129):
        fs = 15000 * N * D
        if fs > MAX_FS:
            break
        for off in _offsets(fs, N):
            o = CH.design(fs, off, N)
            t = capi.chan_taps(fs, [(off, N)], 0)
            assert (t["T"], t["D"], t["P"]) == (o["T"], o["D"], o["P"]) and o["D"] == D, (fs, off)
            for k in ("h", "g", "rot"):
                assert t[k].tobytes() == o[k].tobytes(), (fs, off, k)
            for rational in (False, True):
                d = capi.chan_design(fs, [(off, N)], 0, rational=rational)
                H = o["T"] // 2
                assert (d["L"], d["M"], d["Tp"], d["Kp"], d["Ka"], d["Kb"], d["P"]) == (1, D, o["T"], o["T"], H, H, o["P"]), (fs, off, rational)
                assert d["hp"].tobytes() == o["h"].tobytes() and d["g"][0].tobytes() == o["g"].tobytes(), (fs, off, rational)
                assert d["rot"].tobytes() == o["rot"].tobytes(), (fs, off, rational)
            plans += 1
    assert plans >= 3 * len([D for D in range(2, 129) if 15000 * N * D <= MAX_FS])


def test_rotation_reduced_over_fs_in(phylib):
    """23.04 Msps, N 512 (D 3), offset 5 MHz: r[48] has the angle -pi/2, and its real part is the rounding of cos(-2 pi (3 offset 48 mod fs_in) /
    fs_in), not of cos(-2 pi (offset 48 mod fs_out) / fs_out)"""
    from ltesniffer_b200 import capi
    t = capi.chan_taps(23040000, [(5000000, 512)], 0)
    d = capi.chan_design(23040000, [(5000000, 512)], 0)
    assert t["P"] == d["P"] == 192
    for r in (t["rot"], d["rot"]):
        assert r[48].real == np.float32(float.fromhex("-0x1.72cecep-53")) and r[48].imag == np.float32(-1.0)
