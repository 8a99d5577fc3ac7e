"""Channeliser outputs at capture positions past 2^31, 2^32 and 2^40 on the CPU (DESIGN.md §2 "channeliser"): the oracles lteo_chan_run /
lteo_chan_run_poly against a float64 restatement of the rule whose output, phase and rotation indices are exact Python integers, for integer and
rational carriers.  A 245.76 Msps recording passes sample 2^32 after 17.5 s."""
import numpy as np
import pytest

import chan_lib as CH
import chan_rational_lib as R
from test_chan import _signal

FIRSTS = [(1 << 31) - 12345, (1 << 32) - 12345, (1 << 32) + 4097, (1 << 40) + 65537]
PLANS = [  # fs_in, carriers, nof_rx, samples
    (30720000, [(-7500000, 1024), (3000000, 1536), (9000000, 256)], 2, 20000),
    (25000000, [(-6000000, 1024), (5000000, 512)], 1, 20000),
    (245760000, [(-101377000, 256), (99999000, 128)], 1, 30000),
]


def _reference(fs, off, N, x, first, ms):
    """float64 outputs ms (Python ints) of a carrier from x complex [n], capture samples first ..; n = m M // L, phi = m M mod L and the rotation
    index (offset m) mod fs_out in exact integers, the tables' float prototype hp"""
    d = R.design(fs, off, N)
    hp = d["hp"].astype(np.float64)
    L, M, Tp, Ka, Kb = d["L"], d["M"], d["Tp"], d["Ka"], d["Kb"]
    Hp, fo = (Tp - 1) // 2, 15000 * N
    n = np.array([m * M // L - first for m in ms], np.int64)           # relative to the call
    ph = np.array([m * M % L for m in ms], np.int64)
    rph = -2 * np.pi * np.array([(off * m) % fo for m in ms], np.float64) / fo
    k = np.arange(-Kb, Ka + 1)
    idx = Hp + ph[:, None] + L * k[None, :]
    tap = np.where((idx >= 0) & (idx < Tp), hp[np.clip(idx, 0, Tp - 1)], 0.0)
    s = n[:, None] - k[None, :]
    assert (s >= 0).all() and (s < len(x)).all()
    gph = 2 * np.pi * ((off * (ph[:, None] + L * k[None, :])) % (L * fs)) / (L * fs)
    return np.exp(1j * rph) * (tap * np.exp(1j * gph) * np.asarray(x, np.complex128)[s]).sum(axis=1)


@pytest.mark.parametrize("first", FIRSTS)
@pytest.mark.parametrize("plan", range(len(PLANS)))
def test_oracle_against_float64_past_2_32(plan, first):
    """every output of the call within 2e-5 of the RMS of the float64 rule; the call's range and next_sample from exact integers; an integer
    carrier's outputs from lteo_chan_run equal lteo_chan_run_poly's"""
    fs, carriers, nrx, n = PLANS[plan]
    x = _signal(n, nrx, fs, 61 + plan)
    outs, nxt = R.run(fs, carriers, x, first)
    needs = []
    for (off, N), o in zip(carriers, outs):
        d = R.design(fs, off, N)
        L, M, Ka, Kb = d["L"], d["M"], d["Ka"], d["Kb"]
        assert o["first"] == -(-(first + Ka) * L // M) and o["count"] > 100
        last = o["first"] + o["count"] - 1
        assert last * M // L + Kb <= first + n - 1 < (last + 1) * M // L + Kb
        needs.append((last + 1) * M // L - Ka)
        ms = [o["first"] + i for i in range(o["count"])]
        for a in range(nrx):
            ref = _reference(fs, off, N, x[a], first, ms)
            rms = np.sqrt(np.mean(np.abs(ref) ** 2))
            err = np.abs(o["iq"][a].astype(np.complex128) - ref).max()
            assert err <= 2e-5 * rms, (off, N, err / rms)
    assert nxt == min(needs)
    ints = [c for c in carriers if CH.geometry(fs, c[0], c[1]) is not None]
    if ints:
        ref, nref = CH.run(fs, ints, x, first)
        for c, r in zip(ints, ref):
            o = outs[carriers.index(c)]
            assert r["first"] == o["first"] and r["iq"].tobytes() == o["iq"].tobytes()
