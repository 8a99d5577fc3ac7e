"""Every kernel shape of the channeliser on the GPU, bit for bit against the oracles (DESIGN.md §2 "channeliser", §4 C1): all 313 integer plans,
a rational set chosen by (L, M, Kp, R) from the plan space (every R from 3 to 31, the R >= 32 values, L = M = 1, the boundary plans of the limits
and the largest rotation period P), sc16 / sc8 at full scale, 8 carriers on 2 antennas (16 segments) with calls where some carriers have no
outputs; and capture positions past 2^31 and 2^32: bit for bit against the oracle, a stream of calls that crosses 2^32 through next_sample,
and the outputs of a capture placed at F >= 2^32 equal to those at 0, shifted by F L / M."""
import math

import numpy as np
import pytest

import chan_lib as CH
import chan_rational_lib as R
from test_chan import _signal
from test_chan_plan_space import BOUNDARY
from test_gpu_chan import _same

pytestmark = pytest.mark.gpu

MAX_FS = 245760000


def _host(outs):
    return [dict(first=o["first"], iq=o["iq"].cpu().numpy()) for o in outs]


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _samples(d):
    """a capture long enough for two full tiles of L R outputs and a partial third, whatever the outputs lost to the window"""
    R_ = R.tile_rows(d["L"], d["M"], d["Kp"])
    return (5 * R_ * d["M"]) // 2 + d["Kp"] + d["M"] + 7


def _full_scale(n, nrx, fmt, seed):
    """interleaved int16 / int8 [nrx][2n], half the values at the extremes -32768 / 32767 or -128 / 127, the rest uniform"""
    lo, hi, dt = (-32768, 32767, np.int16) if fmt == "sc16" else (-128, 127, np.int8)
    rng = np.random.default_rng(seed)
    q = rng.integers(lo, hi + 1, (nrx, 2 * n))
    m = rng.random(q.shape) < 0.5
    q[m] = rng.choice([lo, hi], int(m.sum()))
    return np.ascontiguousarray(q.astype(dt))


@pytest.mark.parametrize("N", CH.SYMBOL_SIZES)
def test_every_integer_plan(phylib, N):
    """D = 2..128 up to 245.76 MHz, one and two antennas in turn, an offset that walks across the band: the integer oracle's bytes and
    next_sample, host input, on captures of two full tiles and a partial one"""
    from ltesniffer_b200 import capi
    plans = 0
    for D in range(2, 129):
        fs = 15000 * N * D
        if fs > MAX_FS:
            break
        T_, _, _, f_pass = CH.geometry(fs, 0, N)
        amax = (fs // 2 - f_pass) // 1000 * 1000
        off = [0, amax, -amax, 1000, -(amax // 3000) * 1000][D % 5]
        nrx = 1 + D % 2
        d = dict(L=1, M=D, Kp=T_)
        n = _samples(d)
        x = _signal(n, nrx, fs, N + D)
        ref, nxt = CH.run(fs, [(off, N)], x, 0)
        assert ref[0]["count"] > 2 * R.tile_rows(1, D, T_), (fs, ref[0]["count"])
        ch = capi.Channelizer(fs, [(off, N)], nrx, n)
        got, nxt_g = ch.run(x, 0)
        ch.close()
        assert nxt_g == nxt, (fs, off)
        _same(ref, _host(got))
        plans += 1
    assert plans == len([D for D in range(2, 129) if 15000 * N * D <= MAX_FS])


def _rational_set():
    """(fs, offset, N) chosen by (L, M, Kp, R) from the plan space at offset 0: for each R below 32 and each R from 32 up at L > 1, the plan with
    the largest phase table L Kp; L = M = 1; the boundary plans; and N 2048 at 1 kHz, the largest rotation period P = 30 720"""
    space = R.plan_space()
    best = {}
    for d in space:
        if d["L"] == 1 and d["M"] > 1:
            continue                                 # integer plans: test_every_integer_plan
        key = d["R"]
        if key not in best or d["L"] * d["Kp"] > best[key]["L"] * best[key]["Kp"]:
            best[key] = d
    assert set(range(3, 32)) <= set(best), sorted(best)
    plans = [(d["fs"], 0, d["N"]) for _, d in sorted(best.items())]
    plans += [(d["fs"], 0, d["N"]) for d in space if d["L"] == 1 and d["M"] == 1]
    plans += [(fs, 0, N) for fs, N, _, _ in BOUNDARY]
    plans += [(20000000, 1000, 2048)]
    return sorted(set(plans))


_RSET = None


def _rset():
    global _RSET
    if _RSET is None:
        _RSET = _rational_set()
    return _RSET


def _check_rational(capi, fs, off, N, fmt, nrx, seed, device=False):
    d = R.design(fs, off, N)
    n = _samples(d)
    if fmt == "cf32":
        q = _signal(n, nrx, fs, seed)
    else:
        q = _full_scale(n, nrx, fmt, seed)
    ref, nxt = R.run(fs, [(off, N)], q, 0, fmt)
    assert ref[0]["count"] >= 2 * d["L"] * R.tile_rows(d["L"], d["M"], d["Kp"]), (fs, N, ref[0]["count"])
    ch = capi.Channelizer(fs, [(off, N)], nrx, n, rational=True, iq_format=fmt)
    got, nxt_g = ch.run_device(_dev(q), 0) if device else ch.run(q, 0)
    ch.close()
    assert nxt_g == nxt, (fs, off, N, fmt)
    _same(ref, _host(got))


def test_rational_set(phylib):
    """the rational set in cf32, one and two antennas in turn, host and device input in turn"""
    from ltesniffer_b200 import capi
    plans = _rset()
    assert len(plans) >= 29 + 5 + 2
    for i, (fs, off, N) in enumerate(plans):
        _check_rational(capi, fs, off, N, "cf32", 1 + i % 2, 100 + i, device=bool(i // 2 % 2))
    P = max(R.design(fs, off, N)["P"] for fs, off, N in plans)
    assert P == 30720


@pytest.mark.parametrize("fmt", ["sc16", "sc8"])
def test_integer_samples_at_full_scale(phylib, fmt):
    """every fourth plan of the rational set and four integer plans, on samples half of which sit at the extremes of the format"""
    from ltesniffer_b200 import capi
    plans = _rset()[::4] + [(30720000, -7500000, 1024), (245760000, 99999000, 128), (61440000, 0, 2048), (3840000, 0, 128)]
    for i, (fs, off, N) in enumerate(plans):
        _check_rational(capi, fs, off, N, fmt, 2 - i % 2, 300 + i, device=bool(i % 3 == 0))


# 8 carriers of a 30.72 Msps capture: integer D = 2 / 4 / 8 / 16 and rational 3 / 4, 1 / 1, 3 / 8 and 3 / 16, each with its own tile shape
EIGHT = (30720000, [(-7500000, 1024), (5000000, 512), (11000000, 256), (-12000000, 128), (1000000, 1536), (0, 2048), (3000000, 768),
                    (-4000000, 384)])


def test_eight_carriers_on_two_antennas(phylib):
    """16 segments in one launch: one call of the whole capture, then calls too short for some carriers' windows (those have no outputs, and
    the segments of the others follow them), each equal to the oracle's bytes and next_sample"""
    from ltesniffer_b200 import capi
    fs, carriers = EIGHT
    n = 24000
    x = _signal(n, 2, fs, 21)
    ch = capi.Channelizer(fs, carriers, 2, n, rational=True)
    ref, nxt = R.run(fs, carriers, x, 0)
    got, nxt_g = ch.run(x, 0)
    assert nxt_g == nxt and all(r["count"] > 0 for r in ref)
    _same(ref, _host(got))
    for first, cnt in ((0, 40), (9001, 60), (12345, 100), (20000, 45)):
        xx = x[:, first:first + cnt]
        ref, nxt = R.run(fs, carriers, xx, first)
        counts = [r["count"] for r in ref]
        assert 0 in counts and any(counts), counts
        got, nxt_g = ch.run_device(_dev(xx), first)
        assert nxt_g == nxt, (first, cnt)
        _same(ref, _host(got))
    ch.close()


# ---- positions past 2^31 and 2^32 ---------------------------------------------------------------------------------------------------------
FIRSTS = [(1 << 31) - 12345, (1 << 32) - 12345, (1 << 32) + 4097, (1 << 40) + 65537]
LONG_PLANS = [  # fs_in, carriers, nof_rx, samples: integer and rational carriers
    (30720000, [(-7500000, 1024), (3000000, 1536), (9000000, 256)], 2, 30000),
    (25000000, [(-6000000, 1024), (5000000, 512)], 1, 30000),
    (245760000, [(-101377000, 256), (99999000, 128)], 1, 40000),
]


@pytest.mark.parametrize("first", FIRSTS)
@pytest.mark.parametrize("plan", range(len(LONG_PLANS)))
def test_positions_past_2_32(phylib, plan, first):
    """capture samples first .. first + n: the oracle's bytes, output indices and next_sample, host and device input"""
    from ltesniffer_b200 import capi
    fs, carriers, nrx, n = LONG_PLANS[plan]
    x = _signal(n, nrx, fs, 31 + plan)
    ref, nxt = R.run(fs, carriers, x, first)
    assert all(r["count"] > 0 and r["first"] > 0 for r in ref)
    ch = capi.Channelizer(fs, carriers, nrx, n, rational=True)
    got, nxt_g = ch.run(x, first)
    assert nxt_g == nxt and nxt > first
    _same(ref, _host(got))
    got, nxt_g = ch.run_device(_dev(x), first)
    assert nxt_g == nxt
    _same(ref, _host(got))
    ch.close()


def test_stream_across_2_32(phylib):
    """a stream of calls from 2^32 - 20 000, each re-fed from next_sample, crosses 2^32: the one-call oracle's bytes and next_sample"""
    from ltesniffer_b200 import capi
    fs, carriers, nrx, _ = LONG_PLANS[0]
    first = (1 << 32) - 20000
    x = _signal(45000, nrx, fs, 41)
    ref, nxt = R.run(fs, carriers, x, first)
    ch = capi.Channelizer(fs, carriers, nrx, x.shape[1], rational=True)
    got, nexts = CH.stream(lambda xx, f: ch.run(xx, f), x, [7919, 3001, 8999], first=first)
    ch.close()
    assert nexts[-1] == nxt and any(v < (1 << 32) for v in nexts) and any(v > (1 << 32) for v in nexts)
    _same(ref, got)


def _shift(fs, carriers):
    """F: the smallest multiple >= 2^32 of M lcm(L, P) over every carrier, so that F L / M is a whole number of outputs, a multiple of L (the
    phase phi of every output is kept) and of P (its rotation is kept)"""
    step = 1
    for off, N in carriers:
        d = R.design(fs, off, N)
        step = math.lcm(step, d["M"] * math.lcm(d["L"], d["P"]))
    return -(-(1 << 32) // step) * step


@pytest.mark.parametrize("plan", range(len(LONG_PLANS)))
def test_shift_identity(phylib, plan):
    """the same samples at F and at 0: past the zero-padded head of the run at 0, every output equals the one at F byte for byte, its index
    moved by F L / M; next_sample moves by F"""
    from ltesniffer_b200 import capi
    fs, carriers, nrx, n = LONG_PLANS[plan]
    F = _shift(fs, carriers)
    assert F >= 1 << 32
    x = _signal(n, nrx, fs, 51 + plan)
    ch = capi.Channelizer(fs, carriers, nrx, n, rational=True)
    a, na = ch.run(x, 0)
    a = _host(a)
    for run in (lambda: ch.run(x, F), lambda: ch.run_device(_dev(x), F)):
        b, nb = run()
        b = _host(b)
        assert nb == na + F
        for (off, N), u, v in zip(carriers, a, b):
            d = R.design(fs, off, N)
            s = F * d["L"] // d["M"]
            assert v["first"] >= s and u["first"] == 0
            k = v["first"] - s                      # outputs of the run at 0 whose window reaches before sample 0
            assert k == -(-d["Ka"] * d["L"] // d["M"]) and v["iq"].shape[1] == u["iq"].shape[1] - k
            assert v["iq"].tobytes() == np.ascontiguousarray(u["iq"][:, k:]).tobytes(), (off, N)
    ch.close()
