"""The tracker at capture positions past 2^32 on the GPU (DESIGN.md §2 "tracking"): a DL tracker, and a DL + UL tracker that re-acquires the
cell after one drop (ltephy_track_set_ul, LTEPHY_TRACK_REACQUIRE), started at frame_offset F + fo with 2^32 inside a push and inside a subframe.
Their records equal those of the same capture at fo with start and tau moved by exactly F and every other field identical, their DL and UL cuts
are the same bytes, and they equal the oracle lteo_track at F bit for bit through host and device pushes.  A 30.72 Msps recording passes sample
2^32 after 140 s."""
import numpy as np
import pytest

import track_lib as T
import track_reacq_lib as Q
import track_ul_lib as U
from test_track_reacquire import PCI, T0, drop_capture

pytestmark = pytest.mark.gpu

TWO32 = 1 << 32


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _moved(a, b, F, keys=("iq",)):
    """b is a moved by F: sf.start and hf.tau + F, all else and the cuts byte for byte"""
    sa, ha = a["sf"].copy(), a["hf"].copy()
    assert len(sa) == len(b["sf"]) and len(ha) == len(b["hf"])
    sa["start"] += F
    ha["tau"] += F
    assert sa.tobytes() == b["sf"].tobytes()
    assert ha.tobytes() == b["hf"].tobytes()
    for k in keys:
        assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k


def _same(a, b, keys=("iq",)):
    assert a["sf"].tobytes() == b["sf"].tobytes() and a["hf"].tobytes() == b["hf"].tobytes()
    for k in keys:
        assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k


def _spans():
    """a push wrapper that records the absolute range [first, first + n) of each push"""
    seen = []

    def wrap(push):
        def f(*args):   # (x, first) or (x, x_ul, first)
            seen.append((args[-1], args[-1] + args[0].shape[-1]))
            return push(*args)
        return f
    return seen, wrap


def test_dl_tracker_past_2_32(phylib):
    from ltesniffer_b200 import capi
    N, A, fo = 512, 2, 500
    SF, FR = 15 * N, 150 * N
    x, _, _ = T.capture(N, 100, 120, nrx=A, ppm=20.0, cfo=900.0, snr=20.0, lead=fo, seed=3)
    F = TWO32 - (fo + 37 * SF + SF // 2)
    sizes = [FR + N + 1, 7919, 3 * SF + 17]
    mk = lambda off: capi.Tracker(N, A, 100, off, cfo_hz=900.0, max_subframes=300)
    tr = mk(fo)
    a = T.run_chunks(tr, x, sizes)
    tr.close()
    assert len(a["sf"]) >= 110 and not (a["sf"]["flags"] & capi.TRACK_LOST).any()
    o = T.run_chunks(T.Oracle(N, A, 100, F + fo, cfo_hz=900.0), x, sizes, first=F)
    for device in (False, True):
        tr = mk(F + fo)
        seen, wrap = _spans()
        push = wrap(lambda xx, s: tr.push_device(_dev(xx), s)) if device else wrap(tr.push)
        b = T.run_chunks(tr, x, sizes, first=F, push=push)
        tr.close()
        assert any(s < TWO32 < e for s, e in seen), seen
        assert any(s < TWO32 < s + SF for s in b["sf"]["start"].tolist())
        _moved(a, b, F)
        _same(o, b)


def test_dl_ul_tracker_with_a_drop_past_2_32(phylib):
    from ltesniffer_b200 import capi
    N, off, rho = 384, -(3 * 384 + 5), 0.95
    SF = 15 * N
    x, _, _, _, lead = drop_capture(N, 1, 20.0, "37SF+1234")
    xu = Q.noise(np.random.default_rng(5), 1, x.shape[1], 1.0)[0]
    F = TWO32 - (lead + 70 * SF + SF // 3)      # after the drop and the find
    sizes = [15 * N * 150 + N + 1, 7919]
    mk = lambda fo: capi.Tracker(N, 1, PCI, fo, cfo_hz=900.0, first_tti=T0, flags=capi.TRACK_REACQUIRE, max_subframes=300,
                                 ul=dict(cfo_ratio=rho, ul_offset=off))
    tr = mk(lead)
    a = U.run_chunks_ul(tr, x, xu, sizes)
    tr.close()
    assert ((a["sf"]["flags"] & capi.TRACK_REACQUIRED) != 0).sum() == 1
    o = U.run_chunks_ul(U.OracleUl(N, 1, PCI, F + lead, cfo_hz=900.0, first_tti=T0, flags=Q.REACQUIRE, cfo_ratio=rho, ul_offset=off), x, xu, sizes,
                        first=F)
    for device in (False, True):
        tr = mk(F + lead)
        seen, wrap = _spans()
        push = wrap(lambda xx, xxu, s: tr.push_ul_device(_dev(xx), _dev(xxu), s)) if device else wrap(tr.push_ul)
        b = U.run_chunks_ul(tr, x, xu, sizes, first=F, push=push)
        tr.close()
        assert any(s < TWO32 < e for s, e in seen), seen
        assert any(s < TWO32 < s + SF for s in b["sf"]["start"].tolist())
        _moved(a, b, F, keys=("iq", "ul_iq"))
        _same(o, b, keys=("iq", "ul_iq"))
