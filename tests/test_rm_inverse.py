"""Turbo rate de-matching through inverse tables (CPU): the per-(K, F) inverse table and the per-rv rotation the library builds reproduce
the forward table (36.212 5.1.4.1 in the pair-buffer layout) exactly, and the per-word rule of rm_turbo_rx_kernel gives the words of the
received-order loop on random int16 soft bits, including repeats, saturation and HARQ combining."""
import numpy as np
import pytest

import rm_ref


def _kf_pairs():
    """every (K, F) a code block can have: F = 0 for every K, and the filler count of the first code block of every byte-aligned TBS"""
    kf = {(K, 0) for K in rm_ref.TURBO_K}
    for tbs in range(16, 110000, 8):
        C_, Kp, Km, Cp, Cm, F = rm_ref.check_tables.segm(tbs)
        kf.add((Km if Cm else Kp, F))
    return sorted(kf)


KF = _kf_pairs()


def test_filler_counts_cover_every_block_size():
    assert len({K for K, _ in KF}) == 188 and max(F for _, F in KF) > 0 and all(F < K for K, F in KF)


@pytest.mark.parametrize("chunk", range(4))
def test_inverse_and_rotation_reproduce_forward_order(phylib, chunk):
    for K, F in KF[chunk::4]:
        NW = (K + 31) // 32
        fill, none = rm_ref.filler_words(K, F), rm_ref.none_words(K)
        for rv in range(4):
            order, nn, inv, rot = rm_ref.tables(phylib, K, F, rv)
            assert nn == 3 * (K + 4) - 2 * F and len(inv) == 96 * NW + 16, (K, F, rv)
            assert len(np.unique(order)) == nn, (K, F, rv)
            k = np.arange(nn)
            assert np.array_equal(inv[order].astype(np.int64), (k + int(rot[rv])) % nn), (K, F, rv)
            missed = np.setdiff1d(np.arange(len(inv)), order)
            assert np.array_equal(np.sort(np.concatenate([fill, none])), missed), (K, F, rv)
            assert np.all(inv[fill] == rm_ref.RM_FILLER) and np.all(inv[none] == rm_ref.RM_NONE), (K, F, rv)
        assert rot[0] == 0 or nn == 0


def _compare(phylib, K, F, rv, E, shift, rng, scale=3000, op=rm_ref.HARQ_NONE, hq=None):
    order, nn, inv, rot = rm_ref.tables(phylib, K, F, rv)
    e = rng.integers(-scale, scale + 1, size=E).astype(np.int16)
    old, hq_old = rm_ref.dematch_per_bit(e, E, order, nn, shift, K, F, op, hq)
    new, hq_new = rm_ref.dematch_words(e, E, inv, nn, int(rot[rv]), shift, op, hq)
    w = np.array(sorted(old))
    assert np.array_equal(new[w], np.array([old[x] for x in w], np.int16)), (K, F, rv, E)
    rest = np.setdiff1d(np.arange(len(inv)), w)
    assert np.all(new[rest] == 0), (K, F, rv, E)      # ragged slots and pad words: nothing received
    if op != rm_ref.HARQ_NONE:
        assert np.array_equal(hq_old, hq_new), (K, F, rv, E)
    return nn, hq_new


@pytest.mark.parametrize("K,F", [(40, 0), (40, 16), (512, 0), (560, 8), (1056, 0), (5824, 0), (6144, 0), (6144, 24)])
@pytest.mark.parametrize("rv", range(4))
def test_word_rule_equals_received_order_loop(phylib, K, F, rv):
    rng = np.random.default_rng(K * 16 + F + rv)
    nn = 3 * (K + 4) - 2 * F
    for E in (nn // 3, nn - 1, nn, nn + 7, int(3.5 * nn)):     # punctured, exact, repeated
        for shift in (0, 1, 2):
            _compare(phylib, K, F, rv, E, shift, rng)
    _compare(phylib, K, F, rv, 5 * nn + 3, 0, rng, scale=32767)   # saturation of the int16 sums


@pytest.mark.parametrize("K,F", [(40, 16), (1056, 0), (6144, 0)])
def test_word_rule_harq_combining(phylib, K, F):
    rng = np.random.default_rng(K + F)
    hq = rng.integers(-30000, 30001, size=rm_ref.HARQ_CB_STRIDE).astype(np.int16)   # non-zero accumulators of earlier transmissions
    nn = 3 * (K + 4) - 2 * F
    _, hq = _compare(phylib, K, F, 0, nn // 2, 1, rng, op=rm_ref.HARQ_NEW, hq=hq)
    for rv, E in ((2, nn // 3), (3, 2 * nn + 5), (1, nn)):
        _, hq = _compare(phylib, K, F, rv, E, 2, rng, scale=20000, op=rm_ref.HARQ_RETX, hq=hq)
    _compare(phylib, K, F, 0, nn // 4, 0, rng, op=rm_ref.HARQ_RETX, hq=rng.integers(-32768, 32768, size=rm_ref.HARQ_CB_STRIDE).astype(np.int16))


def test_bad_block_size_rejected(phylib):
    import ctypes as C
    buf = np.zeros(20000, np.uint32)
    nn = C.c_uint32(0)
    phylib.ltephy_rm_turbo_tables.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.c_void_p, C.c_void_p]
    assert phylib.ltephy_rm_turbo_tables(41, 0, 0, buf.ctypes.data, C.byref(nn), buf.ctypes.data, buf.ctypes.data) == -2
