"""The batches of tests/test_gpu_pool_offsets.py, checked without a GPU: from the documented pool layouts alone -- (G + 7) & ~7 soft bits per
codeword, E_r soft bits per code block, 96 * ceil(K / 32) + 16 words per turbo pair in the order ltephy_turbo_pairing returns, and
LTEPHY_HARQ_SLOT_BYTES per HARQ slot -- every region a real transport block writes or reads is placed, once with 64-bit offsets and once with the
offsets truncated to 32 bits.  With 64 bits no two real transport blocks share an element; with 32 bits each case makes one real transport block
land on another, so the GPU tests fail on a library whose descriptors keep 32-bit pool offsets."""
import numpy as np

import ref_dec
import rm_ref
import test_gpu_pool_offsets as P
from test_gpu_dense_pairs import _pairing
from ltesniffer_b200 import capi


def clash(regions, bits):
    """regions: (tag, start, length); True if two regions of different tags overlap once every start is taken mod 2^bits"""
    r = [(t, s % (1 << bits), n) for t, s, n in regions]
    return any(a[0] != b[0] and a[1] < b[1] + b[2] and b[1] < a[1] + a[2] for i, a in enumerate(r) for b in r[i + 1:])


def soft_bit_regions(layout):
    """each real transport block: the codeword the demapper writes (from the grant's offset) and the code blocks the rate de-matcher reads (from
    each code block's own offset)"""
    grants, idx, off, G, E = layout
    out = []
    for k, i in enumerate(idx):
        out.append((k, int(off[i]), G))
        out += [(k, int(off[i]) + sum(E[:r]), E[r]) for r in range(len(E))]
    return out


def check_soft_bits(layout):
    grants, idx, off, G, E = layout
    t1, t2 = int(off[idx[1]]), int(off[idx[2]])
    assert t1 < P.WRAP <= t1 + sum(E[:-1])                 # T1: the grant's offset fits 32 bits, its last code block's does not
    assert P.WRAP <= t2 and t2 - P.WRAP < P.cw_len(G)       # T2: wholly past 2^32, congruent to a point inside T0
    regions = soft_bit_regions(layout)
    assert not clash(regions, 64)
    assert clash(regions, 32)


def test_downlink_soft_bit_layout_wraps_onto_a_real_block():
    check_soft_bits(P.a_layout())


def test_uplink_soft_bit_layout_wraps_onto_a_real_block():
    check_soft_bits(P.b_layout())


def test_turbo_pool_layout_wraps_onto_another_block(phylib):
    grants, G = P.c_layout()
    Cn, Ks, F = ref_dec.segmentation(P.C_TBS)
    assert (Cn, set(Ks), F) == (16, {6144}, 0)
    ncb = Cn * len(grants)
    pair, half, npairs = _pairing(phylib, np.full(ncb, 6144), np.full(ncb, P.C_TBS), np.full(ncb, G))
    cb = np.arange(ncb)
    assert npairs == ncb // 2 and np.array_equal(pair, cb // 2) and np.array_equal(half, cb % 2)   # equal rate: submission order
    pw = rm_ref.pair_words(6144)
    assert pw == 18448 and npairs * pw > P.WRAP
    content = (cb[::2] // Cn) % len(P.C_TTI)               # the transmitted subframe of each pair's transport block
    for bits in (64, 32):
        start = np.arange(npairs, dtype=np.int64) * pw
        if bits == 32:
            start &= 0xFFFFFFFF
        o = np.argsort(start, kind="stable")
        s, t = start[o], content[o]
        over = (s[1:] < s[:-1] + pw) & (t[1:] != t[:-1])   # equal lengths: an overlap of two tags shows between neighbours in start order
        assert over.any() == (bits == 32), bits


def test_harq_layout_wraps_onto_the_other_block():
    G, tbs = P.d_tbs()
    Cn, Ks, F = ref_dec.segmentation(tbs)
    assert 2 <= Cn <= 16 and capi.HARQ_SLOT_BYTES // 2 == rm_ref.HARQ_SLOT_ELEMS
    b1, b2 = P.d_grants(P.D_SLOTS - 1)
    slots = {int(g["rnti"]): int(g["tb"]["harq_slot"][0]) for g in b1}
    assert sorted(slots.values()) == [0, P.D_SLOTS - 1]
    regions = [(rnti, slot * rm_ref.HARQ_SLOT_ELEMS + r * rm_ref.HARQ_CB_STRIDE, rm_ref.pair_words(K))
               for rnti, slot in slots.items() for r, K in enumerate(Ks)]
    assert not clash(regions, 64)
    assert clash(regions, 32)
