"""The oracle's two decoders (lteo_dci_decode, lteo_turbo_decode, lteo_dlsch_decode[_harq]) bit for bit against the integer references of
tests/ref_dec.py, which were written from 36.212 and DESIGN.md §2 by another hand.  The inputs are chosen where the §2 rules decide the
result: garbage decodes of noise, tie-dense LLRs, single non-zero values, the quantiser's scale invariance and its NaN rule, every turbo block
size with inputs that saturate the extrinsic or leave the trellis to the tails, early stopping at every iteration count, and the DL-SCH
assembly (fillers, several code blocks, all redundancy versions and modulations, HARQ combining).  The input generators are shared with
tests/test_gpu_decoder_reference.py, which holds the kernels to the same references."""
import ctypes as C

import numpy as np
import pytest

import ltelib
import ref_dec
from ltelib import Cell

CELLS = [(nprb, ports) for nprb in (6, 15, 25, 50, 75, 100) for ports in (1, 2)]
DCI_E = (72, 144, 288, 576)
TURBO_SNR = [-1.8, -1.2, -0.6, 0.2, 1.0]          # dB, as the GPU shape tests: from most blocks failing to most stopping after one or two
TURBO_KINDS = ("waterfall", "full_scale", "no_parity", "zero_tails", "burst")


def turbo_sizes():
    """the 188 code-block sizes of 36.212 Table 5.1.3-3"""
    return list(range(40, 512, 8)) + list(range(512, 1024, 16)) + list(range(1024, 2048, 32)) + list(range(2048, 6145, 64))


@pytest.fixture(scope="module")
def S(infra):
    L = infra.sim()
    L.lte_turbo_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def dci_sizes(S):
    """every distinct DCI payload size of the formats the library knows, over every bandwidth and port count"""
    return sorted({int(S.lte_dci_sizeof(C.byref(Cell(nprb, ports, 1, 1)), f)) for nprb, ports in CELLS for f in range(9)})


def dci_inputs(S, rng, nbits, E, n):
    """n candidates of E soft bits per kind -> {kind: float32 [n][E]}, plus the planted (bits, rnti) of kind "planted" """
    L = {72: 0, 144: 1, 288: 2, 576: 3}[E]
    out = {"noise": (rng.standard_normal((n, E)) * rng.uniform(0.01, 100, (n, 1))).astype(np.float32)}
    pl = np.zeros((n, E), np.float32)
    truth = []
    for i in range(n):
        b = rng.integers(0, 2, nbits).astype(np.uint8)
        rnti = int(rng.integers(0, 0x10000))
        e = np.zeros(E, np.uint8)
        S.lte_sim_pdcch_encode(ltelib.ptr(b), nbits, rnti, L, ltelib.ptr(e))
        sigma = 1.5 * i / max(1, n - 1)                          # clean to well below the waterfall
        pl[i] = (2.0 * e - 1.0) + sigma * rng.standard_normal(E)
        truth.append((b, rnti, sigma))
    out["planted"] = pl[::-1].copy()
    truth = truth[::-1]
    out["ties"] = rng.integers(-1, 2, (n, E)).astype(np.float32)
    one = np.zeros((n, E), np.float32)
    one[np.arange(n), rng.integers(0, E, n)] = rng.choice([-3.0, -1.0, 0.5, 7.0], n)
    out["single"] = one
    out["full_scale"] = np.where(rng.random((n, E)) < 0.5, -1.0, 1.0).astype(np.float32)
    out["zero"] = np.zeros((max(2, n // 16), E), np.float32)
    return out, truth


def oracle_dci(o, e, nbits):
    n = e.shape[0]
    valid, bits, rem = np.zeros(n, bool), np.zeros((n, nbits), np.uint8), np.zeros(n, np.int64)
    for i in range(n):
        r, b, c = o.dci_decode(e[i], nbits)
        if r == 0:
            valid[i], bits[i], rem[i] = True, b, c
    return valid, bits, rem


def assert_dci_equal(got, want, what):
    gv, gb, gr = got
    wv, wb, wr = want
    bad = np.nonzero((gv != wv) | (wv & ((gb != wb).any(1) | (gr != wr))))[0]
    assert len(bad) == 0, "%s: %d of %d candidates differ, first %d: valid %s / %s, rem %s / %s" % (
        what, len(bad), len(gv), bad[0], gv[bad[0]], wv[bad[0]], hex(int(gr[bad[0]])), hex(int(wr[bad[0]])))


def test_crcs_of_the_reference_against_catalogue_check_values():
    check = np.unpackbits(np.frombuffer(b"123456789", np.uint8))[None]
    assert ref_dec.crc16_lfsr(check)[0] == 0x31C3
    for poly, cv in ((ref_dec.CRC24A, 0xCDE703), (ref_dec.CRC24B, 0x23EF52)):
        word = np.concatenate([check[0], [(cv >> (23 - i)) & 1 for i in range(24)]])[None]
        assert ref_dec.crc24_syndrome(word, poly)[0] == 0
        word[0, -1] ^= 1
        assert ref_dec.crc24_syndrome(word, poly)[0] != 0


def test_dci_decoder_equals_reference_on_every_payload_size(infra, S):
    """every payload size x E = 72 / 144 / 288 / 576 x six input kinds; valid, bits and CRC remainder of every candidate"""
    o = ltelib.Oracle(Cell(100, 2, 5, 1))
    rng = np.random.default_rng(40)
    sizes = dci_sizes(S)
    assert len(sizes) >= 25 and min(sizes) <= 10 and max(sizes) >= 51, sizes
    total, recovered, garbage_valid = 0, 0, 0
    for nbits in sizes:
        for E in DCI_E:
            kinds, truth = dci_inputs(S, rng, nbits, E, 192)
            for kind, e in kinds.items():
                got = ref_dec.dci_decode_ref(e, nbits)
                assert_dci_equal(got, oracle_dci(o, e, nbits), "%s nbits %d E %d" % (kind, nbits, E))
                total += len(e)
                if kind == "zero":
                    assert not got[0].any()
                if kind == "noise":
                    garbage_valid += int(got[0].sum())
                if kind == "planted":
                    for i, (b, rnti, sigma) in enumerate(truth):
                        ok = np.array_equal(got[1][i], b) and got[2][i] == rnti
                        recovered += int(ok)
                        assert ok or sigma > 0.25, (nbits, E, i, sigma)       # the reference decodes what the transmitter sent
    assert total >= 100000 and garbage_valid > 0.9 * len(sizes) * len(DCI_E) * 192, (total, garbage_valid)


def test_dci_quantiser_scale_invariance_and_nan_rule(infra, S):
    """integer-valued soft bits scaled by every power of two that keeps them and 32 / max|x| finite and normal decode as the unscaled ones
    (the scaling is exact there); outside that range (max|x| about 1e-39, 1e-38, sums overflowing at 1e38) and with NaN soft bits the §2 rule
    "NaN quantises to q = 0" decides, and the oracle must follow it"""
    o = ltelib.Oracle(Cell(100, 2, 5, 1))
    rng = np.random.default_rng(41)
    for nbits, E in ((27, 72), (44, 288), (51, 576)):
        e = rng.integers(-8, 9, (24, E)).astype(np.float32)
        e[0] = 0
        e[0, 5] = 1
        base = ref_dec.dci_decode_ref(e, nbits)
        assert base[0][1:].all() and base[0][0]
        ks = 0
        for k in range(-140, 129):
            with np.errstate(all="ignore"):
                es = (e * np.float32(2.0) ** k).astype(np.float32)
                nz = np.abs(e[e != 0])
                exact = nz.min() * 2.0 ** k >= 2.0 ** -126 and 8.0 * 8 * 2.0 ** k < 3.4e38 and 32 / (2.0 ** k) < 3.4e38
            got = ref_dec.dci_decode_ref(es, nbits)
            if exact:
                ks += 1
                assert_dci_equal(got, base, "scale 2^%d" % k)
            if k % 7 == 0 or not exact:
                assert_dci_equal(got, oracle_dci(o, es, nbits), "scale 2^%d against the oracle" % k)
        assert ks >= 240, ks
        ext = []
        for mag in (1e-39, 1e-38, 1e38):
            x = (np.where(rng.random((16, E)) < 0.5, -1, 1) * rng.uniform(0.5, 1, (16, E)) * mag).astype(np.float32)
            x[:4, ::3] = 0                                               # zeros meet an infinite gain: 0 * inf = NaN
            ext.append(x)
        nan = rng.standard_normal((16, E)).astype(np.float32)
        nan[np.arange(16), rng.integers(0, E, 16)] = np.nan
        nan[0] = np.nan
        ext.append(nan)
        inf = rng.standard_normal((4, E)).astype(np.float32)
        inf[:, 0] = np.inf
        ext.append(inf)
        for x in ext:
            assert_dci_equal(ref_dec.dci_decode_ref(x, nbits), oracle_dci(o, x, nbits), "extreme input, nbits %d" % nbits)
    with np.errstate(all="ignore"):
        rm = np.array([[np.nan, 1.0, -1.0, 0.0]], np.float32)
        valid, r = ref_dec.dci_quantise(rm)
    assert valid[0] and r[0].tolist() == [-255, 63, -65, -1]


def encode_turbo(S, rng, K, crc_poly):
    b = rng.integers(0, 2, K).astype(np.uint8)
    crc = S.lte_crc(crc_poly, 24, ltelib.ptr(b), K - 24)
    b[K - 24:] = [(crc >> (23 - j)) & 1 for j in range(24)]
    D = K + 4
    enc = np.zeros(3 * D, np.uint8)
    S.lte_turbo_encode(ltelib.ptr(b), K, ltelib.ptr(enc[0:]), ltelib.ptr(enc[D:]), ltelib.ptr(enc[2 * D:]))
    return b, enc


def turbo_inputs(S, rng, K, n):
    """one code block of each TURBO_KINDS for position n of the K table, with its CRC24A (even n) or CRC24B (odd n) -> (d int16 [5][3 (K + 4)], info)"""
    D = K + 4
    poly = ref_dec.CRC24A if n % 2 == 0 else ref_dec.CRC24B
    d = np.zeros((len(TURBO_KINDS), 3 * D), np.int16)
    info = np.zeros((len(TURBO_KINDS), K), np.uint8)
    for j, kind in enumerate(TURBO_KINDS):
        b, enc = encode_turbo(S, rng, K, poly)
        info[j] = b
        x = 2.0 * enc - 1.0
        if kind == "waterfall":
            v = np.round((x + 10 ** (-TURBO_SNR[(n + j) % len(TURBO_SNR)] / 20) * rng.standard_normal(3 * D)) * 60)
        elif kind == "full_scale":                                     # not a codeword: the metric spreads and the extrinsic saturate
            v = np.where(rng.random(3 * D) < 0.5, -255, 255)
        elif kind == "no_parity":                                      # systematic only, as under heavy puncturing
            v = 255 * x
            v[D:D + K] = 0
            v[2 * D:2 * D + K] = 0
        elif kind == "zero_tails":
            v = np.round((x + 0.5 * rng.standard_normal(3 * D)) * 60)
            for s in range(3):
                v[s * D + K:(s + 1) * D] = 0
        else:                                                          # a burst of large wrong-sign systematic values
            v = np.round((x + 0.3 * rng.standard_normal(3 * D)) * 80)
            n0, nb = int(rng.integers(0, K // 2)), max(8, K // 8)
            v[n0:n0 + nb] = -255 * x[n0:n0 + nb]
        d[j] = np.clip(v, -255, 255)
    return d, info


def oracle_turbo(O, d, K, max_iter, crc_type):
    n = d.shape[0]
    max_iter = np.broadcast_to(max_iter, (n,))
    crc_type = np.broadcast_to(crc_type, (n,))
    bits, iters, ok = np.zeros((n, K), np.uint8), np.zeros(n, np.int64), np.zeros(n, bool)
    for i in range(n):
        o = C.c_int(0)
        iters[i] = O.lteo_turbo_decode(ltelib.ptr(np.ascontiguousarray(d[i])), K, int(max_iter[i]), int(crc_type[i]), ltelib.ptr(bits[i]), C.byref(o))
        ok[i] = bool(o.value)
    return bits, iters, ok


def assert_turbo_equal(got, want, what):
    for i in range(len(got[1])):
        nb = int((got[0][i] != want[0][i]).sum())
        assert nb == 0 and got[1][i] == want[1][i] and got[2][i] == want[2][i], (
            "%s block %d: %d bits differ, iterations %d / %d, crc %d / %d" % (what, i, nb, got[1][i], want[1][i], got[2][i], want[2][i]))


def turbo_settings(n):
    """(max_iter, crc_type) per block of turbo_inputs at table position n: every max_iter 1..8 and crc_type 0 / 1 / 2 across the table; the CRC
    type matches the code blocks' CRC unless it is 0"""
    j = np.arange(len(TURBO_KINDS))
    max_iter = 1 + (n + 3 * j) % 8
    crc_type = np.where((n + j) % 3 == 0, 0, 1 + n % 2)
    return max_iter, crc_type


def test_turbo_decoder_equals_reference_at_every_block_size(infra, S):
    """all 188 K, five input kinds each, max_iter 1..8 and no / CRC24A / CRC24B early stop: bits, iterations and crc_ok of every block"""
    O = infra.oracle()
    seen_iters, seen_settings, stopped, failed, decoded = set(), set(), 0, 0, 0
    for n, K in enumerate(turbo_sizes()):
        rng = np.random.default_rng(50000 + K)
        d, info = turbo_inputs(S, rng, K, n)
        max_iter, crc_type = turbo_settings(n)
        got = ref_dec.turbo_decode_ref(d, K, max_iter, crc_type)
        assert_turbo_equal(got, oracle_turbo(O, d, K, max_iter, crc_type), "K=%d" % K)
        seen_settings.update(zip(max_iter.tolist(), crc_type.tolist()))
        seen_iters.update(int(i) for i, c in zip(got[1], crc_type) if c)
        stopped += int((got[2] & (got[1] < max_iter)).sum())
        failed += int((~got[2] & (crc_type > 0)).sum())
        decoded += int(sum(np.array_equal(got[0][j], info[j]) for j in range(len(info)) if got[2][j]))
    assert {m for m, c in seen_settings} == set(range(1, 9)) and {c for m, c in seen_settings} == {0, 1, 2}
    assert seen_iters == set(range(1, 9)), sorted(seen_iters)
    assert stopped >= 100 and failed >= 50 and decoded >= 300, (stopped, failed, decoded)


def test_turbo_offsets_do_not_change_decisions():
    """§2: every decision is offset-invariant.  A constant added to every boundary metric of one window, or to the tail metrics, shifts all
    alpha / beta of that window alike, so L and the extrinsic must not move; checked on the reference's windowed pass directly"""
    rng = np.random.default_rng(42)
    K = 200
    NW = -(-K // 32)
    xs, par, apr = (rng.integers(-255, 256, (3, K)) for _ in range(3))
    tx, tz = rng.integers(-255, 256, (3, 3)), rng.integers(-255, 256, (3, 3))
    A = rng.integers(-3000, 3000, (3, NW, 8))
    B = rng.integers(-3000, 3000, (3, NW, 8))
    e0, L0, _, _ = ref_dec._siso(xs, par, apr, tx, tz, A, B)
    e1, L1, _, _ = ref_dec._siso(xs, par, apr, tx, tz, A + rng.integers(-9000, 9000, (3, NW, 1)), B + rng.integers(-9000, 9000, (3, NW, 1)))
    assert np.array_equal(L0, L1) and np.array_equal(e0, e1)


def dlsch_cases():
    """(tbs, rv, Qm, NL, laps of the circular buffer, SNR dB, early_stop, amplitude): C = 1 and C > 1, F > 0, both K of a segmentation,
    every rv and Qm, two layers, no early stop, and amplitudes that saturate the int16 accumulation"""
    return [(512, 0, 2, 1, 1.0, 3.0, 1, 100), (1536, 1, 4, 2, 0.7, 4.0, 1, 200), (6208, 2, 6, 1, 0.8, 6.0, 1, 400), (9000, 3, 8, 2, 1.2, 12.0, 1, 400),
            (13000, 0, 2, 1, 0.5, 1.0, 1, 100), (12000, 1, 6, 2, 2.5, 30.0, 0, 30000), (104, 3, 2, 1, 6.0, 20.0, 1, 20000), (7992, 2, 4, 1, 0.9, 0.0, 0, 150)]


def dlsch_llr(S, rng, tbs, rv, Qm, NL, laps, snr, amp):
    """random payload, lte_sim_dlsch_encode, +-amp plus Gaussian noise at snr dB, saturated to int16 -> (G, int16 soft bits, payload)"""
    Cn, Ks, F = ref_dec.segmentation(tbs)
    G = int(sum(3 * (K + 4) for K in Ks) * laps) // (NL * Qm) * (NL * Qm)
    pl = rng.integers(0, 256, tbs // 8).astype(np.uint8)
    e = np.zeros(G, np.uint8)
    assert S.lte_sim_dlsch_encode(ltelib.ptr(pl), tbs, rv, G, Qm, NL, ltelib.ptr(e)) == 0
    x = (2.0 * e - 1.0) + 10 ** (-snr / 20) * rng.standard_normal(G)
    return G, np.clip(np.round(x * amp), -32768, 32767).astype(np.int16), pl


def oracle_dlsch(O, llr, G, tbs, rv, Qm, NL, max_iter, early_stop, soft=None, combine=0):
    Cn, Ks, F = ref_dec.segmentation(tbs)
    out = np.zeros(tbs // 8 + 8, np.uint8)
    it = np.zeros(64, np.uint32)
    O.lteo_dlsch_decode_harq.argtypes = [C.c_void_p] + [C.c_uint32] * 6 + [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    r = O.lteo_dlsch_decode_harq(ltelib.ptr(llr), G, tbs, rv, Qm, NL, max_iter, early_stop, ltelib.ptr(out), ltelib.ptr(it),
                                 None if soft is None else ltelib.ptr(soft), combine)
    return bool(r == 1), out[:tbs // 8], it[:Cn].astype(np.int64)


def test_dlsch_decode_equals_reference(infra, S):
    O = infra.oracle()
    rng = np.random.default_rng(43)
    seen = set()
    for tbs, rv, Qm, NL, laps, snr, early, amp in dlsch_cases():
        G, llr, pl = dlsch_llr(S, rng, tbs, rv, Qm, NL, laps, snr, amp)
        crc, payload, iters, _ = ref_dec.dlsch_decode_ref(llr, G, tbs, rv, Qm, NL, 8, early)
        ocrc, opl, oit = oracle_dlsch(O, llr, G, tbs, rv, Qm, NL, 8, early)
        assert (crc, payload.tolist(), iters.tolist()) == (ocrc, opl.tolist(), oit.tolist()), (tbs, rv, Qm, NL)
        Cn, Ks, F = ref_dec.segmentation(tbs)
        seen.add(("C>1" if Cn > 1 else "C=1", F > 0))
        seen.add(("crc", crc))
        if crc:
            assert np.array_equal(payload, pl), tbs
    assert {("C=1", True), ("C>1", True), ("C=1", False), ("crc", True), ("crc", False)} <= seen, seen


def test_dlsch_harq_combining_equals_reference(infra, S):
    """a first transmission too noisy to decode, then a retransmission with another rv added to its accumulators: crc, payload, iterations
    and the accumulators themselves after both"""
    O = infra.oracle()
    rng = np.random.default_rng(44)
    for tbs, Qm, NL in ((1536, 2, 1), (9000, 4, 2)):
        Cn, Ks, F = ref_dec.segmentation(tbs)
        soft = np.zeros(Cn * ltelib.HARQ_CB_STRIDE, np.int16)
        pl = rng.integers(0, 256, tbs // 8).astype(np.uint8)
        accs, results = None, []
        for rv, snr, combine in ((0, -2.0, 0), (2, -2.0, 1), (3, 0.0, 1)):
            G = int(sum(3 * (K + 4) for K in Ks) * 0.6) // (NL * Qm) * (NL * Qm)
            e = np.zeros(G, np.uint8)
            assert S.lte_sim_dlsch_encode(ltelib.ptr(pl), tbs, rv, G, Qm, NL, ltelib.ptr(e)) == 0
            llr = np.clip(np.round(((2.0 * e - 1.0) + 10 ** (-snr / 20) * rng.standard_normal(G)) * 100), -32768, 32767).astype(np.int16)
            crc, payload, iters, accs = ref_dec.dlsch_decode_ref(llr, G, tbs, rv, Qm, NL, 8, 1, accs, bool(combine))
            ocrc, opl, oit = oracle_dlsch(O, llr, G, tbs, rv, Qm, NL, 8, 1, soft, combine)
            assert (crc, payload.tolist(), iters.tolist()) == (ocrc, opl.tolist(), oit.tolist()), (tbs, rv)
            for r, K in enumerate(Ks):
                o_acc = soft[r * ltelib.HARQ_CB_STRIDE:r * ltelib.HARQ_CB_STRIDE + 3 * (K + 4)]
                assert np.array_equal(o_acc, accs[r]), (tbs, rv, r)
            results.append(crc)
        assert results[0] is False and results[-1] is True, (tbs, results)


def crafted_codeword(S, rng, tbs, G, Qm, NL, rv, bad=None):
    """the coded bits of a random transport block, built here from 36.212 5.1.1 - 5.1.4 with lte_turbo_encode and the reference's circular
    buffer, so that one CRC can be made wrong on purpose: bad = "tb" flips the last bit of the TB CRC24A before segmentation (every CB CRC24B is
    then computed over it and valid), bad = r flips the last bit of code block r's CRC24B -> (e uint8 [G], payload bytes)"""
    a = rng.integers(0, 2, tbs).astype(np.uint8)
    crc = S.lte_crc(ref_dec.CRC24A, 24, ltelib.ptr(a), tbs)
    b = np.concatenate([a, [(crc >> (23 - j)) & 1 for j in range(24)]]).astype(np.uint8)
    if bad == "tb":
        b[-1] ^= 1
    Cn, Ks, F = ref_dec.segmentation(tbs)
    e, pos = [], 0
    for r, K in enumerate(Ks):
        Fr = F if r == 0 else 0
        nd = K - Fr - (24 if Cn > 1 else 0)
        c = np.concatenate([np.zeros(Fr, np.uint8), b[pos:pos + nd]])             # filler bits enter the encoder as 0
        pos += nd
        if Cn > 1:
            crc = S.lte_crc(ref_dec.CRC24B, 24, ltelib.ptr(c), K - 24)
            c = np.concatenate([c, [(crc >> (23 - j)) & 1 for j in range(24)]]).astype(np.uint8)
            if bad == r:
                c[-1] ^= 1
        D = K + 4
        d = np.zeros(3 * D, np.uint8)
        S.lte_turbo_encode(ltelib.ptr(c), K, ltelib.ptr(d[0:]), ltelib.ptr(d[D:]), ltelib.ptr(d[2 * D:]))
        e.append(d[np.resize(ref_dec.turbo_ring(K, Fr, rv), ref_dec.cb_E(G, Cn, r, Qm, NL))])
    assert pos == tbs + 24
    return np.concatenate(e), np.packbits(a)


def test_crafted_transport_blocks_separate_tb_and_cb_crcs(infra, S):
    """the rule "crc needs the TB CRC24A and, when C > 1, every CB CRC24B": (1) every CB CRC valid but the TB CRC wrong: crc 0 and one iteration per
    code block; (2) the TB CRC valid but one CB CRC wrong: crc 0, that code block runs max_iter and the payload is still right; (3) C = 1 with F > 0.
    The construction itself is checked first: without a wrong CRC it equals lte_sim_dlsch_encode bit for bit."""
    O = infra.oracle()
    rng = np.random.default_rng(45)
    for tbs, Qm, NL, rv in ((9000, 2, 1, 0), (13000, 4, 2, 1), (512, 6, 1, 2)):
        Cn, Ks, F = ref_dec.segmentation(tbs)
        assert F > 0
        G = int(sum(3 * (K + 4) for K in Ks) * 0.8) // (NL * Qm) * (NL * Qm)
        state = rng.bit_generator.state
        e, pl = crafted_codeword(S, rng, tbs, G, Qm, NL, rv)
        rng.bit_generator.state = state
        a = rng.integers(0, 2, tbs).astype(np.uint8)
        sim_e = np.zeros(G, np.uint8)
        assert S.lte_sim_dlsch_encode(ltelib.ptr(np.packbits(a)), tbs, rv, G, Qm, NL, ltelib.ptr(sim_e)) == 0
        assert np.array_equal(e, sim_e), tbs
        for bad in [None] + (["tb"] + list(range(Cn)) if Cn > 1 else ["tb"]):
            e, pl = crafted_codeword(S, rng, tbs, G, Qm, NL, rv, bad)
            llr = ((2 * e.astype(np.int16) - 1) * 120).astype(np.int16)
            crc, payload, iters, _ = ref_dec.dlsch_decode_ref(llr, G, tbs, rv, Qm, NL, 8, 1)
            ocrc, opl, oit = oracle_dlsch(O, llr, G, tbs, rv, Qm, NL, 8, 1)
            assert (crc, payload.tolist(), iters.tolist()) == (ocrc, opl.tolist(), oit.tolist()), (tbs, bad)
            assert np.array_equal(payload, pl), (tbs, bad)                        # the information bits always decode
            assert crc == (bad is None), (tbs, bad, crc)
            want_it = [8 if r == bad else 1 for r in range(Cn)]
            if bad == "tb" and Cn == 1:
                want_it = [8]                                                     # C = 1: the CRC24A is the code block's own early-stop CRC
            assert iters.tolist() == want_it, (tbs, bad, iters)
