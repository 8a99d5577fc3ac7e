"""What turbo_kernel does around its trellis steps, against tests/ref_dec.py (integer references from 36.212 and DESIGN.md §2):
  * the CRC24 byte tables of turbo_arith.cuh (no GPU): the remainder of a decision word of 1 .. 32 bits and the byte fold of tb_crc_kernel;
  * on the GPU, bit for bit: pairs whose two code blocks stop at different iterations (the syndromes of both halves are computed in one
    round, a finished half must stay as it was), launches with a single code block, a single pair and fewer pairs than resident CTAs,
    block sizes with a ragged last window (the termination metrics and the last decision word), CRC24A / CRC24B / no CRC, and a
    launch of more pairs than resident CTAs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ltelib
import ref_dec
from ltesniffer_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLY = {1: ref_dec.CRC24A, 2: ref_dec.CRC24B}


# ------------------------------------------------------------------------------------------------ byte tables (no GPU)
@pytest.fixture(scope="module")
def model():
    so = os.path.join(ROOT, "tools", "libturbo_model.so")
    src = [os.path.join(ROOT, "tools", "turbo_model.cpp"), os.path.join(ROOT, "ltesniffer_b200", "csrc", "turbo_arith.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in src):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-o", so, src[0]], check=True)
    L = C.CDLL(so)
    L.turbo_model_crc24_table.argtypes = [C.c_uint32, C.c_void_p]
    for f in (L.turbo_model_crc24_word, L.turbo_model_crc24_byte):
        f.argtypes = [C.c_uint32] * 3
        f.restype = C.c_uint32
    return L


def times_x24(r, poly):
    """r(x) x^24 mod g by 24 shifts of a bitwise register: the syndromes of ref_dec carry this factor, and it is invertible"""
    for _ in range(24):
        r <<= 1
        if r >> 24:
            r ^= poly
    return r


@pytest.mark.parametrize("ct", [1, 2])
def test_byte_table_remainder_of_a_decision_word(model, ct):
    poly = POLY[ct]
    tab = np.zeros(256, np.uint32)
    model.turbo_model_crc24_table(ct - 1, tab.ctypes.data)
    for b in (0, 1, 0x80, 0xFF):                                  # entry b = b(x) x^24 mod g
        assert int(tab[b]) == int(ref_dec.crc24_syndrome(np.unpackbits(np.array([b], np.uint8))[None], poly)[0])
    rng = np.random.default_rng(24 + ct)
    for nb in range(1, 33):
        words = [0, 0xFFFFFFFF, 0x80000000, 1 << (32 - nb)] + [int(x) for x in rng.integers(0, 1 << 32, 60, dtype=np.uint64)]
        bits = np.array([[(w >> (31 - i)) & 1 for i in range(nb)] for w in words], np.uint8)      # the top nb bits, first bit first
        want = ref_dec.crc24_syndrome(bits, poly)
        for w, s in zip(words, want):
            r = model.turbo_model_crc24_word(ct - 1, w, nb)
            assert r < (1 << 24) and times_x24(r, poly) == int(s), (ct, nb, hex(w))


def test_byte_table_fold_of_payload_bytes(model):
    rng = np.random.default_rng(5)
    for n in (1, 2, 3, 4, 7, 61):
        data = rng.integers(0, 256, n).astype(np.uint8)
        r = 0
        for b in data:
            r = model.turbo_model_crc24_byte(0, r, int(b))
        assert times_x24(r, ref_dec.CRC24A) == int(ref_dec.crc24_syndrome(np.unpackbits(data)[None], ref_dec.CRC24A)[0]), n


# ------------------------------------------------------------------------------------------------ the kernel (GPU)
def encode_blocks(S, rng, K, snrs, poly):
    """one random code block per entry of snrs (dB) with a CRC24 (poly) in its last 24 bits, turbo encoded, BPSK over AWGN, scaled and
    clipped as the rate matcher delivers it (|d| <= 255) -> int16 [n][3 (K + 4)]"""
    D = K + 4
    d = np.zeros((len(snrs), 3 * D), np.int16)
    for i, snr in enumerate(snrs):
        b = rng.integers(0, 2, K).astype(np.uint8)
        crc = S.lte_crc(poly, 24, ltelib.ptr(b), K - 24)
        b[K - 24:] = [(crc >> (23 - j)) & 1 for j in range(24)]
        enc = np.zeros(3 * D, np.uint8)
        S.lte_turbo_encode(ltelib.ptr(b), K, ltelib.ptr(enc[0:]), ltelib.ptr(enc[D:]), ltelib.ptr(enc[2 * D:]))
        x = (2.0 * enc - 1.0) + 10 ** (-snr / 20) * rng.standard_normal(3 * D)
        d[i] = np.clip(np.round(x * 60), -255, 255).astype(np.int16)
    return d


def check(phy, d, K, max_iter, crc_type, what):
    bits, iters, ok = phy.turbo_batch(d, K, max_iter, crc_type)
    rb, rit, rok = ref_dec.turbo_decode_ref(d, K, max_iter, crc_type)
    for i in range(d.shape[0]):
        assert np.array_equal(bits[i], rb[i]), "%s K=%d cb %d crc_type %d: %d bits differ from the reference" % (what, K, i, crc_type, int((bits[i] != rb[i]).sum()))
    assert np.array_equal(iters, rit) and np.array_equal(ok.astype(bool), rok), (what, K, crc_type, iters.tolist(), rit.tolist(), ok.tolist(), rok.tolist())
    return rit, rok


@pytest.fixture(scope="module")
def sim(infra):
    S = infra.sim()
    S.lte_turbo_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    return S


@pytest.mark.gpu
@pytest.mark.parametrize("K", [104, 1008, 2112])
def test_halves_of_a_pair_stop_at_different_iterations(sim, phylib, K):
    """clean and marginal code blocks alternate, so a pair holds one of each; with CRC24A, CRC24B, and a half that never passes"""
    phy = capi.LtePhy(100, 1, 1, 1, max_subframes=1)
    split, stopped = 0, set()
    for ct in (1, 2):
        rng = np.random.default_rng(10 * K + ct)
        d = encode_blocks(sim, rng, K, [6.0, -0.4, -0.8, 6.0, -3.0, 6.0, 0.2], POLY[ct])     # 7 blocks: the last pair has an idle half
        rit, rok = check(phy, d, K, 8, ct, "split pair")
        split += sum(int(rit[i] != rit[i + 1]) for i in range(0, 6, 2))
        stopped.update(int(x) for x in rit)
        assert rok[0] and rit[0] <= 2 and (rit[4] == 8 and not rok[4])
    phy.close()
    assert split >= 4 and len(stopped) >= 3, (split, sorted(stopped))


@pytest.mark.gpu
@pytest.mark.parametrize("K", [40, 1008, 6144])
def test_launches_smaller_than_the_grid(sim, phylib, K):
    """1 code block (one pair with an idle half), 2 (one pair) and 5 (three pairs): far fewer pairs than resident CTAs.  K = 40 and 1008 end
    in a window of 8 and 16 steps; every CRC type; 1 and 8 iterations at most"""
    phy = capi.LtePhy(100, 1, 1, 1, max_subframes=1)
    for ncb in (1, 2, 5):
        for ct in (0, 1, 2):
            rng = np.random.default_rng(K + 100 * ncb + ct)
            d = encode_blocks(sim, rng, K, [1.5, 0.0, 5.0, -2.0, 0.8][:ncb], POLY[ct or 2])
            check(phy, d, K, 8, ct, "%d blocks" % ncb)
            check(phy, d, K, 1, ct, "%d blocks, one iteration" % ncb)
    phy.close()


@pytest.mark.gpu
def test_more_pairs_than_resident_ctas(sim, phylib):
    """K = 40 runs 32-thread CTAs, twelve to an SM: 4001 code blocks are more pairs than any H100 holds at once, so pairs are taken from
    the queue by CTAs that have already decoded one; the last pair has an idle half"""
    K, n = 40, 4001
    phy = capi.LtePhy(100, 1, 1, 1, max_subframes=1)
    rng = np.random.default_rng(4001)
    d = encode_blocks(sim, rng, K, list(rng.uniform(-2.0, 4.0, n)), POLY[1])
    rit, rok = check(phy, d, K, 8, 1, "long queue")
    phy.close()
    assert rok.sum() > n // 4 and (~rok).sum() > n // 20 and len(set(rit.tolist())) >= 4
