"""The two decoders stand-alone at every shape the library accepts (pytest -m gpu), bit-exact against the CPU oracle:
  * dci_viterbi_kernel (ltephy_dci_sweep) on the ten standard cells (15 / 25 / 50 / 75 / 100 PRB x 1 / 2 ports): every DCI payload size they
    give (23 in all, 10 bits for format 1C at 15 PRB up to 51 for format 2 at 100 PRB), every aggregation level, the RNTIs 0, 0xFFFE and
    0xFFFF, and LLR blocks that stress the quantiser and the add-compare-select: all zero, constant, one huge value among small ones.
    Every entry of the candidate table is compared, not a sample.
  * turbo_kernel<NT, FULL> (ltephy_turbo_batch) at all 188 code-block sizes of 36.212 Table 5.1.3-3, with CRC24A and CRC24B early stop and
    with a fixed iteration count, an odd number of code blocks per size (one CTA pair has an idle half), and noiseless / all-zero inputs.
Each test asserts its own coverage, so losing a shape fails it."""
import ctypes as C
import numpy as np
import pytest

import ltelib
from ltelib import Cell, Oracle
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu

STD_CELLS = [(nprb, ports) for nprb in (15, 25, 50, 75, 100) for ports in (1, 2)]
SWEEP_CFI = [1, 2, 3, 1, 2, 3]
SPECIAL_RNTIS = [0x0000, 0xFFFF, 0xFFFE]
CRC24A, CRC24B = 0x1864CFB, 0x1800063


def distinct_sizes(phy):
    sizes, sidx = phy.sizes()
    return {sidx[f]: sizes[f] for f in range(capi.NOF_FORMATS)}


def check_table(o, phy, llr, cfis, cands, distinct):
    """every (subframe, location, size) entry of the GPU table against one oracle decode; -> {(sf, location index, size index): (bits, rnti)} of the valid ones"""
    valid = {}
    for i, cfi in enumerate(cfis):
        nc, Ls = phy.locations(cfi)
        for li in range(len(nc)):
            e = llr[i, 72 * int(nc[li]):72 * int(nc[li]) + (72 << int(Ls[li]))]
            for si, nb in distinct.items():
                ret, bits, crc = o.dci_decode(e, nb)
                c = cands[i, li, si]
                if ret != 0:
                    assert c["valid"] == 0, (i, li, si, nb)
                    continue
                assert c["valid"] == 1, (i, li, si, nb)
                assert int(c["rnti"]) == crc, (i, li, si, nb, hex(int(c["rnti"])), hex(crc))
                assert np.array_equal(capi.cand_bits(c["bits"], nb), bits), (i, li, si, nb)
                valid[(i, li, si)] = (bits, crc)
    return valid


def plant_dcis(S, phy, rng, distinct):
    """LLR buffers of len(SWEEP_CFI) subframes: noise everywhere, DCIs encoded into non-overlapping locations, each location taking the size
    planted least often so far at its aggregation level; the first DCIs carry the special RNTIs -> (llr, planted)"""
    n = len(SWEEP_CFI)
    llr = (0.3 * rng.standard_normal((n, capi.LLR_STRIDE))).astype(np.float32)
    planted, count, k = [], {}, 0
    for i, cfi in enumerate(SWEEP_CFI):
        ncce = phy.nof_cce(cfi)
        llr[i, 72 * ncce:] = 0
        nc, Ls = phy.locations(cfi)
        used = np.zeros(ncce, bool)
        first = [int(rng.choice(np.nonzero(Ls == L)[0])) for L in (3, 2, 1, 0) if (Ls == L).any()]   # one location of every level, then any
        for li in first + list(rng.permutation(len(nc))):
            c, L = int(nc[li]), int(Ls[li])
            if used[c:c + (1 << L)].any() or rng.random() < 0.15:
                continue
            used[c:c + (1 << L)] = True
            si = min(distinct, key=lambda s: (count.get((L, s), 0), rng.random()))
            count[(L, si)] = count.get((L, si), 0) + 1
            nb = distinct[si]
            b = rng.integers(0, 2, nb).astype(np.uint8)
            rnti = SPECIAL_RNTIS[k] if k < len(SPECIAL_RNTIS) else int(rng.integers(1, 0xFFFD))
            k += 1
            e = np.zeros(72 << L, np.uint8)
            S.lte_sim_pdcch_encode(ltelib.ptr(b), nb, rnti, L, ltelib.ptr(e))
            llr[i, 72 * c:72 * c + (72 << L)] = (2.0 * e - 1.0) + 0.3 * rng.standard_normal(72 << L)
            planted.append((i, li, L, si, rnti, b))
    return llr, planted


def test_dci_sweep_every_size_and_level(infra, phylib):
    """the ten standard cells in one test, so that the union of the payload sizes decoded can be asserted: exactly the 23 they give"""
    S = infra.sim()
    sizes_seen = set()
    for nprb, ports in STD_CELLS:
        cell = Cell(nprb, ports, 3 * nprb + ports, 1)
        phy = capi.LtePhy(nprb, ports, cell.cell_id, 1, max_subframes=len(SWEEP_CFI))
        o = Oracle(cell)
        distinct = distinct_sizes(phy)
        sizes, _ = phy.sizes()
        assert sizes == [S.lte_dci_sizeof(C.byref(cell), f) for f in range(capi.NOF_FORMATS)]
        nlocs = [len(phy.locations(cfi)[0]) for cfi in (1, 2, 3)]
        assert len({n % 2 for n in nlocs}) == 2, (nprb, ports, nlocs)      # odd and even location counts: one pair of locations is half empty
        rng = np.random.default_rng(1000 + 10 * nprb + ports)
        llr, planted = plant_dcis(S, phy, rng, distinct)
        cands = phy.dci_sweep(llr, np.array(SWEEP_CFI, np.uint32))
        valid = check_table(o, phy, llr, SWEEP_CFI, cands, distinct)
        got = [(L, si, rnti) for (i, li, L, si, rnti, b) in planted
               if (i, li, si) in valid and valid[(i, li, si)][1] == rnti and np.array_equal(valid[(i, li, si)][0], b)]
        levels = {L for (i, li, L, si, rnti, b) in planted}
        assert levels == {0, 1, 2, 3}, (nprb, ports, levels)
        assert {si for L, si, r in got} == set(distinct), (nprb, ports, "sizes never recovered", sorted(distinct[s] for s in set(distinct) - {si for L, si, r in got}))
        assert {L for L, si, r in got} == levels, (nprb, ports)
        assert set(SPECIAL_RNTIS) <= {r for L, si, r in got}, (nprb, ports)
        sizes_seen.update(distinct[si] for L, si, r in got)
        phy.close()
    assert len(sizes_seen) == 23, sorted(sizes_seen)


@pytest.mark.parametrize("kind", ["zero", "constant", "huge"])
@pytest.mark.parametrize("nprb,ports", STD_CELLS)
def test_dci_sweep_edge_blocks(infra, phylib, nprb, ports, kind):
    """zero: every candidate must come back invalid (max |x| = 0); constant: one value everywhere, then one magnitude with random signs, where
    the two competitors of many add-compare-select steps on the surviving path tie (the survivor is the lower predecessor; a single constant
    value has a unique best path and does not exercise that rule); huge: one value 1e4 among values of 1e-2 in each CCE (the uint8 quantiser
    puts almost everything at its midpoint)"""
    cell = Cell(nprb, ports, 5 * nprb + ports, 1)
    phy = capi.LtePhy(nprb, ports, cell.cell_id, 1, max_subframes=3)
    o = Oracle(cell)
    distinct = distinct_sizes(phy)
    cfis = [1, 2, 3]
    rng = np.random.default_rng(2000 + 10 * nprb + ports)
    llr = np.zeros((3, capi.LLR_STRIDE), np.float32)
    for i, cfi in enumerate(cfis):
        ncce = phy.nof_cce(cfi)
        if kind == "constant":
            llr[i, :72 * ncce] = 0.75 if i == 0 else np.where(rng.random(72 * ncce) < 0.5, 0.5 * i, -0.5 * i)
        elif kind == "huge":
            llr[i, :72 * ncce] = (0.01 * rng.standard_normal(72 * ncce)).astype(np.float32)
            for c in range(ncce):
                llr[i, 72 * c + int(rng.integers(0, 72))] = 1e4 if rng.random() < 0.5 else -1e4
    cands = phy.dci_sweep(llr, np.array(cfis, np.uint32))
    valid = check_table(o, phy, llr, cfis, cands, distinct)
    total = sum(len(phy.locations(cfi)[0]) for cfi in cfis) * len(distinct)
    if kind == "zero":
        assert not valid and not cands["valid"].any()
    else:
        assert len(valid) == total
    phy.close()


def turbo_sizes():
    """the 188 code-block sizes of 36.212 Table 5.1.3-3"""
    return list(range(40, 512, 8)) + list(range(512, 1024, 16)) + list(range(1024, 2048, 32)) + list(range(2048, 6145, 64))


def turbo_variant(K):
    """(threads per CTA, every window full) of the turbo_kernel instantiation that decodes K"""
    return 32 * ((K + 1023) // 1024), K % 32 == 0


def encode_blocks(S, rng, K, n, poly, snr):
    """n random code blocks with a CRC24 (poly) in their last 24 bits, turbo encoded, BPSK over AWGN at snr dB, scaled and clipped as
    the rate matcher delivers them (|d| <= 255) -> (int16 [n][3 (K + 4)], bits [n][K])"""
    D = K + 4
    d = np.zeros((n, 3 * D), np.int16)
    info = np.zeros((n, K), np.uint8)
    for i in range(n):
        b = rng.integers(0, 2, K).astype(np.uint8)
        crc = S.lte_crc(poly, 24, ltelib.ptr(b), K - 24)
        for j in range(24):
            b[K - 24 + j] = (crc >> (23 - j)) & 1
        info[i] = b
        enc = np.zeros(3 * D, np.uint8)
        S.lte_turbo_encode(ltelib.ptr(b), K, ltelib.ptr(enc[0:]), ltelib.ptr(enc[D:]), ltelib.ptr(enc[2 * D:]))
        x = (2.0 * enc - 1.0) + 10 ** (-snr / 20) * rng.standard_normal(3 * D)
        d[i] = np.clip(np.round(x * 60), -255, 255).astype(np.int16)
    return d, info


def oracle_turbo(O, d, K, max_iter, crc_type):
    n = d.shape[0]
    bits, iters, ok = np.zeros((n, K), np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.int32)
    for i in range(n):
        o = C.c_int(0)
        iters[i] = O.lteo_turbo_decode(ltelib.ptr(np.ascontiguousarray(d[i])), K, max_iter, crc_type, ltelib.ptr(bits[i]), C.byref(o))
        ok[i] = o.value
    return bits, iters, ok


def check_turbo(phy, O, d, K, max_iter, crc_type, what):
    bits, iters, ok = phy.turbo_batch(d, K, max_iter, crc_type)
    ob, oit, ook = oracle_turbo(O, d, K, max_iter, crc_type)
    for i in range(d.shape[0]):
        assert np.array_equal(bits[i], ob[i]), "%s K=%d cb %d crc_type %d: %d bits differ from the oracle" % (what, K, i, crc_type, int((bits[i] != ob[i]).sum()))
        assert (int(iters[i]), int(ok[i])) == (int(oit[i]), int(ook[i])), (what, K, i, crc_type, int(iters[i]), int(oit[i]), int(ok[i]), int(ook[i]))
    return ob, oit, ook


# SNR (dB) by position in the K table: from where most blocks fail all 8 iterations to where most stop after one or two
TURBO_SNR = [-1.8, -1.2, -0.6, 0.2, 1.0]


def test_turbo_every_block_size(infra, phylib):
    """three noisy code blocks per K (pairs (0, 1) and (2, idle)); even table positions carry CRC24A and stop early on it, odd ones CRC24B;
    every K is decoded again with crc_type 0 (8 iterations, no early stop)"""
    S, O = infra.sim(), infra.oracle()
    S.lte_turbo_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    Ks = turbo_sizes()
    assert len(Ks) == 188 and Ks[-1] == 6144
    phy = capi.LtePhy(100, 1, 1, 1, max_subframes=1)
    iter_counts, split_pair, failed, variants, passed = set(), 0, 0, set(), 0
    for n, K in enumerate(Ks):
        rng = np.random.default_rng(K)
        crc_type, poly = (1, CRC24A) if n % 2 == 0 else (2, CRC24B)
        d, info = encode_blocks(S, rng, K, 3, poly, TURBO_SNR[n % len(TURBO_SNR)])
        ob, oit, ook = check_turbo(phy, O, d, K, 8, crc_type, "early stop")
        iter_counts.update(int(x) for x in oit)
        split_pair += int(oit[0] != oit[1])
        failed += int(((oit == 8) & (ook == 0)).sum())
        passed += int(sum(np.array_equal(ob[i], info[i]) for i in range(3) if ook[i]))
        check_turbo(phy, O, d, K, 8, 0, "fixed iterations")
        variants.add(turbo_variant(K))
    phy.close()
    assert variants == {(32, False), (32, True), (64, True), (96, True), (128, True), (160, True), (192, True)}
    assert len(iter_counts) >= 4, sorted(iter_counts)
    assert split_pair >= 5 and failed >= 20 and passed >= 188, (split_pair, failed, passed)


@pytest.mark.parametrize("kind", ["zero", "noiseless"])
def test_turbo_extreme_inputs(infra, phylib, kind):
    """zero: L = 0 everywhere, so every hard decision is the tie rule's (bit = 0, and CRC24 of all zeros passes); noiseless: +-255 on every
    input, the largest metrics the int16 arithmetic has to hold.  Every K, three blocks, CRC24B early stop and 8 fixed iterations."""
    S, O = infra.sim(), infra.oracle()
    S.lte_turbo_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    phy = capi.LtePhy(100, 1, 1, 1, max_subframes=1)
    for K in turbo_sizes():
        rng = np.random.default_rng(K + 7)
        if kind == "zero":
            d, info = np.zeros((3, 3 * (K + 4)), np.int16), np.zeros((3, K), np.uint8)
        else:
            d, info = encode_blocks(S, rng, K, 3, CRC24B, 200.0)
            d = np.where(d > 0, 255, -255).astype(np.int16)
        for max_iter, crc_type in ((8, 2), (8, 0)):
            ob, oit, ook = check_turbo(phy, O, d, K, max_iter, crc_type, kind)
            assert np.array_equal(ob, info), (kind, K, crc_type)
            if crc_type:
                assert (oit == 1).all() and (ook == 1).all(), (kind, K)
    phy.close()
