"""GPU parity tests (pytest -m gpu): every stage of the CUDA path against the CPU oracle on the same
seeded captures, through the C-ABI.  Bar: bit-exact (float stages included: the oracle fixes the
evaluation order and the kernels are built with -fmad=false)."""
import ctypes as C
import numpy as np
import pytest

import ltelib
from ltelib import Cell, Oracle, FORMATS
from helpers import make_capture, oracle_frontend, to_phy_grant, truth_grants, feq, describe_mismatch
from ltesniffer_b200 import capi

pytestmark = pytest.mark.gpu

CASES = {
    "20MHz_1p1a": dict(cell=Cell(100, 1, 1, 1), n=3, kw=dict(seed=11, cfi=2, nof_ues=4, dl_min=1, dl_max=2, tm=1, mcs_min=3, mcs_max=9, snr_db=28.0, si_period=2)),
    "20MHz_2p2a_tm3": dict(cell=Cell(100, 2, 7, 2), n=3, kw=dict(seed=12, cfi=3, nof_ues=30, dl_min=6, dl_max=10, ul_min=1, ul_max=3, tm=3, mcs_min=10, mcs_max=24, snr_db=27.0, full_band=1, chan_delay=4)),
    "10MHz_2p2a_mix": dict(cell=Cell(50, 2, 301, 2), n=4, kw=dict(seed=13, cfi=3, nof_ues=12, dl_min=3, dl_max=5, ul_min=1, ul_max=2, tm=13, mcs_min=0, mcs_max=22, snr_db=24.0, chan_delay=6, tti0=4)),
    "10MHz_tm4_256qam": dict(cell=Cell(50, 2, 11, 2), n=3, kw=dict(seed=15, cfi=2, nof_ues=8, dl_min=2, dl_max=4, tm=4, mcs_min=4, mcs_max=22, snr_db=33.0, alt_table=1)),
    "10MHz_tm3_tm4_cw_swap": dict(cell=Cell(50, 2, 21, 2), n=4, kw=dict(seed=16, cfi=2, nof_ues=8, dl_min=2, dl_max=4, tm=3, mcs_min=6, mcs_max=24, snr_db=29.0, tb_swap=1)),
    "10MHz_tm4_cw_swap": dict(cell=Cell(50, 2, 11, 2), n=3, kw=dict(seed=17, cfi=2, nof_ues=8, dl_min=2, dl_max=4, tm=4, mcs_min=4, mcs_max=20, snr_db=33.0, tb_swap=1)),
    "5MHz_2p1a": dict(cell=Cell(25, 2, 150, 1), n=3, kw=dict(seed=14, cfi=2, nof_ues=5, dl_min=1, dl_max=3, tm=1, mcs_min=2, mcs_max=12, snr_db=25.0, tti0=9)),
    # Cell(nof_prb, ports, cell id, antennas, symbol size (0: the standard one), phich-Resource Ng (0..3 = 1/6, 1/2, 1, 2), phich-Duration extended).
    # Every case decodes subframe 0 or 5: PBCH / synchronisation REs cut PRBs in half there at odd PRB counts.
    "3MHz_1p1a_cfi3": dict(cell=Cell(15, 1, 31, 1), n=3, kw=dict(seed=41, cfi=3, nof_ues=4, dl_min=1, dl_max=3, tm=1, mcs_min=2, mcs_max=20, snr_db=28.0, si_period=2, tti0=4)),
    "3MHz_2p2a_384": dict(cell=Cell(15, 2, 32, 2, 384), n=3, kw=dict(seed=42, cfi=2, nof_ues=4, dl_min=1, dl_max=3, tm=13, mcs_min=2, mcs_max=20, snr_db=28.0, tti0=9)),
    "15MHz_2p2a_mix_delay": dict(cell=Cell(75, 2, 301, 2), n=3, kw=dict(seed=43, cfi=3, nof_ues=12, dl_min=3, dl_max=6, ul_min=1, ul_max=2, tm=13, mcs_min=0, mcs_max=24, snr_db=25.0, chan_delay=5)),
    "15MHz_1p1a_1536": dict(cell=Cell(75, 1, 76, 1, 1536), n=3, kw=dict(seed=44, cfi=2, nof_ues=6, dl_min=2, dl_max=4, tm=1, mcs_min=2, mcs_max=24, snr_db=28.0, tti0=5)),
    "15MHz_tm4_256qam_1024": dict(cell=Cell(75, 2, 77, 2, 1024), n=3, kw=dict(seed=45, cfi=2, nof_ues=8, dl_min=2, dl_max=4, tm=4, mcs_min=4, mcs_max=22, snr_db=33.0, alt_table=1, tti0=9)),
    "10MHz_1p1a": dict(cell=Cell(50, 1, 9, 1), n=3, kw=dict(seed=46, cfi=2, nof_ues=6, dl_min=2, dl_max=4, tm=1, mcs_min=2, mcs_max=24, snr_db=27.0, si_period=3)),
    "20MHz_ng2": dict(cell=Cell(100, 2, 301, 2, 0, 3), n=3, kw=dict(seed=47, cfi=2, nof_ues=10, dl_min=3, dl_max=6, tm=3, mcs_min=4, mcs_max=22, snr_db=27.0, tti0=4)),
    "5MHz_ng1_ext_cfi3": dict(cell=Cell(25, 2, 150, 2, 0, 2, 1), n=3, kw=dict(seed=48, cfi=3, nof_ues=5, dl_min=1, dl_max=3, tm=13, mcs_min=2, mcs_max=20, snr_db=27.0, tti0=5)),
    "15MHz_ng_half_ext": dict(cell=Cell(75, 2, 17, 2, 0, 1, 1), n=3, kw=dict(seed=49, cfi=3, nof_ues=8, dl_min=2, dl_max=5, tm=3, mcs_min=2, mcs_max=22, snr_db=27.0, tti0=9)),
}


def new_phy(cell, n, flags=0):
    return capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8, flags=flags, symbol_sz=cell.symbol_sz,
                       phich_resources=cell.phich_ng, phich_length=cell.phich_ext)


def new_search(cell):
    return capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, phich_resources=cell.phich_ng | (cell.phich_ext << 8))


@pytest.fixture(scope="module", params=list(CASES))
def case(request, infra, phylib):
    c = CASES[request.param]
    cell = c["cell"]
    sim, iq, tti, truths, payloads = make_capture(cell, c["n"], **c["kw"])
    o = Oracle(cell)
    ref = oracle_frontend(o, iq, tti)
    assert any(int(t) % 5 == 0 for t in tti), "every case decodes subframe 0 or 5"
    phy = new_phy(cell, c["n"])
    phy.submit_iq(iq, tti)
    info, cands = phy.get_phase_a()
    yield dict(name=request.param, alt=c["kw"].get("alt_table", 0), cell=cell, iq=iq, tti=tti, truths=truths, payloads=payloads, o=o, ref=ref, phy=phy, info=info, cands=cands, n=c["n"])
    phy.close()


def test_ofdm_bit_exact(case):
    n, cell, phy = case["n"], case["cell"], case["phy"]
    sym = phy.tap(capi.TAP_SYM, (n, cell.nof_rx, 14 * phy.nsc), np.complex64)
    for i in range(n):
        assert feq(sym[i], case["ref"][i]["sym"]), describe_mismatch(sym[i], case["ref"][i]["sym"], "sym sf%d" % i)


def test_chest_bit_exact(case):
    n, cell, phy = case["n"], case["cell"], case["phy"]
    ce = phy.tap(capi.TAP_CE, (n, cell.nof_ports * cell.nof_rx, 14 * phy.nsc), np.complex64)
    for i in range(n):
        r = case["ref"][i]
        assert feq(ce[i], r["ce"]), describe_mismatch(ce[i], r["ce"], "ce sf%d" % i)
        inf, res = case["info"][i], r["res"]
        for p in range(cell.nof_ports):
            for a in range(cell.nof_rx):
                assert inf.noise[p][a] == res.noise[p][a] and inf.rsrp[p][a] == res.rsrp[p][a], (i, p, a, inf.noise[p][a], res.noise[p][a])
        assert (inf.noise_avg, inf.rsrp_avg, inf.cfo_re, inf.cfo_im) == (res.noise_avg, res.rsrp_avg, res.cfo_re, res.cfo_im)
        assert inf.snr_db == res.snr_db and inf.cfo == res.cfo
        assert feq(np.array(inf.rb_power[:cell.nof_prb], np.float32), r["rb_power"])


def test_pcfich_pdcch_llr_bit_exact(case):
    n, phy = case["n"], case["phy"]
    llr = phy.tap(capi.TAP_LLR, (n, capi.LLR_STRIDE), np.float32)
    for i in range(n):
        r, inf = case["ref"][i], case["info"][i]
        assert inf.cfi == r["cfi"] == case["truths"][i].cfi
        assert feq(np.array(inf.pcfich_corr[:], np.float32), r["corr"])
        ncce = len(r["llr"]) // 72
        assert inf.nof_cce == ncce
        assert feq(llr[i, :72 * ncce], r["llr"]), describe_mismatch(llr[i, :72 * ncce], r["llr"], "pdcch llr sf%d" % i)
        assert feq(np.array(inf.cce_power[:ncce], np.float32), r["cce_power"])


def test_dci_table_bit_exact(case):
    """full blind-decode table vs one oracle decode per (location, size); truth DCIs must be in it"""
    n, phy, o = case["n"], case["phy"], case["o"]
    sizes, sidx = phy.sizes()
    distinct = {}
    for f in range(9):
        distinct[sidx[f]] = sizes[f]
    nchecked = total = 0
    for i in range(n):
        r = case["ref"][i]
        nc, Ls = phy.locations(r["cfi"])
        assert case["info"][i].nof_locations == len(nc)
        total += len(nc) * len(distinct)
        for li in range(len(nc)):
            e = r["llr"][72 * int(nc[li]):72 * int(nc[li]) + (72 << int(Ls[li]))]
            for si, nb in distinct.items():
                ret, bits, crc = o.dci_decode(e, nb)
                c = case["cands"][i, li, si]
                if ret != 0:
                    assert c["valid"] == 0
                    continue
                assert c["valid"] == 1
                assert int(c["rnti"]) == crc, (i, li, si, hex(int(c["rnti"])), hex(crc))
                assert np.array_equal(capi.cand_bits(c["bits"], nb), bits), (i, li, si)
                nchecked += 1
        tr = case["truths"][i]
        for k in range(tr.nof_dci):
            d = tr.dci[k]
            li = [j for j in range(len(nc)) if nc[j] == d.ncce and Ls[j] == d.L]
            if not li:
                continue  # placed beyond the first 84 CCEs
            c = case["cands"][i, li[0], sidx[d.format]]
            assert int(c["rnti"]) == d.rnti, "truth DCI not recovered: sf %d rnti %#x fmt %s" % (i, d.rnti, FORMATS[d.format])
            assert np.array_equal(capi.cand_bits(c["bits"], d.nbits), np.frombuffer(bytes(d.bits), np.uint8)[:d.nbits])
    assert nchecked >= 0.9 * total, (nchecked, total)     # only an all-zero location decodes to nothing


@pytest.mark.parametrize("flags", [0, capi.FLAG_SKIP_LOW_POWER])
def test_survivor_form_matches_host_restatement(case, flags):
    """cand_compact_kernel (search-space validation, zero-RNTI and parent-match tests on the GPU) against
    ltephy_compact_from_table applied to the GPU's own full table: same counts, location records and listed entries;
    and the walk over the survivor form accepts what the walk over the full table accepts."""
    cell, n = case["cell"], case["n"]
    phy = new_phy(cell, n, flags)
    phy.submit_iq(case["iq"], case["tti"])
    info, cands = phy.get_phase_a()
    info_c, comp = phy.get_phase_a_compact()
    assert bytes(info) == bytes(info_c)
    sa = new_search(cell)
    sb = new_search(cell)
    total = 0
    for i in range(n):
        ref = sa.compact_from_table(info[i], cands[i])[0]
        got = comp[i]
        assert int(got["count"]) == int(ref["count"]) and int(got["count"]) <= capi.COMPACT_CAP, (i, int(got["count"]), int(ref["count"]))
        assert got["loc"].tobytes() == ref["loc"].tobytes(), (i, "location records differ")
        k = int(ref["count"])
        assert got["list"][:k].tobytes() == ref["list"][:k].tobytes(), (i, "listed entries differ")
        total += k
        for _ in range(3):     # a few repetitions so that the RNTI histogram crosses its threshold and DCIs are accepted
            a = sa.subframe(info[i], cands[i])
            b = sb.subframe_compact(info[i], comp[i:i + 1])
            assert b is not None and len(a) == len(b) and all(np.array_equal(a[f], b[f]) for f in a.dtype.names)
    assert total > 0
    phy.close()


def test_pdsch_llr_and_tb_bit_exact(case):
    cell, phy, o = case["cell"], case["phy"], case["o"]
    tg = truth_grants(cell, case["truths"], case["tti"], case["alt"])
    if not tg:
        pytest.skip("no DL grants in this capture")
    grants = [to_phy_grant(sf, d.rnti, g) for sf, d, g in tg]
    phy.submit_grants(grants)
    res, pl = phy.get_phase_b()
    # int16 LLRs of every codeword, in submission order
    total = sum(((g.nof_re * g.tb[t].qm + 7) & ~7) for _, _, g in tg for t in range(2) if g.tb[t].enabled)
    gl = phy.tap(capi.TAP_PDSCH_LLR, (total,), np.int16)
    off = 0
    nbad_truth = 0
    for gi, (sf, d, g) in enumerate(tg):
        r = case["ref"][sf]
        ret, ollr, _ = o.pdsch_llr(int(case["tti"][sf]) % 10, r["cfi"], d.rnti, g, r["sym"], r["ce"])
        assert ret == 0
        ret, opl, ook = o.pdsch_decode(int(case["tti"][sf]) % 10, r["cfi"], d.rnti, g, r["sym"], r["ce"], 8)
        cw = 0
        for t in range(2):
            if not g.tb[t].enabled:
                continue
            G = g.nof_re * g.tb[t].qm
            ocw = (1 - cw) if (g.nof_tb == 2 and g.cw_swap) else cw     # the oracle indexes LLRs by CODEWORD, the pool is in TB order
            assert np.array_equal(gl[off:off + G], ollr[ocw][:G]), describe_mismatch(gl[off:off + G], ollr[ocw][:G], "pdsch llr grant %d cw %d" % (gi, ocw))
            off += (G + 7) & ~7
            cw += 1
            rr = res[2 * gi + t]
            nby = g.tb[t].tbs // 8
            assert rr.payload_len == nby
            assert rr.crc == ook[t], "crc differs from oracle: grant %d tb %d gpu %d oracle %d" % (gi, t, rr.crc, ook[t])
            assert np.array_equal(pl[rr.payload_off:rr.payload_off + nby], opl[t][:nby]), "payload differs from oracle grant %d tb %d" % (gi, t)
            if rr.crc:
                tp = case["payloads"][sf][d.payload_off[t]:d.payload_off[t] + nby]
                assert np.array_equal(pl[rr.payload_off:rr.payload_off + nby], tp), "CRC ok but payload != transmitted"
            else:
                nbad_truth += 1
    assert nbad_truth <= max(1, len(tg) // 4), "too many undecodable transport blocks: %d" % nbad_truth


@pytest.mark.parametrize("K,ncb,snr", [(40, 5, 2.0), (512, 4, 1.0), (1056, 3, 0.5), (5824, 13, 0.5), (6144, 4, 0.0)])
def test_turbo_batch_bit_exact(infra, phylib, K, ncb, snr):
    """stand-alone K8: random code blocks through the reference encoder + AWGN, conditioned int16"""
    S = infra.sim()
    rng = np.random.default_rng(K)
    D = K + 4
    d = np.zeros((ncb, 3 * D), np.int16)
    info = np.zeros((ncb, K), np.uint8)
    S.lte_turbo_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    for i in range(ncb):
        b = rng.integers(0, 2, K).astype(np.uint8)
        crc = S.lte_crc(0x1800063, 24, ltelib.ptr(b), K - 24)
        for j in range(24):
            b[K - 24 + j] = (crc >> (23 - j)) & 1
        info[i] = b
        enc = np.zeros(3 * D, np.uint8)
        S.lte_turbo_encode(ltelib.ptr(b), K, ltelib.ptr(enc[0:]), ltelib.ptr(enc[D:]), ltelib.ptr(enc[2 * D:]))
        sigma = 10 ** (-snr / 20)
        x = (2.0 * enc - 1.0) + sigma * rng.standard_normal(3 * D)
        d[i] = np.clip(np.round(x * 60), -255, 255).astype(np.int16)
    phy = capi.LtePhy(100, 1, 1, 1, max_subframes=1)
    for max_iter, crc_type in [(4, 2), (3, 0)]:
        bits, iters, ok = phy.turbo_batch(d, K, max_iter, crc_type)
        O = infra.oracle()
        for i in range(ncb):
            ob = np.zeros(K, np.uint8)
            ook = C.c_int(0)
            oit = O.lteo_turbo_decode(ltelib.ptr(d[i]), K, max_iter, crc_type, ltelib.ptr(ob), C.byref(ook))
            assert np.array_equal(bits[i], ob), "K=%d cb %d: %d bits differ from oracle" % (K, i, int((bits[i] != ob).sum()))
            assert iters[i] == oit and ok[i] == ook.value, (K, i, iters[i], oit, ok[i], ook.value)
    phy.close()


def test_dci_sweep_matches_oracle(infra, phylib):
    """config-3 style: LLR buffers synthesised directly (30 % valid DCIs, rest noise), small batch"""
    S = infra.sim()
    cell = Cell(100, 2, 1, 1)
    phy = capi.LtePhy(100, 2, 1, 1, max_subframes=4)
    o = Oracle(cell)
    rng = np.random.default_rng(3)
    n = 4
    sizes, sidx = phy.sizes()
    llr = (0.3 * rng.standard_normal((n, capi.LLR_STRIDE))).astype(np.float32)
    ncce = phy.nof_cce(3)
    llr[:, 72 * ncce:] = 0
    planted = []
    for i in range(n):
        c = 0
        while c + 8 <= 80:
            L = int(rng.integers(0, 4))
            c = (c + (1 << L) - 1) // (1 << L) * (1 << L)
            if rng.random() < 0.3 and c + (1 << L) <= 84:
                f = int(rng.choice([0, 1, 2, 4, 6, 7]))
                nb = sizes[f]
                b = rng.integers(0, 2, nb).astype(np.uint8)
                rnti = int(rng.integers(1, 65535))
                e = np.zeros(72 << L, np.uint8)
                S.lte_sim_pdcch_encode(ltelib.ptr(b), nb, rnti, L, ltelib.ptr(e))
                llr[i, 72 * c:72 * c + (72 << L)] = (2.0 * e - 1.0) + 0.3 * rng.standard_normal(72 << L)
                planted.append((i, c, L, f, rnti, b))
            c += 1 << L
    cands = phy.dci_sweep(llr, np.full(n, 3, np.uint32))
    nc, Ls = phy.locations(3)
    assert len(nc) == 157
    for (i, c, L, f, rnti, b) in planted:
        li = [j for j in range(len(nc)) if nc[j] == c and Ls[j] == L][0]
        cd = cands[i, li, sidx[f]]
        assert int(cd["rnti"]) == rnti and np.array_equal(capi.cand_bits(cd["bits"], len(b)), b)
    for i in range(n):
        for li in range(0, len(nc), 7):
            e = llr[i, 72 * int(nc[li]):72 * int(nc[li]) + (72 << int(Ls[li]))]
            for f in range(9):
                ret, bits, crc = o.dci_decode(e, sizes[f])
                cd = cands[i, li, sidx[f]]
                assert ret == 0 and cd["valid"] == 1 and int(cd["rnti"]) == crc and np.array_equal(capi.cand_bits(cd["bits"], sizes[f]), bits)
    phy.close()
