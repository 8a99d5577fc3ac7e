"""The GPU decoders held directly to the integer references of tests/ref_dec.py (written from 36.212 and DESIGN.md §2), not through the oracle:
  * dci_viterbi_kernel (ltephy_dci_sweep, which decodes every location): every byte of the candidate table against dci_decode_ref, on LLR
    buffers of every input kind of tests/test_decoder_reference.py, the quantiser's scale and NaN cases, and full-scale patterns that spread the
    path metrics as far as they go (the +765 branch bias and the renormalisation to (state 0) - 9180 every 5 steps must stay invisible);
  * the same kernel in phase A with FLAG_SKIP_LOW_POWER, where the work list leaves out locations below the CCE power floor: decoded entries
    against dci_decode_ref on the tapped PDCCH LLRs, skipped locations all zero;
  * turbo_kernel (ltephy_turbo_batch) at all 188 K on the turbo input kinds, with CRC early stop and fixed iteration counts: bits, iterations, crc;
  * phase B (K7 rate dematch, K8, tb_crc_kernel) on low-SNR downlink and uplink captures: crc, avg_iters, nof_cb and payload of every transport
    block against dlsch_decode_ref on the tapped soft bits;
  * ltephy_mib_decode_combined against the combining loop of tests/mib_lib.py, which decodes with pbch_hyp_ref."""
import ctypes as C

import numpy as np
import pytest

import ltelib
import mib_lib as M
import ref_dec
from helpers import make_capture, to_phy_grant, truth_grants
from ltelib import Cell
from ltesniffer_b200 import capi
from test_decoder_reference import crafted_codeword, dci_inputs, turbo_inputs, turbo_sizes
from test_float64_reference import Case
from test_gpu_pbch_combining import PLAN, expected, run_gpu, sequence

pytestmark = pytest.mark.gpu

SWEEP_KINDS = ("noise", "planted", "ties", "single", "full_scale", "zero", "scale_lo", "scale_hi", "tiny", "denormal", "overflow", "nan",
               "spread_const", "spread_alt", "huge")


def sweep_llr(S, rng, phy, cfis):
    """one LLR buffer per kind: the kind fills every CCE of the subframe"""
    llr = np.zeros((len(SWEEP_KINDS), capi.LLR_STRIDE), np.float32)
    for i, (kind, cfi) in enumerate(zip(SWEEP_KINDS, cfis)):
        n = 72 * phy.nof_cce(cfi)
        x = np.zeros(n, np.float64)
        if kind in ("noise", "ties", "full_scale", "zero"):
            x = dci_inputs(S, rng, 10, 72, n // 72)[0][kind][:n // 72].ravel() if kind != "zero" else x
        elif kind == "planted":                                       # DCIs in level-0 / level-2 blocks, clean to noisy
            x = rng.standard_normal(n) * 0.8
            for c in range(0, n // 72 - 3, 4):
                L = 2 if c % 8 == 0 else 0
                e = np.zeros(72 << L, np.uint8)
                nb = int(rng.choice([27, 31, 43, 51]))
                S.lte_sim_pdcch_encode(ltelib.ptr(rng.integers(0, 2, nb).astype(np.uint8)), nb, int(rng.integers(0, 0x10000)), L, ltelib.ptr(e))
                x[72 * c:72 * c + len(e)] = (2.0 * e - 1.0) + rng.uniform(0, 1.2) * rng.standard_normal(len(e))
        elif kind == "single":                                        # one non-zero soft bit per CCE
            x[72 * np.arange(n // 72) + rng.integers(0, 72, n // 72)] = rng.choice([-3.0, 0.5, 7.0], n // 72)
        elif kind in ("scale_lo", "scale_hi"):                        # integers scaled by 2^-122 / 2^115: near the edges of the exact range
            x = rng.integers(-8, 9, n) * 2.0 ** (-122 if kind == "scale_lo" else 115)
        elif kind in ("tiny", "denormal", "overflow"):                # max|x| ~ 1e-38, 1e-39 (gain overflows), 1e38 (the sums overflow)
            x = np.where(rng.random(n) < 0.5, -1, 1) * rng.uniform(0.5, 1, n) * {"tiny": 1e-38, "denormal": 1e-39, "overflow": 1e38}[kind]
            x[rng.random(n) < 0.2] = 0
        elif kind == "nan":
            x = rng.standard_normal(n)
            x[rng.integers(0, n, n // 50)] = np.nan
        elif kind == "spread_const":                                  # one path far ahead of all others
            x[:] = 1e4
        elif kind == "spread_alt":                                    # full scale with long runs of equal sign
            x = np.where((np.arange(n) // int(rng.integers(3, 40))) % 2 == 0, 1.0, -1.0) * 255
        else:
            x = 0.01 * rng.standard_normal(n)
            x[72 * np.arange(n // 72) + rng.integers(0, 72, n // 72)] = 1e4
        llr[i, :n] = np.asarray(x, np.float32)
    return llr


def expected_table(phy, llr, cfis, cce_power=None):
    """the candidate table dci_decode_ref gives for llr [n][LLR_STRIDE]; with cce_power [n][MAX_CCE], locations with a CCE below the power
    floor 0.7 (the FLAG_SKIP_LOW_POWER rule of §1a) are left all zero"""
    sizes, sidx = phy.sizes()
    distinct = {sidx[f]: sizes[f] for f in range(capi.NOF_FORMATS)}
    want = np.zeros((len(cfis), capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
    shift = np.array([1 << (63 - b) for b in range(64)], np.uint64)
    for i, cfi in enumerate(cfis):
        nc, Ls = phy.locations(cfi)
        for L in sorted(set(Ls.tolist())):
            li = np.nonzero(Ls == L)[0]
            if cce_power is not None:
                li = np.array([j for j in li if (cce_power[i][int(nc[j]):int(nc[j]) + (1 << L)] >= np.float32(0.7)).all()], np.int64)
                if len(li) == 0:
                    continue
            e = np.stack([llr[i, 72 * int(nc[j]):72 * int(nc[j]) + (72 << L)] for j in li])
            for si, nb in distinct.items():
                v, b, rem = ref_dec.dci_decode_ref(e, nb)
                packed = np.bitwise_or.reduce(np.where(b.astype(bool), shift[:nb], np.uint64(0)), axis=1)
                for k, j in enumerate(li):
                    if v[k]:
                        want[i, j, si]["bits"], want[i, j, si]["rnti"], want[i, j, si]["valid"] = packed[k], rem[k], 1
    return want


def assert_table_equal(got, want, names, cfis):
    for i, name in enumerate(names):
        bad = np.argwhere(got[i].view(np.uint8).reshape(capi.MAX_LOC, capi.MAX_SIZES, 16) != want[i].view(np.uint8).reshape(capi.MAX_LOC, capi.MAX_SIZES, 16))
        assert bad.size == 0, "%s (cfi %d): %d bytes differ, first at location %d size %d" % (name, cfis[i], len(bad), bad[0][0], bad[0][1])


@pytest.mark.parametrize("nprb,ports", [(15, 1), (50, 2), (100, 2)])
def test_dci_sweep_equals_reference(infra, phylib, nprb, ports):
    S = infra.sim()
    rng = np.random.default_rng(300 + nprb)
    cfis = [1 + i % 3 for i in range(len(SWEEP_KINDS))]
    probe = capi.LtePhy(nprb, ports, 7, 1, max_subframes=len(cfis))
    llr = sweep_llr(S, rng, probe, cfis)
    want = expected_table(probe, llr, cfis)
    probe.close()
    phy = capi.LtePhy(nprb, ports, 7, 1, max_subframes=len(cfis))
    got = phy.dci_sweep(llr, np.array(cfis, np.uint32))
    counts = [len(phy.locations(c)[0]) for c in (1, 2, 3)]
    phy.close()
    assert_table_equal(got, want, SWEEP_KINDS, cfis)
    assert len({c % 2 for c in counts}) == 2, counts                  # an odd location count leaves a single-candidate item
    nvalid = {k: int(want[i]["valid"].sum()) for i, k in enumerate(SWEEP_KINDS)}
    assert nvalid["zero"] == 0 and all(nvalid[k] > 0 for k in SWEEP_KINDS if k != "zero"), nvalid


def test_phase_a_skipping_low_power_locations_equals_reference(infra, phylib):
    """a capture with a few DCIs per subframe through phase A with FLAG_SKIP_LOW_POWER: CCEs without a DCI fall below the power floor, so the
    work list holds an odd or even number of the locations, or none; every entry against dci_decode_ref on the tapped PDCCH LLRs"""
    cell = Cell(100, 2, 7, 2)
    n = 6
    sim, iq, tti, truths, payloads = make_capture(cell, n, seed=23, cfi=3, nof_ues=20, dl_min=0, dl_max=4, tm=1, mcs_min=5, mcs_max=9, snr_db=25.0)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, flags=capi.FLAG_SKIP_LOW_POWER)
    try:
        phy.submit_iq(iq, tti)
        info, got = phy.get_phase_a()
        llr = phy.tap(capi.TAP_LLR, (n, capi.LLR_STRIDE), np.float32)
        cfis = [int(info[i].cfi) for i in range(n)]
        power = [np.array(info[i].cce_power[:], np.float32) for i in range(n)]
        want = expected_table(phy, llr, cfis, power)
        decodable, nloc = [], []
        for i in range(n):
            nc, Ls = phy.locations(cfis[i])
            nloc.append(len(nc))
            decodable.append(sum(1 for c, L in zip(nc, Ls) if (power[i][int(c):int(c) + (1 << int(L))] >= np.float32(0.7)).all()))
    finally:
        phy.close()
    assert_table_equal(got, want, ["subframe %d" % i for i in range(n)], cfis)
    assert any(d % 2 == 1 for d in decodable) and any(d > 0 and d % 2 == 0 for d in decodable), decodable
    assert all(d < m for d, m in zip(decodable, nloc)), (decodable, nloc)                  # every subframe skips some locations


def test_turbo_batch_equals_reference_at_every_block_size(infra, phylib):
    """per K nine blocks of the turbo input kinds (four pairs and one idle half; two CRC types, so pair halves stop at different iterations),
    once with CRC early stop at 8 iterations and once at a fixed count 1..8"""
    S = infra.sim()
    S.lte_turbo_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    phy = capi.LtePhy(100, 1, 1, 1, max_subframes=1)
    split, iters_seen = 0, set()
    for n, K in enumerate(turbo_sizes()):
        rng = np.random.default_rng(70000 + K)
        d = np.concatenate([turbo_inputs(S, rng, K, n)[0], turbo_inputs(S, rng, K, n + 1)[0][:-2]])   # 8 blocks: four pairs
        d = np.concatenate([d, d[:1]])                                                             # 9: one idle half
        for max_iter, crc_type in ((8, 1 + n % 2), (1 + n % 8, 0)):
            bits, iters, ok = phy.turbo_batch(d, K, max_iter, crc_type)
            rb, ri, ro = ref_dec.turbo_decode_ref(d, K, max_iter, crc_type)
            for i in range(len(d)):
                assert np.array_equal(bits[i], rb[i]) and (int(iters[i]), bool(ok[i])) == (int(ri[i]), bool(ro[i])), (
                    K, i, max_iter, crc_type, int((bits[i] != rb[i]).sum()), int(iters[i]), int(ri[i]), int(ok[i]), bool(ro[i]))
            if crc_type:
                split += sum(int(ri[2 * p] != ri[2 * p + 1]) for p in range(4))
                iters_seen.update(int(x) for x in ri)
    phy.close()
    assert split >= 100 and iters_seen == set(range(1, 9)), (split, sorted(iters_seen))


def _ref_tb(llr, G, tbs, rv, qm, NL):
    crc, payload, iters, _ = ref_dec.dlsch_decode_ref(llr[:G], G, tbs, rv, qm, NL, 8, 1)
    return crc, payload, -(-int(iters.sum()) // len(iters)), len(iters)


def _check(res, pl, want):
    for slot, (crc, payload, avg, ncb) in want:
        rr = res[slot]
        assert (bool(rr.crc), int(rr.avg_iters), int(rr.nof_cb)) == (crc, avg, ncb), (slot, rr.crc, crc, rr.avg_iters, avg, rr.nof_cb, ncb)
        assert np.array_equal(pl[rr.payload_off:rr.payload_off + len(payload)], payload), slot


def test_phase_b_downlink_equals_reference_at_low_snr(infra, phylib):
    cell = Cell(100, 2, 7, 2)
    sim, iq, tti, truths, payloads = make_capture(cell, 2, seed=31, cfi=3, nof_ues=12, dl_min=4, dl_max=6, tm=3, mcs_min=14, mcs_max=28,
                                                  snr_db=17.0, full_band=1)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=2, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
    try:
        phy.submit_iq(iq, tti)
        phy.get_phase_a()
        grants = [to_phy_grant(sf, d.rnti, g) for sf, d, g in truth_grants(cell, truths, tti)]
        phy.submit_grants(grants)
        res, pl = phy.get_phase_b()
        total = sum(((g.nof_re * g.tb[t].qm + 7) & ~7) for g in grants for t in range(2) if g.tb[t].enabled)
        llr = phy.tap(capi.TAP_PDSCH_LLR, (total,), np.int16)
        want, off = [], 0
        for gi, g in enumerate(grants):
            for t in range(2):
                if not g.tb[t].enabled:
                    continue
                G = g.nof_re * g.tb[t].qm
                want.append((2 * gi + t, _ref_tb(llr[off:], G, g.tb[t].tbs, g.tb[t].rv, g.tb[t].qm, 2 if g.tx_scheme == capi.TX_DIVERSITY else 1)))
                off += (G + 7) & ~7
        _check(res, pl, want)
        crcs = [w[1][0] for w in want]
        avgs = {w[1][2] for w in want}
        assert any(crcs) and not all(crcs) and len(avgs) >= 3 and max(w[1][3] for w in want) > 1, (crcs, avgs)
    finally:
        phy.close()


def test_phase_b_uplink_equals_reference(infra, phylib):
    cell = Cell(50, 1, 9, 1)
    ucfg = ltelib.UlCfg(n_dmrs1=3, delta_ss=2)
    s = ltelib.Sim(cell=cell, seed=8, snr_db=9.0, nof_ues=1)                 # some transport blocks fail, the rest need 1 to 3 iterations
    rng = np.random.default_rng(8)
    iq = np.zeros((2, s.sf_len), np.complex64)
    grants, cg = [], []
    for i in range(2):
        gr = ltelib.make_ul_grants(cell, rng, 4, table=1)
        iq[i] = ltelib.sim_ul_subframe(s, i, ucfg, gr)[0]
        grants += gr
        cg += [capi.UlGrant(sf=i, rnti=g.rnti, qm=g.qm, rv=g.rv, L_prb=g.L_prb, n_prb=g.n_prb, n_dmrs2=g.n_dmrs2, tbs=g.tbs, n_prb_slot1=g.n_prb,
                            flags=capi.UL_FLAG_SLOT1, nof_ack=g.nof_ack, ri_len=g.ri_len, cqi_len=g.cqi_len, I_offset_ack=g.I_offset_ack,
                            I_offset_ri=g.I_offset_ri, I_offset_cqi=g.I_offset_cqi) for g in gr]
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=2)
    try:
        phy.set_ul_cfg(3, 2)
        res, ch, payload = phy.decode_ul(iq, np.arange(2, dtype=np.uint32), cg)
        Gs = [ltelib.uci_layout(g).G for g in grants]
        llr = phy.tap(capi.TAP_PDSCH_LLR, (sum((G + 7) & ~7 for G in Gs),), np.int16)
        want, off = [], 0
        for gi, (g, G) in enumerate(zip(grants, Gs)):
            want.append((gi, _ref_tb(llr[off:], G, g.tbs, g.rv, g.qm, 1)))
            off += (G + 7) & ~7
        _check(res, payload, want)
        crcs = [w[1][0] for w in want]
        avgs = {w[1][2] for w in want}
        assert any(crcs) and not all(crcs) and len(avgs) >= 3 and max(w[1][3] for w in want) > 1, (crcs, avgs)
    finally:
        phy.close()


@pytest.mark.parametrize("cellp", [(25, 1, 3, 1), (50, 2, 301, 2), (15, 2, 11, 2)])
def test_mib_combined_equals_reference_loop(infra, phylib, cellp):
    cell = Cell(*cellp)
    iq, tti, fes = sequence(cell, PLAN)
    pc = M.PyCombiner(cell)
    ref = [expected(pc.decode(int(t), f, False)) for t, f in zip(tti, fes)]
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=len(tti), phich_resources=cell.phich_ng,
                      phich_length=cell.phich_ext)
    try:
        assert run_gpu(phy, iq, tti, len(tti), False) == ref
    finally:
        phy.close()
    assert sum(r is not None for r in ref) >= 4


# (tbs, Qm, which CRC is wrong): (1) every CB CRC24B valid, the TB CRC24A wrong; (2) the TB CRC24A valid, code block 1's CRC24B wrong;
# (3) C = 1 with F > 0; (4) the largest transport block of one codeword (TBS index 26 at 100 PRB: 75 376 bits, C = 13)
CRAFTED = [(9000, 2, "tb"), (9000, 2, 1), (512, 2, None), (75376, 6, None)]
CRAFTED_CELL = (100, 1, 1, 1)


def crafted_cases(S, rng):
    """one subframe 1 per CRAFTED entry: the whole band as one port-0 grant, the codeword of crafted_codeword mapped by the float64
    transmitter of tests/test_float64_reference.py over a flat channel at high SNR"""
    cell = Cell(*CRAFTED_CELL)
    out = []
    for i, (tbs, qm, bad) in enumerate(CRAFTED):
        probe = Case(cell, 1, 1, "port0", [qm], range(cell.nof_prb), chan="flat", noise_var=1e-5, seed=80 + i)
        G = probe.grant.nof_re * qm
        e, pl = crafted_codeword(S, rng, tbs, G, qm, 1, 0, bad)
        c = Case(cell, 1, 1, "port0", [qm], range(cell.nof_prb), chan="flat", noise_var=1e-5, seed=80 + i, cw_bits=[e])
        c.grant.tb[0].tbs = tbs
        out.append((c, G, pl))
    return cell, out


def test_phase_b_crafted_transport_blocks_equal_reference(infra, phylib):
    """crc, avg_iters, nof_cb and payload of phase B against dlsch_decode_ref on the tapped soft bits, and what each case is built to show:
    crc = 0 with one iteration per code block when only the TB CRC is wrong; crc = 0 with the bad code block at max_iter when only a CB CRC is wrong"""
    S = infra.sim()
    S.lte_turbo_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    cell, cases = crafted_cases(S, np.random.default_rng(81))
    n = len(cases)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8)
    try:
        phy.submit_iq(np.stack([c.iq for c, _, _ in cases]), np.array([1 + 10 * i for i in range(n)], np.uint32))
        phy.get_phase_a(want_cands=False)
        grants = [to_phy_grant(i, c.rnti, c.grant) for i, (c, _, _) in enumerate(cases)]
        phy.submit_grants(grants)
        res, pl = phy.get_phase_b()
        llr = phy.tap(capi.TAP_PDSCH_LLR, (sum((G + 7) & ~7 for _, G, _ in cases),), np.int16)
        off = 0
        for i, ((c, G, payload), (tbs, qm, bad)) in enumerate(zip(cases, CRAFTED)):
            crc, rpl, iters, _ = ref_dec.dlsch_decode_ref(llr[off:off + G], G, tbs, 0, qm, 1, 8, 1)
            off += (G + 7) & ~7
            rr = res[2 * i]
            avg = -(-int(iters.sum()) // len(iters))
            assert (bool(rr.crc), int(rr.avg_iters), int(rr.nof_cb)) == (crc, avg, len(iters)), (tbs, bad, rr.crc, crc, rr.avg_iters, avg, rr.nof_cb)
            assert np.array_equal(pl[rr.payload_off:rr.payload_off + tbs // 8], rpl), (tbs, bad)
            assert np.array_equal(rpl, payload) and crc == (bad is None), (tbs, bad, crc)
            if bad is not None:
                assert iters.tolist() == [8 if r == bad else 1 for r in range(len(iters))], (tbs, bad, iters)
        assert res[6].nof_cb == 13
    finally:
        phy.close()
