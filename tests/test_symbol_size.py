"""Symbol sizes of srsRAN's default build (3/4 of the standard LTE rate: srsran_symbol_sz = 1536 at 100 PRB, 768 at 50, 384 at 25 -- the rate a
stock LTESniffer records at, srsran_sampling_freq_hz at src/src/LTESniffer_Core.cc:222): the simulator, the oracle and the product handle the
3 * 2^k-point OFDM symbols; GPU: symbols bit-exact against the oracle, and the whole pipeline decodes such a capture.  Also the other sizes a 15 MHz
capture comes in (1536 at the 3GPP rate of 23.04 Msps, 1024 from srsRAN's default build; the library's default there is 2048) and a 3 * 2^k size at 3 MHz."""
import numpy as np
import pytest
import ltelib
from ltelib import Cell
from helpers import make_capture, oracle_frontend, truth_grants

CASES = [(100, 1536), (50, 768), (25, 384), (75, 1536), (75, 1024), (15, 384)]     # 75 PRB: the 3GPP 15 MHz rate, srsRAN's 75 PRB size; 15 PRB: 3 * 2^7
KW = dict(seed=3, cfi=2, nof_ues=3, dl_min=2, dl_max=2, tm=13, mcs_min=8, mcs_max=20, snr_db=28.0)


@pytest.mark.parametrize("nprb,sz", CASES)
def test_oracle_decodes_three_quarter_rate_capture(infra, nprb, sz):
    cell = Cell(nprb, 2, 7, 2, sz)
    sim, iq, tti, truths, payloads = make_capture(cell, 2, **KW)
    assert iq.shape[-1] == 15 * sz
    o = ltelib.Oracle(cell)
    fe = oracle_frontend(o, iq, tti)
    n = ok = 0
    for sf, d, g in truth_grants(cell, truths, tti):
        r, pl, c = o.pdsch_decode(int(tti[sf]) % 10, fe[sf]["cfi"], d.rnti, g, fe[sf]["sym"], fe[sf]["ce"])
        for t in range(2):
            if g.tb[t].enabled:
                n += 1
                ok += c[t]
    assert n >= 4 and ok == n
    # the symbols are the ones a standard-rate receiver sees (same grid, other sampling rate), up to the noise realisation
    cell2 = Cell(nprb, 2, 7, 2, 0)
    _, iq2, _, _, _ = make_capture(cell2, 2, **dict(KW, snr_db=60.0))
    _, iq3, _, _, _ = make_capture(cell, 2, **dict(KW, snr_db=60.0))
    a = ltelib.Oracle(cell2).ofdm(iq2[0])
    b = ltelib.Oracle(cell).ofdm(iq3[0])
    scale = np.sqrt(sz / cell2.fft())          # unitary IFFT in the simulator, unnormalised FFT in the receiver
    assert np.abs(a / np.sqrt(cell2.fft()) - b / np.sqrt(sz)).max() < 0.02 * np.abs(a).max() / np.sqrt(cell2.fft()) + 1e-3, scale


def test_product_rejects_unsupported_symbol_sizes(phylib):
    from ltesniffer_b200 import capi
    for nprb, sz in ((100, 1024), (100, 1200), (50, 3072), (25, 300)):
        with pytest.raises(RuntimeError):
            capi.LtePhy(nprb, 2, 1, 2, symbol_sz=sz)


@pytest.mark.gpu
@pytest.mark.parametrize("nprb,sz", CASES)
def test_gpu_three_quarter_rate_bit_exact(infra, phylib, nprb, sz):
    from ltesniffer_b200 import capi
    cell = Cell(nprb, 2, 7, 2, sz)
    sim, iq, tti, truths, payloads = make_capture(cell, 3, **KW)
    o = ltelib.Oracle(cell)
    fe = oracle_frontend(o, iq, tti)
    phy = capi.LtePhy(nprb, 2, 7, 2, max_subframes=3, symbol_sz=sz, flags=capi.FLAG_SKIP_LOW_POWER)
    assert phy.sf_len == 15 * sz
    phy.submit_iq(iq, tti)
    info, cands = phy.get_phase_a()
    g = 14 * 12 * nprb
    sym = phy.tap(capi.TAP_SYM, (3, 2, g), np.complex64)
    for i in range(3):
        assert np.array_equal(sym[i].view(np.uint32), np.asarray(fe[i]["sym"]).reshape(2, g).view(np.uint32)), "OFDM symbols of subframe %d" % i
        assert info[i].cfi == fe[i]["cfi"]
    srch = capi.Search(nprb, 2, 7, 2)
    inf, dcis, tbs, pl = capi.decode_subframes(phy, srch, iq, tti)
    assert sum(1 for i in range(2 * len(dcis)) if tbs[i].crc) >= 4
    # uplink symbols (7.5 kHz shift + the same radix-3 step)
    ucfg = ltelib.UlCfg(n_dmrs1=3, delta_ss=2)
    ucell = Cell(nprb, 1, 7, 1, sz)
    us = ltelib.Sim(cell=ucell, seed=4, snr_db=30.0, nof_ues=1)
    gr = ltelib.make_ul_grants(ucell, np.random.default_rng(4), 3)
    x, upl, off = ltelib.sim_ul_subframe(us, 5, ucfg, gr)
    uphy = capi.LtePhy(nprb, 1, 7, 1, max_subframes=1, symbol_sz=sz)
    uphy.set_ul_cfg(3, 2)
    res, ch, payload = uphy.decode_ul(x[None, :], np.array([5], np.uint32),
                                      [capi.UlGrant(sf=0, rnti=q.rnti, qm=q.qm, rv=q.rv, L_prb=q.L_prb, n_prb=q.n_prb, n_dmrs2=q.n_dmrs2, tbs=q.tbs) for q in gr])
    usym, ref = ltelib.oracle_ul(ltelib.Oracle(ucell), ucfg, 5, gr, x)
    got = uphy.tap(capi.TAP_UL_SYM, (14 * 12 * nprb,), np.complex64)
    assert np.array_equal(got.view(np.uint32), np.asarray(usym).view(np.uint32))
    for k, (r, opl, ocrc, och, _) in enumerate(ref):
        assert res[k].crc == ocrc == 1
    phy.close(), uphy.close()
