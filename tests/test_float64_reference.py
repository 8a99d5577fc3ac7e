"""The CPU oracle's receive path against the float64 references of tests/ref64.py (written from 36.211 / 36.212 and DESIGN.md section 2, not from
lte_oracle.c).  Every GPU parity test compares the kernels bit for bit with the oracle, so a mistake in a formula both restate -- an extrapolation,
an edge renormalisation, a noise correction, a demodulator threshold, a clamp, the order PDSCH REs are read in -- is invisible to parity.  These
tests pin the oracle from outside; tests/test_gpu_float64_reference.py runs the same references against the kernels.

Inputs are synthesised in numpy (ref64's transmitter: CRS, PDSCH, precoding, scrambling, a designed channel, numpy.fft.ifft), so nothing here goes
through the simulator's transmitter, whose resource-element map the oracle shares."""
import ctypes as C
import numpy as np
import pytest

import ltelib
import ref64
from helpers import make_capture, oracle_frontend
from ltelib import Cell, Oracle

ORACLE_CELLS = [(15, 1, 31, 1), (15, 2, 32, 2), (25, 2, 150, 1), (50, 1, 9, 2), (50, 2, 301, 2), (75, 2, 77, 2, 1536), (75, 1, 76, 1),
                (100, 2, 7, 2), (100, 1, 1, 1, 1536)]
SCHEMES = {"port0": 0, "sfbc": 1, "cdd": 2, "tm4": 3}


def re_map_oracle(cell, sf, cfi, l, prb):
    S = ltelib.sim()
    S.lte_pdsch_re_in_prb.argtypes = [C.POINTER(Cell), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    S.lte_pdsch_re_in_prb.restype = C.c_uint32
    kk = np.zeros(12, np.uint16)
    n = S.lte_pdsch_re_in_prb(C.byref(cell), sf, cfi, l, prb, ltelib.ptr(kk))
    return kk[:n].astype(np.int64)


def pdcch_index(cell, cfi):
    """grid indices l * nsc + k of the PDCCH REs in reading order, and of the 16 PCFICH REs (symbol 0)"""
    O = ltelib.oracle()
    O.lteo_pdcch_re_index.restype = C.c_uint32
    O.lteo_pdcch_re_index.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    o = Oracle(cell)
    idx, pidx = np.zeros(4 * 9 * 88, np.uint16), np.zeros(16, np.uint16)
    ncce = O.lteo_pdcch_re_index(o.h, cfi, ltelib.ptr(idx), ltelib.ptr(pidx))
    return idx[:36 * ncce].astype(np.int64), pidx.astype(np.int64)


def pcfich_index(cell):
    return pdcch_index(cell, 1)[1]


def tbs_of(itbs, nprb):
    return ltelib.sim().lte_tbs_from_idx(itbs, min(nprb, 110))


# ------------------------------------------------------------------------------------------------ synthesis shared with the GPU file
class Case:
    """One synthesised subframe: a cell, a PDSCH grant over prb_mask with the given scheme / codeword modulations, a designed channel, AWGN.
    Attributes: iq complex64 [rx][sf_len], grant (ltelib.DlGrant), l / k (the grant's REs in mapping order), sf, cfi, rnti, qm per codeword.
    cw_bits: the n_RE * Qm coded bits of each codeword (before scrambling); random when None."""

    def __init__(self, cell, sf, cfi, scheme, qms, prbs, chan="selective", noise_var=1e-3, seed=0, cw_swap=0, pmi=0, H=None, rnti=0x4321, cw_bits=None, **_):
        rng = np.random.default_rng(seed)
        N, P, A = cell.nof_prb, cell.nof_ports, cell.nof_rx
        nsc = 12 * N
        self.cell, self.sf, self.cfi, self.scheme, self.rnti, self.qms = cell, sf, cfi, scheme, rnti, list(qms)
        mask = np.zeros((2, 110), np.uint8)
        for s in range(2):
            mask[s, list(prbs)] = 1
        self.l, self.k = ref64.pdsch_res(cell, sf, cfi, mask)
        n = len(self.l)
        self.nof_layers = 2 if scheme == "cdd" else len(qms) if scheme == "tm4" else 1
        grids = np.zeros((P, 14, nsc), complex)
        for p in range(P):
            grids[p] += ref64.crs_grid(cell, sf, p)
            nctrl = cfi + 1 if N <= 10 else cfi
            for l in range(nctrl):                                        # the control region: random QPSK on every RE that is not a pilot
                free = np.ones(nsc, bool)
                if l == 0:
                    for q in range(P):
                        free[ref64.crs_offset(cell, q, 0)::6] = False
                grids[p, l, free] = ref64.qam(rng.integers(0, 2, 2 * free.sum()), 2)
        # PCFICH (36.211 6.7): the CFI codeword scrambled, QPSK, port 0 or SFBC, on the four REGs of lteo_pdcch_re_index (pinned by test_phich_resources)
        pidx = pcfich_index(cell)
        d = ref64.qam(np.array(ref64.CFI_CODEWORDS[cfi - 1][:32], np.uint8) ^ ref64.gold((sf + 1) * (2 * cell.cell_id + 1) * 512 + cell.cell_id, 32), 2)
        grids[:, 0, pidx] = ref64.precode("port0" if P == 1 else "sfbc", d[None], P)
        layers = []
        for q, qm in enumerate(qms):
            bits = rng.integers(0, 2, n * qm).astype(np.uint8)
            if cw_bits is not None:                                       # given coded bits instead of random ones (same draws, so the noise is unchanged)
                bits = np.asarray(cw_bits[q], np.uint8)
            layers.append(ref64.qam(bits ^ ref64.scrambling_seq(cell, sf, rnti, q, n * qm), qm))
        y = ref64.precode(scheme, np.array(layers), P, self.nof_layers, pmi)
        for p in range(y.shape[0]):
            grids[p, self.l, self.k] = y[p]
        self.H = H if H is not None else ref64.channel(chan, A, P, nsc)
        Y = ref64.receive(cell, grids, self.H, noise_var, rng)
        self.iq = np.stack([ref64.ofdm_modulate(cell, Y[a]) for a in range(A)]).astype(np.complex64)
        # the grant, as the oracle and the product take it; TB t goes to codeword t, or to 1 - t when cw_swap is set
        g = ltelib.DlGrant()
        for s in range(2):
            for prb in prbs:
                g.prb_mask[s][prb] = 1
        g.nof_prb = len(prbs)
        g.nof_re = n
        g.tx_scheme = SCHEMES[scheme]
        g.nof_layers = self.nof_layers
        g.pmi = pmi
        g.cw_swap = cw_swap
        g.nof_tb = len(qms)
        for t in range(len(qms)):
            q = (1 - t) if (cw_swap and len(qms) == 2) else t
            g.tb[t].enabled, g.tb[t].qm, g.tb[t].rv = 1, qms[q], 0
            g.tb[t].tbs = tbs_of(5, len(prbs))
            g.tb[t].nof_bits = n * qms[q]
        self.grant = g

    def reference(self, Y=None):
        """float64 receive chain from the same complex64 samples: -> (chest info, llr per codeword, cond per RE)"""
        cell = self.cell
        if Y is None:
            Y = np.stack([ref64.ofdm_demodulate(cell, self.iq[a]) for a in range(cell.nof_rx)])
        ce, info = ref64.chest(cell, self.sf, Y)
        x, cond = ref64.equalise_pdsch(cell, self.scheme, ce, Y, self.l, self.k, self.nof_layers, self.grant.pmi)
        llr = []
        for q, qm in enumerate(self.qms):
            z = ref64.demod_int16(x[q], qm)
            llr.append(ref64.descramble(z, ref64.scrambling_seq(cell, self.sf, self.rnti, q, len(z))))
        return Y, ce, info, llr, cond


def check_llr(got, ref, cond, qm, what):
    """the K6 bar: where cond(H P) <= 100, |diff| <= 1 everywhere, >= 99.5 % exactly equal and saturated values exact; above, the signs where |ref| > 64"""
    got = np.asarray(got, np.int64)[:len(ref)]
    well = np.repeat(cond <= 100, qm)
    d = np.abs(got - ref)
    if well.any():
        assert d[well].max() <= 1, "%s: max |diff| %d at %d (got %d, ref %d)" % (what, d[well].max(), np.argmax(np.where(well, d, 0)),
                                                                             got[np.argmax(np.where(well, d, 0))], ref[np.argmax(np.where(well, d, 0))])
        assert np.mean(d[well] == 0) >= 0.995, "%s: only %.4f exactly equal" % (what, np.mean(d[well] == 0))
        sat = well & (np.abs(ref) == 32767)
        assert np.array_equal(got[sat], ref[sat]), "%s: saturated values differ" % what
    strong = ~well & (np.abs(ref) > 64)
    assert np.all(np.sign(got[strong]) == np.sign(ref[strong])), "%s: %d sign flips on ill-conditioned REs" % (what, int(np.sum(np.sign(got[strong]) != np.sign(ref[strong]))))


def oracle_llr(case, o, sym, ce):
    r, llr, _ = o.pdsch_llr(case.sf, case.cfi, case.rnti, case.grant, sym, ce)
    assert r == 0, r
    return llr


# ------------------------------------------------------------------------------------------------ RE map
@pytest.mark.parametrize("cellp", [(15, 1, 31, 1), (15, 2, 32, 2), (25, 1, 5, 1), (25, 2, 150, 2), (50, 1, 9, 1), (50, 2, 301, 2), (75, 2, 77, 2), (75, 1, 76, 1),
                                   (100, 2, 7, 2), (100, 1, 1, 1)], ids=lambda c: "x".join(map(str, c)))
def test_pdsch_re_map_equals_36211(infra, phylib, cellp):
    """lte_pdsch_re_in_prb (shared by the simulator and the oracle) and the product's nof_re from ltephy_dci_to_grant, PRB by PRB, against the 6.3.5
    map of ref64 on every CFI and on subframes 0, 5 and 3"""
    from ltesniffer_b200 import capi
    cell = Cell(*cellp)
    N = cell.nof_prb
    S = ltelib.sim()
    srch = capi.Search(N, cell.nof_ports, cell.cell_id, cell.nof_rx)
    nb = S.lte_dci_sizeof(C.byref(cell), 2)                                   # format 1A
    for sf in (0, 5, 3):
        for cfi in (1, 2, 3):
            for prb in range(N):
                mask = np.zeros((2, 110), np.uint8)
                mask[:, prb] = 1
                l, k = ref64.pdsch_res(cell, sf, cfi, mask)
                for ll in range(14):
                    assert np.array_equal(re_map_oracle(cell, sf, cfi, ll, prb), k[l == ll]), (sf, cfi, ll, prb)
                d = ltelib.Dci()                                          # a localised one-PRB format 1A grant: riv = start
                d.format, d.rnti, d.alloc_type, d.riv = 2, 0x1234, 2, prb
                bits = np.zeros(64, np.uint8)
                n = C.c_uint32(0)
                assert S.lte_dci_pack(C.byref(cell), C.byref(d), ltelib.ptr(bits), C.byref(n)) == 0 and n.value == nb
                row = np.zeros(1, capi.DCI_DTYPE)[0]
                row["sf"], row["rnti"], row["format"], row["nof_bits"] = 0, 0x1234, 2, nb
                row["bits"] = sum(int(bits[i]) << (63 - i) for i in range(nb))
                r, g, _ = srch.dci_to_grant(row, sf, cfi)
                assert r == 0 and g.prb_mask[0][prb >> 5] == g.prb_mask[1][prb >> 5] == 1 << (prb & 31), (sf, cfi, prb)
                assert g.nof_re == len(l), (sf, cfi, prb, g.nof_re, len(l))
    srch.close()


# ------------------------------------------------------------------------------------------------ K1 / K2
@pytest.mark.parametrize("cellp", ORACLE_CELLS, ids=lambda c: "x".join(map(str, c)))
def test_ofdm_and_chest_equal_the_float64_reference(infra, cellp):
    cell = Cell(*cellp)
    o = Oracle(cell)
    N = ref64.fft_size(cell)
    scheme = "port0" if cell.nof_ports == 1 else "sfbc"
    for sf, chan in ((0, "selective"), (5, "linear_l"), (3, "delay")):
        case = Case(cell, sf, 2, scheme, [4], range(cell.nof_prb), chan=chan, seed=sf)
        sym = o.ofdm(case.iq)
        Y, ce, info, _, _ = case.reference()
        for a in range(cell.nof_rx):
            assert np.allclose(sym[a].reshape(14, -1), Y[a], rtol=0, atol=2e-5 * np.sqrt(N)), (sf, a)
        oce, res = o.chest(sf, sym)
        scale = np.abs(ce).max()
        assert np.abs(oce.reshape(ce.shape) - ce).max() <= 1e-5 * scale, (sf, chan, np.abs(oce.reshape(ce.shape) - ce).max() / scale)
        for p in range(cell.nof_ports):
            for a in range(cell.nof_rx):
                assert abs(res.noise[p][a] - info["noise"][p, a]) <= 1e-5 * info["noise"][p, a], (p, a, res.noise[p][a], info["noise"][p, a])
                assert abs(res.rsrp[p][a] - info["rsrp"][p, a]) <= 1e-5 * info["rsrp"][p, a]
        assert abs(res.snr_db - info["snr_db"]) <= 1e-4
        assert abs(complex(res.cfo_re, res.cfo_im) - info["cfo_sum"]) <= 1e-5 * abs(info["cfo_sum"])


@pytest.mark.parametrize("chan", ["flat", "linear_l", "linear_k"])
def test_noiseless_channel_estimate_is_the_channel(infra, chan):
    """physics anchor: without noise the estimate equals H wherever H is linear between the pilots -- everywhere for a flat channel and for one linear
    in time (symbols 12 and 13 included), and between pilots 2 and 2 N - 3 for one linear in frequency (the renormalised edge taps are not symmetric)"""
    cell = Cell(50, 2, 301, 2)
    o = Oracle(cell)
    case = Case(cell, 3, 2, "sfbc", [2], range(50), chan=chan, noise_var=0.0)
    ce, res = o.chest(3, o.ofdm(case.iq))
    ce = ce.reshape(4, 14, -1)
    H = np.stack([case.H[a, p] for p in range(2) for a in range(2)])
    sel = slice(None)
    if chan == "linear_k":
        lo, hi = 12 + 6, 12 * 50 - 18
        sel = (slice(None), slice(None), slice(lo, hi))
    err = np.abs(ce - H)[sel].max() / np.abs(H).max()
    assert err < 2e-6, err
    Y, rce, info, _, _ = case.reference()
    assert np.abs(rce - H)[sel].max() / np.abs(H).max() < 1e-6                 # the reference itself, from the same complex64 samples


def test_noise_and_snr_estimates_on_a_flat_channel(infra):
    """physics anchor: flat channel, AWGN of variance s2 per RE.  100 PRB, 2 ports x 2 rx, 4 subframes = 4 x 4 x 4 x 200 = 12800 LS residuals, whose
    mean has a relative standard deviation near 1 %: the +-5 % bar on the noise and the +-0.3 dB bar on the SNR are more than 4 sigma wide"""
    cell = Cell(100, 2, 7, 2)
    o = Oracle(cell)
    s2 = 10 ** (-15 / 10)
    nsum = rsum = 0.0
    for sf in (1, 2, 3, 4):
        H = np.ones((2, 2, 14, 1200), complex) * np.array([[1, 1j], [-1j, 1]])[:, :, None, None] / np.sqrt(1.0)
        case = Case(cell, sf, 2, "sfbc", [2], range(100), noise_var=s2, seed=40 + sf, H=H)
        _, res = o.chest(sf, o.ofdm(case.iq))
        nsum += res.noise_avg
        rsum += res.rsrp_avg
    noise = nsum / 4
    assert abs(noise / s2 - 1) < 0.05, noise / s2
    assert abs(10 * np.log10(rsum / nsum) - 15.0) < 0.3, 10 * np.log10(rsum / nsum)


# ------------------------------------------------------------------------------------------------ K3 / K4
@pytest.mark.parametrize("cellp", [(15, 1, 31, 1), (50, 2, 301, 2), (100, 2, 7, 1), (75, 1, 76, 2, 1536)], ids=lambda c: "x".join(map(str, c)))
def test_pcfich_and_pdcch_llrs_equal_the_float64_reference(infra, cellp):
    cell = Cell(*cellp)
    o = Oracle(cell)
    for sf, cfi in ((0, 1), (5, 2), (7, 3)):
        case = Case(cell, sf, cfi, "port0" if cell.nof_ports == 1 else "sfbc", [2], [0], seed=cfi)
        sym = o.ofdm(case.iq)
        ce, _ = o.chest(sf, sym)
        Y, rce, _, _, _ = case.reference()
        idx, pidx = pdcch_index(cell, cfi)
        ocfi, corr = o.pcfich(sf, sym, ce)
        rc = ref64.pcfich_corr(cell, sf, rce, Y, pidx)
        assert ocfi == cfi and np.argmax(rc) == cfi - 1
        assert np.abs(corr - rc).max() <= 1e-5 * np.abs(rc).max(), (corr, rc)
        llr = o.pdcch_llr(sf, cfi, sym, ce)
        rl = ref64.pdcch_llr(cell, sf, rce, Y, idx, (sf << 9) + cell.cell_id)
        assert np.abs(llr - rl).max() <= 1e-5 * np.abs(rl).max(), np.abs(llr - rl).max() / np.abs(rl).max()


# ------------------------------------------------------------------------------------------------ K6
def pdsch_cases():
    """(id, cell, sf, cfi, scheme, qms, prbs, kw): every scheme with Qm 2 / 4 / 6 / 8, two codewords with different Qm, cw_swap, PRB 0 and N - 1,
    deep fades, near-singular 2x2 channels and a dead receive antenna"""
    out = []
    for qm in (2, 4, 6, 8):
        out += [("port0_q%d" % qm, (50, 1, 9, 2), 5, 1, "port0", [qm], range(0, 50, 2), {}),
                ("sfbc_q%d" % qm, (15, 2, 32, 2), 0, 3, "sfbc", [qm], range(15), {}),
                ("cdd_q%d" % qm, (100, 2, 7, 2), 3, 2, "cdd", [qm, 10 - qm if qm != 2 else 6], list(range(6)) + [99], {}),
                ("tm4_1l_q%d" % qm, (25, 2, 150, 2), 0, 2, "tm4", [qm], range(25), dict(pmi=qm // 2 - 1)),
                ("tm4_2l_q%d" % qm, (75, 2, 77, 2, 1536), 5, 1, "tm4", [qm, 2], [0, 37, 74], dict(pmi=(qm // 2) % 2))]
    out += [("cdd_cw_swap", (50, 2, 301, 2), 0, 2, "cdd", [6, 2], range(50), dict(cw_swap=1)),
            ("tm4_cw_swap", (50, 2, 11, 2), 7, 3, "tm4", [4, 8], range(20, 50), dict(cw_swap=1, pmi=1)),
            ("sfbc_1rx_q6", (25, 2, 150, 1), 5, 2, "sfbc", [6], range(25), {}),
            ("port0_1rx_q8_1536", (100, 1, 1, 1, 1536), 0, 3, "port0", [8], range(100), {}),
            ("deep_fade_port0", (50, 1, 9, 2), 3, 2, "port0", [6], range(50), dict(fade=True)),
            ("deep_fade_sfbc", (100, 2, 7, 2), 3, 2, "sfbc", [4], range(100), dict(fade=True)),
            ("near_singular_cdd", (50, 2, 301, 2), 3, 2, "cdd", [4, 6], range(50), dict(singular=True)),
            ("near_singular_tm4", (50, 2, 11, 2), 8, 2, "tm4", [2, 8], range(50), dict(singular=True, pmi=0)),
            ("dead_rx_sfbc", (50, 2, 301, 2), 3, 2, "sfbc", [4], range(50), dict(dead=True))]
    return out


def designed_channel(cell, fade=False, singular=False, dead=False, **_):
    nsc = 12 * cell.nof_prb
    H = ref64.channel("selective", cell.nof_rx, cell.nof_ports, nsc)
    if fade:                                                               # |h| ~ 1e-3 on PRBs 0-3, 20-27 and the last four up to symbol 11; the fade
        N = cell.nof_prb                                                   # ends on 12 and 13, where the estimate extrapolated from pilot symbols 7 and
        for prb in list(range(4)) + list(range(20, 28)) + list(range(N - 4, N)):      # 11 stays deep, so the equalised symbols drive the int16 clamp
            H[:, :, :12, 12 * prb:12 * prb + 12] *= 1e-3
    if singular:                                                           # cond(H P) from 10 to 1e4 across the band: rx 1 close to a copy of rx 0
        eps = np.logspace(-1, -4, nsc)
        H[1] = H[0] * np.exp(0.4j) + eps[None, None, :] * np.exp(1j * np.arange(nsc) * 0.1)[None, None, :] * np.array([1, -1j])[:, None, None]
    if dead:
        H[1] = 0
    return H


@pytest.mark.parametrize("cid,cellp,sf,cfi,scheme,qms,prbs,kw", pdsch_cases(), ids=[c[0] for c in pdsch_cases()])
def test_pdsch_llrs_equal_the_float64_reference(infra, cid, cellp, sf, cfi, scheme, qms, prbs, kw):
    cell = Cell(*cellp)
    kw = dict(kw)
    H = designed_channel(cell, **kw)
    case = Case(cell, sf, cfi, scheme, qms, list(prbs), H=H, noise_var=3e-3, seed=len(cid), cw_swap=kw.get("cw_swap", 0), pmi=kw.get("pmi", 0))
    o = Oracle(cell)
    sym = o.ofdm(case.iq)
    ce, _ = o.chest(sf, sym)
    llr = oracle_llr(case, o, sym, ce)
    _, _, _, ref, cond = case.reference()
    if kw.get("singular"):
        assert cond.min() < 100 < cond.max() and cond.max() > 1e3, (cond.min(), cond.max())
    for q, qm in enumerate(qms):
        check_llr(llr[q], ref[q], cond, qm, "%s cw %d" % (cid, q))
    if kw.get("fade"):
        assert sum(int(np.sum(np.abs(r) == 32767)) for r in ref) > 0, "the deep fades drive the int16 clamp"


# ------------------------------------------------------------------------------------------------ zero-filled samples
ZERO_CELL = Cell(50, 2, 301, 2)
ZERO_KINDS = ["all_zero", "gap_from_symbol_8", "first_two_symbols", "dead_rx1"]


def zero_fill(iq, kind, cell):
    """iq [n][rx][sf_len] -> a copy with the samples of `kind` set to exactly 0"""
    out = iq.copy()
    N = cell.fft()
    start = [sum(ref64.cp_len(N, j) + N for j in range(l)) for l in range(15)]
    if kind == "all_zero":
        out[:] = 0
    elif kind == "gap_from_symbol_8":                                          # a capture gap that zero-fills the rest of the subframe
        out[:, :, start[8]:] = 0
    elif kind == "first_two_symbols":
        out[:, :, :start[2]] = 0
    elif kind == "dead_rx1":
        out[:, 1] = 0
    return out


def zero_channel_res(cell, ce_sf, g, l, k):
    """REs of a grant whose equaliser denominator is exactly 0 (MRC / SFBC: the channel of every port and antenna, 2x2: |det|^2)"""
    H = ref64.h_at(ce_sf.reshape(cell.nof_ports * cell.nof_rx, 14, -1).astype(np.complex128), cell, l, k)
    if g.tx_scheme in (2, 3) and g.nof_layers == 2:
        P = [ref64.port_precoder("cdd" if g.tx_scheme == 2 else "tm4", i, 2, g.pmi) for i in range(len(l))]
        return np.array([np.linalg.det(H[i] @ P[i]) == 0 for i in range(len(l))])
    if g.tx_scheme == 1:
        z = np.all(H == 0, axis=(1, 2))
        return np.repeat(z[0::2] & z[1::2], 2)                               # each symbol of a pair divides by channel power taken from both REs
    return np.all(H == 0, axis=(1, 2))


def zero_capture(kind):
    """three simulated subframes (subframes 9, 0, 1; port 0 / SFBC / CDD grants) with `kind` zeroed"""
    _, iq, tti, truths, _ = make_capture(ZERO_CELL, 3, seed=61, cfi=2, nof_ues=6, dl_min=2, dl_max=3, tm=13, mcs_min=2, mcs_max=20, snr_db=27.0, tti0=9)
    return zero_fill(iq, kind, ZERO_CELL), tti, truths


def grants_at_cfi(cell, truths, tti, cfis):
    """the transmitted DL grants of a capture, with the RE count of the CFI each subframe was decoded with: [(sf, truth dci, DlGrant)]"""
    out = []
    for sf, tr in enumerate(truths):
        for i in range(tr.nof_dci):
            d = tr.dci[i]
            if d.nof_tb == 0:
                continue
            bits = np.frombuffer(bytes(d.bits), np.uint8)[:d.nbits]
            r, _, g = ltelib.unpack_and_grant(cell, d.format, d.rnti, bits, int(tti[sf]) % 10, cfis[sf])
            assert r == 0, r
            out.append((sf, d, g))
    return out


@pytest.mark.parametrize("kind", ZERO_KINDS)
def test_oracle_on_zero_filled_subframes(infra, kind):
    """The oracle on exactly-zero samples: no NaN in the PCFICH correlations or PDCCH LLRs, an SNR that is NaN or <= 6 dB makes the reference's walk
    produce no DCI, and an RE whose equaliser denominator is exactly 0 gets LLR 0 (an erasure) instead of the undefined int16 cast of NaN"""
    cell = ZERO_CELL
    iq, tti, truths = zero_capture(kind)
    o = Oracle(cell)
    ref = oracle_frontend(o, iq, tti)
    for r in ref:
        assert not np.isnan(r["corr"]).any() and not np.isnan(r["llr"]).any() and not np.isnan(r["ce"]).any()
    if kind == "all_zero":
        assert all(np.isnan(r["res"].snr_db) for r in ref)
    if ltelib.ref_buildable():
        walk = ltelib.OracleWalk(cell)
        for i, r in enumerate(ref):
            for _ in range(3):
                out = walk.subframe(int(tti[i]) % 10, r["cfi"], len(r["llr"]) // 72, r["llr"], r["res"].snr_db)
                if not r["res"].snr_db > 6.0:
                    assert len(out) == 0, (kind, i, r["res"].snr_db)
    nzero = 0
    for sf, d, g in grants_at_cfi(cell, truths, tti, [r["cfi"] for r in ref]):
        sf_idx, cfi = int(tti[sf]) % 10, ref[sf]["cfi"]
        ret, llr, _ = o.pdsch_llr(sf_idx, cfi, d.rnti, g, ref[sf]["sym"], ref[sf]["ce"])
        assert ret == 0
        mask = np.array([[g.prb_mask[s][p] for p in range(110)] for s in range(2)])
        l, k = ref64.pdsch_res(cell, sf_idx, cfi, mask)
        zero = zero_channel_res(cell, ref[sf]["ce"], g, l, k)
        for cw in range(2 if g.nof_tb == 2 else 1):
            qm = g.tb[(1 - cw) if g.cw_swap else cw].qm
            assert np.all(llr[cw][:g.nof_re * qm][np.repeat(zero, qm)] == 0), (kind, sf, cw)
        nzero += int(zero.sum())
    if kind != "first_two_symbols":                                       # PDSCH never starts on symbol 0, the only zero-channel symbol there
        assert nzero > 0, kind
