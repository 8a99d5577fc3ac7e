"""Uplink receive diversity for the tests (DESIGN.md §2, "uplink receive diversity"): ctypes bindings of the two-antenna PUSCH oracle
(oracle_ul/liblteopuschrx.so, lteo_pusch_decode_rx) and of the simulator's multi-antenna uplink (lte_sim_ul_subframe_rx), and float64
two-antenna references built on tests/ref64_ul.py's one-antenna pieces.  Imported only by tests/."""
import ctypes as C
import os

import numpy as np

import ltelib
import ref64
import ref64_ul

_rx = None


def rxlib():
    global _rx
    if _rx is None:
        ltelib.build_infra()
        L = C.CDLL(os.path.join(ltelib.ROOT, "oracle_ul", "liblteopuschrx.so"))
        P = C.c_void_p
        L.lteo_pusch_decode_rx.argtypes = [C.POINTER(ltelib.Cell), C.POINTER(ltelib.UlCfg), C.c_uint32, C.POINTER(ltelib.UlGrant), P, C.c_uint32,
                                           C.c_uint32, P, C.POINTER(C.c_int), C.POINTER(ltelib.UlChest), P, P]
        _rx = L
    return _rx


def sim_ul_rx(simobj, tti, ucfg, grants, nof_rx):
    """lte_sim_ul_subframe_rx -> (iq complex64 [nof_rx][sf_len], payload, payload offsets)"""
    S = ltelib.sim()
    iq = np.zeros((nof_rx, simobj.sf_len), np.complex64)
    pl = np.zeros(1 << 16, np.uint8)
    off = np.zeros(max(1, len(grants)), np.uint32)
    arr = (ltelib.UlGrant * max(1, len(grants)))(*grants)
    r = S.lte_sim_ul_subframe_rx(simobj.h, tti, C.byref(ucfg), arr, len(grants), nof_rx, ltelib.ptr(iq), ltelib.ptr(pl), ltelib.ptr(off), len(pl))
    assert r == 0, r
    return iq, pl, off


def ul_ofdm(o, iq):
    """lteo_ul_ofdm of every antenna: iq [A][sf_len] -> sym complex64 [A][14 nsc]"""
    O = ltelib.oracle()
    O.lteo_ul_ofdm.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    iq = np.ascontiguousarray(iq, np.complex64)
    iq = iq[None] if iq.ndim == 1 else iq
    sym = np.zeros((iq.shape[0], 14 * o.nsc), np.complex64)
    for a in range(iq.shape[0]):
        O.lteo_ul_ofdm(o.h, ltelib.ptr(np.ascontiguousarray(iq[a])), ltelib.ptr(sym[a]))
    return sym


def decode_rx(cell, ucfg, sf_idx, g, sym, max_iter=8):
    """lteo_pusch_decode_rx of one grant on the grids sym [A][14 nsc] -> (ret, payload, crc, chest, llr [G], eq [12][M])"""
    sym = [np.ascontiguousarray(s, np.complex64) for s in sym]
    pl = np.zeros(16000, np.uint8)
    ok = C.c_int(0)
    ch = ltelib.UlChest()
    G = ltelib.uci_layout(g).G
    llr = np.zeros(G + 16, np.int16)
    eq = np.zeros((12, 12 * g.L_prb), np.complex64)
    r = rxlib().lteo_pusch_decode_rx(C.byref(cell), C.byref(ucfg), sf_idx, C.byref(g), ltelib.ptr_array(sym), len(sym), max_iter, ltelib.ptr(pl),
                                     C.byref(ok), C.byref(ch), ltelib.ptr(llr), ltelib.ptr(eq))
    return r, pl, ok.value, ch, llr[:G], eq


def oracle_ul_rx(o, ucfg, tti, grants, iq, max_iter=8):
    """ltelib.oracle_ul for [A][sf_len] samples: lteo_ul_ofdm per antenna, lteo_pusch_decode_rx per grant -> (sym [A][14 nsc], results)"""
    sym = ul_ofdm(o, iq)
    return sym, [decode_rx(o.cell, ucfg, tti % 10, g, sym, max_iter) for g in grants]


# ------------------------------------------------------------------------------------------------ float64 references, A antennas
def chest_rx(cell, Ys, grant, sf, ucfg):
    """DESIGN.md §2 "uplink receive diversity" in float64: ref64_ul.chest per antenna; noise and RSRP the mean over (antenna, slot), ta_us from the
    per-slot correlations summed over the antennas -> (smoothed [A][2][M], dict(noise, rsrp, snr_db, ta_us))"""
    M = grant.M
    f = ref64_ul.smooth_taps()
    sms, ls = [], []
    for Y in Ys:
        sm, _ = ref64_ul.chest(cell, Y, grant, sf, ucfg)
        sms.append(sm)
        ls.append(np.array([Y[7 * sl + 3, grant.k0(sl):grant.k0(sl) + M] * np.conj(ref64_ul.dmrs(cell.cell_id, ucfg, 2 * sf + sl, grant.n_dmrs2, M))
                            for sl in range(2)]))
    ls, sms = np.array(ls), np.array(sms)
    noise = np.mean(np.abs(ls - sms) ** 2) / (1 - 2 * f[1] + np.sum(f ** 2))
    rsrp = np.mean(np.abs(sms) ** 2)
    ta = sum(-np.angle(np.sum(ls[:, sl, 1:] * np.conj(ls[:, sl, :-1]))) / (2 * np.pi) / 2 for sl in range(2))
    return sms, dict(noise=noise, rsrp=rsrp, snr_db=10 * np.log10(rsrp / noise), ta_us=ta / 15e-3)


def deprecode_rx(cell, Ys, grant, sms):
    """sum_a conj(h_a) y_a / sum_a |h_a|^2 (0 where the sum is exactly 0), then ref64_ul.deprecode's IDFT -> (eq [12][M], x [12][M], cond [12])"""
    M = grant.M
    eq, x, cond = np.zeros((12, M), complex), np.zeros((12, M), complex), np.zeros(12)
    for c, l in enumerate(ref64_ul.DATA_SYMBOLS):
        k0 = grant.k0(l // 7)
        hs = [ref64_ul.estimate_at(grant, sm, l) for sm in sms]
        num = sum(Y[l, k0:k0 + M] * np.conj(h) for Y, h in zip(Ys, hs))
        p = sum(np.abs(h) ** 2 for h in hs)
        eq[c] = ref64._div(num, p)
        x[c] = np.fft.ifft(eq[c]) * np.sqrt(M)
        with np.errstate(divide="ignore", invalid="ignore"):
            cond[c] = p.max() / p.min() if p.max() > 0 else 1.0
    return eq, x, cond


def decode_ref_rx(cell, Ys, grant, sf, ucfg):
    """the two-antenna receive chain of one grant in float64 -> (chest dict, eq [12][M], llr [G], cond per soft bit [G])"""
    sms, info = chest_rx(cell, Ys, grant, sf, ucfg)
    eq, x, cond = deprecode_rx(cell, Ys, grant, sms)
    llr, col = ref64_ul.soft_bits(cell, x, grant, sf)
    return info, eq, llr, cond[col]
