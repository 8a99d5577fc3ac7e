"""Uplink receive diversity for the tests (DESIGN.md §2, "uplink receive diversity"): ctypes bindings of the two-antenna PUSCH oracle
(oracle_ul/liblteopuschrx.so, lteo_pusch_decode_rx), of the simulator's multi-antenna uplink (lte_sim_ul_subframe_rx) and of the oracle tracker's
UL antenna count (lteo_track_set_ul_rx), and float64 two-antenna references built on tests/ref64_ul.py's one-antenna pieces.  Imported only by
tests/."""
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
    S.lte_sim_ul_subframe_rx.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(ltelib.UlCfg), C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_uint32]
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


def track_set_ul_rx(L, t, cfo_ratio, ul_offset, nof_rx):
    L.lteo_track_set_ul_rx.argtypes = [C.c_void_p, C.c_double, C.c_int32, C.c_uint32]
    return L.lteo_track_set_ul_rx(t, cfo_ratio, ul_offset, nof_rx)


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


# ------------------------------------------------------------------------------------------------ the oracle tracker with A UL antennas
class OracleUlRx:
    """track_ul_lib.OracleUl with nof_rx UL antennas (lteo_track_set_ul_rx): push_ul takes xu [A][n] and returns ul_iq [k][A][15 N]"""

    def __init__(self, N, nrx, pci, frame_offset, cfo_hz=0.0, first_tti=0, flags=0, cfo_ratio=1.0, ul_offset=0, ul_nof_rx=2):
        import track_lib as T
        import track_ul_lib as U
        self.T, self.U = T, U
        self.o = T.Oracle(N, nrx, pci, frame_offset, cfo_hz=cfo_hz, first_tti=first_tti, flags=flags)
        U.lib()
        assert track_set_ul_rx(T.lib(), self.o.t, cfo_ratio, ul_offset, ul_nof_rx) == 0
        self.N, self.A, self.UA = N, nrx, ul_nof_rx
        self.next_sample = min(frame_offset, frame_offset + ul_offset)

    def push_ul(self, x, xu, first, max_sf=1000):
        T = self.T
        x = np.ascontiguousarray(x, np.complex64)
        xu = np.ascontiguousarray(xu, np.complex64).reshape(self.UA, -1)
        assert xu.shape[1] == x.shape[1]
        sf, hf = np.zeros(max_sf, T.SF_DTYPE), np.zeros(max_sf // 5 + 1, T.HF_DTYPE)
        iq = np.zeros((max_sf, self.A, 15 * self.N), np.complex64)
        iqu = np.zeros((max_sf, self.UA, 15 * self.N), np.complex64)
        nsf, nhf, nxt = C.c_uint32(), C.c_uint32(), C.c_uint64()
        r = T.lib().lteo_track_push_ul(self.o.t, ltelib.ptr(x), ltelib.ptr(xu), first, x.shape[1], max_sf, ltelib.ptr(sf), C.byref(nsf), ltelib.ptr(hf),
                                       C.byref(nhf), ltelib.ptr(iq), ltelib.ptr(iqu), C.byref(nxt))
        assert r == 0, r
        self.next_sample = nxt.value
        k = nsf.value
        return dict(sf=sf[:k], hf=hf[:nhf.value], iq=iq[:k], ul_iq=iqu[:k], next_sample=nxt.value)


def run_chunks_ul_rx(tr, x, xu, sizes, first=0, push=None):
    """track_ul_lib.run_chunks_ul with xu [A][n]: pieces of the given sizes (cycled), each push from the tracker's next_sample to what has arrived"""
    push = push or tr.push_ul
    outs, recv, i, end = [], first, 0, first + x.shape[1]
    while True:
        if recv < end:
            recv = min(recv + sizes[i % len(sizes)], end)
            i += 1
        start = tr.next_sample
        if start < recv:
            o = push(x[:, start - first:recv - first], xu[:, start - first:recv - first], start)
            outs.append(o)
            if recv == end and not len(o["sf"]):
                break
        elif recv == end:
            break
    host = lambda q: q if isinstance(q, np.ndarray) else q.cpu().numpy()
    got = [o for o in outs if len(o["sf"])]
    return dict(sf=np.concatenate([o["sf"] for o in outs]), hf=np.concatenate([o["hf"] for o in outs]),
                iq=np.concatenate([host(o["iq"]) for o in got]), ul_iq=np.concatenate([host(o["ul_iq"]) for o in got]))


# ------------------------------------------------------------------------------------------------ a two-carrier recording with two UL antennas
class TwoCarrierRx:
    """track_ul_lib.TwoCarrier with the uplink received on two antennas: x complex64 [1][L] (downlink), xu complex64 [2][L] (uplink, antenna-major).
    The UEs' subframes come from lte_sim_ul_subframe_rx without noise; antenna 1 is scaled to antenna 0's power (the simulator's cross-port gain is
    0.35), and each antenna gets its own white noise of power 10^(-ul_snr / 10) before the common clock and carrier offsets.  dl, ul ([k] complex64
    [2][15 N], aligned and offset-free, with the noise), grants, sent, as TwoCarrier."""

    def __init__(self, N, pci, nsf, ppm=0.0, cfo=0.0, rho=1.0, lead=1000, ul_offset=0, snr=25.0, ul_snr=24.0, seed=1, nof_ues=3, pbch=0,
                 nof_ports=1, mcs_max=16):
        import sync_lib as S
        import track_lib as T
        import track_ul_lib as U
        self.N, self.SF, self.nsf = N, 15 * N, nsf
        prb = T.PRB_OF[N]
        self.cell = ltelib.Cell(prb, nof_ports, pci, 1, N)
        self.ul_cell = ltelib.Cell(prb, 1, pci, 2, N)
        s = S.sim(sync=1, cell=self.cell, seed=seed, snr_db=snr, nof_ues=nof_ues, dl_min=1, dl_max=2, ul_min=1, ul_max=2, ul_pusch=1, pbch=pbch,
                  tm=1 if nof_ports == 1 else 2, mcs_min=2, mcs_max=mcs_max)
        self.dl = [s.subframe(t) for t in range(nsf)]
        ue = ltelib.Sim(cell=self.ul_cell, seed=seed + 100, snr_db=300.0, nof_ues=1, chan_delay=2)
        self.ucfg = ltelib.UlCfg(**U.UCFG)
        ul, self.grants, self.sent = [], [], {}
        for k in range(nsf):
            gl = U.ul_grants_of(self.cell, self.dl[k - 4][1]) if k >= 4 else []
            u, pl, off = sim_ul_rx(ue, k, self.ucfg, gl, 2)
            ul.append(u)
            self.grants.append(gl)
            for g, of in zip(gl, off):
                self.sent[(k, int(g.rnti), int(g.n_prb))] = bytes(pl[of:of + g.tbs // 8])
        ul = np.array(ul)                                                   # [nsf][2][15 N]
        ul[:, 1] *= np.sqrt(np.mean(np.abs(ul[:, 0]) ** 2) / np.mean(np.abs(ul[:, 1]) ** 2))
        rng = np.random.default_rng(seed + 200)
        sigma = 10 ** (-ul_snr / 20) * np.sqrt(0.5)
        ul = ul + sigma * (rng.standard_normal(ul.shape) + 1j * rng.standard_normal(ul.shape))
        self.ul = ul.astype(np.complex64)
        tx = np.concatenate([np.zeros((1, lead))] + [q[0][:1] for q in self.dl], axis=1)
        txu = np.concatenate([np.zeros((2, lead + ul_offset))] + list(self.ul), axis=1)
        Ltot = min(tx.shape[1], txu.shape[1]) - 2 * T.TAPS
        x = T.resample(tx, ppm, Ltot) if ppm else tx[:, :Ltot].astype(complex)
        xu = T.resample(txu, ppm, Ltot) if ppm else txu[:, :Ltot].astype(complex)
        ts = np.arange(Ltot) / (15000.0 * N)
        ph = 2 * np.pi * cfo * ts
        self.x = (x * np.exp(1j * ph)).astype(np.complex64)
        self.xu = (xu * np.exp(1j * rho * ph)).astype(np.complex64)

