"""Two-carrier captures for the uplink tracker tests (DESIGN.md §2, "tracking", uplink): the downlink of a simulated cell with its sync signals and
DCI-0s, the uplink of the UEs those DCI-0s schedule (PUSCH in subframe n + 4), both resampled with one sampling clock, the downlink rotated by
f(t) and the uplink by rho f(t), and the uplink starting ul_offset samples after the downlink.  Also the oracle tracker with its uplink set
(lteo_track_set_ul / lteo_track_push_ul), and an oracle PUSCH decode of given uplink subframes.  Imported only by tests/."""
import ctypes as C

import numpy as np

import ltelib
import sync_lib as S
import track_lib as T

UCFG = dict(n_dmrs1=2, delta_ss=1)


def lib():
    L = T.lib()
    if not getattr(L, "_ul_bound", False):
        L.lteo_track_set_ul.argtypes = [C.c_void_p, C.c_double, C.c_int32]
        L.lteo_track_push_ul.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32),
                                         C.c_void_p, C.POINTER(C.c_uint32), C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        L._ul_bound = True
    return L


class OracleUl(T.Oracle):
    """lteo_track_* with the uplink set: the arguments of capi.Tracker(..., ul=dict(cfo_ratio, ul_offset))"""

    def __init__(self, N, nrx, pci, frame_offset, cfo_hz=0.0, first_tti=0, flags=0, cfo_ratio=1.0, ul_offset=0):
        super().__init__(N, nrx, pci, frame_offset, cfo_hz=cfo_hz, first_tti=first_tti, flags=flags)
        assert lib().lteo_track_set_ul(self.t, cfo_ratio, ul_offset) == 0
        self.next_sample = min(frame_offset, frame_offset + ul_offset)

    def push_ul(self, x, xu, first, max_sf=1000, cut=True):
        x = np.ascontiguousarray(x, np.complex64)
        xu = np.ascontiguousarray(xu, np.complex64).reshape(-1)
        assert xu.shape[0] == x.shape[1]
        sf, hf = np.zeros(max_sf, T.SF_DTYPE), np.zeros(max_sf // 5 + 1, T.HF_DTYPE)
        iq = np.zeros((max_sf, self.A, 15 * self.N), np.complex64) if cut else None
        iqu = np.zeros((max_sf, 15 * self.N), np.complex64) if cut else None
        nsf, nhf, nxt = C.c_uint32(), C.c_uint32(), C.c_uint64()
        r = lib().lteo_track_push_ul(self.t, ltelib.ptr(x), ltelib.ptr(xu), first, x.shape[1], max_sf, ltelib.ptr(sf), C.byref(nsf), ltelib.ptr(hf),
                                     C.byref(nhf), ltelib.ptr(iq) if cut else None, ltelib.ptr(iqu) if cut else None, C.byref(nxt))
        assert r == 0, r
        self.next_sample = nxt.value
        k = nsf.value
        return dict(sf=sf[:k], hf=hf[:nhf.value], iq=iq[:k] if cut else None, ul_iq=iqu[:k] if cut else None, next_sample=nxt.value)


def run_chunks_ul(tr, x, xu, sizes, first=0, push=None):
    """track_lib.run_chunks for both carriers: the recording arrives in pieces of the given sizes (cycled) and each push passes everything from
    the tracker's next_sample to the end of what has arrived -> concatenated records, DL cut and UL cut"""
    push = push or tr.push_ul
    outs, recv, i, end = [], first, 0, first + x.shape[1]
    while True:
        if recv < end:
            recv = min(recv + sizes[i % len(sizes)], end)
            i += 1
        start = tr.next_sample
        if start < recv:
            o = push(x[:, start - first:recv - first], xu[start - first:recv - first], start)
            outs.append(o)
            if recv == end and not len(o["sf"]):
                break
        elif recv == end:
            break
    cat = lambda k: np.concatenate([o[k] for o in outs])
    host = lambda q: q if isinstance(q, np.ndarray) else q.cpu().numpy()
    iq = [host(o["iq"]) for o in outs if len(o["sf"])]
    iqu = [host(o["ul_iq"]) for o in outs if len(o["sf"])]
    return dict(sf=cat("sf"), hf=cat("hf"), iq=np.concatenate(iq) if iq else np.zeros(0, np.complex64),
                ul_iq=np.concatenate(iqu) if iqu else np.zeros(0, np.complex64))


def ul_grants_of(cell, truth):
    """the PUSCH grants (ltelib.UlGrant) of the DCI-0s the simulator sent in one downlink subframe"""
    Sm = ltelib.sim()
    Sm.lte_dci_unpack.argtypes = [C.POINTER(ltelib.Cell), C.c_int, C.c_uint16, C.c_void_p, C.c_uint32, C.POINTER(ltelib.Dci)]
    Sm.lte_ul_dci_to_grant.argtypes = [C.POINTER(ltelib.Cell), C.POINTER(ltelib.Dci), C.c_int, C.POINTER(ltelib.UlGrant)]
    out = []
    for k in range(truth.nof_dci):
        d = truth.dci[k]
        if d.format != 0:
            continue
        bits = np.frombuffer(bytes(d.bits), np.uint8)[:d.nbits].copy()
        dd, g = ltelib.Dci(), ltelib.UlGrant()
        assert Sm.lte_dci_unpack(C.byref(cell), 0, d.rnti, ltelib.ptr(bits), d.nbits, C.byref(dd)) == 0
        assert Sm.lte_ul_dci_to_grant(C.byref(cell), C.byref(dd), 1, C.byref(g)) == 0
        out.append(g)
    return out


class TwoCarrier:
    """A two-carrier capture of nsf subframes.  x complex64 [nrx][L] (downlink), xu complex64 [L] (uplink, one antenna), both in receiver samples
    of a clock ppm off; the downlink's subframe 0 starts at `lead` transmit samples, the uplink's at lead + ul_offset.  dl[k] = (iq, truth,
    payload) of DL subframe k; ul[k] = the aligned, offset-free UL subframe k (complex64 [15 N]); grants[k] = its PUSCH grants (from the DCI-0s of
    DL subframe k - 4); sent[(k, rnti, n_prb)] = the transport block bytes; tti[k] = k."""

    def __init__(self, N, pci, nsf, nrx=1, ppm=0.0, cfo=0.0, ramp=0.0, rho=1.0, lead=1000, ul_offset=0, snr=25.0, ul_snr=24.0, seed=1, nof_ues=3,
                 pbch=0, nof_ports=1, mcs_max=16):
        self.N, self.SF, self.nsf, self.lead, self.ul_offset = N, 15 * N, nsf, lead, ul_offset
        prb = T.PRB_OF[N]
        self.cell = ltelib.Cell(prb, nof_ports, pci, nrx, N)
        self.ul_cell = ltelib.Cell(prb, 1, pci, 1, N)
        s = S.sim(sync=1, cell=self.cell, seed=seed, snr_db=snr, nof_ues=nof_ues, dl_min=1, dl_max=2, ul_min=1, ul_max=2, ul_pusch=1, pbch=pbch,
                  tm=1 if nof_ports == 1 else 2, mcs_min=2, mcs_max=mcs_max)
        self.dl = [s.subframe(t) for t in range(nsf)]
        ue = ltelib.Sim(cell=self.ul_cell, seed=seed + 100, snr_db=ul_snr, nof_ues=1, chan_delay=2)
        self.ucfg = ltelib.UlCfg(**UCFG)
        self.ul, self.grants, self.sent = [], [], {}
        for k in range(nsf):
            gl = ul_grants_of(self.cell, self.dl[k - 4][1]) if k >= 4 else []
            u, pl, off = ltelib.sim_ul_subframe(ue, k, self.ucfg, gl)
            self.ul.append(u)
            self.grants.append(gl)
            for g, of in zip(gl, off):
                self.sent[(k, int(g.rnti), int(g.n_prb))] = bytes(pl[of:of + g.tbs // 8])
        self.tti = np.arange(nsf, dtype=np.uint32)
        tx = np.concatenate([np.zeros((nrx, lead))] + [q[0] for q in self.dl], axis=1)
        txu = np.concatenate([np.zeros(lead + ul_offset)] + list(self.ul))[None, :]
        Ltot = min(tx.shape[1], txu.shape[1]) - 2 * T.TAPS
        x = T.resample(tx, ppm, Ltot) if ppm else tx[:, :Ltot].astype(complex)
        xu = T.resample(txu, ppm, Ltot)[0] if ppm else txu[0, :Ltot].astype(complex)
        ts = np.arange(Ltot) / (15000.0 * N)
        ph = 2 * np.pi * (cfo * ts + 0.5 * ramp * ts ** 2)
        self.x = (x * np.exp(1j * ph)).astype(np.complex64)
        self.xu = (xu * np.exp(1j * rho * ph)).astype(np.complex64)


def decode_ul(cap, iq_of, ks, cfo_hz=0.0):
    """oracle PUSCH decode (lteo_ul_ofdm + lteo_pusch_decode, after lteo_cfo_correct when cfo_hz) of the grants of UL subframes ks, iq_of(k) giving
    the subframe's samples -> set of (k, rnti, n_prb) whose CRC passed with the sent bytes"""
    o = ltelib.Oracle(cap.ul_cell)
    ok = set()
    for k in ks:
        if not cap.grants[k]:
            continue
        iq = np.ascontiguousarray(iq_of(k), np.complex64)
        if cfo_hz:
            iq = o.cfo_correct(cfo_hz, iq[None, :])[0]
        gs = [ltelib.UlGrant.from_buffer_copy(g) for g in cap.grants[k]]
        _, res = ltelib.oracle_ul(o, cap.ucfg, k, gs, iq)
        for g, (r, pl, crc, _, _) in zip(gs, res):
            key = (k, int(g.rnti), int(g.n_prb))
            if r == 0 and crc and bytes(pl[:g.tbs // 8]) == cap.sent[key]:
                ok.add(key)
    return ok
