"""ctypes bindings for the tracker's oracle (oracle_track/liblteotrack.so, lteo_track_*) and the captures the tracker tests feed it: simulator
subframes with their sync signals, a sampling-clock offset applied with a band-limited resampler, a continuous carrier offset that may ramp, and
the true start of every subframe in receiver samples.  Also two-carrier captures (DESIGN.md §2, "tracking", uplink): the downlink of a simulated
cell with its DCI-0s and the uplink of the UEs those DCI-0s schedule, on one or two UL antennas, and an oracle PUSCH decode of given uplink
subframes.  Imported only by tests/."""
import ctypes as C
import os

import numpy as np

import ltelib
import pusch_rx_lib as X
import ref64_sync as R
import sync_lib as S

SF_DTYPE = np.dtype([("start", "<i8"), ("tti", "<u4"), ("cfo_hz", "<f4"), ("flags", "<u4"), ("index", "<u4")])
HF_DTYPE = np.dtype([("tau", "<i8"), ("index", "<u4"), ("delta", "<i4"), ("peak", "<f4"), ("s_re", "<f4"), ("s_im", "<f4"), ("f_meas", "<f4"),
                     ("flags", "<u4"), ("pad", "<u4")])
NO_CFO, LOCKED, LOST = 1, 1, 2
PRB_OF = {128: 6, 256: 15, 384: 25, 512: 25, 768: 50, 1024: 50, 1536: 75, 2048: 100}
TAPS = 64          # resampler length: a Kaiser-windowed sinc
BETA = 9.0
UCFG = dict(n_dmrs1=2, delta_ss=1)

_lib = None


def lib():
    global _lib
    if _lib is None:
        ltelib.build_infra()
        L = C.CDLL(os.path.join(ltelib.ROOT, "oracle_track", "liblteotrack.so"))
        P, U32, U64 = C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
        L.lteo_track_create.restype = P
        L.lteo_track_create.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_float, C.c_uint32]
        L.lteo_track_destroy.argtypes = [P]
        L.lteo_track_set_ul.argtypes = [P, C.c_double, C.c_int32]
        L.lteo_track_set_ul_rx.argtypes = [P, C.c_double, C.c_int32, C.c_uint32]
        L.lteo_track_push.argtypes = [P, P, C.c_uint64, C.c_uint64, C.c_uint32, P, U32, P, U32, P, U64]
        L.lteo_track_push_ul.argtypes = [P, P, P, C.c_uint64, C.c_uint64, C.c_uint32, P, U32, P, U32, P, P, U64]
        L.lteo_track_finds.restype = C.c_uint32
        L.lteo_track_finds.argtypes = [P]
        _lib = L
    return _lib


class Oracle:
    """lteo_track_* with the arguments of capi.Tracker: ul=dict(cfo_ratio, ul_offset, nof_rx) sets the uplink (lteo_track_set_ul_rx), push_ul then
    takes xu [n] ([A][n] with A = 2 UL antennas) and returns ul_iq [k][15 N] ([k][A][15 N]).  Every push reports finds, the find windows it
    searched (ltephy_track_out_t.finds)."""

    def __init__(self, N, nrx, pci, frame_offset, cfo_hz=0.0, first_tti=0, flags=0, ul=None):
        self.N, self.A = N, nrx
        self.t = lib().lteo_track_create(N, nrx, pci, first_tti, frame_offset, cfo_hz, flags)
        assert self.t, "lteo_track_create refused the arguments"
        self.next_sample = frame_offset
        self.UA = None
        if ul is not None:
            ratio, off, self.UA = float(ul.get("cfo_ratio", 1.0)), int(ul.get("ul_offset", 0)), max(1, int(ul.get("nof_rx", 1)))
            assert lib().lteo_track_set_ul_rx(self.t, ratio, off, self.UA) == 0
            self.next_sample = min(frame_offset, frame_offset + off)

    def close(self):
        if self.t:
            lib().lteo_track_destroy(self.t)
            self.t = None

    def __del__(self):
        self.close()

    def push(self, x, first, max_sf=1000, cut=True):
        return self._push(x, None, first, max_sf, cut)

    def push_ul(self, x, xu, first, max_sf=1000, cut=True):
        return self._push(x, xu, first, max_sf, cut)

    def _push(self, x, xu, first, max_sf, cut):
        x = np.ascontiguousarray(x, np.complex64)
        sf, hf = np.zeros(max_sf, SF_DTYPE), np.zeros(max_sf // 5 + 1, HF_DTYPE)
        iq = np.zeros((max_sf, self.A, 15 * self.N), np.complex64) if cut else None
        nsf, nhf, nxt = C.c_uint32(), C.c_uint32(), C.c_uint64()
        out = (ltelib.ptr(sf), C.byref(nsf), ltelib.ptr(hf), C.byref(nhf), ltelib.ptr(iq) if cut else None)
        finds = lib().lteo_track_finds(self.t)
        if xu is None:
            r = lib().lteo_track_push(self.t, ltelib.ptr(x), first, x.shape[1], max_sf, *out, C.byref(nxt))
        else:
            xu = np.ascontiguousarray(xu, np.complex64).reshape(self.UA, -1)
            assert xu.shape[1] == x.shape[1]
            iqu = np.zeros((max_sf, self.UA, 15 * self.N), np.complex64) if cut else None
            r = lib().lteo_track_push_ul(self.t, ltelib.ptr(x), ltelib.ptr(xu), first, x.shape[1], max_sf, *out, ltelib.ptr(iqu) if cut else None,
                                         C.byref(nxt))
        assert r == 0, r
        self.next_sample, k = nxt.value, nsf.value
        o = dict(sf=sf[:k], hf=hf[:nhf.value], iq=iq[:k] if cut else None, next_sample=nxt.value, finds=lib().lteo_track_finds(self.t) - finds)
        if xu is not None:
            o["ul_iq"] = (iqu[:k, 0] if self.UA == 1 else iqu[:k]) if cut else None
        return o


def run_chunks(tr, x, sizes, first=0, xu=None, push=None):
    """stream x (absolute samples first ...), and with xu ([n] or [A][n]) the uplink with it, into a tracker (Oracle or capi.Tracker): the
    recording arrives in pieces of the given sizes (cycled), and each push passes everything from the tracker's next_sample to the end of what has
    arrived -> the concatenated records and cuts, the summed finds and the tracker's last next_sample"""
    push = push or (tr.push if xu is None else tr.push_ul)
    outs, recv, i, end = [], first, 0, first + x.shape[1]
    while True:
        if recv < end:
            recv = min(recv + sizes[i % len(sizes)], end)
            i += 1
        start = tr.next_sample
        if start < recv:
            a, b = start - first, recv - first
            if xu is None:
                o = push(x[:, a:b], start)
            else:   # xu has an antenna axis when it has as many axes as x ([A][n], or [A][n][2] for integer samples)
                o = push(x[:, a:b], xu[:, a:b] if xu.ndim == x.ndim else xu[a:b], start)
            outs.append(o)
            if recv == end and not len(o["sf"]):
                break
        elif recv == end:
            break
    host = lambda q: q if isinstance(q, np.ndarray) else q.cpu().numpy()
    cut = lambda k: np.concatenate([host(o[k]) for o in outs if o[k] is not None and len(o["sf"])] or [np.zeros(0, np.complex64)])
    r = dict(sf=np.concatenate([o["sf"] for o in outs]), hf=np.concatenate([o["hf"] for o in outs]), iq=cut("iq"),
             finds=sum(o["finds"] for o in outs), next_sample=tr.next_sample)
    if xu is not None:
        r["ul_iq"] = cut("ul_iq")
    return r


def kernel(frac):
    """TAPS coefficients of the Kaiser-windowed sinc that delays by frac in [0, 1): taps at integer offsets -TAPS/2 + 1 .. TAPS/2"""
    i = np.arange(-TAPS // 2 + 1, TAPS // 2 + 1)
    t = i - np.asarray(frac)[..., None]
    w = np.kaiser(TAPS + 1, BETA)
    wt = np.interp(t, np.arange(-TAPS // 2, TAPS // 2 + 1), w)
    return np.sinc(t) * wt


PHASES = 8192
_tab = None


def _table():
    global _tab
    if _tab is None:
        _tab = kernel(np.arange(PHASES) / PHASES)
    return _tab


def resample(x, ppm, L):
    """receiver samples n = 0 .. L - 1 of a transmit signal x [A][M] sampled with a clock off by ppm: sample n is at transmit time n (1 + ppm 1e-6),
    interpolated with the TAPS-tap windowed sinc (samples outside x count as 0)"""
    x = np.asarray(x, complex)
    t = np.arange(L) * (1.0 + ppm * 1e-6)
    base = np.floor(t).astype(np.int64)
    ph = np.rint((t - base) * PHASES).astype(np.int64)   # the delay rounded to 1 / PHASES of a sample
    base, ph = base + ph // PHASES, ph % PHASES
    h = _table()[ph]                                # [L][TAPS]
    out = np.zeros((x.shape[0], L), complex)
    xp = np.concatenate([np.zeros((x.shape[0], TAPS)), x, np.zeros((x.shape[0], TAPS))], axis=1)
    for j, i in enumerate(range(-TAPS // 2 + 1, TAPS // 2 + 1)):
        idx = np.clip(base + i + TAPS, 0, xp.shape[1] - 1)
        out += xp[:, idx] * h[None, :, j]
    return out


def capture(N, pci, nsf, nrx=1, ppm=0.0, cfo=0.0, ramp=0.0, snr=40.0, lead=0, seed=1, chan_delay=0, t0=0, gap=None, nof_ues=3):
    """nsf sync = 1 subframes (the first is subframe t0) per antenna after `lead` zero samples, at a receiver clock ppm off, with the carrier offset
    cfo + ramp t (Hz, t in seconds of receiver time) applied in float64, an optional zero-filled gap (first, count) in receiver samples.
    -> (x complex64 [nrx][L], truth starts of the subframes in receiver samples, truth carrier offset at each subframe start)"""
    SF = 15 * N
    if N == 128:
        rng = np.random.default_rng(seed)
        tx = np.array([R.synth(N, pci, nsf, rng, t0) for _ in range(nrx)])
        tx = tx + (rng.standard_normal(tx.shape) + 1j * rng.standard_normal(tx.shape)) * np.sqrt(0.5 * 10 ** (-snr / 10))
    else:
        cell = ltelib.Cell(PRB_OF[N], 1, pci, nrx, N)
        s = S.sim(sync=1, cell=cell, seed=seed, snr_db=snr, nof_ues=nof_ues, dl_min=1, dl_max=3, chan_delay=chan_delay)
        tx = np.concatenate([s.subframe(t0 + i)[0] for i in range(nsf)], axis=1).astype(complex)
    tx = np.concatenate([np.zeros((nrx, lead)), tx], axis=1)
    L = int(np.floor((tx.shape[1] - TAPS) / (1.0 + ppm * 1e-6)))
    x = resample(tx, ppm, L) if ppm else tx[:, :L]
    n = np.arange(L)
    ts = n / (15000.0 * N)
    x = x * np.exp(2j * np.pi * (cfo * ts + 0.5 * ramp * ts ** 2))
    if gap:
        x[:, gap[0]:gap[0] + gap[1]] = 0
    truth = (lead + np.arange(nsf) * SF) / (1.0 + ppm * 1e-6)
    f_truth = cfo + ramp * truth / (15000.0 * N)
    return x.astype(np.complex64), truth, f_truth


def ul_grants_of(cell, truth):
    """the PUSCH grants (ltelib.UlGrant) of the DCI-0s the simulator sent in one downlink subframe"""
    Sm = ltelib.sim()
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
    """A two-carrier capture of nsf subframes.  x complex64 [nrx][L] (downlink), xu complex64 [L] (uplink, one antenna; [2][L] antenna-major with
    ul_nof_rx = 2), both in receiver samples of a clock ppm off; the downlink's subframe 0 starts at `lead` transmit samples, the uplink's at
    lead + ul_offset.  dl[k] = (iq, truth, payload) of DL subframe k; ul[k] = the aligned, offset-free UL subframe k (complex64 [15 N]; [2][15 N]
    with two antennas); grants[k] = its PUSCH grants (from the DCI-0s of DL subframe k - 4); sent[(k, rnti, n_prb)] = the transport block bytes;
    tti[k] = k.  One UL antenna carries the simulator's noise at ul_snr.  Two come from lte_sim_ul_subframe_rx without noise; antenna 1 is scaled
    to antenna 0's power (the simulator's cross-port gain is 0.35), and each antenna gets its own white noise of power 10^(-ul_snr / 10) before
    the common clock and carrier offsets."""

    def __init__(self, N, pci, nsf, nrx=1, ppm=0.0, cfo=0.0, ramp=0.0, rho=1.0, lead=1000, ul_offset=0, snr=25.0, ul_snr=24.0, seed=1, nof_ues=3,
                 pbch=0, nof_ports=1, mcs_max=16, ul_nof_rx=1):
        assert ul_nof_rx == 1 or ramp == 0.0, "the two-antenna uplink has no carrier-offset ramp"
        self.N, self.SF, self.nsf, self.lead, self.ul_offset = N, 15 * N, nsf, lead, ul_offset
        prb = PRB_OF[N]
        self.cell = ltelib.Cell(prb, nof_ports, pci, nrx, N)
        self.ul_cell = ltelib.Cell(prb, 1, pci, ul_nof_rx, N)
        s = S.sim(sync=1, cell=self.cell, seed=seed, snr_db=snr, nof_ues=nof_ues, dl_min=1, dl_max=2, ul_min=1, ul_max=2, ul_pusch=1, pbch=pbch,
                  tm=1 if nof_ports == 1 else 2, mcs_min=2, mcs_max=mcs_max)
        self.dl = [s.subframe(t) for t in range(nsf)]
        ue = ltelib.Sim(cell=self.ul_cell, seed=seed + 100, snr_db=ul_snr if ul_nof_rx == 1 else 300.0, nof_ues=1, chan_delay=2)
        self.ucfg = ltelib.UlCfg(**UCFG)
        self.ul, self.grants, self.sent = [], [], {}
        for k in range(nsf):
            gl = ul_grants_of(self.cell, self.dl[k - 4][1]) if k >= 4 else []
            u, pl, off = ltelib.sim_ul_subframe(ue, k, self.ucfg, gl) if ul_nof_rx == 1 else X.sim_ul_rx(ue, k, self.ucfg, gl, ul_nof_rx)
            self.ul.append(u)
            self.grants.append(gl)
            for g, of in zip(gl, off):
                self.sent[(k, int(g.rnti), int(g.n_prb))] = bytes(pl[of:of + g.tbs // 8])
        if ul_nof_rx > 1:
            ul = np.array(self.ul)                                              # [nsf][2][15 N]
            ul[:, 1] *= np.sqrt(np.mean(np.abs(ul[:, 0]) ** 2) / np.mean(np.abs(ul[:, 1]) ** 2))
            rng = np.random.default_rng(seed + 200)
            sigma = 10 ** (-ul_snr / 20) * np.sqrt(0.5)
            self.ul = (ul + sigma * (rng.standard_normal(ul.shape) + 1j * rng.standard_normal(ul.shape))).astype(np.complex64)
        self.tti = np.arange(nsf, dtype=np.uint32)
        tx = np.concatenate([np.zeros((nrx, lead))] + [q[0] for q in self.dl], axis=1)
        txu = np.concatenate([np.zeros((ul_nof_rx, lead + ul_offset))] + [np.reshape(u, (ul_nof_rx, -1)) for u in self.ul], axis=1)
        Ltot = min(tx.shape[1], txu.shape[1]) - 2 * TAPS
        x = resample(tx, ppm, Ltot) if ppm else tx[:, :Ltot].astype(complex)
        xu = resample(txu, ppm, Ltot) if ppm else txu[:, :Ltot].astype(complex)
        ts = np.arange(Ltot) / (15000.0 * N)
        # each recipe keeps the grouping its recordings were made with: the roundings of the two differ in the last bit
        ph = 2 * np.pi * (cfo * ts + 0.5 * ramp * ts ** 2) if ul_nof_rx == 1 else 2 * np.pi * cfo * ts
        self.x = (x * np.exp(1j * ph)).astype(np.complex64)
        self.xu = ((xu[0] if ul_nof_rx == 1 else xu) * np.exp(1j * rho * ph)).astype(np.complex64)


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
