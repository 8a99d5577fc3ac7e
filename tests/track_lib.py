"""ctypes bindings for the tracker's oracle (oracle_track/liblteotrack.so, lteo_track_*) and the captures the tracker tests feed it: simulator
subframes with their sync signals, a sampling-clock offset applied with a band-limited resampler, a continuous carrier offset that may ramp, and
the true start of every subframe in receiver samples.  Imported only by tests/."""
import ctypes as C
import os

import numpy as np

import ltelib
import ref64_sync as R
import sync_lib as S

SF_DTYPE = np.dtype([("start", "<i8"), ("tti", "<u4"), ("cfo_hz", "<f4"), ("flags", "<u4"), ("index", "<u4")])
HF_DTYPE = np.dtype([("tau", "<i8"), ("index", "<u4"), ("delta", "<i4"), ("peak", "<f4"), ("s_re", "<f4"), ("s_im", "<f4"), ("f_meas", "<f4"),
                     ("flags", "<u4"), ("pad", "<u4")])
NO_CFO, LOCKED, LOST = 1, 1, 2
PRB_OF = {128: 6, 256: 15, 384: 25, 512: 25, 768: 50, 1024: 50, 1536: 75, 2048: 100}
TAPS = 64          # resampler length: a Kaiser-windowed sinc
BETA = 9.0

_lib = None


def lib():
    global _lib
    if _lib is None:
        ltelib.build_infra()
        L = C.CDLL(os.path.join(ltelib.ROOT, "oracle_track", "liblteotrack.so"))
        L.lteo_track_create.restype = C.c_void_p
        L.lteo_track_create.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_float, C.c_uint32]
        L.lteo_track_destroy.argtypes = [C.c_void_p]
        L.lteo_track_push.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.c_void_p,
                                      C.POINTER(C.c_uint32), C.c_void_p, C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


class Oracle:
    """lteo_track_* with the arguments of capi.Tracker"""

    def __init__(self, N, nrx, pci, frame_offset, cfo_hz=0.0, first_tti=0, flags=0):
        self.N, self.A = N, nrx
        self.t = lib().lteo_track_create(N, nrx, pci, first_tti, frame_offset, cfo_hz, flags)
        assert self.t, "lteo_track_create refused the arguments"
        self.next_sample = frame_offset

    def close(self):
        if self.t:
            lib().lteo_track_destroy(self.t)
            self.t = None

    def __del__(self):
        self.close()

    def push(self, x, first, max_sf=1000, cut=True):
        x = np.ascontiguousarray(x, np.complex64)
        sf, hf = np.zeros(max_sf, SF_DTYPE), np.zeros(max_sf // 5 + 1, HF_DTYPE)
        iq = np.zeros((max_sf, self.A, 15 * self.N), np.complex64) if cut else None
        nsf, nhf, nxt = C.c_uint32(), C.c_uint32(), C.c_uint64()
        r = lib().lteo_track_push(self.t, ltelib.ptr(x), first, x.shape[1], max_sf, ltelib.ptr(sf), C.byref(nsf), ltelib.ptr(hf), C.byref(nhf),
                                  ltelib.ptr(iq) if cut else None, C.byref(nxt))
        assert r == 0, r
        self.next_sample = nxt.value
        return dict(sf=sf[:nsf.value], hf=hf[:nhf.value], iq=iq[:nsf.value] if cut else None, next_sample=nxt.value)


def run_chunks(tr, x, sizes, first=0, push=None, **kw):
    """stream x (absolute samples first ...) into a tracker (Oracle or capi.Tracker): the recording arrives in pieces of the given sizes (cycled),
    and each push passes everything from the tracker's next_sample to the end of what has arrived; returns the concatenated records and cut"""
    push = push or tr.push
    outs, recv, i, end = [], first, 0, first + x.shape[1]
    while True:
        if recv < end:
            recv = min(recv + sizes[i % len(sizes)], end)
            i += 1
        start = tr.next_sample
        if start < recv:
            o = push(x[:, start - first:recv - first], start, **kw)
            outs.append(o)
            if recv == end and not len(o["sf"]):
                break
        elif recv == end:
            break
    cat = lambda k: np.concatenate([o[k] for o in outs])
    iqs = [o["iq"] for o in outs if o["iq"] is not None and len(o["iq"])]
    if iqs and not isinstance(iqs[0], np.ndarray):
        iqs = [q.cpu().numpy() for q in iqs]
    return dict(sf=cat("sf"), hf=cat("hf"), iq=np.concatenate(iqs) if iqs else np.zeros(0, np.complex64))


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
