"""ctypes bindings for the channeliser's rational oracle (oracle/liblteochanpoly.so, lteo_chan_*_poly), a float64 numpy restatement of the
rational rule (DESIGN.md §2 "channeliser"), integer sample conversion, and a composer of wideband captures at any rate: narrowband simulator cells
resampled to the capture rate by a long scipy filter that shares nothing with the rule.  Imported only by tests/."""
import ctypes as C
import math
import os

import numpy as np

import chan_lib as CH
import ltelib
import track_lib as T

RATIONAL = 1
FORMATS = {"cf32": 0, "sc16": 1, "sc8": 2}
MAX_L, MAX_TABLE = 1024, 1 << 15


class Poly(C.Structure):
    _fields_ = [(k, C.c_uint32) for k in ("L", "M", "Tp", "Kp", "Ka", "Kb", "P")]


_lib = None


def lib():
    global _lib
    if _lib is None:
        ltelib.build_infra()
        L = C.CDLL(os.path.join(ltelib.ROOT, "oracle", "liblteochanpoly.so"))
        L.lteo_chan_design_poly.argtypes = [C.c_uint32, C.c_int32, C.c_uint32, C.c_uint32, C.POINTER(Poly), C.c_void_p, C.c_void_p, C.c_void_p]
        L.lteo_chan_run_poly.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                         C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


def _geo(q):
    return {k: getattr(q, k) for k, _ in Poly._fields_}


def design(fs_in, offset_hz, N, flags=RATIONAL):
    """lteo_chan_design_poly -> dict(L, M, Tp, Kp, Ka, Kb, P, hp f32 [Tp], g complex64 [L][Kp], rot complex64 [P]), or None when refused"""
    q = Poly()
    if lib().lteo_chan_design_poly(fs_in, offset_hz, N, flags, C.byref(q), None, None, None) != 0:
        return None
    d = _geo(q)
    hp, g, rot = np.zeros(q.Tp, np.float32), np.zeros((q.L, q.Kp), np.complex64), np.zeros(q.P, np.complex64)
    assert lib().lteo_chan_design_poly(fs_in, offset_hz, N, flags, C.byref(q), ltelib.ptr(hp), ltelib.ptr(g), ltelib.ptr(rot)) == 0
    d.update(hp=hp, g=g, rot=rot)
    return d


def to_format(x, fmt, seed=0):
    """x complex [nof_rx][n] (|re|, |im| below 1) -> (samples in fmt: complex64, or int16 / int8 [nof_rx][2n], and the exact complex64 they stand for)"""
    if fmt == "cf32":
        x = np.ascontiguousarray(x, np.complex64)
        return x, x
    scale, dt = (32768.0, np.int16) if fmt == "sc16" else (128.0, np.int8)
    iq = np.empty(x.shape[:-1] + (2 * x.shape[-1],), np.float64)
    iq[..., 0::2], iq[..., 1::2] = x.real, x.imag
    q = np.clip(np.round(iq * scale), np.iinfo(dt).min, np.iinfo(dt).max).astype(dt)
    f = q.astype(np.float32) / np.float32(scale)
    return np.ascontiguousarray(q), np.ascontiguousarray(f[..., 0::2] + 1j * f[..., 1::2]).astype(np.complex64)


def run(fs_in, carriers, x, first, fmt="cf32", flags=RATIONAL):
    """lteo_chan_run_poly on x (complex64 [nof_rx][n], or int16 / int8 [nof_rx][2n] in fmt) -> ([dict(first, count, iq)], next_sample)"""
    x = np.ascontiguousarray(x)
    A = x.shape[0]
    n = x.shape[1] if fmt == "cf32" else x.shape[1] // 2
    cap = 0
    for off, N in carriers:
        d = design(fs_in, off, N, flags)
        assert d is not None, (fs_in, off, N)
        cap = max(cap, n * d["L"] // d["M"] + 2)
    outs = [np.zeros((A, cap), np.complex64) for _ in carriers]
    ptrs = (C.c_void_p * len(carriers))(*[o.ctypes.data for o in outs])
    off = np.array([c[0] for c in carriers], np.int32)
    Ns = np.array([c[1] for c in carriers], np.uint32)
    m0, cnt, nxt = np.zeros(len(carriers), np.uint64), np.zeros(len(carriers), np.uint64), C.c_uint64()
    r = lib().lteo_chan_run_poly(fs_in, flags, FORMATS[fmt], A, len(carriers), ltelib.ptr(off), ltelib.ptr(Ns), x.ctypes.data, first, n, ptrs, cap,
                                 ltelib.ptr(m0), ltelib.ptr(cnt), C.byref(nxt))
    assert r == 0, r
    res = []
    for c in range(len(carriers)):
        k = int(cnt[c])
        res.append(dict(first=int(m0[c]), count=k, iq=outs[c].ravel()[:A * k].reshape(A, k).copy()))
    return res, nxt.value


# ---- float64 restatement of the rational rule ------------------------------------------------------------------------------------------
def geometry(fs_in, offset_hz, N):
    """dict(L, M, Tp, Kp, Ka, Kb, P, f_pass, w) of a rational carrier from the rule (scipy.signal.kaiserord), or None when it refuses"""
    import scipy.signal as ss
    if N not in CH.MAX_PRB or not 0 < fs_in <= 245760000 or offset_hz % 1000:
        return None
    fs_out = 15000 * N
    g = math.gcd(fs_out, fs_in)
    L, M = fs_out // g, fs_in // g
    f_pass = 90000 * CH.MAX_PRB[N]
    if L > MAX_L or M > 128 * L or L > 2 * M or abs(offset_hz) + f_pass > fs_in / 2:
        return None
    w = (min(fs_in, fs_out) - 2 * f_pass) / (L * fs_in / 2)
    Tp = ss.kaiserord(CH.ATTEN, w)[0] | 1
    Hp = (Tp - 1) // 2
    Ka, Kb = Hp // L, -(-Hp // L)
    if L * (Ka + Kb + 1) > MAX_TABLE:
        return None
    P = fs_out // math.gcd(offset_hz % fs_out, fs_out)
    return dict(L=L, M=M, Tp=Tp, Kp=Ka + Kb + 1, Ka=Ka, Kb=Kb, P=P, f_pass=f_pass, w=w)


def reference(fs_in, offset_hz, N, x, ms):
    """float64 outputs ms of a rational carrier from x complex [n] (capture samples 0 .., zero before 0), with the float prototype hp of the rule"""
    d = design(fs_in, offset_hz, N)
    hp = d["hp"].astype(np.float64)
    L, M, Tp, Ka, Kb = d["L"], d["M"], d["Tp"], d["Ka"], d["Kb"]
    Hp = (Tp - 1) // 2
    ms = np.asarray(ms, np.int64)
    n, ph = ms * M // L, ms * M % L
    k = np.arange(-Kb, Ka + 1)
    idx = Hp + ph[:, None] + L * k[None, :]
    tap = np.where((idx >= 0) & (idx < Tp), hp[np.clip(idx, 0, Tp - 1)], 0.0)
    s = n[:, None] - k[None, :]
    xs = np.where(s >= 0, np.asarray(x, np.complex128)[np.clip(s, 0, len(x) - 1)], 0)
    gph = 2 * np.pi * ((offset_hz * (ph[:, None] + L * k[None, :])) % (L * fs_in)) / (L * fs_in)
    fs_out = 15000 * N
    rph = -2 * np.pi * ((offset_hz * ms) % fs_out) / fs_out
    return np.exp(1j * rph) * (tap * np.exp(1j * gph) * xs).sum(axis=1)


# ---- wideband captures at any rate -------------------------------------------------------------------------------------------------------
def _resample(x, fs_from, fs_to):
    """x complex [A][n] at fs_from -> fs_to by scipy.signal.resample_poly with a long Kaiser filter (beta 12, 40 zero crossings a side)"""
    import scipy.signal as ss
    g = math.gcd(fs_from, fs_to)
    up, down = fs_to // g, fs_from // g
    h = ss.firwin(2 * 40 * max(up, down) + 1, 1.0 / max(up, down), window=("kaiser", 12.0)) * up
    return ss.resample_poly(x.astype(np.complex128), up, down, axis=1, window=h)


def compose(fs_in, carriers, nsf, nrx=1, ppm=0.0, noise_db=-40.0, seed=1):
    """chan_lib.compose at any fs_in: each carrier (cell_capture when decode=True, else track_lib.capture) resampled from 15 kHz * N to fs_in
    with _resample, shifted by offset_hz and scaled by gain_db, plus complex noise.  -> (x complex64 [nrx][L], [dict(truth starts in carrier
    samples, narrow, sub)])"""
    rng = np.random.default_rng(seed)
    parts, truths = [], []
    for i, c in enumerate(carriers):
        N = c["N"]
        sub = None
        if c.get("decode"):
            xn, truth, sub = CH.cell_capture(c, nsf, nrx, ppm, seed * 17 + i)
        else:
            xn, truth, _ = T.capture(N, c["pci"], nsf, nrx=nrx, ppm=ppm, cfo=c.get("cfo", 0.0), snr=c.get("snr", 60.0), lead=c.get("lead", 0),
                                     seed=seed * 17 + i)
        pw = np.mean(np.abs(xn[:, c.get("lead", 0):]) ** 2)
        up = _resample(xn / np.sqrt(pw), 15000 * N, fs_in)
        parts.append(up * 10 ** (c.get("gain_db", 0.0) / 20))
        truths.append(dict(truth=truth, narrow=xn, sub=sub))
    L = min(p.shape[1] for p in parts)
    n = np.arange(L)
    x = np.zeros((nrx, L), np.complex128)
    for c, p in zip(carriers, parts):
        x += p[:, :L] * np.exp(2j * np.pi * ((c["offset_hz"] * n) % fs_in) / fs_in)
    sig = 10 ** (noise_db / 20) * np.sqrt(0.5)
    x += sig * (rng.standard_normal(x.shape) + 1j * rng.standard_normal(x.shape))
    return x.astype(np.complex64), truths
