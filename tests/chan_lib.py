"""ctypes bindings for the channeliser's oracle (oracle/liblteochan.so, lteo_chan_*), a float64 numpy restatement of its rule (DESIGN.md §2
"channeliser"), and a composer of wideband captures: several narrowband carriers from track_lib.capture, each upsampled to the capture rate,
shifted to its offset and summed, with wideband noise.  Imported only by tests/."""
import ctypes as C
import math
import os

import numpy as np

import ltelib
import sync_lib as S
import track_lib as T

MAX_PRB = {128: 6, 256: 15, 384: 25, 512: 25, 768: 50, 1024: 50, 1536: 100, 2048: 100}
SYMBOL_SIZES = sorted(MAX_PRB)
ATTEN = 70.0
BETA = 0.1102 * (ATTEN - 8.7)

_lib = None


def lib():
    global _lib
    if _lib is None:
        ltelib.build_infra()
        L = C.CDLL(os.path.join(ltelib.ROOT, "oracle", "liblteochan.so"))
        L.lteo_chan_design.argtypes = [C.c_uint32, C.c_int32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32),
                                       C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.lteo_chan_run.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p,
                                    C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


def design(fs_in, offset_hz, N):
    """lteo_chan_design -> dict(h, g, rot, T, D, P), or None when the rule refuses the carrier"""
    T_, D, P = C.c_uint32(), C.c_uint32(), C.c_uint32()
    if lib().lteo_chan_design(fs_in, offset_hz, N, None, None, None, C.byref(T_), C.byref(D), C.byref(P)) != 0:
        return None
    h, g, rot = np.zeros(T_.value, np.float32), np.zeros(T_.value, np.complex64), np.zeros(P.value, np.complex64)
    lib().lteo_chan_design(fs_in, offset_hz, N, ltelib.ptr(h), ltelib.ptr(g), ltelib.ptr(rot), C.byref(T_), C.byref(D), C.byref(P))
    return dict(h=h, g=g, rot=rot, T=T_.value, D=D.value, P=P.value)


def run(fs_in, carriers, x, first):
    """lteo_chan_run on x complex64 [nof_rx][n] (capture samples first ...) -> ([dict(first, count, iq complex64 [nof_rx][count])], next_sample)"""
    x = np.ascontiguousarray(x, np.complex64)
    A, n = x.shape
    cap = n // 2 + 2
    outs = [np.zeros((A, cap), np.complex64) for _ in carriers]
    ptrs = (C.c_void_p * len(carriers))(*[o.ctypes.data for o in outs])
    off = np.array([c[0] for c in carriers], np.int32)
    Ns = np.array([c[1] for c in carriers], np.uint32)
    m0, cnt, nxt = np.zeros(len(carriers), np.uint64), np.zeros(len(carriers), np.uint64), C.c_uint64()
    r = lib().lteo_chan_run(fs_in, A, len(carriers), ltelib.ptr(off), ltelib.ptr(Ns), ltelib.ptr(x), first, n, ptrs, cap, ltelib.ptr(m0),
                            ltelib.ptr(cnt), C.byref(nxt))
    assert r == 0, r
    res = []
    for c in range(len(carriers)):
        k = int(cnt[c])
        res.append(dict(first=int(m0[c]), count=k, iq=outs[c].ravel()[:A * k].reshape(A, k).copy()))
    return res, nxt.value


# ---- float64 restatement of DESIGN.md §2 "channeliser" -----------------------------------------------------------------------------------
def geometry(fs_in, offset_hz, N):
    """(T, D, P, f_pass) from the rule, or None when it refuses the carrier"""
    if N not in MAX_PRB or not 0 < fs_in <= 245760000 or offset_hz % 1000:
        return None
    fs_out = 15000 * N
    if fs_in % fs_out or not 2 <= fs_in // fs_out <= 128:
        return None
    D, f_pass = fs_in // fs_out, 90000 * MAX_PRB[N]
    if abs(offset_hz) + f_pass > fs_in / 2:
        return None
    import scipy.signal as ss
    T_, _ = ss.kaiserord(ATTEN, (fs_out - 2 * f_pass) / (fs_in / 2))
    P = fs_in // math.gcd((D * offset_hz) % fs_in, fs_in)
    return T_ | 1, D, P, f_pass


def reference(fs_in, offset_hz, N, x, ms):
    """float64 outputs ms of carrier (offset_hz, N) from x complex [n] (capture samples 0 .., zero before 0), with the float taps h of the rule"""
    t = design(fs_in, offset_hz, N)
    h = t["h"].astype(np.float64)
    T_, D = t["T"], t["D"]
    H = (T_ - 1) // 2
    k = np.arange(-H, H + 1)
    ms = np.asarray(ms, np.int64)
    idx = ms[:, None] * D - k[None, :]
    xp = np.where(idx >= 0, np.asarray(x, np.complex128)[np.clip(idx, 0, len(x) - 1)], 0)
    ph_g = 2 * np.pi * ((offset_hz * k) % fs_in) / fs_in
    ph_r = -2 * np.pi * ((offset_hz * D * ms) % fs_in) / fs_in
    return np.exp(1j * ph_r) * (xp * (h * np.exp(1j * ph_g))[None, :]).sum(axis=1)


# ---- wideband captures ---------------------------------------------------------------------------------------------------------------
def cell_capture(c, nsf, nrx, ppm, seed):
    """a decodable carrier: the simulator's subframes with PBCH and PDSCH for several UEs (2 ports, transmission modes 1 to 3), after c["lead"]
    zero samples, at a receiver clock ppm off, with the carrier offset c["cfo"] applied in float64.  -> (x complex64 [nrx][L], truth starts in
    receiver samples, [(iq, truth, payload)] of the subframes as the simulator made them)"""
    N, lead = c["N"], c.get("lead", 0)
    cell = ltelib.Cell(T.PRB_OF[N], 2, c["pci"], nrx, N)
    s = S.sim(sync=1, cell=cell, seed=seed, pbch=1, snr_db=c.get("snr", 30.0), nof_ues=6, dl_min=2, dl_max=4, tm=13, mcs_min=2, mcs_max=16)
    sub = [s.subframe(t) for t in range(nsf)]
    tx = np.concatenate([np.zeros((nrx, lead))] + [q[0] for q in sub], axis=1)
    L = int(np.floor((tx.shape[1] - T.TAPS) / (1.0 + ppm * 1e-6)))
    x = T.resample(tx, ppm, L) if ppm else tx[:, :L]
    n = np.arange(L)
    x = x * np.exp(2j * np.pi * c.get("cfo", 0.0) * n / (15000.0 * N))
    truth = (lead + np.arange(nsf) * 15 * N) / (1.0 + ppm * 1e-6)
    return x.astype(np.complex64), truth, sub


def compose(fs_in, carriers, nsf, nrx=1, ppm=0.0, noise_db=-40.0, seed=1):
    """carriers: [dict(offset_hz, N, pci, cfo, lead, gain_db, decode)]; decode=True makes the carrier with cell_capture (truth transport blocks in
    "sub" of its truth entry).  Each is a track_lib.capture of nsf subframes (its own PCI, carrier offset and lead
    in carrier samples; all share the clock offset ppm), upsampled by D with scipy.signal.resample_poly, shifted by offset_hz and scaled by gain_db;
    the sum gets complex noise of power noise_db (dB relative to a 0 dB carrier's mean power) over the whole capture band.
    -> (x complex64 [nrx][L], [dict(truth starts in carrier samples, D, narrow: the carrier's own capture at its rate)])"""
    import scipy.signal as ss
    rng = np.random.default_rng(seed)
    parts, truths = [], []
    for i, c in enumerate(carriers):
        N = c["N"]
        D = fs_in // (15000 * N)
        sub = None
        if c.get("decode"):
            xn, truth, sub = cell_capture(c, nsf, nrx, ppm, seed * 17 + i)
        else:
            xn, truth, _ = T.capture(N, c["pci"], nsf, nrx=nrx, ppm=ppm, cfo=c.get("cfo", 0.0), snr=c.get("snr", 60.0), lead=c.get("lead", 0),
                                     seed=seed * 17 + i)
        pw = np.mean(np.abs(xn[:, c.get("lead", 0):]) ** 2)
        up = ss.resample_poly(xn.astype(np.complex128) / np.sqrt(pw), D, 1, axis=1, window=("kaiser", 10.0))
        parts.append(up * 10 ** (c.get("gain_db", 0.0) / 20))
        truths.append(dict(truth=truth, D=D, narrow=xn, sub=sub))
    L = min(p.shape[1] for p in parts)
    n = np.arange(L)
    x = np.zeros((nrx, L), np.complex128)
    for c, p in zip(carriers, parts):
        x += p[:, :L] * np.exp(2j * np.pi * ((c["offset_hz"] * n) % fs_in) / fs_in)
    sig = 10 ** (noise_db / 20) * np.sqrt(0.5)
    x += sig * (rng.standard_normal(x.shape) + 1j * rng.standard_normal(x.shape))
    return x.astype(np.complex64), truths


def stream(run_fn, x, sizes, first=0):
    """feed x (capture samples first ...) to run_fn(span, span_first) -> (outs, next) in pieces of the given sizes (cycled), each call re-fed from
    the last next_sample; returns per carrier the concatenated outputs with repeats dropped, and the list of next_sample values"""
    recv, nxt, i, end = first, first, 0, first + x.shape[1]
    got, nexts = None, []
    while recv < end:
        recv = min(recv + sizes[i % len(sizes)], end)
        i += 1
        outs, n2 = run_fn(x[:, nxt - first:recv - first], nxt)
        nexts.append(n2)
        if got is None:
            got = [dict(first=o["first"], iq=[]) for o in outs]
        for g, o in zip(got, outs):
            have = g["first"] + sum(q.shape[1] for q in g["iq"])
            iq = o["iq"] if isinstance(o["iq"], np.ndarray) else o["iq"].cpu().numpy()
            assert o["first"] <= have or not o["count"], (o["first"], have)
            if o["count"] and o["first"] + o["count"] > have:
                g["iq"].append(iq[:, have - o["first"]:])
        nxt = n2
    return [dict(first=g["first"], iq=np.concatenate(g["iq"], axis=1) if g["iq"] else np.zeros((x.shape[0], 0), np.complex64)) for g in got], nexts
