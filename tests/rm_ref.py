"""numpy restatements of the turbo rate de-matcher (36.212 5.1.4.1) in the pair-buffer layout of the library: the per-soft-bit loop over
the forward table (received order) and the per-word rule over the inverse table that rm_turbo_rx_kernel runs, plus the code-block
and pair bookkeeping of phase B, so that LTEPHY_TAP_TURBO_IN can be predicted word for word."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import check_tables  # noqa: E402

RM_FILLER, RM_NONE = 0xFFFE, 0xFFFF
HARQ_NONE, HARQ_NEW, HARQ_RETX = 0, 1, 2
HARQ_CB_STRIDE = 18448                 # int16 accumulators per code block in a HARQ slot
HARQ_SLOT_ELEMS = 16 * HARQ_CB_STRIDE
TURBO_K = [check_tables.qpp_K(i) for i in range(188)]


def pair_words(K):
    return 96 * ((K + 31) // 32) + 16


def tables(lib, K, F, rv):
    """(order [nn] of rv, nn, inv [96 NW + 16], rot [4]) as the library builds them"""
    lib.ltephy_rm_turbo_tables.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32), C.c_void_p, C.c_void_p]
    order = np.zeros(3 * (K + 4), np.uint32)
    inv = np.zeros(pair_words(K), np.uint16)
    rot = np.zeros(4, np.uint32)
    nn = C.c_uint32(0)
    r = lib.ltephy_rm_turbo_tables(K, F, rv, order.ctypes.data, C.byref(nn), inv.ctypes.data, rot.ctypes.data)
    assert r == 0, (K, F, rv)
    return order[:nn.value].astype(np.int64), nn.value, inv, rot


def filler_words(K, F):
    NW = (K + 31) // 32
    i = np.arange(F)
    return np.concatenate([st * 32 * NW + (i & 31) * NW + (i >> 5) for st in range(2)]).astype(np.int64)


def none_words(K):
    """ragged window slots i in [K, 32 NW) of the three streams and the 4 pad words"""
    NW = (K + 31) // 32
    i = np.arange(K, 32 * NW)
    return np.concatenate([st * 32 * NW + (i & 31) * NW + (i >> 5) for st in range(3)] + [np.arange(96 * NW + 12, 96 * NW + 16)]).astype(np.int64)


def _sat16(v):
    return np.clip(v, -32768, 32767)


def _condition(acc, shift):
    return np.clip(acc >> shift, -255, 255)


def dematch_per_bit(e, E, order, nn, shift, K, F, op=HARQ_NONE, hq=None):
    """the received-order loop: soft bit k and its repeats k + nn, ... < E are summed (saturating, ascending) onto word order[k].
    -> (values of the words it writes, dict word -> value; updated accumulators or None)"""
    acc = hq[order].astype(np.int64) if op == HARQ_RETX else np.zeros(nn, np.int64)
    for m in range(-(-E // nn) if E else 0):
        kk = np.arange(nn) + m * nn
        sel = kk < E
        acc[sel] = _sat16(acc[sel] + e[kk[sel]].astype(np.int64))
    out = {}
    v = _condition(acc, shift)
    for w, x in zip(order.tolist(), v.tolist()):
        out[w] = x
    for w in filler_words(K, F).tolist():
        out[w] = -255
    hq2 = None
    if op != HARQ_NONE:
        hq2 = hq.copy()
        hq2[order] = acc
    return out, hq2


def dematch_words(e, E, inv, nn, rot, shift, op=HARQ_NONE, hq=None):
    """the per-word rule of rm_turbo_rx_kernel: every word of the pair buffer -> int16 value; updated accumulators or None"""
    inv = inv.astype(np.int64)
    valid = inv < nn
    k = np.where(valid, (inv - rot) % max(nn, 1), 0)
    acc = np.where(valid, hq[:len(inv)].astype(np.int64), 0) if op == HARQ_RETX else np.zeros(len(inv), np.int64)
    m = 0
    while True:
        kk = k + m * nn
        sel = valid & (kk < E)
        if not sel.any():
            break
        acc[sel] = _sat16(acc[sel] + e[kk[sel]].astype(np.int64))
        m += 1
    v = np.where(valid, _condition(acc, shift), 0)
    v[inv == RM_FILLER] = -255
    hq2 = None
    if op != HARQ_NONE:
        hq2 = hq.copy()
        hq2[:len(inv)][valid] = acc[valid]
    return v.astype(np.int16), hq2


def rm_E(G, C_, r, qm, NL):
    Gp = G // (NL * qm)
    gamma = Gp % C_
    return NL * qm * (Gp // C_) if r + gamma + 1 <= C_ else NL * qm * (-(-Gp // C_))


class PhaseB:
    """phase-B bookkeeping restated: transport blocks -> code blocks -> pairs of equal K in the turbo pool, in submission order, and the
    expected contents of the pool after the rate de-matcher.  HARQ accumulators persist across batches (one dict for the handle)."""

    def __init__(self, lib):
        self.lib, self.harq, self.cache = lib, {}, {}

    def begin(self):
        self.cbs, self.pairs, self.open, self.words, self.uses = [], [], {}, 0, {}

    def add_tb(self, tbs, G, qm, rv, NL, llr_off, op=HARQ_NONE, slot=0):
        C_, Kp, Km, Cp, Cm, F = check_tables.segm(tbs)
        gen = 0
        if op != HARQ_NONE:
            gen = self.uses.get(slot, 0)
            self.uses[slot] = gen + 1
        rp = llr_off
        for r in range(C_):
            K = Km if r < Cm else Kp
            E = rm_E(G, C_, r, qm, NL)
            cb = dict(K=K, F=F if r == 0 else 0, E=E, llr=rp, rv=rv, shift={2: 0, 4: 1}.get(qm, 2), op=op, slot=slot, r=r, gen=gen)
            rp += E
            if K in self.open:
                p = self.open.pop(K)
                p["cbs"].append(cb)
            else:
                p = dict(K=K, off=self.words, cbs=[cb])
                self.words += pair_words(K)
                self.pairs.append(p)
                self.open[K] = p
            self.cbs.append(cb)

    def expected(self, llr):
        """int16 view of the turbo pool words the batch writes ([2 w + half]); HARQ state advanced generation by generation"""
        out = np.zeros(2 * self.words, np.int16)
        for gen in range(max([cb["gen"] for cb in self.cbs] + [0]) + 1):
            for p in self.pairs:
                for h, cb in enumerate(p["cbs"]):
                    if cb["gen"] != gen:
                        continue
                    key = (cb["K"], cb["F"])
                    if key not in self.cache:
                        self.cache[key] = tables(self.lib, cb["K"], cb["F"], 0)
                    _, nn, inv, rot = self.cache[key]
                    hq = None
                    if cb["op"] != HARQ_NONE:
                        hq = self.harq.setdefault(cb["slot"], np.zeros(HARQ_SLOT_ELEMS, np.int16))[cb["r"] * HARQ_CB_STRIDE:(cb["r"] + 1) * HARQ_CB_STRIDE]
                    e = llr[cb["llr"]:cb["llr"] + cb["E"]]
                    v, hq2 = dematch_words(e, cb["E"], inv, nn, int(rot[cb["rv"] & 3]), cb["shift"], cb["op"], hq)
                    if hq2 is not None:
                        hq[:] = hq2
                    out[2 * p["off"] + h:2 * (p["off"] + pair_words(p["K"])):2] = v
        return out
