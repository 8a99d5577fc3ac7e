"""Integer references of the two decoders that consume the receive path's LLRs, written from 36.212 and the DESIGN.md §2 rows "Viterbi",
"PBCH combining", "rate dematch" and "turbo" (numpy only; nothing here calls the oracle, the simulator or the product library).

Where the oracle has a formulation, this file uses another one, so that a mistake the two share cannot cancel:
  * rate matching from the matrix form of the sub-block interleavers (36.212 5.1.4.1.1 / 5.1.4.2.1), not from lookup tables;
  * trellises evaluated from the shift registers of 36.212 5.1.3.1 (generators 133 / 171 / 165) and 5.1.3.2.1 (feedback 1 + D^2 + D^3,
    parity 1 + D + D^3), with this file's own state numbering for the turbo code;
  * path and state metrics in int64, never renormalised (§2 claims every decision is offset-invariant; these references test that claim);
  * CRC16 as a bitwise LFSR, CRC24A / CRC24B as GF(2)-linear maps (x^(24 + j) mod g per bit position);
  * QPP parameters and code-block segmentation from tools/check_tables.py.
Everything is vectorised: DCI candidates along the first axis, turbo code blocks along the first axis and the 32-step windows along the second.
Imported only by tests/."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import check_tables  # noqa: E402

P_TURBO = [0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30, 1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31]   # 36.212 Table 5.1.4-1
P_CONV = [1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31, 0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30]    # Table 5.1.4-2
CRC16, CRC24A, CRC24B = 0x11021, 0x1864CFB, 0x1800063                                                 # 36.212 5.1.1
PBCH_PORT_MASK = {1: 0x0000, 2: 0xFFFF, 4: 0x5555}                                                   # 36.212 Table 5.3.1.1-1
NEG_INF = -8192                                                                                       # §2 turbo row
WL = 32                                                                                               # turbo window length


def subblock(y, P):
    """sub-block interleaver as the matrix of 36.212 5.1.4.1.1: NULLs (-1) in front, rows of 32, columns permuted, read column by column"""
    D = len(y)
    R = -(-D // 32)
    m = np.concatenate([np.full(32 * R - D, -1, np.int64), np.asarray(y, np.int64)]).reshape(R, 32)
    return m[:, P].T.reshape(-1), R


# ------------------------------------------------------------------------------------------------ CRC
def crc16_lfsr(bits):
    """bits [N][n] -> CRC16 (gCRC16 = D^16 + D^12 + D^5 + 1) of each row, a bitwise shift register with zero initial state"""
    bits = np.asarray(bits, np.int64)
    reg = np.zeros(bits.shape[0], np.int64)
    for i in range(bits.shape[1]):
        fb = ((reg >> 15) & 1) ^ bits[:, i]
        reg = ((reg << 1) & 0xFFFF) ^ (fb * (CRC16 & 0xFFFF))
    return reg


_XPOW = {}


def _xpow24(poly, n):
    """x^(24 + j) mod g(x) for j < n, as 24-bit integers"""
    if poly not in _XPOW or len(_XPOW[poly]) < n:
        out = np.zeros(max(n, 6144), np.int64)
        v = poly & 0xFFFFFF                                            # x^24 = g(x) - x^24 mod g
        for j in range(len(out)):
            out[j] = v
            v <<= 1
            if v >> 24:
                v = (v ^ poly) & 0xFFFFFF
        _XPOW[poly] = out
    return _XPOW[poly][:n]


def crc24_syndrome(bits, poly):
    """bits [N][n] -> remainder of (sum_i b_i x^(n-1-i)) x^24 mod g: zero exactly when the last 24 bits of a row are the CRC of the rest"""
    bits = np.asarray(bits).astype(bool)
    h = _xpow24(poly, bits.shape[1])[::-1]
    return np.bitwise_xor.reduce(np.where(bits, h[None, :], 0), axis=1)


# ------------------------------------------------------------------------------------------------ DCI: rate dematch, quantiser, Viterbi
G_CONV = np.array([[1, 0, 1, 1, 0, 1, 1], [1, 1, 1, 1, 0, 0, 1], [1, 1, 1, 0, 1, 0, 1]])   # 133, 171, 165 (octal); tap j multiplies c_{k-j}


def _conv_branches():
    """for every state S' = sum_{j=1..6} c_{k+1-j} 2^(j-1) after a step: its two predecessors (dropped register bit 0, then 1) and the
    +-1 signs of the three coded bits on each of those branches"""
    pred = np.zeros((64, 2), np.int64)
    sgn = np.zeros((64, 2, 3), np.int64)
    for n in range(64):
        c = n & 1                                                    # c_k, the bit that entered the register
        for b in (0, 1):
            S = (n >> 1) | (b << 5)                                  # b = c_{k-6}, the bit that left it
            reg = np.array([c] + [(S >> (j - 1)) & 1 for j in range(1, 7)])
            pred[n, b] = S
            sgn[n, b] = 2 * ((G_CONV @ reg) % 2) - 1
    return pred, sgn


CONV_PRED, CONV_SGN = _conv_branches()


def conv_dematch_order(K):
    """positions (in d0 | d1 | d2 order, 3 K values) of the circular buffer of 36.212 5.1.4.2: three interleaved streams, NULLs removed"""
    w = np.concatenate([subblock(np.arange(s * K, (s + 1) * K), P_CONV)[0] for s in range(3)])
    return w[w >= 0]


def dci_quantise(rm):
    """rm float32 [N][3K] -> (valid, r int64 [N][3K]): gain = 32 / max|rm| (NaN ignored), v = rm * gain + 127.5 rounded twice in float32, NaN -> 0,
    clamp to [0, 255], truncate, r = 2 q - 255; a candidate with max|rm| = 0 is invalid"""
    with np.errstate(all="ignore"):
        mx = np.where(np.isnan(rm), np.float32(0), np.abs(rm)).max(axis=1)
        gain = np.float32(32) / mx
        v = (rm * gain[:, None]).astype(np.float32) + np.float32(127.5)
    v = np.where(np.isnan(v), np.float32(0), v)
    q = np.clip(v, 0, 255).astype(np.int64)
    return mx > 0, 2 * q - 255


def viterbi_tb(r, K):
    """tail-biting Viterbi over three concatenated copies of r int64 [N][3 K] (d0 | d1 | d2 order): 3 K steps from all-zero metrics, ties keep
    the predecessor whose dropped bit is 0, the best end state is the lowest index among the maxima, the middle copy is the output -> bits [N][K]"""
    N = r.shape[0]
    rr = r.reshape(N, 3, K)
    pm = np.zeros((N, 64), np.int64)
    dec = np.zeros((2 * K, N, 64), bool)
    flat = CONV_SGN.reshape(128, 3)
    for t in range(3 * K):
        bm = (rr[:, :, t % K] @ flat.T).reshape(N, 64, 2)
        m = pm[:, CONV_PRED] + bm
        take1 = m[:, :, 1] > m[:, :, 0]
        pm = np.where(take1, m[:, :, 1], m[:, :, 0])
        if t >= K:
            dec[t - K] = take1
    st = np.argmax(pm, axis=1)
    out = np.zeros((N, K), np.uint8)
    ar = np.arange(N)
    for t in range(3 * K - 1, K - 1, -1):
        if t < 2 * K:
            out[:, t - K] = st & 1
        st = (st >> 1) | (dec[t - K][ar, st].astype(np.int64) << 5)
    return out


def dci_decode_ref(e, nbits):
    """e float32 [N][E] (or [E]) -> (valid [N], bits uint8 [N][nbits], crc_rem [N]): 36.212 5.1.4.2 dematch with float32 accumulation in ascending k,
    the §2 quantiser, tail-biting Viterbi, CRC16 remainder = received CRC XOR computed CRC.  Invalid candidates get zero bits and remainder."""
    e = np.atleast_2d(np.asarray(e, np.float32))
    N, E = e.shape
    K = nbits + 16
    w = conv_dematch_order(K)
    rm = np.zeros((N, 3 * K), np.float32)
    with np.errstate(all="ignore"):
        for j0 in range(0, E, 3 * K):                                # one lap at a time: positions are distinct within a lap
            idx = w[:min(3 * K, E - j0)]
            rm[:, idx] = rm[:, idx] + e[:, j0:j0 + len(idx)]
    valid, r = dci_quantise(rm)
    bits = np.zeros((N, K), np.uint8)
    rem = np.zeros(N, np.int64)
    for c0 in range(0, N, 4096):
        sl = slice(c0, min(N, c0 + 4096))
        bits[sl] = viterbi_tb(r[sl], K)
    rx = np.zeros(N, np.int64)
    for i in range(16):
        rx = (rx << 1) | bits[:, nbits + i]
    rem = rx ^ crc16_lfsr(bits[:, :nbits])
    bits[~valid] = 0
    rem[~valid] = 0
    return valid, bits[:, :nbits], rem


def pbch_hyp_ref(frames, src, dst, n, scr):
    """one PBCH combining hypothesis (§2 "PBCH combining"): held frames src .. src+n-1 (480 soft bits each) descrambled with the cell's bits
    [480 (dst + j), 480 (dst + j) + 480) of scr and placed at 40 ms positions dst .. dst+n-1 of a 1920-value buffer, 0 elsewhere, then
    decoded as a 24-bit payload -> (valid, bits [24], crc_rem); the hypothesis passes with k ports when crc_rem == PBCH_PORT_MASK[k]"""
    e = np.zeros(1920, np.float32)
    for j in range(n):
        sl = slice(480 * (dst + j), 480 * (dst + j + 1))
        e[sl] = np.where(scr[sl], -np.asarray(frames[src + j], np.float32), np.asarray(frames[src + j], np.float32))
    v, b, rem = dci_decode_ref(e, 24)
    return bool(v[0]), b[0], int(rem[0])


# ------------------------------------------------------------------------------------------------ turbo decoder
def _rsc_trellis():
    """36.212 5.1.3.2.1 with this file's state numbering s = a_{k-1} + 2 a_{k-2} + 4 a_{k-3} (a = the register input):
    branches b = 2 s + u -> (from, to, u, z)"""
    frm, to, uu, zz = [], [], [], []
    for s in range(8):
        a1, a2, a3 = s & 1, (s >> 1) & 1, (s >> 2) & 1
        for u in (0, 1):
            a = u ^ a2 ^ a3                                          # feedback 1 + D^2 + D^3
            frm.append(s)
            to.append(a | (a1 << 1) | (a2 << 2))
            uu.append(u)
            zz.append(a ^ a1 ^ a3)                                   # parity 1 + D + D^3
    frm, to, uu, zz = (np.array(x, np.int64) for x in (frm, to, uu, zz))
    into = np.array([np.nonzero(to == s)[0] for s in range(8)])      # [8][2] branches entering each state
    return frm, to, 2 * uu - 1, 2 * zz - 1, into


T_FROM, T_TO, T_SU, T_SZ, T_INTO = _rsc_trellis()

# 36.212 5.1.3.2.2: the 12 tail values by stream and position K .. K+3 -> (systematic / parity, constituent encoder, step)
TAIL_MAP = {0: [("x", 0, 0), ("z", 0, 1), ("x", 1, 0), ("z", 1, 1)],
            1: [("z", 0, 0), ("x", 0, 2), ("z", 1, 0), ("x", 1, 2)],
            2: [("x", 0, 1), ("z", 0, 2), ("x", 1, 1), ("z", 1, 2)]}


def qpp(K):
    i = [j for j in range(188) if check_tables.qpp_K(j) == K]
    assert len(i) == 1, K
    f1, f2, _, _ = check_tables.load()
    n = np.arange(K, dtype=np.int64)
    return (f1[i[0]] * n + f2[i[0]] * n * n) % K


def _siso(xs, par, apr, tx, tz, A, B):
    """one windowed max-log-MAP pass over code blocks [N][K]: windows of 32 steps, alpha of window w > 0 starting from A[:, w] and beta of
    window w < NW - 1 from B[:, w] (the previous iteration's boundaries), the first window from state 0 and the last from the tail.
    Doubled metrics: a branch adds u' xa + z' p with u', z' = +-1 and xa = systematic + a-priori.  -> (ext, L, new A, new B)"""
    N, K = xs.shape
    NW = -(-K // WL)
    pad = NW * WL - K
    xa = np.pad(xs + apr, ((0, 0), (0, pad))).reshape(N, NW, WL)
    pp = np.pad(par, ((0, 0), (0, pad))).reshape(N, NW, WL)
    live = (np.arange(NW * WL) < K).reshape(NW, WL)
    g = xa[..., None] * T_SU + pp[..., None] * T_SZ                  # [N][NW][32][16]
    bt = np.full((N, 8), NEG_INF, np.int64)                          # beta at K + 3: the register is empty
    bt[:, 0] = 0
    for k in (2, 1, 0):
        gt = tx[:, k, None] * T_SU + tz[:, k, None] * T_SZ
        bt = (bt[:, T_TO] + gt).reshape(N, 8, 2).max(-1)
    al = np.zeros((N, NW, WL + 1, 8), np.int64)
    al[:, :, 0] = A
    al[:, 0, 0] = NEG_INF
    al[:, 0, 0, 0] = 0
    for j in range(WL):
        m = al[:, :, j][..., T_FROM] + g[:, :, j]
        al[:, :, j + 1] = m[..., T_INTO].max(-1)
    be = B.copy()
    be[:, NW - 1] = bt
    L = np.zeros((N, NW, WL), np.int64)
    for j in range(WL - 1, -1, -1):
        v = be[..., T_TO] + g[:, :, j]
        tot = al[:, :, j][..., T_FROM] + v
        L[:, :, j] = tot[..., 1::2].max(-1) - tot[..., 0::2].max(-1)
        be = np.where(live[None, :, j, None], v.reshape(N, NW, 8, 2).max(-1), be)   # steps past K (short last window) leave beta alone
    ext = np.clip(np.floor_divide(3 * (L - 2 * xa), 8), -511, 511)
    An = np.zeros_like(A)
    An[:, 1:] = al[:, :-1, WL]
    Bn = np.zeros_like(B)
    Bn[:, :-1] = be[:, 1:]
    return ext.reshape(N, -1)[:, :K], L.reshape(N, -1)[:, :K], An, Bn


def turbo_decode_ref(d, K, max_iter, crc_type):
    """d int [N][3 (K + 4)] (streams d0 | d1 | d2 of 36.212 5.1.3.2), max_iter and crc_type (0 none, 1 CRC24A, 2 CRC24B) scalars or per block
    -> (bits uint8 [N][K], iterations [N], crc_ok [N]).  An iteration is decoder 1 on the natural order, then decoder 2 on the QPP order;
    hard decisions are decoder 2's L > 0, de-interleaved; after each iteration the CRC (if any) may stop a block; at least one iteration."""
    d = np.atleast_2d(np.asarray(d, np.int64))
    N, D = d.shape[0], K + 4
    assert d.shape[1] == 3 * D
    max_iter = np.maximum(np.broadcast_to(np.asarray(max_iter, np.int64), (N,)), 1)
    crc_type = np.broadcast_to(np.asarray(crc_type, np.int64), (N,))
    pi = qpp(K)
    xs, p1, p2 = d[:, :K], d[:, D:D + K], d[:, 2 * D:2 * D + K]
    tail = {(kind, enc): np.zeros((N, 3), np.int64) for kind in "xz" for enc in (0, 1)}
    for s, row in TAIL_MAP.items():
        for i, (kind, enc, step) in enumerate(row):
            tail[(kind, enc)][:, step] = d[:, s * D + K + i]
    NW = -(-K // WL)
    A1, B1, A2, B2 = (np.zeros((N, NW, 8), np.int64) for _ in range(4))
    apr1 = np.zeros((N, K), np.int64)
    bits = np.zeros((N, K), np.uint8)
    iters = np.zeros(N, np.int64)
    ok = np.zeros(N, bool)
    done = np.zeros(N, bool)
    for it in range(1, int(max_iter.max()) + 1):
        ext1, _, A1, B1 = _siso(xs, p1, apr1, tail[("x", 0)], tail[("z", 0)], A1, B1)
        ext2, L2, A2, B2 = _siso(xs[:, pi], p2, ext1[:, pi], tail[("x", 1)], tail[("z", 1)], A2, B2)
        apr1 = np.zeros_like(apr1)
        apr1[:, pi] = ext2
        b = np.zeros((N, K), np.uint8)
        b[:, pi] = L2 > 0
        act = ~done
        bits[act], iters[act] = b[act], it
        passed = np.zeros(N, bool)
        for ct, poly in ((1, CRC24A), (2, CRC24B)):
            sel = act & (crc_type == ct)
            if sel.any():
                passed[sel] = crc24_syndrome(b[sel], poly) == 0
        ok |= passed
        done |= passed | (it >= max_iter)
        if done.all():
            break
    return bits, iters, ok


# ------------------------------------------------------------------------------------------------ DL-SCH: segmentation, rate dematch, turbo, CRCs
def segmentation(tbs):
    """36.212 5.1.2 -> (C, [K_r], F)"""
    Cn, Kp, Km, Cp, Cm, F = check_tables.segm(tbs)
    return Cn, [Km if r < Cm else Kp for r in range(Cn)], F


def cb_E(G, Cn, r, Qm, NL):
    """36.212 5.1.4.1.2: E_r"""
    Gp = G // (NL * Qm)
    gam = Gp % Cn
    return NL * Qm * (Gp // Cn) if r <= Cn - gam - 1 else NL * Qm * (-(-Gp // Cn))


def turbo_ring(K, F, rv):
    """one lap of the circular buffer of 36.212 5.1.4.1.2 from k0 as positions in d (stream-major, 3 (K + 4)); NULLs and fillers removed"""
    D = K + 4
    lab = [np.arange(s * D, (s + 1) * D, dtype=np.int64) for s in range(3)]
    lab[0][:F] = -1
    lab[1][:F] = -1
    v0, R = subblock(lab[0], P_TURBO)
    v1, _ = subblock(lab[1], P_TURBO)
    Kpi = 32 * R
    y2 = np.concatenate([np.full(Kpi - D, -1, np.int64), lab[2]])
    k = np.arange(Kpi)
    v2 = y2[(np.array(P_TURBO)[k // R] + 32 * (k % R) + 1) % Kpi]
    w = np.empty(3 * Kpi, np.int64)
    w[:Kpi] = v0
    w[Kpi::2] = v1
    w[Kpi + 1::2] = v2
    k0 = R * (2 * -(-3 * Kpi // (8 * R)) * rv + 2)
    ring = np.roll(w, -k0)
    return ring[ring >= 0]


def rm_turbo_rx_ref(e, K, F, rv, Qm, acc=None):
    """§2 "rate dematch": received values added into the circular buffer in received order with int16 saturation at every addition, onto acc
    (the HARQ accumulators of a retransmission) or onto zeros; turbo input = clamp(floor(w / 2^sh), +-255), sh = 0 / 1 / 2 / 2 for
    Qm = 2 / 4 / 6 / 8, filler positions of d0 and d1 = -255 -> (d [3 (K + 4)], accumulators)"""
    D = K + 4
    ring = turbo_ring(K, F, rv)
    w = np.zeros(3 * D, np.int64) if acc is None else np.asarray(acc, np.int64).copy()
    e = np.asarray(e, np.int64)
    for j0 in range(0, len(e), len(ring)):
        idx = ring[:min(len(ring), len(e) - j0)]
        w[idx] = np.clip(w[idx] + e[j0:j0 + len(idx)], -32768, 32767)
    sh = {2: 0, 4: 1, 6: 2, 8: 2}[Qm]
    dd = np.clip(np.floor_divide(w, 1 << sh), -255, 255)
    dd[:F] = -255
    dd[D:D + F] = -255
    return dd, w


def dlsch_decode_ref(e, G, tbs, rv, Qm, NL, max_iter, early_stop, soft=None, combine=False):
    """one transport block from its G int16 soft bits -> (crc, payload bytes, iterations per code block, accumulators per code block).
    Code blocks stop early on CRC24B (CRC24A when C = 1) if early_stop; crc = TB CRC24A passes and, when C > 1, every CB CRC24B passes.
    soft / combine: the accumulators of an earlier transmission, which a retransmission (combine) adds to."""
    Cn, Ks, F = segmentation(tbs)
    e = np.asarray(e, np.int64)
    ds, accs, rp = [], [], 0
    for r, K in enumerate(Ks):
        E = cb_E(G, Cn, r, Qm, NL)
        dd, w = rm_turbo_rx_ref(e[rp:rp + E], K, F if r == 0 else 0, rv, Qm, soft[r] if (soft is not None and combine) else None)
        rp += E
        ds.append(dd)
        accs.append(w)
    ct = (2 if Cn > 1 else 1) if early_stop else 0
    cb_bits, iters, cb_ok = [None] * Cn, np.zeros(Cn, np.int64), np.zeros(Cn, bool)
    for K in sorted(set(Ks)):
        rs = [r for r in range(Cn) if Ks[r] == K]
        b, it, ok = turbo_decode_ref(np.stack([ds[r] for r in rs]), K, max_iter, ct)
        for j, r in enumerate(rs):
            cb_bits[r], iters[r], cb_ok[r] = b[j], it[j], ok[j]
    if Cn > 1 and not early_stop:
        cb_ok = np.array([crc24_syndrome(b[None], CRC24B)[0] == 0 for b in cb_bits])
    tb = np.concatenate([cb_bits[r][(F if r == 0 else 0):Ks[r] - (24 if Cn > 1 else 0)] for r in range(Cn)])
    crc = bool(crc24_syndrome(tb[None, :tbs + 24], CRC24A)[0] == 0) and (Cn == 1 or bool(cb_ok.all()))
    return crc, np.packbits(tb[:tbs]), iters, accs
