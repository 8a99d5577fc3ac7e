"""Float64 references for the uplink (PUSCH) receive path, written from 36.211 / 36.212 / 36.213 and the PUSCH rows of DESIGN.md section 2, not from
oracle/lte_oracle.c.  numpy / scipy only: nothing here calls the simulator, the oracle or the product (the DMRS, the control-information layout and
map and the Gold sequences of sim/lte_common.c are what is under test).

Two halves:
  * a transmitter: the PUSCH DMRS (5.5.1 / 5.5.2 with group and sequence hopping), Q' of HARQ-ACK / RI / CQI and G (36.212 5.2.2.6, beta offsets of
    36.213 Tables 8.6.3-1..3), the channel interleaver with the RI / CQI / ACK placement (5.2.2.8), scrambling (5.3.1), Gray-PAM QAM, transform
    precoding with a DFT scaled by 1 / sqrt M (5.3.3), resource mapping and the SC-FDMA modulator with its half-subcarrier shift (5.6);
  * the receiver in float64: UL grid, least-squares estimate at the two reference symbols, (w, 1 - 2w, w) smoothing, noise / RSRP / SNR / timing
    offset, linear interpolation in time (or one estimate per slot under type-1 hopping), zero forcing, the 1 / sqrt M inverse DFT, srsRAN's int16
    demodulator, descrambling, control-information de-multiplexing and the channel de-interleaver.

Grids are complex128 arrays [14][12 N] (l, k); k counts the subcarriers from the lowest one, as in 36.211."""
import math
import os
import sys
from fractions import Fraction

import numpy as np

import ref64
from ref64 import gold, qam, cp_len, fft_size, demod_int16, descramble

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import check_tables  # noqa: E402

DATA_SYMBOLS = (0, 1, 2, 4, 5, 6, 7, 8, 9, 11, 12, 13)      # normal CP: the DMRS sits on l = 3 of each slot
SMOOTH_W = 0.3333                                          # DESIGN.md section 2: taps (w, 1 - 2w, w), edges renormalised
N_DMRS1 = (0, 2, 3, 4, 6, 8, 9, 10)                        # cyclicShift -> n_DMRS^(1), 36.211 Table 5.5.2.1.1-2
BETA_ACK = ("2.000", "2.500", "3.125", "4.000", "5.000", "6.250", "8.000", "10.000", "12.625", "15.875", "20.000", "31.000", "50.000", "80.000", "126.000")
BETA_RI = ("1.250", "1.625", "2.000", "2.500", "3.125", "4.000", "5.000", "6.250", "8.000", "10.000", "12.625", "15.875", "20.000")
BETA_CQI = (None, None, "1.125", "1.250", "1.375", "1.625", "1.750", "2.000", "2.250", "2.500", "2.875", "3.125", "3.500", "4.000", "5.000", "6.250")
RI_COLUMNS, ACK_COLUMNS = (1, 4, 7, 10), (2, 3, 8, 9)      # 36.212 Tables 5.2.2.8-1 / -2, normal CP
DATA, CQI, RI, ACK_DATA, ACK_CQI = 0, 1, 2, 3, 4


# ------------------------------------------------------------------------------------------------ DMRS (36.211 5.5)
def largest_prime_below(m):
    return max(p for p in range(2, m) if all(p % d for d in range(2, int(p ** 0.5) + 1)))


def dmrs(cell_id, ucfg, ns, n_dmrs2, M):
    """r^PUSCH(n), n < M, of slot ns: r_{u,v}^(alpha)(n) = e^{j alpha n} x_q(n mod N_zc) for M >= 36 (5.5.1.1); u = (f_gh(ns) + f_ss) mod 30 (5.5.1.3);
    v = c(ns) without group hopping from 6 PRB on (5.5.1.4); alpha = 2 pi ((n_DMRS^(1) + n_DMRS^(2) + n_PRS(ns)) mod 12) / 12 (5.5.2.1.1).
    ucfg: (cyclicShift, delta_ss, group_hopping, seq_hopping)"""
    cs, delta_ss, gh, sh = ucfg
    fss = (cell_id + delta_ss) % 30
    fgh = sum(int(b) << i for i, b in enumerate(gold(cell_id // 30, 8 * ns + 8)[8 * ns:])) % 30 if gh else 0
    u = (fgh + fss) % 30
    c_ss = gold((cell_id // 30) * 32 + fss, 8 * 7 * ns + 8)
    v = int(c_ss[ns]) if (not gh and sh and M >= 72) else 0
    nzc = largest_prime_below(M)
    qbar = nzc * (u + 1) / 31.0
    q = int(math.floor(qbar + 0.5)) + v * (-1) ** int(math.floor(2 * qbar))
    m = np.arange(M) % nzc
    nprs = sum(int(b) << i for i, b in enumerate(c_ss[8 * 7 * ns:8 * 7 * ns + 8]))
    alpha = 2 * np.pi * ((N_DMRS1[cs] + n_dmrs2 + nprs) % 12) / 12
    return np.exp(1j * alpha * np.arange(M)) * np.exp(-1j * np.pi * q * m * (m + 1) / nzc)


# ------------------------------------------------------------------------------------------------ control information (36.212 5.2.2.6 / 5.2.2.8)
def sum_k(tbs):
    """sum of the code-block sizes K_r of a transport block (36.212 5.1.2, tools/check_tables.segm)"""
    C, Kp, Km, Cp, Cm, F = check_tables.segm(tbs)
    return Cp * Kp + Cm * Km


def layout(M, qm, tbs, nof_ack=0, ri_len=0, cqi_len=0, I_ack=0, I_ri=0, I_cqi=0):
    """-> (Q'_ACK, Q'_RI, Q'_CQI, G).  Q' = min(ceil(O M N_symb beta / sum K_r), 4 M) for ACK and RI, Q'_CQI = min(ceil((O + L) M N_symb beta / sum K_r),
    M N_symb - Q'_RI) with the CRC length L = 8 from 12 CQI bits on; in exact rational arithmetic.  G = (M N_symb - Q'_CQI - Q'_RI) Qm"""
    K = sum_k(tbs)
    nsymb = 12

    def q(o, beta):
        return math.ceil(Fraction(o * M * nsymb) * Fraction(beta) / K)
    qa = min(q(nof_ack, BETA_ACK[I_ack]), 4 * M) if nof_ack else 0
    qr = min(q(ri_len, BETA_RI[I_ri]), 4 * M) if ri_len else 0
    qc = min(q(cqi_len + (8 if cqi_len > 11 else 0), BETA_CQI[I_cqi]), M * nsymb - qr) if cqi_len else 0
    return qa, qr, qc, (M * nsymb - qc - qr) * qm


def interleaver_map(M, qa, qr, qc):
    """the R' = M rows x 12 columns of the channel interleaver (5.2.2.8) step by step: RI symbols from the bottom row up in the columns {1, 4, 7, 10}
    taken in the order 0, 3, 2, 1; the CQI symbols and then the UL-SCH symbols row by row around them; HARQ-ACK symbols from the bottom row up in the
    columns {2, 3, 8, 9} in the same order, overwriting.  -> kind [M][12] (DATA, CQI, RI, ACK_DATA, ACK_CQI) and pos [M][12], the index of the symbol in
    the UL-SCH stream (DATA, ACK_DATA) or the CQI stream (CQI, ACK_CQI)"""
    kind = np.full((M, 12), -1, np.int64)
    pos = np.full((M, 12), -1, np.int64)
    for i in range(qr):
        kind[M - 1 - i // 4, RI_COLUMNS[(3 * i) % 4]] = RI
    n = 0
    for r in range(M):
        for c in range(12):
            if kind[r, c] == RI:
                continue
            kind[r, c], pos[r, c] = (CQI, n) if n < qc else (DATA, n - qc)
            n += 1
    for i in range(qa):
        r, c = M - 1 - i // 4, ACK_COLUMNS[(3 * i) % 4]
        kind[r, c] = ACK_DATA if kind[r, c] == DATA else ACK_CQI
    return kind, pos


def scrambling(cell_id, sf, rnti, n):
    """36.211 5.3.1: c_init = n_RNTI 2^14 + floor(ns / 2) 2^9 + N_cell"""
    return gold((rnti << 14) + (sf << 9) + cell_id, n)


# ------------------------------------------------------------------------------------------------ grants
class Grant:
    """one PUSCH allocation: L PRB from n_prb (slot 0) and n_prb1 (slot 1; = n_prb without hopping), Qm, the transport block size the control
    information is sized with, n_DMRS^(2) and the UCI of 36.212 5.2.2.6"""

    def __init__(self, L, n_prb, qm, tbs, rnti=0x1234, n_dmrs2=0, n_prb1=None, nof_ack=0, ri_len=0, cqi_len=0, I_ack=0, I_ri=0, I_cqi=0):
        self.L, self.n_prb, self.qm, self.tbs, self.rnti, self.n_dmrs2 = L, n_prb, qm, tbs, rnti, n_dmrs2
        self.n_prb1 = n_prb if n_prb1 is None else n_prb1
        self.uci = dict(nof_ack=nof_ack, ri_len=ri_len, cqi_len=cqi_len, I_ack=I_ack, I_ri=I_ri, I_cqi=I_cqi)
        self.M = 12 * L
        self.qa, self.qr, self.qc, self.G = layout(self.M, qm, tbs, **self.uci)
        self.kind, self.pos = interleaver_map(self.M, self.qa, self.qr, self.qc)

    @property
    def hop(self):
        return self.n_prb1 != self.n_prb

    def k0(self, sl):
        return 12 * (self.n_prb1 if sl else self.n_prb)


def transmit(cell, grant, sf, ucfg, bits, rng):
    """the grid contribution [14][12 N] of one grant.  bits: the G UL-SCH bits (None: random); CQI, RI and ACK carry random bits.
    -> (grid, d) with d [12][M] the modulation symbols before transform precoding (column c of the interleaver = data symbol c)"""
    M, qm = grant.M, grant.qm
    if bits is None:
        bits = rng.integers(0, 2, grant.G).astype(np.uint8)
    h = rng.integers(0, 2, (M, 12, qm)).astype(np.uint8)                   # RI, CQI and ACK symbols: random content
    data = grant.kind == DATA
    h[data] = np.asarray(bits, np.uint8).reshape(-1, qm)[grant.pos[data]]
    tx = h.transpose(1, 0, 2).reshape(-1)                                  # read out column by column: bit (c M + k) Qm + b
    tx = tx ^ scrambling(cell.cell_id, sf, grant.rnti, len(tx))
    d = qam(tx, qm).reshape(12, M)
    grid = np.zeros((14, 12 * cell.nof_prb), complex)
    for c, l in enumerate(DATA_SYMBOLS):
        k0 = grant.k0(l // 7)
        grid[l, k0:k0 + M] = np.fft.fft(d[c]) / np.sqrt(M)                 # transform precoding, 5.3.3
    for sl in range(2):
        k0 = grant.k0(sl)
        grid[7 * sl + 3, k0:k0 + M] = dmrs(cell.cell_id, ucfg, 2 * sf + sl, grant.n_dmrs2, M)
    return grid, d


def scfdma_modulate(cell, grid, delay=0):
    """36.211 5.6: s_l(t) = sum_k a_{k,l} e^{j 2 pi (k + 1/2) df (t - N_CP Ts)} with k = -N_sc / 2 .. N_sc / 2 - 1, evaluated at t = (n + N_CP) Ts over
    the cyclic prefix and the symbol (n = -N_CP .. N - 1), scaled by 1 / N so that an unscaled FFT gives the grid back.  delay: a delay of whole samples
    applied to every symbol as s_l(n - delay) (|delay| < CP: the receive window sees no neighbouring symbol)"""
    N, nsc = fft_size(cell), 12 * cell.nof_prb
    k = np.arange(nsc) - nsc // 2
    out = []
    for l in range(14):
        n = np.arange(-cp_len(N, l), N) - delay
        X = np.zeros(N, complex)
        X[k % N] = grid[l]
        out.append(np.fft.ifft(X)[n % N] * np.exp(1j * np.pi * n / N))
    return np.concatenate(out)


def ul_grid(cell, iq):
    """the UL grid [14][nsc] of one subframe: remove the half-subcarrier shift e^{-j pi n / N}, FFT of the N samples after each cyclic prefix"""
    N, nsc = fft_size(cell), 12 * cell.nof_prb
    out, p = np.zeros((14, nsc), complex), 0
    n = np.arange(N)
    for l in range(14):
        p += cp_len(N, l)
        X = np.fft.fft(np.asarray(iq[p:p + N], np.complex128) * np.exp(-1j * np.pi * n / N))
        out[l] = X[(np.arange(nsc) - nsc // 2) % N]
        p += N
    return out


# ------------------------------------------------------------------------------------------------ designed channels H[14][nsc] (one rx antenna)
def channel(kind, nsc, **kw):
    l = np.arange(14)[:, None].astype(float)
    k = np.arange(nsc)[None, :].astype(float)
    g = np.exp(0.6j) * 0.9
    if kind == "flat":
        return g * np.ones((14, nsc), complex)
    if kind == "selective":                                               # frequency-selective, with its fastest changes at the band edges
        return g * (1.0 + 0.45 * np.cos(2 * np.pi * k / 29.0) + 0.3 * np.exp(-k / 9.0) + 0.3 * np.exp(-(nsc - 1 - k) / 9.0)) * np.exp(-2j * np.pi * k * 2.5 / 2048) + 0 * l
    if kind == "linear_l":                                                # linear in time: the interpolation is exact on every data symbol, 0-2 and 11-13 too
        return g * (1.0 + (0.3 - 0.25j) * (l - 6.5) / 7.0) + 0 * k
    if kind == "late_change":                                             # constant up to symbol 10, then turning: symbols 11-13 are mis-extrapolated
        return g * np.where(l <= 10, 1.0, np.exp(0.35j * (l - 10)) * (1 + 0.2 * (l - 10))) + 0 * k
    if kind == "per_slot":                                                # type-1 hopping: an unrelated channel in each slot
        a = g * (1.0 + 0.3 * np.cos(2 * np.pi * k / 41.0))
        b = np.exp(-2.1j) * 0.6 * (1.0 + 0.4 * np.sin(2 * np.pi * k / 23.0))
        return np.where(l < 7, a, b)
    if kind == "fade":                                                    # |h| ~ 1e-3 on some PRBs up to symbol 10: the estimate extrapolated to 11-13
        H = channel("selective", nsc)                                     # stays deep where the data symbols are not, and the IDFT spreads the
        for prb in kw.get("prbs", ()):                                    # quotients over the whole symbol, past the int16 clamp
            H[:11, 12 * prb:12 * prb + 12] *= 1e-3
        return H
    raise ValueError(kind)


def receive(grid, H, noise_var, rng):
    Y = H * grid
    if noise_var:
        Y = Y + np.sqrt(noise_var / 2) * (rng.standard_normal(Y.shape) + 1j * rng.standard_normal(Y.shape))
    return Y


# ------------------------------------------------------------------------------------------------ receiver
def smooth_taps():
    return np.array([SMOOTH_W, 1.0 - 2.0 * SMOOTH_W, SMOOTH_W])


def chest(cell, Y, grant, sf, ucfg):
    """DESIGN.md section 2, PUSCH: LS at l = 3 of each slot, (w, 1 - 2w, w) smoothing with renormalised edges, noise = mean |LS - smoothed|^2 /
    (1 - 2 f_1 + sum f^2), RSRP = mean |smoothed|^2 over both slots, ta_us = -arg(sum ls[n+1] conj(ls[n])) / 2 pi averaged over the slots, / 15e-3.
    -> (smoothed [2][M], dict(noise, rsrp, snr_db, ta_us))"""
    M = grant.M
    f = smooth_taps()
    ls, sm = np.zeros((2, M), complex), np.zeros((2, M), complex)
    ta = 0.0
    for sl in range(2):
        k0 = grant.k0(sl)
        ls[sl] = Y[7 * sl + 3, k0:k0 + M] * np.conj(dmrs(cell.cell_id, ucfg, 2 * sf + sl, grant.n_dmrs2, M))
        sm[sl] = np.convolve(ls[sl], f, mode="same") / np.convolve(np.ones(M), f, mode="same")
        ta += -np.angle(np.sum(ls[sl, 1:] * np.conj(ls[sl, :-1]))) / (2 * np.pi) / 2
    noise = np.mean(np.abs(ls - sm) ** 2) / (1 - 2 * f[1] + np.sum(f ** 2))
    rsrp = np.mean(np.abs(sm) ** 2)
    with np.errstate(divide="ignore", invalid="ignore"):
        snr = 10 * np.log10(rsrp / noise)
    return sm, dict(noise=noise, rsrp=rsrp, snr_db=snr, ta_us=ta / 15e-3)


def estimate_at(grant, sm, l):
    """the estimate used on data symbol l: per slot under hopping, else A + (B - A) t with t = (l - 3) / 7 (extrapolated on 0-2 and 11-13)"""
    if grant.hop:
        return sm[l // 7]
    return sm[0] + (sm[1] - sm[0]) * ((l - 3) / 7.0)


def deprecode(cell, Y, grant, sm):
    """zero forcing (an exactly zero |h|^2 gives 0) and the inverse DFT scaled by 1 / sqrt M -> x [12][M] and cond [12] = max |h|^2 / min |h|^2 of each
    data symbol (the IDFT spreads the noise enhancement of its worst RE over the whole symbol)"""
    M = grant.M
    x, cond = np.zeros((12, M), complex), np.zeros(12)
    for c, l in enumerate(DATA_SYMBOLS):
        k0 = grant.k0(l // 7)
        h = estimate_at(grant, sm, l)
        p = np.abs(h) ** 2
        z = ref64._div(Y[l, k0:k0 + M] * np.conj(h), p)
        x[c] = np.fft.ifft(z) * np.sqrt(M)
        with np.errstate(divide="ignore", invalid="ignore"):
            cond[c] = p.max() / p.min() if p.max() > 0 else 1.0
    return x, cond


def soft_bits(cell, x, grant, sf):
    """int16 demodulation of every de-precoded sample, descrambling at bit (c M + k) Qm + b (the transmitted order), then the UL-SCH codeword in
    de-interleaved order: ACK over data -> 0, CQI / RI / ACK over CQI dropped.  -> (llr int64 [G], index of the data symbol of each soft bit [G])"""
    M, qm = grant.M, grant.qm
    z = demod_int16(x.reshape(-1), qm).reshape(12, M, qm)                  # [c][k][b]
    z = descramble(z.reshape(-1), scrambling(cell.cell_id, sf, grant.rnti, 12 * M * qm)).reshape(12, M, qm)
    llr = np.zeros((grant.G // qm, qm), np.int64)
    col = np.zeros(grant.G // qm, np.int64)
    for kd in (DATA, ACK_DATA):
        k, c = np.nonzero(grant.kind == kd)
        p = grant.pos[k, c]
        llr[p] = 0 if kd == ACK_DATA else z[c, k]
        col[p] = c
    return llr.reshape(-1), np.repeat(col, qm)


def decode(cell, Y, grant, sf, ucfg):
    """the whole receive chain of one grant -> (chest dict, llr [G], cond per soft bit [G])"""
    sm, info = chest(cell, Y, grant, sf, ucfg)
    x, cond = deprecode(cell, Y, grant, sm)
    llr, col = soft_bits(cell, x, grant, sf)
    return info, llr, cond[col]
