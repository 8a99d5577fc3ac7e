"""Float64 reference of WHERE the control channels and the PBCH sit in the downlink grid, and a numpy eNB that puts them there, written from
36.211 (6.2.4 REGs, 6.6 PBCH, 6.7 PCFICH, 6.8 PDCCH, 6.9 PHICH, 6.10.1.2 CRS positions), 36.212 (5.1.3.1, 5.1.4.2, 5.3.1, 5.3.3, 5.3.4) and
36.331 (MasterInformationBlock).  numpy only, on top of tests/ref64.py and tests/ref_dec.py: nothing here calls the simulator, the oracle or the
product, so a mistake the three share in their C statements of the map cannot hide behind agreement between them.

Where the C code walks the grid with counters and lookup tables, this file uses other formulations:
  * REGs as arrays of (l, k) built per symbol, the PDCCH order as a lexicographic sort of the REG representatives on (k, l);
  * the quadruplet interleaver as the 36.212 5.1.4.2.1 matrix (ref_dec.subblock with Table 5.1.4-2), the cyclic shift as an index rotation;
  * pilot positions from the per-port rule of 6.10.1.2, so the PBCH exclusion of ports 0..3 is stated once for every port.

Grid indices are l * 12 N + k (k counts the occupied subcarriers from the lowest one, as in ref64).  Cells are duck-typed: nof_prb, nof_ports,
cell_id, nof_rx, symbol_sz, phich_ng (phich-Resource 0..3 = 1/6, 1/2, 1, 2), phich_ext (phich-Duration extended).  One and two CRS ports are
implemented; four raise NotImplementedError where the geometry differs (the symbol-1 REGs and SFBC-FSTD)."""
import functools
from types import SimpleNamespace

import numpy as np

import ref64
import ref64_sync
from ref64 import CFI_CODEWORDS, gold, precode, qam
from ref_dec import G_CONV, P_CONV, PBCH_PORT_MASK, conv_dematch_order, crc16_lfsr, subblock

NG = {0: (1, 6), 1: (1, 2), 2: (1, 1), 3: (2, 1)}          # 36.331 phich-Resource -> Ng as a fraction
BW_CODE = {6: 0, 15: 1, 25: 2, 50: 3, 75: 4, 100: 5}       # 36.331 dl-Bandwidth n6 .. n100; codes 6 and 7 are not in the enumeration


def _check_ports(nof_ports):
    if nof_ports == 4:
        raise NotImplementedError("4 CRS ports: symbol-1 REGs of six REs around the port 2/3 pilots, SFBC-FSTD")
    if nof_ports not in (1, 2):
        raise ValueError(nof_ports)


# ------------------------------------------------------------------------------------------------ pilot positions (6.10.1.2)
def crs_k(port, pci, ns, l, nsc):
    """the subcarriers of port `port`'s pilots in symbol l (0..6) of slot ns, or an empty array when the port has none there"""
    if port in (0, 1):
        if l not in (0, 4):
            return np.zeros(0, np.int64)
        v = (0 if l == 0 else 3) if port == 0 else (3 if l == 0 else 0)
    elif port in (2, 3):
        if l != 1:
            return np.zeros(0, np.int64)
        v = 3 * (ns % 2) + (0 if port == 2 else 3)
    else:
        raise ValueError(port)
    return np.arange((v + pci % 6) % 6, nsc, 6, dtype=np.int64)


def reg_pilot_ports(l, nof_ports):
    """the ports whose pilot REs 6.2.4 keeps out of the REGs of control symbol l: ports 0 and 1 in symbol 0 whatever the port count (a one-port
    cell assumes the port 1 pilots), ports 2 and 3 in symbol 1 of a four-port cell"""
    _check_ports(nof_ports)
    return (0, 1) if l == 0 else ()


# ------------------------------------------------------------------------------------------------ REGs (6.2.4)
@functools.lru_cache(maxsize=None)
def reg_table(N, nof_ports, pci):
    """every REG of symbols 0..2: SimpleNamespace(l [n], k0 [n] (the representative: lowest k of the REG), re [n][4] (the k of its four data REs,
    increasing)), ordered by symbol, then frequency"""
    nsc = 12 * N
    ls, k0s, res = [], [], []
    for l in range(3):
        res_l = np.zeros(nsc, bool)
        for p in reg_pilot_ports(l, nof_ports):
            res_l[crs_k(p, pci, 0, l, nsc)] = True
        size = 4 + 2 * bool(res_l.any())                   # six REs around two pilots, four without
        k0 = np.arange(0, nsc, size, dtype=np.int64)
        kk = k0[:, None] + np.arange(size)[None, :]
        kk = kk[~res_l[kk]].reshape(len(k0), 4)
        ls.append(np.full(len(k0), l, np.int64))
        k0s.append(k0)
        res.append(kk)
    return SimpleNamespace(l=np.concatenate(ls), k0=np.concatenate(k0s), re=np.concatenate(res))


def _reg_of(T, l, k0):
    """index in reg_table of the REG of symbol l represented by subcarrier k0"""
    i = np.nonzero((T.l == l) & (T.k0 == k0))[0]
    assert len(i) == 1, (l, k0)
    return int(i[0])


# ------------------------------------------------------------------------------------------------ PCFICH (6.7.4), PHICH (6.9)
def pcfich_k0(N, pci):
    """the representatives of the four PCFICH REGs of symbol 0: k = kbar + floor(i N / 2) * 6 mod 12 N, kbar = 6 (PCI mod 2 N)"""
    kbar = 6 * (pci % (2 * N))
    return [(kbar + (i * N // 2) * 6) % (12 * N) for i in range(4)]


def n_group(N, ng):
    """N_group = ceil(Ng N / 8), normal cyclic prefix"""
    num, den = NG[ng]
    return -(-num * N // (8 * den))


@functools.lru_cache(maxsize=None)
def phich_regs(N, nof_ports, pci, ng, ext):
    """[N_group][3] reg_table indices of PHICH group m, quadruplet i.  The REGs of symbol l' not taken by the PCFICH are numbered 0 .. n_l' - 1 in
    increasing frequency; normal duration: nbar_i = (PCI + m + floor(i n_0 / 3)) mod n_0 in symbol 0; extended (FDD, not MBSFN): symbol l' = i and
    nbar_i = (floor(PCI n_l' / n_0) + m + floor(i n_l' / 3)) mod n_l'"""
    T = reg_table(N, nof_ports, pci)
    pc = {_reg_of(T, 0, k) for k in pcfich_k0(N, pci)}
    avail = [np.array([r for r in np.nonzero(T.l == l)[0] if r not in pc], np.int64) for l in range(3)]
    n = [len(a) for a in avail]
    G = n_group(N, ng)
    out = np.zeros((G, 3), np.int64)
    for m in range(G):
        for i in range(3):
            if ext:
                lp = i
                nb = (pci * n[lp] // n[0] + m + i * n[lp] // 3) % n[lp]
            else:
                lp = 0
                nb = (pci + m + i * n[0] // 3) % n[0]
            out[m, i] = avail[lp][nb]
    return out


# ------------------------------------------------------------------------------------------------ PDCCH (6.8.5)
@functools.lru_cache(maxsize=None)
def control_map(N, nof_ports, pci, ng, ext, cfi):
    """the control region of a cell at one CFI (N > 10: the region is `cfi` symbols).  -> SimpleNamespace:
    pdcch [ncce][36]: grid indices of every CCE's REs, quadruplet by quadruplet (the layout of the product's and the oracle's CCE tables);
    pcfich [16]: quadruplet i on its REG;  phich [N_group][3][4]: group m, quadruplet i (REs of a REG outside the region included);
    nil [M_quad mod 9][4]: the REGs the interleaved, shifted quadruplets 9 ncce .. M_quad - 1 land on (no CCE owns them);
    mquad, ncce, and reg_order (reg_table indices of the PDCCH REGs in the k-outer / l-inner mapping order)"""
    T = reg_table(N, nof_ports, pci)
    nsc = 12 * N
    grid = T.l[:, None] * nsc + T.re                       # [nreg][4]
    pc = [_reg_of(T, 0, k) for k in pcfich_k0(N, pci)]
    ph = phich_regs(N, nof_ports, pci, ng, ext)
    taken = np.zeros(len(T.l), bool)
    taken[pc] = True
    taken[ph.ravel()] = True
    cand = np.nonzero((T.l < cfi) & ~taken)[0]
    order = cand[np.lexsort((T.l[cand], T.k0[cand]))]     # k' outer, l' inner: 6.8.5 steps 1-10
    M = len(order)
    v, _ = subblock(np.arange(M), P_CONV)                  # 36.212 5.1.4.2.1 on quadruplets, NULLs in front
    w = v[v >= 0]                                          # w(j): the quadruplet at position j of the permuted sequence
    wbar = w[(np.arange(M) + pci) % M]                     # wbar(i) = w((i + N_ID) mod M_quad), mapped to REG i of the order
    reg_of_quad = np.empty(M, np.int64)
    reg_of_quad[wbar] = order
    ncce = M // 9
    return SimpleNamespace(pdcch=grid[reg_of_quad[:9 * ncce]].reshape(ncce, 36), pcfich=grid[pc].reshape(16), phich=grid[ph],
                           nil=grid[reg_of_quad[9 * ncce:]], mquad=M, ncce=ncce, reg_order=order, grid=grid)


def cell_map(cell, cfi):
    return control_map(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.phich_ng, cell.phich_ext, cfi)


# ------------------------------------------------------------------------------------------------ PBCH (6.6.4) and MIB (36.331)
@functools.lru_cache(maxsize=None)
def pbch_re(N, pci):
    """the 240 grid indices of the PBCH in mapping order: symbols 0..3 of slot 1 (7..10), the 72 subcarriers around DC, k first, then l; the pilot
    REs of ports 0..3 are left out whatever the cell's port count"""
    nsc = 12 * N
    out = []
    for l in range(4):
        k = np.arange(6 * N - 36, 6 * N + 36, dtype=np.int64)
        res = np.zeros(nsc, bool)
        for p in range(4):
            res[crs_k(p, pci, 1, l, nsc)] = True
        out.append((7 + l) * nsc + k[~res[k]])
    out = np.concatenate(out)
    assert len(out) == 240
    return out


def mib_bits(bw_code, ext, ng, sfn, spare=0):
    """MasterInformationBlock, unaligned PER: dl-Bandwidth (3 bits), phich-Duration (1), phich-Resource (2), systemFrameNumber = the 8 MSBs of the
    SFN (8), spare (10), each field MSB first -> uint8 [24]"""
    fields = [(bw_code, 3), (ext, 1), (ng, 2), (sfn >> 2, 8), (spare, 10)]
    return np.array([(v >> (n - 1 - i)) & 1 for v, n in fields for i in range(n)], np.uint8)


def mib_fields(bits):
    """-> (bw_code, ext, ng, sfn MSBs << 2, spare)"""
    b = [int(x) for x in bits]

    def take(a, n):
        return int("".join(map(str, b[a:a + n])), 2)
    return take(0, 3), take(3, 1), take(4, 2), take(6, 8) << 2, take(14, 10)


# ------------------------------------------------------------------------------------------------ coding (36.212)
def conv_encode(c):
    """5.1.3.1 tail-biting: the register starts with the last six bits, d_s(k) = sum_j G_s(j) c((k - j) mod K) -> [3][K]"""
    c = np.asarray(c, np.int64)
    K = len(c)
    taps = c[(np.arange(K)[:, None] - np.arange(7)[None, :]) % K]
    return ((taps @ G_CONV.T) % 2).T.astype(np.uint8)


def conv_rate_match(d, E):
    """5.1.4.2: the circular buffer of the three interleaved streams, NULLs skipped, read E times from the start"""
    ring = conv_dematch_order(d.shape[1])
    return d.reshape(-1)[ring[np.arange(E) % len(ring)]]


def crc_bits(bits, mask):
    """the 16 parity bits of 5.1.1 (CRC16) XOR mask, MSB of the mask on the first parity bit (5.3.3.2 / 5.3.1.1)"""
    r = int(crc16_lfsr(np.asarray(bits, np.uint8)[None])[0]) ^ mask
    return np.array([(r >> (15 - i)) & 1 for i in range(16)], np.uint8)


def dci_encode(bits, rnti, E):
    bits = np.asarray(bits, np.uint8)
    return conv_rate_match(conv_encode(np.concatenate([bits, crc_bits(bits, rnti)])), E)


def pbch_encode(mib, nof_ports):
    return conv_rate_match(conv_encode(np.concatenate([np.asarray(mib, np.uint8), crc_bits(mib, PBCH_PORT_MASK[nof_ports])])), 1920)


# ------------------------------------------------------------------------------------------------ the numpy eNB
def _scheme(cell):
    _check_ports(cell.nof_ports)
    return "port0" if cell.nof_ports == 1 else "sfbc"


def _put(grids, idx, y, nsc):
    idx = np.asarray(idx).ravel()
    grids[:, idx // nsc, idx % nsc] = y


def enb_subframe(cell, sf, cfi, dcis, rng, sfn=0, spare=0, trap_amp=4.0, bw_code=None):
    """one downlink subframe of a cell -> (port grids [P][14][12 N], truth).
    dcis: [(bits, rnti, L, ncce)], each on CCEs ncce .. ncce + L - 1.  The grid holds: CRS of the cell's ports, PSS / SSS (subframes 0 / 5, port 0),
    the PCFICH, random QPSK on every REG of every PHICH group, the PDCCH (NIL on unused CCEs), and in subframe 0 the PBCH quarter of frame sfn with
    `trap_amp` QPSK on every other RE of symbols 7..10 in the central 72 subcarriers that is not a transmitted pilot (the port 1 / 2 / 3 pilot REs
    of cells without those ports), so a receiver that reads a wrong RE there reads energy.  truth: cfi, dcis, mib, sfn"""
    N, P, pci = cell.nof_prb, cell.nof_ports, cell.cell_id
    assert N > 10 and 1 <= cfi <= 3
    scheme = _scheme(cell)
    nsc = 12 * N
    grids = np.zeros((P, 14, nsc), complex)
    for p in range(P):
        grids[p] += ref64.crs_grid(cell, sf, p)
    if sf in (0, 5):                                       # 6.11: SSS in symbol 5, PSS in symbol 6 (FDD), d(n) on -31..-1, 1..31
        f = ref64_sync.subcarriers()
        k = np.where(f < 0, 6 * N + f, 6 * N + f - 1)
        grids[0, 6, k] = ref64_sync.pss(pci % 3)
        grids[0, 5, k] = ref64_sync.sss(pci // 3, pci % 3, sf == 5)
    m = cell_map(cell, cfi)
    # PCFICH (6.7)
    b = np.array(CFI_CODEWORDS[cfi - 1][:32], np.uint8) ^ gold((sf + 1) * (2 * pci + 1) * 512 + pci, 32)
    _put(grids, m.pcfich, precode(scheme, qam(b, 2)[None], P), nsc)
    # PHICH: energy on every REG of every group, at the PDCCH's power
    ph = m.phich.reshape(-1, 4)
    ph = ph[ph[:, 0] // nsc < cfi].ravel()
    _put(grids, ph, precode(scheme, qam(rng.integers(0, 2, 2 * len(ph)), 2)[None], P), nsc)
    # PDCCH (6.8.2 - 6.8.5): multiplex with NIL, scramble over M_tot = 8 M_quad, QPSK, precode, quadruplets onto their REGs
    M = m.mquad
    bb = np.zeros(8 * M, np.uint8)
    used = np.zeros(m.ncce, bool)
    for bits, rnti, L, ncce in dcis:
        assert ncce % L == 0 and ncce + L <= m.ncce and not used[ncce:ncce + L].any(), (L, ncce, m.ncce)
        bb[72 * ncce:72 * (ncce + L)] = dci_encode(bits, rnti, 72 * L)
        used[ncce:ncce + L] = True
    y = precode(scheme, qam(bb ^ gold((sf << 9) + pci, 8 * M), 2)[None], P)[:, :36 * m.ncce].reshape(P, m.ncce, 36)
    _put(grids, m.pdcch[used], y[:, used].reshape(P, -1), nsc)
    truth = SimpleNamespace(cfi=cfi, dcis=list(dcis), mib=None, sfn=sfn)
    if sf == 0:                                            # PBCH (6.6): quarter sfn mod 4 of the scrambled 1920 bits
        mib = mib_bits(BW_CODE[N] if bw_code is None else bw_code, cell.phich_ext, cell.phich_ng, sfn, spare)
        q = sfn % 4
        e = pbch_encode(mib, P) ^ gold(pci, 1920)
        pb = pbch_re(N, pci)
        centre = np.zeros((14, nsc), bool)
        centre[7:11, 6 * N - 36:6 * N + 36] = True
        for p in range(P):
            for l in range(7, 11):
                centre[l, crs_k(p, pci, 1, l - 7, nsc)] = False
        centre.ravel()[pb] = False
        tl, tk = np.nonzero(centre)
        grids[0, tl, tk] = trap_amp * qam(rng.integers(0, 2, 2 * len(tl)), 2)
        _put(grids, pb, precode(scheme, qam(e[480 * q:480 * (q + 1)], 2)[None], P), nsc)
        truth.mib = mib
    return grids, truth


def capture(cell, grids, H, noise_var, rng):
    """port grids -> (received grids Y [rx][14][nsc], complex64 samples [rx][sf_len]) through H [rx][ports][14][nsc] with AWGN"""
    Y = ref64.receive(cell, grids, H, noise_var, rng)
    return Y, np.stack([ref64.ofdm_modulate(cell, Y[a]) for a in range(cell.nof_rx)]).astype(np.complex64)


# ------------------------------------------------------------------------------------------------ PBCH receive reference
def pbch_llr(cell, ce, Y, nof_ports):
    """the 480 soft bits of the PBCH assuming nof_ports: MRC (1) or pairwise SFBC (2) on pbch_re, -sqrt2 (re, im); not descrambled"""
    N = cell.nof_prb
    idx = pbch_re(N, cell.cell_id)
    nsc = 12 * N
    l, k = idx // nsc, idx % nsc
    H = ref64.h_at(ce, cell, l, k)[:, :, :nof_ports]
    r = np.stack([Y[a][l, k] for a in range(cell.nof_rx)], 1)
    d = ref64.equalise_mrc(H[:, :, 0], r) if nof_ports == 1 else ref64.equalise_sfbc(H, r)
    out = np.empty(480)
    out[0::2], out[1::2] = -np.sqrt(2) * d.real, -np.sqrt(2) * d.imag
    return out
