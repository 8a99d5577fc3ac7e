"""The control-region and PBCH geometry of the simulator, the oracle and the product against tests/ref64_ctrl.py, a statement of it written from
36.211 / 36.212 / 36.331 alone.  The simulator transmits with the map of sim/lte_common.c and the oracle receives with it; the product builds its own
copy (build_ctrl_map in lte_host.cpp, the PBCH table of ltephy_capi.cu).  Agreement between the three says nothing about the standard, so:
  * the exported CCE / PCFICH maps equal the spec's, RE by RE, for every PCI at 25 PRB and at PCIs that reach the formulas' edges on every bandwidth;
  * the PHICH REGs, which no one exports, are pinned through the complement of those maps;
  * the PBCH resource elements and the MIB bit layout equal the spec's;
  * the simulator's transmitter decodes with a float64 receiver that reads the spec's positions, and the oracle decodes a numpy eNB that writes them.
No GPU: the product's map comes from ltephy_ctrl_region_map; its PBCH table and MIB unpack need a device handle
(tests/test_gpu_control_region_36211.py)."""
import ctypes as C

import numpy as np
import pytest

import ltelib
import ref64
import ref64_ctrl
import ref_dec
from ltelib import Cell, Oracle, Sim

MAX_CCE = 8 * 110 // 9                      # room for the largest control region: 110 PRB, CFI 3, no PHICH


# ------------------------------------------------------------------------------------------------ the maps as the two C statements export them
def product_map(N, P, pci, ng, ext, cfi):
    """ltephy_ctrl_region_map -> (return code, pdcch [ncce][36], pcfich [16])"""
    from ltesniffer_b200 import capi
    L = capi.load_library()
    capi._bind_search(L)
    idx = np.zeros(MAX_CCE * 36, np.uint16)
    pc = np.zeros(16, np.uint16)
    n = C.c_uint32(0)
    r = L.ltephy_ctrl_region_map(N, P, pci, ng | (ext << 8), cfi, idx.ctypes.data_as(C.c_void_p), len(idx), C.byref(n), pc.ctypes.data_as(C.c_void_p))
    return r, idx[:36 * n.value].astype(np.int64).reshape(-1, 36), pc.astype(np.int64)


def oracle_map(o, cfi):
    O = ltelib.oracle()
    O.lteo_pdcch_re_index.restype = C.c_uint32
    O.lteo_pdcch_re_index.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    idx, pc = np.zeros(MAX_CCE * 36, np.uint16), np.zeros(16, np.uint16)
    n = O.lteo_pdcch_re_index(o.h, cfi, ltelib.ptr(idx), ltelib.ptr(pc))
    return idx[:36 * n].astype(np.int64).reshape(-1, 36), pc.astype(np.int64)


def region_cfis(ext):
    """36.211 Table 6.9.3-1: the extended duration needs three control symbols (N > 10, not MBSFN)"""
    return (3,) if ext else (1, 2, 3)


def check_complement(N, P, pci, ng, ext, cfi, pdcch, pcfich, who):
    """the control-region REs that belong to a REG but to neither exported map are exactly the spec's PHICH REGs plus the REGs of the
    interleaved quadruplets past the last full CCE; the spec's PHICH REGs meet neither map"""
    m = ref64_ctrl.control_map(N, P, pci, ng, ext, cfi)
    nsc = 12 * N
    reg_re = m.grid[ref64_ctrl.reg_table(N, P, pci).l < cfi].ravel()
    left = np.zeros(3 * nsc, bool)
    left[reg_re] = True
    left[pdcch.ravel()] = False
    left[pcfich] = False
    phich = m.phich.reshape(-1, 4)
    phich = phich[phich[:, 0] // nsc < cfi].ravel()
    want = np.zeros(3 * nsc, bool)
    want[phich] = True
    want[m.nil.ravel()] = True
    assert not np.isin(phich, pdcch).any() and not np.isin(phich, pcfich).any(), (who, N, P, pci, ng, ext, cfi)
    assert np.array_equal(left, want), (who, N, P, pci, ng, ext, cfi, np.nonzero(left != want)[0][:8])


def check_cell_maps(N, P, pci, ng, ext, o=None):
    for cfi in region_cfis(ext):
        m = ref64_ctrl.control_map(N, P, pci, ng, ext, cfi)
        r, pi, pp = product_map(N, P, pci, ng, ext, cfi)
        assert r == 0, (N, P, pci, ng, ext, cfi, r)
        assert pi.shape[0] == m.ncce, ("product nof_cce", N, P, pci, ng, ext, cfi, pi.shape[0], m.ncce)
        assert np.array_equal(pp, m.pcfich), ("product PCFICH", N, P, pci, ng, ext, cfi)
        assert np.array_equal(pi, m.pdcch), ("product PDCCH", N, P, pci, ng, ext, cfi, np.argwhere(pi != m.pdcch)[:4])
        check_complement(N, P, pci, ng, ext, cfi, pi, pp, "product")
        if o is not None:
            oi, op = oracle_map(o, cfi)
            assert oi.shape[0] == m.ncce, ("oracle nof_cce", N, P, pci, ng, ext, cfi, oi.shape[0], m.ncce)
            assert np.array_equal(op, m.pcfich), ("oracle PCFICH", N, P, pci, ng, ext, cfi)
            assert np.array_equal(oi, m.pdcch), ("oracle PDCCH", N, P, pci, ng, ext, cfi)
            check_complement(N, P, pci, ng, ext, cfi, oi, op, "oracle")


# ------------------------------------------------------------------------------------------------ maps
@pytest.mark.parametrize("ports", [1, 2])
def test_control_maps_equal_36211_for_every_pci_at_25_prb(infra, ports):
    """all 504 PCIs, every Ng, both durations, CFI 1..3 (3 with the extended duration): PCI mod 3 moves the symbol-0 pilots, PCI mod 50 the PCFICH,
    PCI the PHICH groups and the PDCCH shift (which wraps past M_quad for most of them)"""
    for pci in range(504):
        for ng in range(4):
            for ext in (0, 1):
                check_cell_maps(25, ports, pci, ng, ext, Oracle(Cell(25, ports, pci, 1, 0, ng, ext)))


def edge_pcis(N):
    """PCIs that reach the edges of the formulas at N PRB: every PCI mod 3, PCI >= 2 N (the PCFICH wraps), PCI >= M_quad (the PDCCH shift wraps),
    PCI = 503 and PCIs whose PHICH start lands near the end of symbol 0"""
    nreg0 = 2 * N - 4
    return sorted({0, 1, 2, 2 * N - 1, 2 * N, 2 * N + 1, 2 * N + 2, nreg0 - 1, nreg0 + 1, 503, 3 * N + 7} & set(range(504)))


def test_control_maps_equal_36211_at_every_bandwidth(infra):
    """every N_RB the product accepts (11..110): odd N (floor(i N / 2)), n_0 = 2 N - 4 not a multiple of 3, M_quad below the PCI (at 11 PRB, CFI 1 and
    Ng 1/6, M_quad is 15)"""
    assert ref64_ctrl.control_map(11, 1, 20, 0, 0, 1).mquad == 15
    assert any((2 * N - 4) % 3 for N in range(11, 111)) and any(N % 2 for N in range(11, 111))
    for N in range(11, 111):
        for i, pci in enumerate(edge_pcis(N)):
            P = 1 + (i + N) % 2
            for ng in range(4):
                for ext in (0, 1):
                    check_cell_maps(N, P, pci, ng, ext, Oracle(Cell(N, P, pci, 1, 0, ng, ext)) if (i + ng) % 3 == 0 else None)
                    if (i + ng + ext) % 4 == 0:
                        check_cell_maps(N, 3 - P, pci, ng, ext)


def test_product_map_refusals(infra):
    """cells the product does not serve stay refusals: 10 PRB or fewer, three or four ports, phich-Resource above 3"""
    for N, P, ng in ((10, 1, 0), (6, 2, 0), (25, 3, 0), (25, 4, 0), (25, 2, 4), (50, 1, 7)):
        assert product_map(N, P, 1, ng, 0, 1)[0] != 0, (N, P, ng)
    assert product_map(11, 1, 1, 0, 0, 1)[0] == 0 and product_map(110, 2, 503, 3, 1, 3)[0] == 0


def test_four_ports_are_not_implemented_here():
    with pytest.raises(NotImplementedError):
        ref64_ctrl.reg_table(25, 4, 1)


def test_reference_geometry_anchors():
    """the closed forms the reference must also satisfy: 2 / 3 / 3 REGs per PRB in symbols 0 / 1 / 2, PCFICH on four REGs spread by a quarter of the band,
    N_group = ceil(Ng N / 8), every REG used once"""
    for N, pci, ng in ((25, 7, 0), (50, 301, 3), (11, 20, 1), (110, 503, 2), (15, 1, 0)):
        T = ref64_ctrl.reg_table(N, 2, pci)
        assert [int(np.sum(T.l == l)) for l in range(3)] == [2 * N, 3 * N, 3 * N]
        assert all((k % 3) != pci % 3 for k in T.re[T.l == 0].ravel())
        G = ref64_ctrl.n_group(N, ng)
        assert G == int(np.ceil({0: 1 / 6, 1: 0.5, 2: 1.0, 3: 2.0}[ng] * N / 8 - 1e-9))
        for ext in (0, 1):
            m = ref64_ctrl.control_map(N, 2, pci, ng, ext, 3)
            assert m.mquad == 8 * N - 4 - 3 * G and m.ncce == m.mquad // 9
            used = np.concatenate([m.pdcch.ravel(), m.pcfich, m.phich.ravel(), m.nil.ravel()])
            assert len(np.unique(used)) == len(used) == 4 * (8 * N)
    assert ref64_ctrl.pcfich_k0(25, 7) == [42, 42 + 6 * 12, 42 + 6 * 25, 42 + 6 * 37]          # kbar = 6 * 7, floor(i * 25 / 2) = 0, 12, 25, 37
    assert ref64_ctrl.pcfich_k0(25, 99) == [294, 366 - 300, 444 - 300, 516 - 300]            # PCI mod 50 = 49: three REGs wrap to the band start


# ------------------------------------------------------------------------------------------------ PBCH and MIB
def sim_pbch_re(cell):
    S = ltelib.sim()
    S.lte_pbch_re.argtypes = [C.POINTER(Cell), C.c_void_p, C.c_void_p]
    S.lte_pbch_re.restype = C.c_uint32
    k, l = np.zeros(240, np.uint16), np.zeros(240, np.uint8)
    n = S.lte_pbch_re(C.byref(cell), ltelib.ptr(k), ltelib.ptr(l))
    return n, l.astype(np.int64) * 12 * cell.nof_prb + k


def test_pbch_resource_elements_equal_36211(infra):
    """slot 1 symbols 0..3 over the central 72 subcarriers, k first, without the pilot REs of ports 0..3 whatever the port count"""
    for N in (6, 11, 15, 25, 27, 50, 75, 99, 100, 110):
        for pci in list(range(6)) + [503, 250]:
            for P in (1, 2):
                n, got = sim_pbch_re(Cell(N, P, pci, 1))
                assert n == 240 and np.array_equal(got, ref64_ctrl.pbch_re(N, pci)), (N, pci, P)


def test_mib_layout_equals_36331(infra):
    """lte_mib_pack (the simulated eNB) and lte_mib_unpack (the oracle) against 36.331 MasterInformationBlock for every bandwidth code, both
    durations, every Ng and SFN 0..1023; the unpack ignores the spare bits and refuses the reserved codes 6 and 7"""
    S = ltelib.sim()
    S.lte_mib_pack.argtypes = [C.c_uint32] * 4 + [C.c_void_p]
    S.lte_mib_unpack.argtypes = [C.c_void_p] + [C.POINTER(C.c_uint32)] * 4
    S.lte_mib_unpack.restype = C.c_int
    rng = np.random.default_rng(3)
    bits = np.zeros(24, np.uint8)
    out = [C.c_uint32() for _ in range(4)]
    bw = {v: k for k, v in ref64_ctrl.BW_CODE.items()}
    for code in range(8):
        for ext in (0, 1):
            for ng in range(4):
                for sfn in range(1024):
                    want = ref64_ctrl.mib_bits(code, ext, ng, sfn)
                    if code in bw:
                        S.lte_mib_pack(bw[code], ext, ng, sfn, ltelib.ptr(bits))
                        assert np.array_equal(bits, want), (code, ext, ng, sfn, bits, want)
                    spare = int(rng.integers(0, 1024))
                    tx = ref64_ctrl.mib_bits(code, ext, ng, sfn, spare)
                    r = S.lte_mib_unpack(ltelib.ptr(tx), *[C.byref(x) for x in out])
                    if code in bw:
                        assert r == 0 and [x.value for x in out] == [bw[code], ext, ng, sfn & ~3], (code, ext, ng, sfn, [x.value for x in out])
                    else:
                        assert r != 0, (code, ext, ng, sfn)


# ------------------------------------------------------------------------------------------------ the simulator, read at the spec's positions
SIM_CELLS = [(25, 1, 150, 1, 0, 0, 0), (50, 2, 301, 2, 0, 3, 0), (15, 2, 503, 1, 0, 1, 1), (75, 1, 77, 2, 0, 2, 1), (100, 2, 2, 1, 0, 0, 0),
             (27, 2, 55, 1, 0, 2, 0)]


@pytest.mark.parametrize("cellp", SIM_CELLS, ids=lambda c: "x".join(map(str, c)))
def test_simulator_decodes_at_the_spec_positions(infra, cellp):
    """every DCI the simulated eNB sends is found by a float64 receiver (ref64 channel estimate and PDCCH LLRs on the ref64_ctrl indices,
    ref_dec's Viterbi) at its CCEs with its RNTI, and its PBCH decodes from the spec's 240 REs"""
    cell = Cell(*cellp)
    cfi = 3 if cell.phich_ext else 2
    s = Sim(cell=cell, seed=17 + cellp[2], cfi=cfi, nof_ues=6, dl_min=3, dl_max=5, tm=2 if cell.nof_ports == 2 else 1, mcs_min=4, mcs_max=12,
            snr_db=25.0, pbch=1)
    total = 0
    for tti in range(0, 12):
        iq, tr, _ = s.subframe(tti)
        sf = tti % 10
        Y = np.stack([ref64.ofdm_demodulate(cell, iq[a]) for a in range(cell.nof_rx)])
        ce, _ = ref64.chest(cell, sf, Y)
        m = ref64_ctrl.cell_map(cell, tr.cfi)
        assert tr.cfi == cfi
        assert np.argmax(ref64.pcfich_corr(cell, sf, ce, Y, m.pcfich)) == cfi - 1
        llr = ref64.pdcch_llr(cell, sf, ce, Y, m.pdcch.ravel(), (sf << 9) + cell.cell_id)
        for i in range(tr.nof_dci):
            d = tr.dci[i]
            L = 1 << d.L
            v, bits, rem = ref_dec.dci_decode_ref(llr[72 * d.ncce:72 * (d.ncce + L)], d.nbits)
            want = np.frombuffer(bytes(d.bits), np.uint8)[:d.nbits]
            assert v[0] and rem[0] == d.rnti and np.array_equal(bits[0], want), (tti, i, d.rnti, d.ncce, L)
            total += 1
        if sf == 0:
            q = (tti // 10) % 4
            frame = ref64_ctrl.pbch_llr(cell, ce, Y, cell.nof_ports)
            ok, mib, rem = ref_dec.pbch_hyp_ref([frame], 0, q, 1, ref64.gold(cell.cell_id, 1920).astype(bool))
            want = ref64_ctrl.mib_bits(ref64_ctrl.BW_CODE.get(cell.nof_prb, 0), cell.phich_ext, cell.phich_ng, tti // 10)
            assert ok and rem == ref_dec.PBCH_PORT_MASK[cell.nof_ports], (tti, rem)
            if cell.nof_prb in ref64_ctrl.BW_CODE:
                assert np.array_equal(mib, want), (tti, mib, want)
    assert total >= 20, total


# ------------------------------------------------------------------------------------------------ the oracle on the numpy eNB
def plant(ncce, rng, sizes=(27, 43), locs=None, first=0):
    """DCIs over the whole CCE space: first the smallest of the locations that end last (on the last CCE unless locs leave it out), then aggregation levels 8 / 4 / 2 / 1 in turn
    (starting at entry `first` of that cycle) from CCE 0 up, sizes in turn.  locs: the allowed (first CCE, L), every aligned one by default.
    -> [(bits, rnti, L, first CCE)]"""
    if locs is None:
        locs = [(n, L) for L in (1, 2, 4, 8) for n in range(0, ncce - L + 1, L)]
    used = np.zeros(ncce, bool)
    out = []

    def take(n, L, j):
        used[n:n + L] = True
        out.append((rng.integers(0, 2, sizes[j % len(sizes)]).astype(np.uint8), int(rng.integers(1, 0xFFF4)), L, n))
    take(*min(locs, key=lambda x: (-(x[0] + x[1]), x[1])), 1)          # ends on the last CCE when a location does
    pos, j, misses = 0, first, 0
    while misses < 4:
        L = (8, 4, 2, 1)[j % 4]
        c = sorted(n for n, LL in locs if LL == L and n >= pos and not used[n:n + L].any())
        j += 1
        if not c:
            misses += 1
            continue
        misses = 0
        take(c[0], L, j)
        pos = c[0] + L + j % 3
    return out


ENB_CELLS = [(25, 1, 0, 1, 0, 0, 0), (25, 2, 151, 2, 0, 3, 0), (15, 2, 44, 1, 0, 1, 1), (50, 1, 302, 2, 0, 2, 1), (75, 2, 500, 1, 0, 0, 0),
             (100, 1, 7, 2, 0, 3, 1)]


def enb_capture(cell, sf, cfi, sfn, seed, noise_var=1e-3, chan="selective"):
    rng = np.random.default_rng(seed)
    m = ref64_ctrl.cell_map(cell, cfi)
    dcis = plant(m.ncce, rng, first=seed)
    grids, truth = ref64_ctrl.enb_subframe(cell, sf, cfi, dcis, rng, sfn=sfn, spare=int(rng.integers(0, 1024)))
    H = ref64.channel(chan, cell.nof_rx, cell.nof_ports, 12 * cell.nof_prb)
    Y, iq = ref64_ctrl.capture(cell, grids, H, noise_var, rng)
    return iq, truth


@pytest.mark.parametrize("cellp", ENB_CELLS, ids=lambda c: "x".join(map(str, c)))
def test_oracle_decodes_the_numpy_enb(infra, cellp):
    """the oracle finds the CFI, every planted DCI at its CCEs with its RNTI, and in subframe 0 the MIB and the port count at every SFN mod 4"""
    cell = Cell(*cellp)
    o = Oracle(cell)
    for i in range(12):
        sf, sfn = i % 10, 2 * i
        if i >= 10:
            sf, sfn = 0, 2 * i + 1
        cfi = 3 if cell.phich_ext else 1 + i % 3
        iq, truth = enb_capture(cell, sf, cfi, sfn, seed=100 * i + cellp[2])
        sym = o.ofdm(iq)
        ce, _ = o.chest(sf, sym)
        got, _ = o.pcfich(sf, sym, ce)
        assert got == cfi, (i, got, cfi)
        llr = o.pdcch_llr(sf, cfi, sym, ce)
        for bits, rnti, L, n in truth.dcis:
            r, b, crc = o.dci_decode(llr[72 * n:72 * (n + L)], len(bits))
            assert r == 0 and crc == rnti and np.array_equal(b, bits), (i, rnti, L, n)
        if sf == 0:
            found, mib, nports, q = o.pbch_decode(sym, ce)
            assert found == 1 and nports == cell.nof_ports and q == sfn % 4, (i, found, nports, q)
            assert np.array_equal(mib, truth.mib), (i, mib, truth.mib)
