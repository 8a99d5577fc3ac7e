"""Shared helpers for the parity tests: run the CPU oracle over a capture, convert grants, and the UL-mode batch step of the examples driven
through the binding."""
import ctypes as C

import numpy as np
import ltelib
from ltelib import Sim
from ltesniffer_b200 import capi


def make_capture(cell, n, **simkw):
    s = Sim(cell=cell, **simkw)
    iq = np.zeros((n, cell.nof_rx, s.sf_len), np.complex64)
    truths, payloads = [], []
    tti0 = simkw.get("tti0", 0)
    for i in range(n):
        x, tr, pl = s.subframe(tti0 + i)
        iq[i] = x
        truths.append(tr)
        payloads.append(pl)
    return s, iq, np.arange(tti0, tti0 + n, dtype=np.uint32), truths, payloads


def oracle_frontend(o, iq, tti):
    """-> list of dicts with sym, ce, res, cfi, corr, llr, rb_power, cce_power per subframe"""
    out = []
    for i in range(len(tti)):
        sf_idx = int(tti[i]) % 10
        sym = o.ofdm(iq[i])
        ce, res = o.chest(sf_idx, sym)
        cfi, corr = o.pcfich(sf_idx, sym, ce)
        llr = o.pdcch_llr(sf_idx, cfi, sym, ce)
        ncce = len(llr) // 72
        pw = np.zeros(ncce, np.float32)
        ltelib.oracle().lteo_cce_power(ltelib.ptr(llr), ncce, ltelib.ptr(pw))
        out.append(dict(sym=sym, ce=ce, res=res, cfi=cfi, corr=corr, llr=llr, rb_power=o.rb_power(sym[0]), cce_power=pw))
    return out


def to_phy_grant(sf, rnti, g):
    """ltelib.DlGrant (oracle/sim) -> capi.Grant (product C-ABI)"""
    pg = capi.Grant()
    pg.sf = sf
    pg.rnti = rnti
    pg.tx_scheme = g.tx_scheme
    pg.nof_tb = g.nof_tb
    pg.nof_re = g.nof_re
    pg.pmi = g.pmi
    for s in range(2):
        for prb in range(110):
            if g.prb_mask[s][prb]:
                pg.prb_mask[s][prb >> 5] |= (1 << (prb & 31))
    for t in range(2):
        pg.tb[t].tbs = g.tb[t].tbs
        pg.tb[t].qm = g.tb[t].qm
        pg.tb[t].rv = g.tb[t].rv
        pg.tb[t].enabled = g.tb[t].enabled
    en = [t for t in range(2) if g.tb[t].enabled]
    for k, t in enumerate(en):
        pg.tb[t].cw_idx = (1 - k) if (len(en) == 2 and g.cw_swap) else k
    return pg


def truth_grants(cell, truths, tti, alt=0):
    """ground-truth DL grants of a capture: list of (sf, truth_dci, DlGrant)"""
    out = []
    for sf, tr in enumerate(truths):
        for i in range(tr.nof_dci):
            d = tr.dci[i]
            if d.nof_tb == 0:
                continue
            bits = np.frombuffer(bytes(d.bits), np.uint8)[:d.nbits]
            r, dd, g = ltelib.unpack_and_grant(cell, d.format, d.rnti, bits, int(tti[sf]) % 10, tr.cfi, alt)
            assert r == 0, r
            out.append((sf, d, g))
    return out


def feq(a, b):
    """float arrays equal as values (so -0.0 == +0.0), no NaNs allowed."""
    a = np.asarray(a)
    b = np.asarray(b)
    return a.shape == b.shape and not np.isnan(a).any() and bool(np.all(a == b))


def describe_mismatch(a, b, name):
    a = np.asarray(a).ravel()
    b = np.asarray(b).ravel()
    bad = np.nonzero(a != b)[0]
    if len(bad) == 0:
        return "%s: identical" % name
    d = np.abs(a.astype(np.complex128) - b.astype(np.complex128))
    return "%s: %d/%d differ, first at %d (%r vs %r), max abs diff %.3g, rel %.3g" % (
        name, len(bad), len(a), bad[0], a[bad[0]], b[bad[0]], d.max(), d.max() / (np.abs(b).max() + 1e-30))


def ul_records(grants, res, pl, tti):
    """the UL records (0, rnti, tti, payload) of one ltephy_submit_ul: the first attempt of a DCI-0 that passed (PUSCH_Decoder::decode stops
    there), as the examples write them"""
    out, passed = [], False
    for k, g in enumerate(grants):
        if k == 0 or grants[k - 1].rnti != g.rnti or grants[k - 1].sf != g.sf:
            passed = False
        ok = res[k].crc and not passed
        passed = passed or res[k].crc != 0
        if ok and res[k].payload_len:
            out.append((0, int(g.rnti), int(tti[g.sf]), bytes(pl[res[k].payload_off:res[k].payload_off + res[k].payload_len])))
    return out


class UlModeStep:
    """The UL-mode batch step of examples/cell_chain.h driven through the binding: decode a batch of DL subframes in UL mode and record their DL
    blocks; split the carried grants into this batch's and later ones; take msg-3 grants from RAR payloads (sf + 6) and activate their C-RNTIs;
    take DCI-0 grants from ul_grants_from_dcis; shift the carry; decode the uplink and keep the first attempt of a DCI-0 that passed.  It owns
    the search handle in UL mode, the DL and UL handles (the UL one with ul_nof_rx antennas), the scratch buffers and the carry.  beyond: the
    largest number of carried grants that fell beyond a batch; carry: the grants still carried; now: the grants of the last batch's UL decode."""

    def __init__(self, prb, ports, pci, B, ul_nof_rx=1, symbol_sz=0, phich_resources=0, phich_length=0):
        import track_lib as T
        mk = lambda A: capi.LtePhy(prb, ports, pci, 1, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER, symbol_sz=symbol_sz,
                                   phich_resources=phich_resources, phich_length=phich_length, ul_nof_rx=A)
        self.phy, self.ul = mk(1), mk(ul_nof_rx)
        self.ul.set_ul_cfg(**T.UCFG)
        self.srch = capi.Search(prb, ports, pci, 1, phich_resources=phich_resources)
        self.L = self.phy.L
        self.L.ltephy_search_set_ul_mode(self.srch.h, 1, 0)
        self.L.ltephy_search_set_ul_hopping(self.srch.h, 0)
        self.L.ltephy_search_activate.argtypes = [C.c_void_p, C.c_uint16, C.c_uint32, C.c_int]
        self.md = 32 * B
        self.info, self.cands = (capi.SfInfo * B)(), np.zeros((B, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE)
        self.dcis, self.tbs, self.pay = np.zeros(self.md, capi.DCI_DTYPE), (capi.TbResult * (2 * self.md))(), np.zeros(B * 64 * 1024, np.uint8)
        self.carry, self.beyond, self.now = [], 0, []

    def close(self):
        self.phy.close(), self.ul.close(), self.srch.close()

    def __call__(self, dl, tti, ul_iq):
        """one batch: dl torch complex64 [m][1][15 N] on the device, tti its m ttis, ul_iq torch complex64 [m][15 N] ([m][A][15 N]) on the device
        -> the batch's records in the examples' order: its DL blocks (1, rnti, tti, payload), then its UL blocks (0, rnti, tti, payload)"""
        tti, m, L, tbs, pay = np.ascontiguousarray(tti, np.uint32), len(tti), self.L, self.tbs, self.pay
        block = lambda rr: bytes(pay[rr.payload_off:rr.payload_off + rr.payload_len])
        nd = C.c_uint32(0)
        assert L.ltephy_decode_subframes_device(self.phy.h, self.srch.h, C.c_void_p(dl.data_ptr()), capi._p(tti), m, capi.SEQ_NONE, self.info,
                                                capi._p(self.cands), capi._p(self.dcis), self.md, C.byref(nd), tbs, capi._p(pay), pay.nbytes) == 0
        dcis = self.dcis[:nd.value].copy()
        now, self.carry = [g for g in self.carry if g.sf < m], [g for g in self.carry if g.sf >= m]
        self.beyond = max(self.beyond, len(self.carry))
        out = []
        for i, d in enumerate(dcis):
            for t in range(2):
                rr = tbs[2 * i + t]
                if rr.crc and rr.payload_len:
                    out.append((1, int(d["rnti"]), int(tti[int(d["sf"])]), block(rr)))
        for i, d in enumerate(dcis):
            rr = tbs[2 * i]
            if not (1 <= int(d["rnti"]) <= 10 and rr.crc and rr.payload_len):
                continue
            rc, rars, _ = capi.rar_unpack(self.srch, block(rr))
            if rc != 0:
                continue
            for a in rars:
                L.ltephy_search_activate(self.srch.h, a.t_crnti, 0, 2)
                if a.valid:
                    g = capi.UlGrant.from_buffer_copy(a.grant)
                    g.sf = int(d["sf"]) + 6
                    (now if g.sf < m else self.carry).append(g)
        for _, _, g in capi.ul_grants_from_dcis(self.srch, self.info, dcis):
            (now if g.sf < m else self.carry).append(g)
        for g in self.carry:
            g.sf -= m
        self.now = now
        if now:
            res, _, pl = self.ul.decode_ul_device(ul_iq, tti, now)
            out += ul_records(now, res, pl, tti)
        return out
