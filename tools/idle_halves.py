"""Idle int16x2 halves of the two paired decoders on the headline workload, counted on the CPU oracle (no GPU).

  Viterbi: warp decodes per (subframe, payload size) with FLAG_SKIP_LOW_POWER -- fixed location pairs (2p, 2p+1) holding any decodable
           location, against decodable locations packed densely (vit_worklist_kernel).
  Turbo:   sum over pairs of K x max(iterations of the two halves), iteration counts from lteo_dlsch_decode, for the submission-order
           pairing of equal K, the code-rate pairing (ltephy_turbo_pairing, host only) and pairing by the true iteration count.

The simulator settings are bench.py's SIM_KW, repeated here as data.  Prints one JSON object.
usage: python tools/idle_halves.py [--subframes N]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

CELL = dict(nof_prb=100, nof_ports=2, cell_id=7, nof_rx=2)
SIM_KW = dict(seed=2, cfi=3, nof_ues=150, dl_min=8, dl_max=12, tm=3, mcs_min=17, mcs_max=28, snr_db=25.0, full_band=1)
MAX_LOC, SEARCH_MAX_CCE, POWER_FLOOR = 160, 84, np.float32(0.7)


def locations(nof_cce):
    """(first CCE, log2 L) of every blind-search location, in the library's order (ltehost::all_locations)"""
    out = []
    lim = min(nof_cce, SEARCH_MAX_CCE)
    for l in (3, 2, 1, 0):
        L = 1 << l
        for i in range(lim // L):
            if len(out) < MAX_LOC and nof_cce // L:
                out.append((L * (i % (nof_cce // L)), l))
    return out


def turbo_cost(K, it, pair):
    cost = {}
    for k, n, p in zip(K, it, pair):
        c = cost.setdefault(p, [k, 0])
        c[1] = max(c[1], n)
    return sum(k * n for k, n in cost.values())


def submission_order_pairs(K):
    pair, open_, n = [], {}, 0
    for k in K:
        if k in open_:
            pair.append(open_.pop(k))
        else:
            open_[k] = n
            pair.append(n)
            n += 1
    return pair


def sorted_pairs(K, key):
    pair, n, open_k = [0] * len(K), 0, None      # open_k: K of the last pair while it has a free half
    for i in sorted(range(len(K)), key=lambda i: (K[i], key[i], i)):
        if open_k == K[i]:
            pair[i], open_k = n - 1, None
        else:
            pair[i], n, open_k = n, n + 1, K[i]
    return pair


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subframes", type=int, default=40)
    args = ap.parse_args()
    import ctypes as C
    import ltelib
    import rm_ref
    from helpers import make_capture, oracle_frontend, truth_grants
    from ltesniffer_b200 import capi, load_library
    cell = ltelib.Cell(CELL["nof_prb"], CELL["nof_ports"], CELL["cell_id"], CELL["nof_rx"])
    sim, iq, tti, truths, payloads = make_capture(cell, args.subframes, **SIM_KW)
    o = ltelib.Oracle(cell)
    ref = oracle_frontend(o, iq, tti)
    O = ltelib.oracle()

    # ---- Viterbi items per (subframe, size)
    fixed = dense = nvalid = nloc = 0
    for r in ref:
        locs = locations(len(r["cce_power"]))
        ok = [bool(np.all(r["cce_power"][n0:n0 + (1 << l)] >= POWER_FLOOR)) for n0, l in locs]
        nloc += len(locs)
        nvalid += sum(ok)
        fixed += sum(1 for p in range((len(ok) + 1) // 2) if any(ok[2 * p:2 * p + 2]))
        dense += (sum(ok) + 1) // 2
    n = len(ref)

    # ---- turbo: per code block K, iterations, code rate of its transport block
    K, it, tbs_l, G_l = [], [], [], []
    for sf, d, g in truth_grants(cell, truths, tti):
        rr = ref[sf]
        ret, llr, _ = o.pdsch_llr(int(tti[sf]) % 10, rr["cfi"], d.rnti, g, rr["sym"], rr["ce"])
        cw = 0
        for t in range(2):
            if not g.tb[t].enabled:
                continue
            ocw = (1 - cw) if (g.nof_tb == 2 and g.cw_swap) else cw
            cw += 1
            tb = g.tb[t]
            G = g.nof_re * tb.qm
            C_, Kp, Km, Cp, Cm, F = rm_ref.check_tables.segm(tb.tbs)
            its = np.zeros(64, np.uint32)
            pl = np.zeros(tb.tbs // 8 + 16, np.uint8)
            O.lteo_dlsch_decode(ltelib.ptr(np.ascontiguousarray(llr[ocw][:G])), G, tb.tbs, tb.rv, tb.qm, 2 if g.tx_scheme == capi.TX_DIVERSITY else 1, 8, 1,
                                ltelib.ptr(pl), ltelib.ptr(its))
            for r_ in range(C_):
                K.append(Km if r_ < Cm else Kp)
                it.append(int(its[r_]))
                tbs_l.append(tb.tbs)
                G_l.append(G)
    lib = load_library()
    lib.ltephy_turbo_pairing.argtypes = [C.c_uint32] + [C.c_void_p] * 5 + [C.POINTER(C.c_uint32)]
    arr = [np.ascontiguousarray(a, np.uint32) for a in (K, tbs_l, G_l)]
    pair, half, npairs = np.zeros(len(K), np.uint32), np.zeros(len(K), np.uint32), C.c_uint32(0)
    assert lib.ltephy_turbo_pairing(len(K), *[a.ctypes.data for a in arr], pair.ctypes.data, half.ctypes.data, C.byref(npairs)) == 0
    old = turbo_cost(K, it, submission_order_pairs(K))
    new = turbo_cost(K, it, pair.tolist())
    best = turbo_cost(K, it, sorted_pairs(K, it))
    refill = sum(k * n for k, n in zip(K, it)) / 2          # both halves always busy
    print(json.dumps({
        "subframes": n, "sim": SIM_KW,
        "viterbi": {"locations_per_sf": nloc / n, "decodable_per_sf": nvalid / n, "items_per_sf_size_fixed_pairs": fixed / n,
                    "items_per_sf_size_dense": dense / n, "dense_over_fixed": dense / fixed if fixed else None},
        "turbo": {"code_blocks": len(K), "distinct_K": len(set(K)), "mean_iters": float(np.mean(it)) if it else None,
                  "cost_submission_order": 1.0, "cost_code_rate": new / old, "cost_true_iterations": best / old,
                  "idle_share_submission_order": 1 - refill / old, "idle_share_code_rate": 1 - refill / new}}, indent=1))


if __name__ == "__main__":
    main()
