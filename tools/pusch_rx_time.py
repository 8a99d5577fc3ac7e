"""Cost of the second uplink antenna: bench.py's cfg-5 PUSCH workload (100 PRB, 256 subframes, 16 distinct subframes tiled, 6-10 DCI-0 grants per
subframe with MCS 10-24, a third with HARQ-ACK / CQI multiplexed) through ltephy_submit_ul(_device) / ltephy_get_ul, with ul_nof_rx = 1 and
ul_nof_rx = 2 on the same grants, alternating in one process, each twice: from pageable host IQ (ltephy_submit_ul: the H2D copy of the samples,
UL OFDM, PUSCH kernel, rate-dematch, turbo, CRC) and from IQ already in HBM (ltephy_submit_ul_device: the same without the copy, which is what
the second antenna costs in the kernels).  device_ms is the handle's CUDA-event time of the submit; the median over the repetitions is reported
with its spread.  Prints the device and its power limit.  Needs a GPU; there is no CPU fallback.

    python tools/pusch_rx_time.py [--reps 9]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def workload(capi, ltelib, X, n=256, n_u=16):
    """the cfg-5 grants of bench.bench_pusch and their subframes received on two antennas.  bench.py builds its workload inside the timed function,
    so it is restated here; antenna 0 is checked against bench's own generator call (ltelib.sim_ul_subframe on the same simulator seed) and the
    grant count against the 1 248 grants bench reports"""
    import numpy as np
    cell = ltelib.Cell(100, 2, 7, 2)
    ucfg = ltelib.UlCfg(n_dmrs1=3, delta_ss=2)
    s = ltelib.Sim(cell=cell, seed=5, snr_db=25.0, nof_ues=1)
    s1 = ltelib.Sim(cell=cell, seed=5, snr_db=25.0, nof_ues=1)
    rng = np.random.default_rng(5)
    iq = np.zeros((n_u, 2, s.sf_len), np.complex64)
    per_sf = []
    for i in range(n_u):
        gr = []
        for g in ltelib.make_ul_grants(cell, rng, int(rng.integers(6, 11)), table=1):
            if not 10 <= g.mcs <= 24:
                continue
            if rng.random() < 0.33:
                g.nof_ack, g.I_offset_ack = int(rng.integers(1, 3)), 9
                if rng.random() < 0.5:
                    g.cqi_len, g.I_offset_cqi, g.ri_len, g.I_offset_ri = 30, 6, 1, 5
            gr.append(g)
        iq[i] = X.sim_ul_rx(s, i, ucfg, gr, 2)[0]
        assert iq[i, 0].tobytes() == ltelib.sim_ul_subframe(s1, i, ucfg, gr)[0].tobytes(), "antenna 0 is not bench's sample stream"
        per_sf.append(gr)
    iq = np.ascontiguousarray(np.tile(iq, (n // n_u, 1, 1)))
    tti = (np.arange(n) % n_u).astype(np.uint32)
    grants = [capi.UlGrant(sf=i, rnti=g.rnti, qm=g.qm, rv=g.rv, L_prb=g.L_prb, n_prb=g.n_prb, n_dmrs2=g.n_dmrs2, tbs=g.tbs, n_prb_slot1=g.n_prb,
                           flags=capi.UL_FLAG_SLOT1, nof_ack=g.nof_ack, ri_len=g.ri_len, cqi_len=g.cqi_len, I_offset_ack=g.I_offset_ack,
                           I_offset_ri=g.I_offset_ri, I_offset_cqi=g.I_offset_cqi) for i in range(n) for g in per_sf[i % n_u]]
    assert len(grants) == 1248, len(grants)
    return cell, iq, tti, grants


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    args = ap.parse_args()
    import numpy as np
    import torch
    import ltelib
    import pusch_rx_lib as X
    from ltesniffer_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q))
    cell, iq, tti, grants = workload(capi, ltelib, X)
    n = len(tti)
    phys, inputs = {}, {1: np.ascontiguousarray(iq[:, 0]), 2: iq}
    dev_in = {A: torch.from_numpy(inputs[A]).cuda() for A in (1, 2)}
    legs = [(A, d) for A in (1, 2) for d in ("host", "device")]
    for A in (1, 2):
        phys[A] = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=n, turbo_max_iter=8, ul_nof_rx=A)
        phys[A].set_ul_cfg(3, 2)
        phys[A].decode_ul(inputs[A], tti, grants)                       # warm-up: module load, table pools, buffers
        phys[A].decode_ul_device(dev_in[A], tti, grants)
    torch.cuda.synchronize()
    dev = {k: [] for k in legs}
    ok = {}
    for _ in range(args.reps):
        for A, d in legs:
            res, _, _ = phys[A].decode_ul(inputs[A], tti, grants) if d == "host" else phys[A].decode_ul_device(dev_in[A], tti, grants)
            dev[(A, d)].append(phys[A].timing()[1])
            ok[(A, d)] = sum(1 for r in res[:len(grants)] if r.crc)
    out = {}
    for A, d in legs:
        v = np.array(dev[(A, d)])
        out["A%d_%s" % (A, d)] = dict(device_ms_median=float(np.median(v)), device_ms_min=float(v.min()), device_ms_max=float(v.max()), tb_crc_ok=ok[(A, d)])
    for A in (1, 2):
        phys[A].close()
    med = lambda k: out[k]["device_ms_median"]
    out.update(subframes=n, grants=len(grants), ratio_A2_over_A1_host=med("A2_host") / med("A1_host"),
               ratio_A2_over_A1_device=med("A2_device") / med("A1_device"), device=q)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
