"""What integer samples save end to end: ltephy_decode_subframes on bench.py's cfg-2 workload (1000 subframes of a 20 MHz, 100 PRB 2x2 cell per batch) from
pinned host memory, with bench's e2e pipeline count, in cf32, sc16 and sc8.  The capture is bench's generator output, quantised once per format
with one scale: the largest I or Q component of the capture lands at half of full scale (q = rint(x * 0.5 / max|x| * 2^15) for sc16, * 2^7 for
sc8), and cf32 runs on the unquantised capture.  Each repetition times every format once, in turn, so drift on a shared host hits all three alike;
the median over repetitions is printed with the lowest and highest value.  Also: the H2D-plus-phase-A time of one batch on one pipeline from
ltephy_last_timing, the decoded transport blocks (TB CRC passes) of one batch per format, and one 1 s push of tools/track_time.py's recording
(N = 2048, 2 antennas, 1000 subframes) through ltephy_track_push from pinned host memory per format.  Prints the device and its power limit.
Needs a GPU; there is no CPU fallback.

    python tools/iq_format_time.py [--reps 7] [--steps 12]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FORMATS = ("cf32", "sc16", "sc8")
PIPELINES = 6   # bench.py's e2e default (--pipelines 0)
BATCH = 1000    # bench.py's --batch default


def quantise(x, fmt, scale):
    """complex64 [...] -> the format's host layout: complex64 as is, int16 / int8 [...][2] = rint(x * scale * 2^bits)"""
    if fmt == "cf32":
        return x
    b = 15 if fmt == "sc16" else 7
    v = x.view(np.float32).reshape(x.shape + (2,)).astype(np.float64) * (scale * 2.0 ** b)
    return np.clip(np.rint(v), -2 ** b, 2 ** b - 1).astype(np.int16 if fmt == "sc16" else np.int8)


def pinned(a):
    """a pinned host copy of a numpy array (what a live binding hands the library)"""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    return t, t.numpy()


def stats(v):
    return dict(median=round(float(np.median(v)), 3), min=round(float(np.min(v)), 3), max=round(float(np.max(v)), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=12, help="batches per timed run (over the pipelines)")
    args = ap.parse_args()
    import torch
    import bench
    from ltesniffer_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q), flush=True)

    cell, iq_u = bench.generate_capture(BATCH, min(os.cpu_count() or 4, 16))
    scale = 0.5 / float(np.abs(iq_u.view(np.float32)).max())
    B, T = BATCH, PIPELINES
    tti = np.ascontiguousarray(np.arange(B, dtype=np.uint32))
    L = capi.load_library()
    capi._bind_search(L)
    max_dcis = 24 * B
    run = {}
    for fmt in FORMATS:
        _, host = pinned(quantise(iq_u, fmt, scale))
        phys = [capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=B, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER,
                            iq_format=fmt) for _ in range(T)]
        scr = [dict(info=(capi.SfInfo * B)(), cands=np.zeros((B, capi.MAX_LOC, capi.MAX_SIZES), capi.CAND_DTYPE), dcis=np.zeros(max_dcis, capi.DCI_DTYPE),
                    tbs=(capi.TbResult * (2 * max_dcis))(), payload=pinned(np.zeros(B * 48000, np.uint8))[1], nd=C.c_uint32(0)) for _ in range(T)]
        run[fmt] = dict(host=host, phys=phys, scr=scr, search=capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx), seq=0,
                        rate=[], h2d_a=[])
    print("capture: %d subframes, %.1f MB per batch in cf32; scale %.6g (peak component at 0.5 full scale)"
          % (B, iq_u.nbytes / 1e6, scale), flush=True)

    def step(r, t, seq):
        S = r["scr"][t]
        rc = L.ltephy_decode_subframes(r["phys"][t].h, r["search"].h, capi._p(r["host"]), capi._p(tti), B, seq, S["info"], capi._p(S["cands"]),
                                       capi._p(S["dcis"]), max_dcis, C.byref(S["nd"]), S["tbs"], capi._p(S["payload"]), S["payload"].nbytes)
        if rc != 0:
            raise RuntimeError("ltephy_decode_subframes: %s" % L.ltephy_last_error().decode())

    def steps(r, n):
        base = r["seq"]
        r["seq"] += n

        def worker(t):
            torch.cuda.set_device(0)
            for k in range(t, n, T):
                step(r, t, base + k)
        with ThreadPoolExecutor(T) as ex:
            list(ex.map(worker, range(T)))

    for fmt in FORMATS:   # warm-up: every pipeline once, then the decoded blocks and phase A of one batch on one pipeline
        r = run[fmt]
        steps(r, T)
        step(r, 0, r["seq"])
        r["seq"] += 1
        S = r["scr"][0]
        nd = S["nd"].value
        r["tb_crc_pass"] = int(sum(S["tbs"][i].crc != 0 for i in range(2 * nd)))
        r["dcis"] = nd
    for _ in range(args.reps):
        for fmt in FORMATS:
            r = run[fmt]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            steps(r, args.steps)
            torch.cuda.synchronize()
            r["rate"].append(args.steps * B / (time.perf_counter() - t0))
            step(r, 0, r["seq"])    # one batch alone on its pipeline: H2D + phase A without the other pipelines' copies in the way
            r["seq"] += 1
            ms = (C.c_float * 4)()
            L.ltephy_last_timing(r["phys"][0].h, ms)
            r["h2d_a"].append(ms[0])
    out = dict(workload="bench cfg-2: %d subframes per batch, %d PRB, %d ports, %d rx, %d pipelines" % (B, cell.nof_prb, cell.nof_ports, cell.nof_rx, T),
               reps=args.reps, steps=args.steps)
    for fmt in FORMATS:
        r = run[fmt]
        out[fmt] = dict(h2d_bytes_per_batch=int(r["host"].nbytes), e2e_subframes_per_s=stats(r["rate"]), h2d_plus_phase_a_ms=stats(r["h2d_a"]),
                        dcis=r["dcis"], tb_crc_pass=r["tb_crc_pass"])
        r["search"].close()
        for p in r["phys"]:
            p.close()
    out["sc16_tb_crc_pass_equals_cf32"] = out["sc16"]["tb_crc_pass"] == out["cf32"]["tb_crc_pass"]
    print(json.dumps(out), flush=True)
    track(args.reps)


def track(reps):
    """one 1 s push (N = 2048, 2 antennas, 1000 subframes) of tools/track_time.py's recording from pinned host memory, per format"""
    import torch
    from ltesniffer_b200 import capi
    N, A, K = 2048, 2, 1000
    Ls = (K + 1) * 15 * N
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((A, Ls), dtype=torch.complex64, device="cuda", generator=g).cpu().numpy()
    scale = 0.5 / float(np.abs(x.view(np.float32)).max())
    out = dict(N=N, nof_rx=A, subframes=K)
    hosts = {fmt: pinned(quantise(x, fmt, scale))[1] for fmt in FORMATS}
    ms = {fmt: [] for fmt in FORMATS}
    for rep in range(reps + 1):
        for fmt in FORMATS:
            tr = capi.Tracker(N, A, 0, 100, max_subframes=K, iq_format=fmt)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = tr.push(hosts[fmt], 0)
            t1 = time.perf_counter()
            assert len(r["sf"]) == K
            if rep:                               # rep 0 is the warm-up
                ms[fmt].append((t1 - t0) * 1e3)
            tr.close()
    for fmt in FORMATS:
        out[fmt] = dict(h2d_bytes=int(hosts[fmt].nbytes), push_ms=stats(ms[fmt]))
    print(json.dumps(dict(track_push=out)), flush=True)


if __name__ == "__main__":
    main()
