"""Time the raster scan (ltephy_scan_run_device) against the per-point composition through the public API (per point, ltephy_chan_run_device with
the one carrier, then ltephy_cell_search_device) on the same 2-antenna, 40 ms capture in HBM, at 100 Msps (rational, 989 points) and 245.76 Msps
(integer D = 128, 2 447 points).  Host clocks around calls that block until their stream is done; the two forms alternate, and each time is the
median of --reps.  The composition's handles are made before its clock starts (a channeliser handle per point, one cell-search handle), so
it is timed on its device work and its host round trips only.  The time ltephy_scan_create takes (every point's filter taps, on the host) is
printed apart.  Both forms must give identical results at every point.  Prints the card's name, power limit and clock, read in the same run, and
one JSON line per capture.

    python tools/scan_time.py [--reps 3] [--ms 40]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from chan_time import card  # noqa: E402

CAPTURES = [("100 Msps", 100000000), ("245.76 Msps", 245760000)]
CENTER = 1850000000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ms", type=float, default=40.0)
    args = ap.parse_args()
    import torch
    from ltesniffer_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to time")
    print("card: %s (%s)" % (card(), torch.cuda.get_device_name(0)))
    rng = np.random.default_rng(1)
    for name, fs in CAPTURES:
        n = int(fs * args.ms / 1000)
        # noise with a few strong tones: the scan's work does not depend on what the capture holds
        x = (rng.standard_normal((2, n), np.float32) + 1j * rng.standard_normal((2, n), np.float32)).astype(np.complex64) * np.float32(0.05)
        t = np.arange(n)
        for f in (-20e6, 3.3e6, 31e6):
            x += (0.2 * np.exp(2j * np.pi * ((f * t) % fs) / fs)).astype(np.complex64)
        xd = torch.from_numpy(x).cuda()
        t0 = time.perf_counter()
        sc = capi.Scanner(fs, 2, CENTER, n)
        t_create = time.perf_counter() - t0
        offs = [int(o) for o in sc.plan()]
        sc.run_device(xd)   # warm-up
        cnt = None
        ts, tc = [], []
        for rep in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sc.run_device(xd)
            ts.append(time.perf_counter() - t0)
            pts = sc.points()
            # the composition, point by point
            comp, dt = [], 0.0
            cs = None
            for o in offs:
                ch = capi.Channelizer(fs, [(o, 128)], 2, n, rational=True)
                if cs is None:
                    res, _ = ch.run_device(xd, 0, copy=False)   # warm-up, and the stream length
                    cnt = res[0]["count"]
                    cs = capi.CellSearch(128, 2, cnt)
                    cs.search_device(res[0]["iq"])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res, _ = ch.run_device(xd, 0, copy=False)
                cells = cs.search_device(res[0]["iq"])
                dt += time.perf_counter() - t0
                comp.append(cells)
                ch.close()
            cs.close()
            tc.append(dt)
            same = all([bytes(c) for c in a] == [bytes(c) for c in b] for a, b in zip(pts, comp))
            assert same, "the scan and the per-point composition differ"
        s, c = statistics.median(ts), statistics.median(tc)
        print(json.dumps(dict(capture=name, fs_in=fs, ms=args.ms, nof_rx=2, points=len(offs), stream_samples=cnt, scan_s=round(s, 4),
                              composition_s=round(c, 4), speedup=round(c / s, 2), scan_create_s=round(t_create, 3), reps=args.reps,
                              identical=True, scan_all_s=[round(v, 4) for v in ts], composition_all_s=[round(v, 4) for v in tc])), flush=True)
        sc.close()
        del xd
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
