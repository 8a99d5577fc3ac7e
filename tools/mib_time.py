"""Time of one ltephy_mib_decode_combined call over 1000 consecutive subframes 0 (noise: every hypothesis job is evaluated whatever the content),
and of ltephy_mib_decode on the same batch.  25 PRB, 2-port handle, 1 antenna, with and without the port search.  Reports the elapsed time on the
handle's stream between ltephy_mark events around the call (the call's host-side job table and result walk included) and the host wall time,
after a warm-up, median of --reps.  Prints the device and its power limit.  Needs a GPU; there is no CPU fallback.

    python tools/mib_time.py [--reps 20] [--frames 1000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--frames", type=int, default=1000)
    args = ap.parse_args()
    from ltesniffer_b200 import capi
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("nvidia-smi: %s" % q)
    n = args.frames
    phy = capi.LtePhy(25, 2, 3, 1, max_subframes=n)
    rng = np.random.default_rng(1)
    iq = (rng.standard_normal((n, 1, phy.sf_len)) + 1j * rng.standard_normal((n, 1, phy.sf_len))).astype(np.complex64)
    tti = (np.arange(n, dtype=np.uint32) % 1024) * 10
    phy.submit_iq(iq, tti)
    phy.get_phase_a(want_cands=False)
    phy.L.ltephy_mark.argtypes = [capi.C.c_void_p, capi.C.c_int]
    calls = [("mib_decode", lambda: phy.mib_decode()),
             ("mib_decode_combined", lambda: (phy.mib_reset(), phy.mib_decode_combined(False))),
             ("mib_decode_combined_search_ports", lambda: (phy.mib_reset(), phy.mib_decode_combined(True)))]
    for name, fn in calls:
        for _ in range(3):
            fn()
        dev, wall = [], []
        for _ in range(args.reps):
            phy.mib_reset()
            phy.L.ltephy_mark(phy.h, 0)
            t0 = time.perf_counter()
            fn()
            wall.append(time.perf_counter() - t0)
            phy.L.ltephy_mark(phy.h, 1)
            dev.append(phy.L.ltephy_mark_elapsed_ms(phy.h))
        print(json.dumps(dict(call=name, frames=n, stream_ms=round(float(np.median(dev)), 3), wall_ms=round(1e3 * float(np.median(wall)), 3))))
    phy.close()


if __name__ == "__main__":
    main()
