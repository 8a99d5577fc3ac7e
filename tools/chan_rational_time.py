"""Device time of ltephy_chan_run_device with LTEPHY_CHAN_RATIONAL over 1 s of 2-antenna input already in HBM, for rational plans in cf32 and sc16,
and the 30.72 Msps integer plan of tools/chan_time.py in cf32 and sc16.  Median of --reps calls; the call blocks until its stream is done, so a
host clock around it measures the device work plus its launches.  The bytes are the algorithm's, from shapes: the input read once per carrier
and the outputs written once.  Prints the card's name, power limit and clock, read in the same run.

    python tools/chan_rational_time.py [--reps 20] [--seconds 1.0]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from chan_time import card  # noqa: E402

WORKLOADS = [
    ("25 Msps, one N 1024 carrier (384 / 625)", 25000000, [(0, 1024)]),
    ("100 Msps, three N 2048 carriers at -30, 0, +30 MHz (192 / 625)", 100000000, [(-30000000, 2048), (0, 2048), (30000000, 2048)]),
    ("200 Msps, N 2048 at +30 MHz and N 128 at -60 MHz (96 / 625, 6 / 625)", 200000000, [(30000000, 2048), (-60000000, 128)]),
    ("30.72 Msps, 20/10/5 MHz carriers (N 1024, 512, 256), integer", 30720000, [(-7500000, 1024), (5000000, 512), (11000000, 256)]),
]
SAMPLE_BYTES = {"cf32": 8, "sc16": 4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seconds", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    from ltesniffer_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to time")
    print("card: %s (%s)" % (card(), torch.cuda.get_device_name(0)))
    nrx = 2
    for name, fs, carriers in WORKLOADS:
        n = int(fs * args.seconds)
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn((nrx, n), dtype=torch.complex64, device="cuda", generator=g) * 0.1
        for fmt in ("cf32", "sc16"):
            if fmt == "sc16":
                xi = torch.view_as_real(x).reshape(nrx, 2 * n).mul(32767.0).round().clamp(-32768, 32767).to(torch.int16).contiguous()
            else:
                xi = x
            torch.cuda.synchronize()                  # the handle reads its input on its own stream
            ch = capi.Channelizer(fs, carriers, nrx, n, rational=True, iq_format=fmt)
            geo = [ch.design(c) for c in range(len(carriers))]
            for _ in range(3):
                ch.run_device(xi, 0, copy=False)
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                ch.run_device(xi, 0, copy=False)
                ts.append(time.perf_counter() - t0)
            ts.sort()
            med = ts[len(ts) // 2]
            outs = [n * q["L"] // q["M"] for q in geo]
            byts = sum(nrx * n * SAMPLE_BYTES[fmt] + nrx * o * 8 for o in outs)
            macs = sum(nrx * o * q["Kp"] for o, q in zip(outs, geo))
            print(json.dumps(dict(workload=name, fmt=fmt, fs_in=fs, nof_rx=nrx, seconds=args.seconds, L=[q["L"] for q in geo], M=[q["M"] for q in geo],
                                  Kp=[q["Kp"] for q in geo], ms_median=round(med * 1e3, 3), ms_min=round(ts[0] * 1e3, 3), ms_max=round(ts[-1] * 1e3, 3),
                                  algorithmic_GB=round(byts / 1e9, 3), GB_per_s=round(byts / med / 1e9, 1), complex_MACs_G=round(macs / 1e9, 2),
                                  realtime_factor=round(args.seconds / med, 1))))
            ch.close()
            del xi
        del x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
