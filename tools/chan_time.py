"""Device time of ltephy_chan_run_device over 1 s of 2-antenna input already in HBM, for two carrier plans, with the achieved bandwidth against the
bytes the algorithm needs (computed from shapes: the input read once per carrier, the outputs written once).  The call blocks until its stream
is done, so a host clock around it measures the device work plus one launch.  Prints the card's name and power limit, read in the same run.

    python tools/chan_time.py [--reps 20] [--seconds 1.0]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [
    ("30.72 Msps, 20/10/5 MHz carriers (N 1024, 512, 256)", 30720000, [(-7500000, 1024), (5000000, 512), (11000000, 256)]),
    ("61.44 Msps, three 20 MHz carriers (N 2048) at -19.8, 0, +19.8 MHz", 61440000, [(-19800000, 2048), (0, 2048), (19800000, 2048)]),
]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # the measurement still runs; the line says what is missing
        return "nvidia-smi unavailable (%s)" % e


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
        x = torch.randn((nrx, n), dtype=torch.complex64, device="cuda", generator=g)
        torch.cuda.synchronize()                      # the handle reads x on its own stream
        ch = capi.Channelizer(fs, carriers, nrx, n)
        Ds = [ch.taps(c)["D"] for c in range(len(carriers))]
        Ts = [ch.taps(c)["T"] for c in range(len(carriers))]
        for _ in range(3):
            ch.run_device(x, 0, copy=False)
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            ch.run_device(x, 0, copy=False)
            ts.append(time.perf_counter() - t0)
        ts.sort()
        med = ts[len(ts) // 2]
        byts = sum(nrx * n * 8 + nrx * (n // D) * 8 for D in Ds)
        print(json.dumps(dict(workload=name, fs_in=fs, nof_rx=nrx, seconds=args.seconds, D=Ds, T=Ts, ms_median=round(med * 1e3, 3),
                              ms_min=round(ts[0] * 1e3, 3), ms_max=round(ts[-1] * 1e3, 3), algorithmic_GB=round(byts / 1e9, 3),
                              GB_per_s=round(byts / med / 1e9, 1), realtime_factor=round(args.seconds / med, 1))))
        ch.close()
        del x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
