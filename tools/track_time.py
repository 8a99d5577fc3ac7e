"""Device time of the tracker's kernels (T1 metric windows, T2 CFO sums, T3 cut) per 1000-subframe push at N = 2048 with 2 antennas, from a
recording resident in HBM, and the wall time of the whole ltephy_track_push_device (prediction, host replay, copies).  Kernel times come from
torch.profiler; the cut's share of the HBM peak counts one read and one write of every cut sample.  Then the find state
(LTEPHY_TRACK_REACQUIRE): at N = 1536 and 2048 with 2 antennas, one push over 1 s of a cell whose middle 500 ms is noise (the tracker is lost
and searches about 50 windows of a frame), against the same push on the loss-free recording; the device time of the cell-search kernels per find
window, and both pushes' wall times.  Prints the device and its power limit.  Needs a GPU; there is no CPU fallback.

    python tools/track_time.py [--reps 5] [--subframes 1000]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_PEAK = 3.35e12   # H100 SXM data sheet, HBM3 bytes per second


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--subframes", type=int, default=1000)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from ltesniffer_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q))
    N, A, K = 2048, 2, args.subframes
    L = (K + 1) * 15 * N
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((A, L), dtype=torch.complex64, device="cuda", generator=g)
    trs = [capi.Tracker(N, A, 0, 100, max_subframes=K) for _ in range(args.reps + 1)]
    trs[0].push_device(x, 0)                  # warm-up
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0.record()
        for tr in trs[1:]:
            r = tr.push_device(x, 0)
        t1.record()
        torch.cuda.synchronize()
    assert len(r["sf"]) == K
    wall = t0.elapsed_time(t1) / args.reps
    dev = {}
    for e in prof.key_averages():
        for name in ("track_metric_kernel", "track_sums_kernel", "track_cut_kernel"):
            if name in e.key:
                dev[name] = dev.get(name, 0.0) + e.device_time_total / args.reps * 1e-3   # ms per push
    cut_bytes = 2 * K * A * 15 * N * 8
    t3 = dev.get("track_cut_kernel", float("nan"))
    print(json.dumps(dict(N=N, nof_rx=A, subframes=K, push_ms=round(wall, 3), kernel_ms={k: round(v, 3) for k, v in dev.items()},
                          kernels_total_ms=round(sum(dev.values()), 3), cut_hbm_share=round(cut_bytes / (t3 * 1e-3) / HBM_PEAK, 3))))
    for tr in trs:
        tr.close()
    for N in (1536, 2048):
        outage(N, args.reps)


def outage(N, reps):
    """the find state's cost: 1 s of a frame-periodic PSS / SSS cell (ref64_sync.synth), the middle 500 ms replaced by noise of the same power"""
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import ref64_sync as R
    from ltesniffer_b200 import capi
    A, SF, pci = 2, 15 * N, 17
    rng = np.random.default_rng(N)
    fr = np.stack([R.synth(N, pci, 10, rng) for _ in range(A)])
    clean = np.tile(fr, (1, 100))
    lost = clean.copy()
    lost[:, 250 * SF:750 * SF] = (rng.standard_normal((A, 500 * SF)) + 1j * rng.standard_normal((A, 500 * SF))) * np.sqrt(0.5 * np.mean(np.abs(fr) ** 2))
    out = dict(N=N, nof_rx=A, push_subframes=1000)
    for name, x in (("loss_free", clean), ("outage", lost)):
        xd = torch.from_numpy(x.astype(np.complex64)).cuda()
        trs = [capi.Tracker(N, A, pci, 0, max_subframes=1000, flags=capi.TRACK_REACQUIRE) for _ in range(reps + 1)]
        trs[0].push_device(xd, 0)           # warm-up
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0.record()
            for tr in trs[1:]:
                r = tr.push_device(xd, 0)
            t1.record()
            torch.cuda.synchronize()
        sync_ms = sum(e.device_time_total for e in prof.key_averages() if e.key.startswith("sync_")) / reps * 1e-3
        out[name] = dict(push_ms=round(t0.elapsed_time(t1) / reps, 3), subframes_cut=len(r["sf"]), finds=r["finds"])
        if r["finds"]:
            out[name]["find_device_ms_per_window"] = round(sync_ms / r["finds"], 4)
        for tr in trs:
            tr.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
