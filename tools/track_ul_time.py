"""Cost of the uplink carrier in the tracker and in the uplink decoder, at N = 2048 (100 PRB) with one downlink antenna:
  * a 1000-subframe push, ltephy_track_push_device (DL only) against ltephy_track_push_ul_device (DL + UL), called through the C entry points
    (the binding's Tracker copies the cuts into torch tensors, which is not the tracker's cost): push_ms is the host wall time of the call, which
    blocks until the cut is complete (prediction, host replay of the rule, table building, copies and kernels), kernel_ms the device time per kernel from
    torch.profiler, and the UL cut's share of the HBM peak (one read and one write of every cut sample);
  * ltephy_submit_ul_device against ltephy_submit_ul (pinned host memory) on the same 1000 subframes, without grants: the UL OFDM and, for the
    host entry point, the copy of the samples; timed with CUDA events around submit + ltephy_get_ul.
Prints the device and its power limit.  Needs a GPU; there is no CPU fallback.

    python tools/track_ul_time.py [--reps 6] [--subframes 1000]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12   # H100 SXM data sheet, HBM3 bytes per second


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--subframes", type=int, default=1000)
    args = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from ltesniffer_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q))
    N, K, R = 2048, args.subframes, args.reps
    SF = 15 * N
    L = (K + 1) * SF
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((1, L), dtype=torch.complex64, device="cuda", generator=g)
    xu = torch.randn(L, dtype=torch.complex64, device="cuda", generator=g)
    out = dict(N=N, nof_rx=1, subframes=K)
    for mode in ("dl", "dl_ul"):
        ul = dict(cfo_ratio=1747.5 / 1842.5, ul_offset=N) if mode == "dl_ul" else None
        trs = [capi.Tracker(N, 1, 0, 100, max_subframes=K, ul=ul) for _ in range(R + 1)]
        o, u = capi.TrackOut(), C.c_void_p()

        def push(tr):
            if ul:
                r = tr.L.ltephy_track_push_ul_device(tr.h, C.c_void_p(x.data_ptr()), C.c_void_p(xu.data_ptr()), 0, L, C.byref(o), C.byref(u))
            else:
                r = tr.L.ltephy_track_push_device(tr.h, C.c_void_p(x.data_ptr()), 0, L, C.byref(o))
            assert r == 0, tr.L.ltephy_last_error()
            return o.nof_subframes
        push(trs[0])                                     # warm-up
        torch.cuda.synchronize()
        wall = []
        for tr in trs[1:R // 2 + 1]:                     # wall time with the profiler off
            t = time.perf_counter()
            nsf = push(tr)
            wall.append((time.perf_counter() - t) * 1e3)
        assert nsf == K, nsf
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for tr in trs[R // 2 + 1:]:
                push(tr)
            torch.cuda.synchronize()
        nprof = R - R // 2
        dev = {}
        for e in prof.key_averages():
            for name in ("track_metric_kernel", "track_sums_kernel", "track_cut_kernel"):
                if name in e.key:
                    dev[name] = dev.get(name, 0.0) + e.device_time_total / nprof * 1e-3   # ms per push
        out[mode] = dict(push_ms=round(float(np.median(wall)), 3), kernel_ms={k: round(v, 3) for k, v in dev.items()},
                         kernels_total_ms=round(sum(dev.values()), 3))
        for tr in trs:
            tr.close()
    # the UL cut is the second half of the cut kernel's time in dl_ul (both cuts move the same bytes with one DL antenna)
    ul_cut = out["dl_ul"]["kernel_ms"]["track_cut_kernel"] - out["dl"]["kernel_ms"]["track_cut_kernel"]
    out["ul_cut_ms"] = round(ul_cut, 3)
    out["ul_cut_hbm_share"] = round(2 * K * SF * 8 / (ul_cut * 1e-3) / HBM_PEAK, 3) if ul_cut > 0 else None
    # uplink decoder: host against device samples
    phy = capi.LtePhy(100, 1, 0, 1, max_subframes=K, symbol_sz=N)
    phy.set_ul_cfg()
    tti = np.arange(K, dtype=np.uint32)
    dev_iq = xu[:K * SF].reshape(K, SF).contiguous()
    host_iq = dev_iq.cpu().pin_memory()
    host_np = host_iq.numpy()
    ms = {}
    for name, run in (("submit_ul", lambda: phy.decode_ul(host_np, tti, [])), ("submit_ul_device", lambda: phy.decode_ul_device(dev_iq, tti, []))):
        run()
        torch.cuda.synchronize()
        t = []
        for _ in range(R):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            run()
            t1.record()
            torch.cuda.synchronize()
            t.append(t0.elapsed_time(t1))
        ms[name] = round(float(np.median(t)), 3)
    phy.close()
    out["ul_decode_ms"] = ms
    print(json.dumps(out))


if __name__ == "__main__":
    main()
