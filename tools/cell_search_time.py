"""Device time of ltephy_cell_search_device on recordings resident in HBM: 40 ms and 1 s, 1 and 2 antennas, N = 2048 and 1536.  Times with CUDA
events after a warm-up, and prints the device, its power limit, the real-time factor (recording length / search time) and the share of the FP32
bound from the coarse search's operation count (8 non-fused FP32 operations per complex MAC, 4 per energy term, 3 replicas).
Needs a GPU; there is no CPU fallback.

    python tools/cell_search_time.py [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP32_PEAK = 67e12   # H100 SXM data sheet, dense FP32, at up to 700 W


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch
    from ltesniffer_b200 import capi
    if not torch.cuda.is_available():
        sys.exit("no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q))
    g = torch.Generator(device="cuda").manual_seed(1)
    for N in (2048, 1536):
        for ms in (40, 1000):
            for A in (1, 2):
                L = ms * 15 * N
                x = torch.randn((A, L), dtype=torch.complex64, device="cuda", generator=g)
                cs = capi.CellSearch(N, A, L)
                for _ in range(2):
                    cs.search_device(x)
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(args.reps):
                    cs.search_device(x)
                t1.record()
                torch.cuda.synchronize()
                t = t0.elapsed_time(t1) / args.reps * 1e-3
                D = N // 128
                J = (L - N) // D + 1
                flops = J * N * A * (3 * 8 + 4)
                print(json.dumps(dict(N=N, capture_ms=ms, nof_rx=A, search_ms=round(t * 1e3, 3), realtime_factor=round(ms * 1e-3 / t, 1),
                                      coarse_gflop=round(flops / 1e9, 2), fp32_share=round(flops / FP32_PEAK / t, 3))))
                cs.close()
                del x


if __name__ == "__main__":
    main()
