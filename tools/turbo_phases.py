"""Where a code-block pair spends its time inside turbo_kernel: the kernel's per-phase clock64() counters (k_turbo.cu, compiled in with
-DLTEPHY_TURBO_PHASES) summed over every CTA of
  * one cfg-2 step (bench.generate_capture, 1000 subframes through ltephy_decode_subframes on one pipeline), and
  * the cfg-4 sub-record shape (26 000 code blocks of K = 5824, 8 fixed iterations, no CRC).
The instrumented kernel is built into a shared object of its own in a temporary directory (k_turbo.cu recompiled with the macro, the other
objects as ltesniffer_b200/build.py made them); the normal library is not replaced.  The counters are thread 0's clock between two marks,
so a phase includes the barrier that ends it.  Needs a GPU and fails without one.  Prints one JSON object.
usage: python tools/turbo_phases.py [--batch N]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import bench  # noqa: E402
from ltesniffer_b200 import build as B  # noqa: E402

PHASES = ["queue", "staging", "btail", "natural", "interleaved", "crc", "emit"]   # the PH_* enum of k_turbo.cu
TRELLIS = ("natural", "interleaved")


def build_instrumented(out_dir):
    B.build()                                                    # the other objects, if they are not there yet
    obj = os.path.join(out_dir, "k_turbo_phases.o")
    so = os.path.join(out_dir, "libltephy_b200_phases.so")
    nvcc = B.nvcc_path()
    subprocess.run([nvcc] + B.NVCC_FLAGS + ["-DLTEPHY_TURBO_PHASES", "-c", "-o", obj, os.path.join(B.CSRC, "k_turbo.cu")], check=True,
                   capture_output=True)
    objs = [obj if s == "k_turbo.cu" else B._obj_of(s) for s in B._sources()]
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "--shared", "-o", so] + objs + ["-ldl"], check=True, capture_output=True)
    return so


def shares(cyc):
    tot = float(sum(cyc))
    out = {"cycles": int(tot), "share": {p: round(c / tot, 4) for p, c in zip(PHASES, cyc)}}
    out["non_trellis_share"] = round(1.0 - sum(out["share"][p] for p in TRELLIS), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("turbo_phases.py measures on the GPU: no CUDA device found")
    from ltesniffer_b200 import capi
    tmp = tempfile.TemporaryDirectory()
    capi.LIB_PATH = build_instrumented(tmp.name)
    L = capi.load_library(build_if_missing=False)
    L.ltephy_turbo_phases.argtypes = [C.c_void_p, C.c_int]

    def read(reset=1):
        v = (C.c_ulonglong * len(PHASES))()
        if L.ltephy_turbo_phases(v, reset) != len(PHASES):
            raise RuntimeError("ltephy_turbo_phases failed")
        return list(v)

    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit_max_sm_clock": q.strip().splitlines()[0] if q.strip() else None,
           "note": "clock64() of thread 0 between marks, summed over all CTAs; a phase includes the barrier that ends it"}

    cell, iq = bench.generate_capture(args.batch, min(bench.effective_cores(), 16))
    tti = np.arange(args.batch, dtype=np.uint32)
    phy = capi.LtePhy(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx, max_subframes=args.batch, turbo_max_iter=8, flags=capi.FLAG_SKIP_LOW_POWER)
    srch = capi.Search(cell.nof_prb, cell.nof_ports, cell.cell_id, cell.nof_rx)
    capi.decode_subframes(phy, srch, iq, tti)                    # warm-up: tables, pools
    read()
    capi.decode_subframes(phy, srch, iq, tti)
    out["cfg2_step"] = dict(shares(read()), subframes=args.batch)

    K, ncb = 5824, 13 * 2000
    d = np.random.default_rng(4).integers(-40, 41, size=(ncb, 3 * (K + 4)), dtype=np.int16)
    phy.turbo_batch(d, K, 8, 0)
    read()
    phy.turbo_batch(d, K, 8, 0)
    out["cfg4_turbo_fixed8"] = dict(shares(read()), K=K, code_blocks=ncb, kernel_ms=phy.timing()[2])
    phy.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
