"""Builds libltephy_b200.so (hand-written sm_90a CUDA + C++ host code) in-tree with nvcc / g++.
Used by __graft_entry__.build() and by the tests' session fixture.  No JIT cache: the .so sits next
to this file so that it travels to the GPU box with the repo snapshot.  Every source is compiled to its
own object (in parallel, only when it or a header changed), then linked."""
import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INC = os.path.join(HERE, "..", "include")
OBJ = os.path.join(HERE, "_obj")
OUT = os.path.join(HERE, "libltephy_b200.so")
COMPAT_OUT = os.path.join(HERE, "libltephy_srsran_compat.so")
SOURCES = ["k_frontend.cu", "k_viterbi.cu", "k_pdsch.cu", "k_turbo.cu", "k_pusch.cu", "k_pbch.cu", "k_sync.cu", "k_track.cu", "k_chan.cu", "ltephy_capi.cu", "sync.cu", "track.cu", "chan.cu", "scan.cu", "shard.cu", "lte_host.cpp",
           "host_search.cpp", "sinks.cpp", "harq.cpp"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-fmad=false",
              "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math,-Wall,-Wno-unused-function", "-Xptxas", "-v"]
CXX_FLAGS = ["-O3", "-g", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function"]


def nvcc_path():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found: libltephy_b200 cannot be built (there is no CPU fallback)")
    return p


def _headers():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".hpp", ".h"))] + \
           [os.path.join(INC, f) for f in os.listdir(INC)] + [os.path.abspath(__file__)]


def _sources():
    return [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def _obj_of(src):
    return os.path.join(OBJ, src + ".o")


def _obj_stale(src, hdr_time):
    o = _obj_of(src)
    if not os.path.exists(o):
        return True
    t = os.path.getmtime(o)
    return os.path.getmtime(os.path.join(CSRC, src)) > t or hdr_time > t


def stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(INC, f) for f in os.listdir(INC)]
    comp = os.path.join(HERE, "..", "compat")
    deps += [os.path.join(r, f) for r, _, fs in os.walk(comp) for f in fs]
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src):
    path = os.path.join(CSRC, src)
    if src.endswith(".cu"):
        cmd = [nvcc_path()] + NVCC_FLAGS + ["-c", "-o", _obj_of(src), path]
    else:
        cmd = [shutil.which("g++") or "g++"] + CXX_FLAGS + ["-c", "-o", _obj_of(src), path]
    r = subprocess.run(cmd, capture_output=True, text=True)
    return src, " ".join(cmd), r.returncode, r.stdout + r.stderr


def build(force=False, verbose=False):
    if not force and not stale():
        if not os.path.exists(COMPAT_OUT):
            build_compat()
        return OUT
    os.makedirs(OBJ, exist_ok=True)
    hdr_time = max(os.path.getmtime(h) for h in _headers())
    srcs = _sources()
    todo = [s for s in srcs if force or _obj_stale(s, hdr_time)]
    logs = {}
    old = os.path.join(HERE, "build.log")
    if os.path.exists(old) and not force:   # keep the ptxas -v output of the objects that are not recompiled
        cur = None
        for line in open(old):
            if line.startswith("### "):
                cur = line[4:].strip()
                logs[cur] = ""
            elif cur:
                logs[cur] += line
    with ThreadPoolExecutor(max(1, min(len(todo), os.cpu_count() or 4))) as ex:
        for src, cmd, rc, log in ex.map(_compile, todo):
            logs[src] = cmd + "\n" + log
            if rc != 0:
                raise RuntimeError("compiling %s failed:\n%s" % (src, log[-6000:]))
    cmd = [nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "--shared", "-o", OUT] + [_obj_of(s) for s in srcs] + ["-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    logs["link"] = " ".join(cmd) + "\n" + r.stdout + r.stderr
    with open(os.path.join(HERE, "build.log"), "w") as f:
        for k in srcs + ["link"]:
            if k in logs:
                f.write("### %s\n%s\n" % (k, logs[k].rstrip("\n")))
    if r.returncode != 0:
        raise RuntimeError("linking libltephy_b200.so failed:\n" + (r.stdout + r.stderr)[-6000:])
    if verbose:
        print(open(os.path.join(HERE, "build.log")).read())
    build_compat()
    return OUT


def build_compat():
    """tier-2 shim (srsRAN / FALCON names over the tier-1 C-ABI): host code only, links libltephy_b200.so"""
    cxx = shutil.which("g++") or "g++"
    comp = os.path.join(HERE, "..", "compat")
    cmd = [cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + comp, "-o", COMPAT_OUT,
           os.path.join(comp, "src", "srsran_host.cpp"), os.path.join(comp, "src", "srsran_phy.cpp"), "-L" + HERE, "-lltephy_b200", "-Wl,-rpath,$ORIGIN"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building the srsRAN compatibility shim failed:\n" + (r.stdout + r.stderr)[-4000:])
    return COMPAT_OUT


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
