"""The ordered turns of concurrent batches (ltesniffer_b200/csrc/turn.hpp) on the CPU: tests/turn_check.cpp drives the four sections of a
sharded call from host threads -- a duplicate seq racing its owner, a stale seq, batches arriving in reverse order, batches failing before a
section, LTEPHY_SEQ_NONE -- and checks the order every section was entered in.  No GPU and no library needed."""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_turns_order_batches_and_refuse_duplicate_and_stale_seqs(tmp_path):
    exe = str(tmp_path / "turn_check")
    subprocess.run([shutil.which("g++") or "g++", "-std=c++17", "-O2", "-Wall", "-pthread", "-I", os.path.join(ROOT, "ltesniffer_b200", "csrc"),
                    "-o", exe, os.path.join(ROOT, "tests", "turn_check.cpp")], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stdout, r.stderr)
