#!/usr/bin/env python3
"""Random-gather bandwidth probe: builds tools/gather_probe.cu for sm_90a in a temporary directory, runs it
on GPU 0 and prints its JSON lines, preceded by one line with the card name and power limit read in the
same call.

  python tools/gather_probe.py [--gib 16] [--reps 20]

The question it answers: does a random 16- or 32-byte read cost about as much HBM time as a random
64- or 128-byte one? If records/s is about the same for every size, storing a path's fields in one
record (one line) saves time; if records/s scales inversely with size, it does not."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=16.0, help="size of the gathered array")
    ap.add_argument("--reps", type=int, default=20, help="timed launches per case")
    a = ap.parse_args()
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = f"nvidia-smi unavailable: {e}"
    print(json.dumps({"gpu": q}), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "gather_probe")
        subprocess.run(["nvcc", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                        os.path.join(HERE, "gather_probe.cu")], check=True)
        r = subprocess.run([exe, str(a.gib), str(a.reps)], text=True)
    return r.returncode


if __name__ == "__main__":
    sys.exit(main())
