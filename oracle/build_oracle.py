#!/usr/bin/env python3
"""ORACLE / TEST INFRASTRUCTURE - builds oracle/_build/libmcrt_oracle.so, the scalar float64 CPU
restatement (oracle/mcrt_oracle.cpp). -ffp-contract=off: the reference build never contracts to FMA."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "_build", "libmcrt_oracle.so")


def build(force=False):
    src = os.path.join(HERE, "mcrt_oracle.cpp")
    hdr = os.path.join(ROOT, "include", "mcrt_abi.h")
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I", os.path.join(ROOT, "include"),
                               src, "-o", LIB])
    return LIB


if __name__ == "__main__":
    print(build(force=True))
