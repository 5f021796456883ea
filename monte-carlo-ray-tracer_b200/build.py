"""Builds libmcrt_b200.so (the C-ABI product library) in-tree with nvcc for sm_90a (H100).

kernels_f64.cu is compiled with --fmad=false (parity with the reference's non-contracting CPU build);
everything else with default FMA contraction. -lineinfo keeps ncu's source page usable."""
import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
ROOT = os.path.dirname(HERE)
LIB = os.path.join(HERE, "libmcrt_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", CSRC]

UNITS = [
    ("kernels_f64.cu", ["--fmad=false"]),
    ("kernels_f32.cu", []),
    ("bvh_build.cu", ["--fmad=false"]),
    ("image.cu", ["--fmad=false"]),
    ("obj_abi.cu", ["--fmad=false"]),
    ("denoise.cu", ["--fmad=false"]),
    ("lpe.cu", []),
    ("abi.cu", []),
]


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr + "\n")
        raise RuntimeError("nvcc failed")
    return r.stdout + r.stderr


def build(force=False, verbose=False, defines=(), suffix=""):
    """defines/suffix: tuning variants, e.g. build(defines=["-DMCRT_TRACE_MINBLOCKS=3"], suffix="_t3")
    writes libmcrt_b200_t3.so (select it at run time with MCRT_LIB)."""
    global LIB
    lib = os.path.join(HERE, f"libmcrt_b200{suffix}.so")
    objdir = os.path.join(HERE, "build" + suffix)
    os.makedirs(objdir, exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "mcrt_abi.h"),
                                                              os.path.join(HERE, "host", "obj_loader.cpp"),
                                                              os.path.join(HERE, "host", "obj_loader.hpp")]
    newest = max(os.path.getmtime(d) for d in deps)
    jobs, objs = [], []
    for src, extra in UNITS:
        obj = os.path.join(objdir, src[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < newest:
            cmd = ["nvcc"] + ARCH + COMMON + list(defines) + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
            jobs.append(cmd)
    with cf.ThreadPoolExecutor(max_workers=4) as ex:
        outs = list(ex.map(_run, jobs))
    if verbose:
        for o in outs:
            sys.stderr.write(o)
    if jobs or not os.path.exists(lib):
        _run(["nvcc"] + ARCH + ["-shared", "-o", lib] + objs + ["-Xcompiler", "-pthread"])
    return lib


if __name__ == "__main__":
    defs = [a for a in sys.argv[1:] if a.startswith("-D")]
    suf = [a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--suffix=")]
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, defines=defs, suffix=suf[0] if suf else ""))
