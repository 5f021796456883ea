#!/usr/bin/env python3
"""Adaptive against uniform sampling at equal error: the C2 workload of bench.py (hexagon_room, 1920x1080, parity
mode, 32 Mi-path pool) rendered in passes of 16 samples.

  python tools/adaptive_bench.py [--reps 2] [--pass-samples 16] [--target T] [--out result.json]

Uniform: Progressive.add to 256 spp. Its measured error E is taken between the frames of two seeds,
sqrt(sum (I1 - I2)^2 / 2 / sum I1^2). Adaptive: Progressive.render_adaptive with target T, by default the uniform
render's own two-half estimate at 256 spp (the target at which uniform sampling stops at 256 spp); its error is
measured between two seeds in the same way, so T can be adjusted until both measured errors match. Each repetition
renders uniform and adaptive for both seeds, alternated.

Reported per run: device ms (CUDA events of the wavefront passes), camera paths, wavefront iterations, the host time
per pass outside the device window (for adaptive passes it includes building and uploading the pixel list), and the
wall time of a resolve (kernel plus the frame's copy to the host). Also the kernel time of the resolve with per-tile
counts on the 1920x1080 frame (torch.profiler). Prints the card name and power limit read in the same call, one JSON
line per run and a summary line."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEEDS = (0x12345678, 0x9E3779B9)
UNIFORM_SPP = 256


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"nvidia-smi unavailable: {e}"


class Timed:
    """Progressive whose passes and resolves are timed."""

    def __init__(self, m, pt, cam):
        self.prog = m.Progressive(pt, cam)
        self.passes, self.resolve_s = [], []
        add, resolve = self.prog.add, self.prog._resolve

        def timed_add(samples):
            t0 = time.perf_counter()
            st = add(samples)
            wall = time.perf_counter() - t0
            self.passes.append({"samples": int(samples), "active": int(self.prog.active.sum()), "device_ms": st["gpu_ms_total"],
                                "host_ms": wall * 1e3 - st["gpu_ms_total"], "paths": st["paths"],
                                "iterations": st["wavefront_iterations"]})
            return st

        def timed_resolve(sums=False):
            t0 = time.perf_counter()
            fresh = self.prog._resolved is None or (sums and self.prog._resolved[3] is None)
            r = resolve(sums)
            if fresh:
                self.resolve_s.append(time.perf_counter() - t0)
            return r
        self.prog.add, self.prog._resolve = timed_add, timed_resolve

    def summary(self):
        p = self.passes
        tile_passes = [x for x in p if x["active"] < self.prog.active.size]
        full_passes = [x for x in p if x["active"] == self.prog.active.size]
        med = lambda xs: float(np.median(xs)) if xs else None
        return {"device_ms": sum(x["device_ms"] for x in p), "paths": sum(x["paths"] for x in p),
                "iterations": sum(x["iterations"] for x in p), "passes": len(p),
                "host_ms_per_full_pass": med([x["host_ms"] for x in full_passes]),
                "host_ms_per_tile_pass": med([x["host_ms"] for x in tile_passes]),
                "resolve_ms": med([s * 1e3 for s in self.resolve_s]),
                "spp_mean": sum(x["paths"] for x in p) / (self.prog.rows * self.prog.camera.width),
                "active_per_pass": [x["active"] for x in p], "estimate": self.prog.error()[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2, help="repetitions of every case (alternated)")
    ap.add_argument("--pass-samples", type=int, default=16)
    ap.add_argument("--min-samples", type=int, default=16)
    ap.add_argument("--max-samples", type=int, default=1024)
    ap.add_argument("--target", type=float, default=None,
                    help="adaptive target error (default: the uniform render's estimate at 256 spp)")
    ap.add_argument("--resolve-reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    import torch
    m = importlib.import_module("monte-carlo-ray-tracer_b200")
    info = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0)}
    print(json.dumps(info), flush=True)

    scene = m.Scene.from_pack(os.path.join(ROOT, "bench_data", "c2_hexagon_room.mcrtpack"))
    cam = scene.cameras()[0].resized(1920, 1080, 16)
    tracers = {}
    for seed in SEEDS:
        tracers[seed] = m.PathTracer(scene, precision=m.PRECISION_F64, global_seed=seed)
        tracers[seed].set_option("pool_paths", float(1 << 25))     # as bench.py: 32 Mi paths in flight

    def uniform(seed):
        t = Timed(m, tracers[seed], cam)
        for _ in range(UNIFORM_SPP // a.pass_samples):
            t.prog.add(a.pass_samples)
        t.prog.tile_sums()       # the resolve render_adaptive runs after every pass, timed once here
        return t

    def adaptive(seed, target):
        t = Timed(m, tracers[seed], cam)
        t.prog.render_adaptive(a.pass_samples, a.max_samples, target, min_samples=a.min_samples)
        return t

    def measured(f1, f2):
        return float(np.sqrt(np.sum((f1 - f2) ** 2) / 2 / np.sum(f1 ** 2)))

    warm = m.Progressive(tracers[SEEDS[0]], cam)   # warm-up: module load, buffers, both generate instantiations
    warm.add(1)
    warm.retire(np.arange(warm.active.size).reshape(warm.active.shape) % 2 == 0)
    warm.add(1)
    warm.frame()
    del warm

    runs = {"uniform": [], "adaptive": []}
    errors = {"uniform": [], "adaptive": []}
    target = a.target
    for rep in range(a.reps):
        frames = {"uniform": [], "adaptive": []}
        for seed in SEEDS:
            for case in ("uniform", "adaptive"):
                if case == "adaptive" and target is None:
                    target = runs["uniform"][0]["estimate"]
                t = uniform(seed) if case == "uniform" else adaptive(seed, target)
                r = dict(case=case, rep=rep, seed=seed, **t.summary())
                if case == "adaptive":
                    r.update(stop_reason=t.prog.stop_reason, target=target)
                runs[case].append(r)
                frames[case].append(t.prog.frame())
                print(json.dumps(r), flush=True)
                del t
        for case in frames:
            errors[case].append(measured(*frames[case]))
        print(json.dumps({"rep": rep, "measured_error": {c: errors[c][-1] for c in errors}}), flush=True)

    # kernel time of the resolve with per-tile counts on the 1920x1080 frame (sums of random tiles), from the profiler
    from torch.profiler import ProfilerActivity, profile
    W, H, pt = cam.width, cam.height, tracers[SEEDS[0]]
    A = torch.rand((H, W, 3), dtype=torch.float64, device="cuda") * 128
    B = torch.rand((H, W, 3), dtype=torch.float64, device="cuda") * 128
    out = torch.empty_like(A)
    grid = m.tile_grid(H, W, 16)
    counts = np.random.default_rng(0).integers(16, 128, grid + (2,))
    tiles, sums = (torch.empty(grid + extra, dtype=torch.float64, device="cuda") for extra in ((), (2,)))
    torch.cuda.synchronize()

    def resolve():
        return pt.progressive_resolve_tiles_dev(A.data_ptr(), None, B.data_ptr(), None, counts, W, H, 16, out.data_ptr(),
                                                tiles.data_ptr(), sums.data_ptr())
    resolve()
    t0 = time.perf_counter()
    for _ in range(a.resolve_reps):
        resolve()
    call_ms = (time.perf_counter() - t0) / a.resolve_reps * 1e3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.resolve_reps):
            resolve()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "progressive" in e.name:
            key = "k_progressive_tile_error<true>" if "tile_error" in e.name else "k_progressive_resolve<true>"
            kern.setdefault(key, []).append(e.device_time_total / 1e3)   # microseconds -> ms
    resolve_kernels = {"frame": f"{W}x{H}", "tile": 16, "call_ms": call_ms, "kernel_ms": {k: float(np.median(v)) for k, v in kern.items()}}
    for pt in tracers.values():
        pt.close()

    summary = {"workload": f"c2 hexagon_room 1920x1080 parity, passes of {a.pass_samples}, min_samples {a.min_samples}",
               **info, "uniform_spp": UNIFORM_SPP, "target": target, "measured_error": errors,
               "resolve_tiles": resolve_kernels}
    for case in runs:
        summary[case] = {k: [r[k] for r in runs[case]] for k in ("device_ms", "paths", "iterations", "passes", "spp_mean",
                                                                 "host_ms_per_full_pass", "host_ms_per_tile_pass", "resolve_ms")}
    summary["device_ms_ratio_adaptive_over_uniform"] = (float(np.median(summary["adaptive"]["device_ms"]))
                                                        / float(np.median(summary["uniform"]["device_ms"])))
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"runs": runs, "summary": summary}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
