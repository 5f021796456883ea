#!/usr/bin/env python3
"""Cost of rendering in progressive passes: the C2 workload of bench.py (hexagon_room, 1920x1080, 256 spp, parity
mode) rendered one-shot and as 1x256, 4x64, 16x16 and 64x4 passes (Progressive.add), each repetition of the cases
alternated in one call. Every pass drains the wavefront's tail before the next starts, so small passes cost something;
this measures how much. Also times the resolve + noise-estimate kernel on the 1920x1080 frame.

  python tools/progressive_bench.py [--reps 2] [--out result.json]

Prints one JSON line per case and a summary line, preceded by the card name and power limit read in the same call.
Rates are camera-path rays (extension + shadow) over the summed device time of the passes (CUDA events)."""
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

CASES = [("one_shot", None), ("1x256", [256]), ("4x64", [64] * 4), ("16x16", [16] * 16), ("64x4", [4] * 64)]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2, help="repetitions of every case (alternated)")
    ap.add_argument("--resolve-reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    import torch
    m = importlib.import_module("monte-carlo-ray-tracer_b200")
    info = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0)}
    print(json.dumps(info), flush=True)

    scene = m.Scene.from_pack(os.path.join(ROOT, "bench_data", "c2_hexagon_room.mcrtpack"))
    cam = scene.cameras()[0].resized(1920, 1080, 16)
    pt = m.PathTracer(scene, precision=m.PRECISION_F64, global_seed=0x12345678)
    pt.set_option("pool_paths", float(1 << 25))     # as bench.py: 32 Mi paths in flight
    W, H, n = cam.width, cam.height, cam.sqrtspp ** 2
    one = torch.empty((H, W, 3), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()

    def run(passes):
        t0 = time.perf_counter()
        if passes is None:
            st = pt.render_rows_dev(cam, one.data_ptr())
            sts, frame = [st], None
        else:
            prog = m.Progressive(pt, cam)
            sts = [prog.add(s) for s in passes]
            frame = prog
        wall = time.perf_counter() - t0
        ms = sum(s["gpu_ms_total"] for s in sts)
        rays = sum(s["extension_rays"] + s["shadow_rays"] for s in sts)
        return {"device_ms": ms, "wall_s": wall, "rays": rays, "paths": sum(s["paths"] for s in sts),
                "iterations": sum(s["wavefront_iterations"] for s in sts), "mray_s": rays / ms / 1e3}, frame

    run([1])                                        # warm-up: module load, buffers of every size
    results = {name: [] for name, _ in CASES}
    equal = {}
    for _ in range(a.reps):
        for name, passes in CASES:
            r, prog = run(passes)
            results[name].append(r)
            if prog is not None:
                frame = prog.frame()
                ref = one.cpu().numpy()
                equal[name] = bool(np.allclose(frame, ref, rtol=1e-12, atol=1e-14))
                r["frame_error"] = prog.error()[0]
            print(json.dumps(dict(case=name, **r)), flush=True)

    # resolve + noise estimate of the full frame (two halves of sums), kernel time from the profiler
    A = torch.rand((H, W, 3), dtype=torch.float64, device="cuda") * 128
    B = torch.rand((H, W, 3), dtype=torch.float64, device="cuda") * 128
    out = torch.empty_like(A)
    tiles = torch.empty(((H + 15) // 16, (W + 15) // 16), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()

    def resolve():
        return pt.progressive_resolve_dev(A.data_ptr(), None, 128, B.data_ptr(), None, 128, W, H, 16, out.data_ptr(), tiles.data_ptr())
    resolve()
    t0 = time.perf_counter()
    for _ in range(a.resolve_reps):
        resolve()
    call_ms = (time.perf_counter() - t0) / a.resolve_reps * 1e3
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.resolve_reps):
            resolve()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "progressive" in e.name:
            key = "k_progressive_tile_error" if "tile_error" in e.name else "k_progressive_resolve"
            kern.setdefault(key, []).append(e.device_time_total / 1e3)   # microseconds -> ms
    kernel_ms = {k: float(np.median(v)) for k, v in kern.items()}
    bytes_moved = H * W * (3 * 8 * 3)                # read A and B, write the frame
    pt.close()

    best_one = min(r["device_ms"] for r in results["one_shot"])
    summary = {"workload": "c2 hexagon_room 1920x1080 256 spp parity", **info, "cases": {}}
    for name, _ in CASES:
        ms = [r["device_ms"] for r in results[name]]
        summary["cases"][name] = {"device_ms": ms, "mray_s": [r["mray_s"] for r in results[name]],
                                  "overhead_vs_one_shot": [x / best_one - 1.0 for x in ms],
                                  "iterations": results[name][0]["iterations"], "equals_one_shot": equal.get(name, True),
                                  "frame_error": results[name][0].get("frame_error")}
    summary["resolve"] = {"frame": f"{W}x{H}", "tile": 16, "call_ms": call_ms, "kernel_ms": kernel_ms,
                          "resolve_gb_s": bytes_moved / (kernel_ms.get("k_progressive_resolve", float("nan")) * 1e-3) / 1e9}
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"runs": results, "summary": summary}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
