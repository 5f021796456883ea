#!/usr/bin/env python3
"""Cost of light-path AOVs on the C2 workload of bench.py (hexagon_room, 1920x1080, parity mode, 32 Mi-path pool): device
time of a 16-spp accumulate pass into one plane (mcrt_render_accumulate_dev) and into the 8 AOV planes
(mcrt_render_accumulate_aovs_dev), alternated, with the stage times of stage_timing; and the combine kernel
(mcrt_light_groups_combine_dev) on the 8 planes of 1080p.

  python tools/aov_bench.py [--reps 2] [--combine-reps 200] [--out result.json]

Prints the card name and power limit read in the same call, one JSON line per pass and a summary line. The planes of every
AOV pass are checked against the one-plane pass of the same samples (sum of planes, rtol 1e-12)."""
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


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2, help="repetitions of each case (alternated)")
    ap.add_argument("--spp", type=int, default=16, help="samples per pixel of a pass")
    ap.add_argument("--combine-reps", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    import torch
    m = importlib.import_module("monte-carlo-ray-tracer_b200")
    info = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0)}
    print(json.dumps(info), flush=True)

    scene = m.Scene.from_pack(os.path.join(ROOT, "bench_data", "c2_hexagon_room.mcrtpack"))
    cam = scene.cameras()[0].resized(1920, 1080, 4)
    pt = m.PathTracer(scene, precision=m.PRECISION_F64, global_seed=0x12345678)
    pt.set_option("pool_paths", float(1 << 25))     # as bench.py: 32 Mi paths in flight
    pt.set_option("stage_timing", 1)
    n_planes = len(m.AOV_NAMES)
    W, H = cam.width, cam.height
    beauty = torch.zeros((H, W, 3), dtype=torch.float64, device="cuda")
    planes = torch.zeros((n_planes, H, W, 3), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()

    def run(case):
        buf = beauty if case == "beauty" else planes
        buf.zero_()
        torch.cuda.synchronize()
        if case == "beauty":
            st = pt.render_accumulate_dev(cam, buf.data_ptr(), None, 0, a.spp)
        else:
            st = pt.render_accumulate_aovs_dev(cam, buf.data_ptr(), 0, a.spp)
        return {"case": case, "device_ms": st["gpu_ms_total"], "shade_ms": st["gpu_ms_shade"], "shadow_ms": st["gpu_ms_shadow"],
                "extend_ms": st["gpu_ms_extend"], "rays": st["extension_rays"] + st["shadow_rays"],
                "mray_s": (st["extension_rays"] + st["shadow_rays"]) / st["gpu_ms_total"] / 1e3}

    run("beauty"); run("aovs")                      # warm-up: module load, buffers
    results = {"beauty": [], "aovs": []}
    equal = True
    for _ in range(a.reps):
        for case in ("beauty", "aovs"):
            r = run(case)
            results[case].append(r)
            print(json.dumps(r), flush=True)
        total = m.light_groups_combine(planes.cpu().numpy(), np.ones(n_planes))
        equal = equal and bool(np.allclose(total, beauty.cpu().numpy(), rtol=1e-12, atol=1e-14 * a.spp))
    pt.set_option("stage_timing", 0)

    # combine kernel: the 8 planes of the 1080p frame in, one frame out
    rnd = torch.rand((n_planes, H, W, 3), dtype=torch.float64, device="cuda")
    out = torch.empty((H, W, 3), dtype=torch.float64, device="cuda")
    w = np.linspace(0.5, 2.0, 3 * n_planes).reshape(n_planes, 3)
    torch.cuda.synchronize()

    def combine():
        pt.light_groups_combine_dev(rnd.data_ptr(), n_planes, out.numel(), w, out.data_ptr())
    combine()
    t0 = time.perf_counter()
    for _ in range(a.combine_reps):
        combine()
    call_ms = (time.perf_counter() - t0) / a.combine_reps * 1e3
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.combine_reps):
            combine()
        torch.cuda.synchronize()
    kern = [e.device_time_total / 1e3 for e in prof.events() if e.device_type.name == "CUDA" and "light_groups_combine" in e.name]
    kernel_ms = float(np.median(kern)) if kern else float("nan")
    bytes_moved = (n_planes + 1) * H * W * 3 * 8    # every plane read once, the frame written once
    pt.close()

    def stat(case, k):
        return [r[k] for r in results[case]]
    summary = {"workload": f"c2 hexagon_room {W}x{H} {a.spp} spp parity, 32 Mi-path pool", **info,
               "planes": n_planes, "aovs_equal_beauty": equal, "plane_mb_per_half": n_planes * H * W * 3 * 8 / 1e6}
    for case in ("beauty", "aovs"):
        summary[case] = {k: stat(case, k) for k in ("device_ms", "shade_ms", "shadow_ms", "extend_ms", "mray_s")}
    summary["aovs_over_beauty"] = float(np.median(stat("aovs", "device_ms")) / np.median(stat("beauty", "device_ms")) - 1.0)
    summary["combine"] = {"frame": f"{W}x{H}", "planes": n_planes, "call_ms": call_ms, "kernel_ms": kernel_ms,
                          "kernel_launches": len(kern), "gb_s": bytes_moved / (kernel_ms * 1e-3) / 1e9}
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"runs": results, "summary": summary}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
