#!/usr/bin/env python3
"""Stage times of the C2 workload of bench.py (hexagon_room, 1920x1080, 256 spp, 32 Mi-path pool) under the wavefront's
sort settings, alternated in one process, with stage_timing on (DESIGN.md §3 and §10, item 8):

  wavefront  the default: the ray-coherence sort of every queue, k_shade walking its queue in buffer order
  classsort  + sort_shade_class = 1: k_shade walks the paths grouped by the material class of their hit
  pathorder  sort_shade = 1: k_shade walks the paths in ray-coherence order
  unsorted   sort_rays = 0: no sorting at all, so its k_extend + k_shade + k_shadow kernel times are what the same
             work costs in the order the camera generates it - the order a kernel that carries each path in
             registers would trace and shade it in

  python tools/fused_paths_bench.py [--arms wavefront,classsort,unsorted] [--reps 3] [--sqrtspp 16] [--precision f64]

Prints the card name and power limit read in the same call, one JSON line per render and a summary line per arm. Every
arm's frame is compared with the first arm's (rtol 1e-12: only the order of the film's float64 atomics differs), and the
ray counts must agree exactly."""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from aov_bench import gpu_info  # noqa: E402

_SORTS = dict(sort_rays=1, sort_shade=0, sort_shade_class=0)     # mcrt_ctx defaults (abi.cu)
ARMS = {"wavefront": _SORTS, "classsort": dict(_SORTS, sort_shade_class=1), "pathorder": dict(_SORTS, sort_shade=1),
        "unsorted": dict(_SORTS, sort_rays=0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arms", default="wavefront,classsort,unsorted")
    ap.add_argument("--reps", type=int, default=3, help="timed renders of each arm (alternated)")
    ap.add_argument("--sqrtspp", type=int, default=16, help="sqrt of the samples per pixel (16: bench.py's 256 spp)")
    ap.add_argument("--precision", default="f64", choices=["f64", "f32"])
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    arms = a.arms.split(",")
    import torch
    m = importlib.import_module("monte-carlo-ray-tracer_b200")
    info = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0)}
    print(json.dumps(info), flush=True)

    scene = m.Scene.from_pack(os.path.join(ROOT, "bench_data", "c2_hexagon_room.mcrtpack"))
    cam = scene.cameras()[0].resized(1920, 1080, a.sqrtspp)
    prec = m.PRECISION_F64 if a.precision == "f64" else m.PRECISION_F32
    pt = m.PathTracer(scene, precision=prec, global_seed=0x12345678)
    pt.set_option("pool_paths", float(1 << 25))     # as bench.py: 32 Mi paths in flight
    pt.set_option("stage_timing", 1)
    W, H = cam.width, cam.height
    frames = {arm: torch.zeros((H, W, 3), dtype=torch.float64, device="cuda") for arm in arms}

    def run(arm):
        for k, v in ARMS[arm].items():
            pt.set_option(k, v)
        st = pt.render_rows_dev(cam, frames[arm].data_ptr())
        torch.cuda.synchronize()
        kern = st["gpu_ms_extend"] + st["gpu_ms_shade"] + st["gpu_ms_shadow"] + st["gpu_ms_generate"]
        rays = st["extension_rays"] + st["shadow_rays"]
        return {"arm": arm, "device_ms": st["gpu_ms_total"], "extend_ms": st["gpu_ms_extend"], "shade_ms": st["gpu_ms_shade"],
                "shadow_ms": st["gpu_ms_shadow"], "generate_ms": st["gpu_ms_generate"],
                "staged_ms": kern, "launches": st["kernel_launches"], "rays": rays, "mray_s": rays / st["gpu_ms_total"] / 1e3,
                "counts": [st["extension_rays"], st["shadow_rays"], st["replayed_rays"], st["paths"], st["max_depth"]]}

    for arm in arms:                                # warm-up: module load, buffers
        run(arm)
    results = {arm: [] for arm in arms}
    for _ in range(a.reps):
        for arm in arms:
            r = run(arm)
            results[arm].append(r)
            print(json.dumps(r), flush=True)
    ref = frames[arms[0]].cpu().numpy()
    summary = {"info": info, "arms": {}}
    for arm in arms:
        f = frames[arm].cpu().numpy()
        rs = results[arm]
        ms = [r["device_ms"] for r in rs]
        summary["arms"][arm] = {
            "device_ms_min": min(ms), "device_ms_max": max(ms), "device_ms_mean": sum(ms) / len(ms),
            **{k: sum(r[k] for r in rs) / len(rs) for k in ("extend_ms", "shade_ms", "shadow_ms", "generate_ms")},
            "launches": rs[0]["launches"], "counts": rs[0]["counts"],
            "counts_equal_first_arm": rs[0]["counts"] == results[arms[0]][0]["counts"],
            "frame_equal_first_arm": bool(np.allclose(f, ref, rtol=1e-12, atol=0.0)),
            "frame_max_rel": float(np.max(np.abs(f - ref) / np.maximum(np.abs(ref), 1e-300))),
        }
        print(json.dumps({"summary": arm, **summary["arms"][arm]}), flush=True)
    pt.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump({"summary": summary, "runs": results}, fh, indent=1)


if __name__ == "__main__":
    main()
