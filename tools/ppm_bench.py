#!/usr/bin/env python3
"""Cost of a progressive photon mapping pass: pm_hexagon_room_64 resized to 1920x1080, parity mode, passes of
--spp samples with a new photon map of 1e5 or 1e6 emissions each (ProgressivePhotonMapping.add). Per pass it reports
the photon pass (emission wavefront + octree build, device ms), the render (device ms) with its photon-lookup stage
(gpu_ms_knn: k_gather), and the camera-path rate. The k-NN estimate (k_knn) renders the same samples on the same
map for comparison. Stage times come from CUDA events between the stages (stage_timing), which add a little time.

  python tools/ppm_bench.py [--passes 4] [--spp 4] [--out result.json]

Prints the card name and power limit read in the same call, one JSON line per pass and a summary line."""
import argparse
import importlib
import json
import os
import subprocess
import sys

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
    ap.add_argument("--passes", type=int, default=4)
    ap.add_argument("--spp", type=int, default=4, help="samples per pixel of each pass")
    ap.add_argument("--emissions", type=float, nargs="+", default=[1e5, 1e6])
    ap.add_argument("--out", default=None, help="also write the summary as JSON here")
    a = ap.parse_args()
    import torch
    m = importlib.import_module("monte-carlo-ray-tracer_b200")
    info = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0)}
    print(json.dumps(info), flush=True)

    scene = m.Scene.from_pack(os.path.join(ROOT, "tests", "golden", "pm_hexagon_room_64.mcrtpack"))
    ep = scene.extra["photon_emit_params"]
    cf, leaf = float(ep[1]), int(ep[2])
    cam = scene.cameras()[0].resized(1920, 1080)
    summary = {"workload": f"pm_hexagon_room_64 1920x1080, {a.spp} spp per pass, parity", **info, "cases": {}}
    for emissions in a.emissions:
        pm = m.PhotonMapper(scene, precision=m.PRECISION_F64)
        pm.set_option("stage_timing", 1.0)
        run = m.ProgressivePhotonMapping(pm, cam, int(emissions), cf, leaf)
        run.add(a.spp)   # warm-up: module load, buffers of every size
        rows = []
        for _ in range(a.passes):
            i = run.passes
            run._emit(i)
            emit = dict(pm.last_stats)
            pm.gather_radius(*run.pass_radii(i))
            # the k-NN estimate on the same map and samples, rendered into a scratch frame
            scratch = m.Progressive(pm, cam)
            pm.gather_radius(0, 0)
            knn_on_map = scratch.add(a.spp)
            pm.gather_radius(*run.pass_radii(i))
            del scratch
            st = m.Progressive.add(run, a.spp)   # the pass itself, on the map emitted above
            rays = st["extension_rays"] + st["shadow_rays"]
            r = {"emissions": int(emissions), "pass": i, "photons": list(pm.n_photons),
                 "emit_build_ms": emit["gpu_ms_total"] + emit["gpu_ms_knn"], "emit_ms": emit["gpu_ms_total"],
                 "build_ms": emit["gpu_ms_knn"], "render_ms": st["gpu_ms_total"], "gather_ms": st["gpu_ms_knn"],
                 "knn_render_ms": knn_on_map["gpu_ms_total"], "knn_ms": knn_on_map["gpu_ms_knn"],
                 "mray_s": rays / st["gpu_ms_total"] / 1e3, "radii": list(run.pass_radii(i))}
            rows.append(r)
            print(json.dumps(r), flush=True)
        pm.close()
        summary["cases"][str(int(emissions))] = {k: float(np.median([r[k] for r in rows]))
                                                 for k in ("emit_build_ms", "emit_ms", "build_ms", "render_ms", "gather_ms",
                                                           "knn_render_ms", "knn_ms", "mray_s")}
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
