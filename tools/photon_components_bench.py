#!/usr/bin/env python3
"""Cost of photon-mapper components on pm_hexagon_room (1920x1080, parity mode, 1e6 emissions, the pack's caustic factor,
leaf size and k): a 16-spp accumulate pass into one plane (mcrt_render_accumulate_dev) against the four component planes
(mcrt_render_accumulate_photon_components_dev), alternated, for the k-NN estimate and for the fixed-radius gather, with the
shade and k-NN stage times of stage_timing.

  python tools/photon_components_bench.py [--reps 3] [--out result.json]

Prints the card name, power limit and max SM clock read in the same call, one JSON line per run and a summary line. The
planes of every component pass are checked against the one-plane pass of the same samples (sum of planes, rtol 1e-12)."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PACK = os.path.join(ROOT, "tests", "golden", "pm_hexagon_room_64.mcrtpack")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="repetitions of each case (alternated)")
    ap.add_argument("--spp", type=int, default=16, help="samples per pixel of a pass")
    ap.add_argument("--emissions", type=float, default=1e6)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()

    import torch
    sys.path.insert(0, ROOT)
    m = importlib.import_module("monte-carlo-ray-tracer_b200")
    info = {"gpu": gpu_info(), "torch_device": torch.cuda.get_device_name(0)}
    print(json.dumps(info), flush=True)
    scene = m.Scene.from_pack(PACK)
    ep = scene.extra["photon_emit_params"]
    sqrt_spp = int(round(a.spp ** 0.5))
    cam = scene.cameras()[0].resized(1920, 1080, sqrt_spp)
    spp = sqrt_spp * sqrt_spp
    pm = m.PhotonMapper(scene, precision=m.PRECISION_F64, global_seed=0x12345678,
                        emit=dict(emissions=int(a.emissions), caustic_factor=float(ep[1]), max_photons_per_octree_leaf=int(ep[2]),
                                  k_nearest_photons=int(scene.photon_maps()[2])))
    pm.set_option("stage_timing", 1)
    n_planes = len(m.PHOTON_COMPONENT_NAMES)
    # the fixed radius: the median distance to the k-th nearest photon at 4096 photons of each map
    radii = []
    for which in (0, 1):
        pos = np.asarray(pm._maps[which]["photons"], np.float32).reshape(-1, 8)[:, 3:6].astype(np.float64)
        _, d2, cnt = pm.knn(which, pos[:: max(1, len(pos) // 4096)])
        radii.append(float(np.median(np.sqrt(np.where(np.arange(d2.shape[1])[None] < cnt[:, None], d2, 0).max(axis=1)))))
    W, H = cam.width, cam.height
    beauty = torch.zeros((H, W, 3), dtype=torch.float64, device="cuda")
    planes = torch.zeros((n_planes, H, W, 3), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()

    def run(estimate, case):
        pm.gather_radius(*(radii if estimate == "gather" else (0.0, 0.0)))
        buf = beauty if case == "beauty" else planes
        buf.zero_()
        torch.cuda.synchronize()
        if case == "beauty":
            st = pm.render_accumulate_dev(cam, buf.data_ptr(), None, 0, spp)
        else:
            st = pm.render_accumulate_components_dev(cam, buf.data_ptr(), 0, spp)
        return {"estimate": estimate, "case": case, "device_ms": st["gpu_ms_total"], "knn_ms": st["gpu_ms_knn"],
                "shade_ms": st["gpu_ms_shade"], "shadow_ms": st["gpu_ms_shadow"], "knn_queries": st["knn_queries"]}

    results, equal = {}, True
    for estimate in ("knn", "gather"):
        run(estimate, "beauty"); run(estimate, "components")     # warm-up: module load, buffers
        for _ in range(a.reps):
            for case in ("beauty", "components"):
                r = run(estimate, case)
                results.setdefault(f"{estimate}_{case}", []).append(r)
                print(json.dumps(r), flush=True)
            equal = equal and bool((planes >= 0).all()) and bool(torch.allclose(planes.sum(dim=0), beauty, rtol=1e-12,
                                                                                   atol=1e-14 * spp))
    pm.close()

    med = lambda rs, k: float(np.median([r[k] for r in rs]))
    summary = {"workload": f"pm_hexagon_room {W}x{H} {spp} spp parity, {a.emissions:.0e} emissions", **info,
               "planes": n_planes, "radii": radii, "components_equal_beauty": equal}
    for key, rs in results.items():
        summary[key] = {k: [r[k] for r in rs] for k in ("device_ms", "knn_ms", "shade_ms", "shadow_ms")}
    for estimate in ("knn", "gather"):
        b, c = results[f"{estimate}_beauty"], results[f"{estimate}_components"]
        for stage in ("device_ms", "knn_ms", "shade_ms", "shadow_ms"):
            summary[f"{estimate}_{stage}_components_over_beauty"] = med(c, stage) / med(b, stage) - 1.0
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"runs": results, "summary": summary}, f, indent=1)
    return 0 if equal else 1


if __name__ == "__main__":
    sys.exit(main())
