#!/usr/bin/env python3
"""Cost of the photon mapper's light path expressions on pm_hexagon_room (1920x1080, parity mode, 1e6 emissions, the
pack's caustic factor, leaf size and k). For the k-NN estimate and for the fixed-radius gather, a 16-spp accumulate
pass into one plane (mcrt_render_accumulate_dev), into the four component planes
(mcrt_render_accumulate_photon_components_dev) and into the LPE planes of PM_COMPONENT_LPES(False) + "C.*"
(mcrt_render_accumulate_lpe_dev), alternated, with the shade and k-NN stage times of stage_timing. The emission pass
is timed on its own, with and without an LPE table set (the photons carry their states only with one).

  python tools/pm_lpe_bench.py [--reps 3] [--out result.json]

Prints the card name, power limit and max SM clock read in the same call, one JSON line per run and a summary line.
Every LPE pass is checked against the other passes of the same samples: its "C.*" plane against the one-plane pass
and its component expressions against the component planes, rtol 1e-12."""
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

    import time
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
    emit = dict(emissions=int(a.emissions), caustic_factor=float(ep[1]), max_photons_per_octree_leaf=int(ep[2]),
                k_nearest_photons=int(scene.photon_maps()[2]))
    pm = m.PhotonMapper(scene, precision=m.PRECISION_F64, global_seed=0x12345678, emit=emit)
    pm.set_option("stage_timing", 1)
    exprs = list(m.PM_COMPONENT_LPES(False)) + ["C.*"]

    # emission: the same pass without and with a table, alternated (wall time around a synchronising call)
    def emit_once(table):
        pm.set_light_path_expressions(exprs if table else None)
        t0 = time.perf_counter()
        pm.emit(**emit)
        ms = (time.perf_counter() - t0) * 1e3
        return {"case": "emit_lpe" if table else "emit", "wall_ms": ms, "device_ms": pm.last_stats["gpu_ms_total"],
                "build_ms": pm.last_stats["gpu_ms_knn"]}

    results = {}
    emit_once(False); emit_once(True)
    for _ in range(a.reps):
        for table in (False, True):
            r = emit_once(table)
            results.setdefault(r["case"], []).append(r)
            print(json.dumps(r), flush=True)
    assert pm.has_photon_lpe_states   # the last pass ran under the table: the LPE renders below take its maps

    radii = []
    for which in (0, 1):
        pos = np.asarray(pm._maps[which]["photons"], np.float32).reshape(-1, 8)[:, 3:6].astype(np.float64)
        _, d2, cnt = pm.knn(which, pos[:: max(1, len(pos) // 4096)])
        radii.append(float(np.median(np.sqrt(np.where(np.arange(d2.shape[1])[None] < cnt[:, None], d2, 0).max(axis=1)))))
    W, H = cam.width, cam.height
    beauty = torch.zeros((H, W, 3), dtype=torch.float64, device="cuda")
    comps = torch.zeros((4, H, W, 3), dtype=torch.float64, device="cuda")
    lpe = torch.zeros((len(exprs), H, W, 3), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()

    def run(estimate, case):
        pm.gather_radius(*(radii if estimate == "gather" else (0.0, 0.0)))
        buf = {"beauty": beauty, "components": comps, "lpe": lpe}[case]
        buf.zero_()
        torch.cuda.synchronize()
        if case == "beauty":
            st = pm.render_accumulate_dev(cam, buf.data_ptr(), None, 0, spp)
        elif case == "components":
            st = pm.render_accumulate_components_dev(cam, buf.data_ptr(), 0, spp)
        else:
            st = pm.render_accumulate_lpe_dev(cam, buf.data_ptr(), len(exprs), 0, spp)
        return {"estimate": estimate, "case": case, "device_ms": st["gpu_ms_total"], "knn_ms": st["gpu_ms_knn"],
                "shade_ms": st["gpu_ms_shade"], "shadow_ms": st["gpu_ms_shadow"], "knn_queries": st["knn_queries"]}

    cases = ("beauty", "components", "lpe")
    equal = True
    for estimate in ("knn", "gather"):
        for case in cases:
            run(estimate, case)   # warm-up: module load, buffers
        for _ in range(a.reps):
            for case in cases:
                r = run(estimate, case)
                results.setdefault(f"{estimate}_{case}", []).append(r)
                print(json.dumps(r), flush=True)
            equal = equal and bool(torch.allclose(lpe[-1], beauty, rtol=1e-12, atol=1e-14 * spp)) and \
                bool(torch.allclose(lpe[:4], comps, rtol=1e-12, atol=1e-14 * spp))
    pm.close()

    med = lambda rs, k: float(np.median([r[k] for r in rs]))
    summary = {"workload": f"pm_hexagon_room {W}x{H} {spp} spp parity, {a.emissions:.0e} emissions", **info,
               "expressions": exprs, "radii": radii, "lpe_equal_beauty_and_components": equal,
               "emit_wall_ms_median": med(results["emit"], "wall_ms"), "emit_lpe_wall_ms_median": med(results["emit_lpe"], "wall_ms"),
               "emit_device_ms_median": med(results["emit"], "device_ms"),
               "emit_lpe_device_ms_median": med(results["emit_lpe"], "device_ms")}
    for estimate in ("knn", "gather"):
        b = results[f"{estimate}_beauty"]
        for case in ("components", "lpe"):
            c = results[f"{estimate}_{case}"]
            for stage in ("device_ms", "knn_ms", "shade_ms"):
                summary[f"{estimate}_{stage}_{case}_over_beauty"] = med(c, stage) / med(b, stage) - 1.0
        summary[f"{estimate}_device_ms_median"] = {case: med(results[f"{estimate}_{case}"], "device_ms") for case in cases}
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"runs": results, "summary": summary}, f, indent=1)
    return 0 if equal else 1


if __name__ == "__main__":
    sys.exit(main())
