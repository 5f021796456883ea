#!/usr/bin/env python3
"""Cost of light groups in the photon mapper on pm_hexagon_room (1920x1080, parity mode, 1e6 emissions, the pack's caustic
factor, leaf size and k): the photon pass (emission + octree build, which now also records and reorders each photon's light
index) of this build against a parent build, alternated; and a 16-spp accumulate pass into one plane
(mcrt_render_accumulate_dev) against the light-group planes (mcrt_render_accumulate_groups_dev, one group per light
triangle plus the sky: 3 planes), alternated, for the k-NN estimate and for the fixed-radius gather, with the k-NN stage
time (gpu_ms_knn) of stage_timing.

  python tools/photon_light_groups_bench.py [--reps 3] [--parent-tree DIR] [--out result.json]

DIR: a built checkout of the parent commit; its photon pass runs in a subprocess with its own package. Prints the card name
and power limit read in the same call, one JSON line per run and a summary line. The planes of every groups pass are checked
against the one-plane pass of the same samples (sum of planes, rtol 1e-12)."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PACK = os.path.join(ROOT, "tests", "golden", "pm_hexagon_room_64.mcrtpack")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"nvidia-smi unavailable: {e}"


def package(tree):
    sys.path.insert(0, tree)
    return importlib.import_module("monte-carlo-ray-tracer_b200")


def emit_args(scene, emissions):
    ep = scene.extra["photon_emit_params"]
    return dict(emissions=int(emissions), caustic_factor=float(ep[1]), max_photons_per_octree_leaf=int(ep[2]),
                k_nearest_photons=int(scene.photon_maps()[2]))


def photon_pass(tree, emissions, reps):
    """Child: the photon pass of the package in `tree`, once to warm up, then `reps` times. -> JSON line per run."""
    m = package(tree)
    scene = m.Scene.from_pack(PACK)
    pm = m.PhotonMapper(scene, precision=m.PRECISION_F64, global_seed=0x12345678, emit=emit_args(scene, emissions))
    for _ in range(reps):
        t0 = time.perf_counter()
        n = pm.emit(**emit_args(scene, emissions))           # returns after the octree build has synchronised
        wall = (time.perf_counter() - t0) * 1e3
        print(json.dumps({"tree": tree, "photon_pass_ms": wall, "emit_ms": pm.last_stats["gpu_ms_total"],
                          "build_ms": pm.last_stats["gpu_ms_knn"], "photons": list(n)}), flush=True)
    pm.close()


def run_photon_pass(tree, emissions, reps):
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--photon-pass", tree, "--emissions", str(emissions),
                          "--reps", str(reps)], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError(out.stdout + out.stderr)
    return [json.loads(l) for l in out.stdout.splitlines() if l.startswith("{")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="repetitions of each case (alternated)")
    ap.add_argument("--spp", type=int, default=16, help="samples per pixel of a pass")
    ap.add_argument("--emissions", type=float, default=1e6)
    ap.add_argument("--parent-tree", default=None, help="built checkout of the parent commit (photon pass comparison)")
    ap.add_argument("--photon-pass", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    if a.photon_pass:
        photon_pass(a.photon_pass, int(a.emissions), a.reps)
        return 0

    info = {"gpu": gpu_info()}
    print(json.dumps(info), flush=True)
    # photon pass, alternated with the parent build (each run a process of its own, 2 timed passes after a warm-up)
    passes = {"this": [], "parent": []}
    for _ in range(a.reps):
        for case, tree in (("this", ROOT), ("parent", a.parent_tree)):
            if tree is None:
                continue
            for r in run_photon_pass(tree, int(a.emissions), 2):
                r["case"] = case
                passes[case].append(r)
                print(json.dumps(r), flush=True)

    import torch
    m = package(ROOT)
    info["torch_device"] = torch.cuda.get_device_name(0)
    scene = m.Scene.from_pack(PACK)
    sqrt_spp = int(round(a.spp ** 0.5))
    cam = scene.cameras()[0].resized(1920, 1080, sqrt_spp)
    spp = sqrt_spp * sqrt_spp
    pm = m.PhotonMapper(scene, precision=m.PRECISION_F64, global_seed=0x12345678, emit=emit_args(scene, a.emissions))
    pm.set_option("stage_timing", 1)
    ids = np.arange(scene.n_lights, dtype=np.uint32)   # one group per light triangle
    n_planes = len(ids) + 1
    pm.set_light_groups(ids)
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
            st = pm.render_accumulate_groups_dev(cam, buf.data_ptr(), n_planes, 0, spp)
        return {"estimate": estimate, "case": case, "device_ms": st["gpu_ms_total"], "knn_ms": st["gpu_ms_knn"],
                "shade_ms": st["gpu_ms_shade"], "knn_queries": st["knn_queries"]}

    results, equal = {}, True
    for estimate in ("knn", "gather"):
        run(estimate, "beauty"); run(estimate, "groups")          # warm-up: module load, buffers
        for _ in range(a.reps):
            for case in ("beauty", "groups"):
                r = run(estimate, case)
                results.setdefault(f"{estimate}_{case}", []).append(r)
                print(json.dumps(r), flush=True)
            total = planes.sum(dim=0)
            equal = equal and bool(torch.allclose(total, beauty, rtol=1e-12, atol=1e-14 * spp))
    pm.close()

    med = lambda rs, k: float(np.median([r[k] for r in rs]))
    summary = {"workload": f"pm_hexagon_room {W}x{H} {spp} spp parity, {a.emissions:.0e} emissions", **info,
               "planes": n_planes, "radii": radii, "groups_equal_beauty": equal}
    for case, rs in passes.items():
        if rs:
            summary[f"photon_pass_{case}"] = {k: [r[k] for r in rs] for k in ("photon_pass_ms", "emit_ms", "build_ms")}
    for key, rs in results.items():
        summary[key] = {k: [r[k] for r in rs] for k in ("device_ms", "knn_ms", "shade_ms")}
    for estimate in ("knn", "gather"):
        b, g = results[f"{estimate}_beauty"], results[f"{estimate}_groups"]
        summary[f"{estimate}_stage_groups_over_beauty"] = med(g, "knn_ms") / med(b, "knn_ms") - 1.0
        summary[f"{estimate}_pass_groups_over_beauty"] = med(g, "device_ms") / med(b, "device_ms") - 1.0
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"photon_pass": passes, "runs": results, "summary": summary}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
