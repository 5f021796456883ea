#!/usr/bin/env python3
"""Cost of light path expressions on the C2 workload of bench.py (hexagon_room, 1920x1080, parity mode, 32 Mi-path pool):
device time of a 16-spp accumulate pass three ways, alternated - the beauty frame (mcrt_render_accumulate_dev), the 8
AOV planes (mcrt_render_accumulate_aovs_dev) and the LPE render of the 8 AOV expressions plus "C.*"
(mcrt_render_accumulate_lpe_dev) - with the stage times of stage_timing.

  python tools/lpe_bench.py [--reps 2] [--spp 16] [--out result.json]

Prints the card name and power limit read in the same call, one JSON line per pass and a summary line. Every LPE pass is
checked against the AOV and beauty passes of the same samples (rtol 1e-12)."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2, help="repetitions of each case (alternated)")
    ap.add_argument("--spp", type=int, default=16, help="samples per pixel of a pass")
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
    exprs = list(m.AOV_LPES) + ["C.*"]
    pt.set_light_path_expressions(exprs)
    W, H = cam.width, cam.height
    bufs = {"beauty": torch.zeros((H, W, 3), dtype=torch.float64, device="cuda"),
            "aovs": torch.zeros((len(m.AOV_NAMES), H, W, 3), dtype=torch.float64, device="cuda"),
            "lpe": torch.zeros((len(exprs), H, W, 3), dtype=torch.float64, device="cuda")}
    torch.cuda.synchronize()

    def run(case):
        buf = bufs[case]
        buf.zero_()
        torch.cuda.synchronize()
        if case == "beauty":
            st = pt.render_accumulate_dev(cam, buf.data_ptr(), None, 0, a.spp)
        elif case == "aovs":
            st = pt.render_accumulate_aovs_dev(cam, buf.data_ptr(), 0, a.spp)
        else:
            st = pt.render_accumulate_lpe_dev(cam, buf.data_ptr(), len(exprs), 0, a.spp)
        return {"case": case, "device_ms": st["gpu_ms_total"], "shade_ms": st["gpu_ms_shade"], "shadow_ms": st["gpu_ms_shadow"],
                "extend_ms": st["gpu_ms_extend"], "rays": st["extension_rays"] + st["shadow_rays"],
                "mray_s": (st["extension_rays"] + st["shadow_rays"]) / st["gpu_ms_total"] / 1e3}

    cases = ("beauty", "aovs", "lpe")
    for c in cases:                                  # warm-up: module load, buffers
        run(c)
    results = {c: [] for c in cases}
    equal = True
    for _ in range(a.reps):
        for c in cases:
            r = run(c)
            results[c].append(r)
            print(json.dumps(r), flush=True)
        lpe = bufs["lpe"].cpu().numpy()
        equal = equal and bool(np.allclose(lpe[:8], bufs["aovs"].cpu().numpy(), rtol=1e-12, atol=1e-14 * a.spp))
        equal = equal and bool(np.allclose(lpe[8], bufs["beauty"].cpu().numpy(), rtol=1e-12, atol=1e-14 * a.spp))
        equal = equal and len({results[c][-1]["rays"] for c in cases}) == 1
    pt.set_option("stage_timing", 0)
    pt.close()

    def stat(case, k):
        return [r[k] for r in results[case]]
    summary = {"workload": f"c2 hexagon_room {W}x{H} {a.spp} spp parity, 32 Mi-path pool", **info,
               "expressions": exprs, "lpe_equal_aovs_and_beauty": equal}
    for c in cases:
        summary[c] = {k: stat(c, k) for k in ("device_ms", "shade_ms", "shadow_ms", "extend_ms", "mray_s")}
    base = np.median(stat("beauty", "device_ms"))
    summary["aovs_over_beauty"] = float(np.median(stat("aovs", "device_ms")) / base - 1.0)
    summary["lpe_over_beauty"] = float(np.median(stat("lpe", "device_ms")) / base - 1.0)
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"runs": results, "summary": summary}, f, indent=1)
    return 0 if equal else 1


if __name__ == "__main__":
    sys.exit(main())
