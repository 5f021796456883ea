#!/usr/bin/env python3
"""Cost and benefit of denoising film planes with the beauty frame's weights (mcrt_denoise_planes_dev) on the C2
workload of bench.py (hexagon_room, 1920x1080, parity mode), default filter parameters, 8 feature samples.

  python tools/denoise_planes_bench.py [--reps 20] [--ref-spp 1024] [--planes 1,4,8,16,31] [--no-quality] [--out r.json]

Time: CUDA events around each call (the library synchronises its stream inside the call), median of --reps, for
mcrt_denoise_dev on the beauty frame and mcrt_denoise_planes_dev on P planes. The planes are the 8 AOV planes of a
16-spp render, repeated to make P; the cost does not depend on their content. The weight and plane passes are timed
per kernel with torch.profiler in a separate run. The card name and power limit are read in the same call.

Quality (unless --no-quality): a 16-spp AOV render of seed s1 against --ref-spp of seed s2. For each AOV plane, the
relative error sqrt(sum (I - R)^2 / sum R^2) of the noisy plane, of the plane from denoise_planes and of
denoise(weights=e_k) (the plane filtered alone with weights of its own); for the recomposite RECOMPOSITE, the noisy,
relight_denoised and denoise(weights=...) errors. The reference's own noise is included in every error."""
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

S1, S2 = 0x12345678, 0x9E3779B9
RECOMPOSITE = [1, 1, 1, 1, 0, 0, 1, 1]   # the AOV planes without the reflections


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"nvidia-smi unavailable: {e}"


def timed(call, reps):
    import torch
    for _ in range(3):
        call()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        times.append((e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3))
    return {"events_median": float(np.median([t[0] for t in times])), "wall_median": float(np.median([t[1] for t in times])),
            "events_min": float(np.min([t[0] for t in times])), "events_max": float(np.max([t[0] for t in times]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--planes", default="1,4,8,16,31")
    ap.add_argument("--no-quality", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    m = importlib.import_module("monte-carlo-ray-tracer_b200")
    scene = m.Scene.from_pack(os.path.join(ROOT, "bench_data", "c2_hexagon_room.mcrtpack"))
    cam = scene.cameras()[0].resized(args.width, args.height, 16)
    pt = m.PathTracer(scene, precision=m.PRECISION_F64, global_seed=S1)
    pt.set_option("pool_paths", float(1 << 25))     # as bench.py: 32 Mi paths in flight
    result = {"gpu": gpu_info(), "lib": m.LIB_PATH, "width": cam.width, "height": cam.height}
    prog = m.Progressive(pt, cam, aovs=True)
    prog.render(8, 16)
    n_aov = len(m.AOV_NAMES)
    guide = prog._halves()
    f = prog._feature_sums(8)
    params = m.DenoiseParams(m.DENOISE_DEFAULTS["iterations"], 0, m.DENOISE_DEFAULTS["sigma_color"], m.DENOISE_DEFAULTS["sigma_normal"],
                             m.DENOISE_DEFAULTS["sigma_depth"], m.DENOISE_DEFAULTS["sigma_albedo"])
    out = torch.empty_like(guide[0])
    torch.cuda.synchronize()

    def beauty():
        return pt.denoise_dev(guide[0].data_ptr(), None, guide[1].data_ptr(), None, prog.tile_counts, prog.tile, f.data_ptr(),
                              cam.width, cam.height, out.data_ptr(), params)
    result["denoise_dev_ms"] = timed(beauty, args.reps)
    print(json.dumps({"denoise_dev_ms": result["denoise_dev_ms"]}), flush=True)

    def planes_call(n, src, dst, with_frame):
        def call():
            return pt.denoise_planes_dev(guide[0].data_ptr(), guide[1].data_ptr(), src[0].data_ptr(), src[1].data_ptr(), n,
                                         prog.tile_counts, prog.tile, f.data_ptr(), cam.width, cam.height, dst[0].data_ptr(),
                                         dst[1].data_ptr(), params, out.data_ptr() if with_frame else None)
        return call
    result["denoise_planes_dev_ms"] = {}
    for n in (int(p) for p in args.planes.split(",")):
        reps = -(-n // n_aov)
        src = [prog.rgb[h].repeat((reps, 1, 1, 1))[:n].contiguous() for h in (0, 1)]
        dst = [torch.empty_like(s) for s in src]
        torch.cuda.synchronize()
        result["denoise_planes_dev_ms"][n] = timed(planes_call(n, src, dst, False), args.reps)
        print(json.dumps({"planes": n, "ms": result["denoise_planes_dev_ms"][n]}), flush=True)
        del src, dst
        torch.cuda.empty_cache()
    if n_aov in result["denoise_planes_dev_ms"]:
        bar = n_aov * result["denoise_dev_ms"]["events_median"]
        result["bar"] = {"aov_planes_ms": result["denoise_planes_dev_ms"][n_aov]["events_median"],
                         "eight_denoise_dev_calls_ms": bar,
                         "passes": result["denoise_planes_dev_ms"][n_aov]["events_median"] < bar}

    # per kernel, in a run of its own: the 8 AOV planes
    dst = [torch.empty_like(prog.rgb[h]) for h in (0, 1)]
    torch.cuda.synchronize()
    call = planes_call(n_aov, prog.rgb, dst, True)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(5):
            call()
        torch.cuda.synchronize()
    kernels = {}
    for ev in p.key_averages():
        if "denoise" in ev.key or "memcpy" in ev.key.lower() or "memset" in ev.key.lower():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            kernels[ev.key[:90]] = {"calls": ev.count, "us_per_call": t / max(ev.count, 1), "us_per_planes_call": t / 5}
    result["planes_kernels_8_planes"] = kernels
    print(json.dumps({"planes_kernels_8_planes": kernels}), flush=True)

    if not args.no_quality:
        other = m.PathTracer(scene, precision=m.PRECISION_F64, global_seed=S2)
        other.set_option("pool_paths", float(1 << 25))
        ref_prog = m.Progressive(other, cam, aovs=True)
        ref_prog.render(256, args.ref_spp)
        ref_planes, _ = ref_prog.aov_frames()
        ref_recomposite = ref_prog.relight(RECOMPOSITE)[0]
        other.close()
        del ref_prog

        def rel(x, ref):
            return float(np.sqrt(np.sum((x - ref) ** 2) / np.sum(ref ** 2)))
        noisy_planes, _ = prog.aov_frames()
        planes, _ = prog.denoise_planes()
        beauty_energy = float(ref_planes.sum())
        rows = []
        for k, name in enumerate(m.AOV_NAMES):
            e = np.eye(n_aov)[k]
            ref = ref_planes[k]
            row = {"plane": name, "share": float(ref.sum()) / beauty_energy}
            if ref.any():
                row.update(noisy=rel(noisy_planes[k], ref), denoise_planes=rel(planes[k], ref),
                           denoise_alone=rel(prog.denoise(weights=e)[0], ref))
            rows.append(row)
            print(json.dumps(row), flush=True)
        result["quality_planes"] = rows
        result["quality_recomposite"] = {"weights": RECOMPOSITE, "noisy": rel(prog.relight(RECOMPOSITE)[0], ref_recomposite),
                                         "relight_denoised": rel(prog.relight_denoised(RECOMPOSITE)[0], ref_recomposite),
                                         "denoise_weights": rel(prog.denoise(weights=RECOMPOSITE)[0], ref_recomposite)}
        print(json.dumps(result["quality_recomposite"]), flush=True)
    result["gpu_after"] = gpu_info()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as fo:
            json.dump(result, fo, indent=1)
    pt.close()


if __name__ == "__main__":
    main()
