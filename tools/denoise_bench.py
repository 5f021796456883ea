#!/usr/bin/env python3
"""Cost and benefit of the denoiser on the C2 workload of bench.py (hexagon_room, 1920x1080, parity mode, 32 Mi-path
pool).

  python tools/denoise_bench.py [--reps 20] [--ref-spp 1024] [--specular-depth 0,1,2,4] [--out result.json]

Reported: the device time of the feature pass at 8 spp (CUDA events of mcrt_render_features_dev); the device time of
mcrt_denoise_dev at the default parameters (CUDA events around the call, median of --reps) and per kernel
(torch.profiler, separate run); the card name and power limit, read in the same call.

Equal-error comparison: noisy frames at 16, 32 and 64 spp with seed s1 and a reference of --ref-spp with seed s2. The
relative error sqrt(sum (I - R)^2 / sum R^2) of each noisy and denoised frame against the reference, the denoised
residual estimate beside it (it sees noise, not the filter's bias), and the spp a noisy render needs to match the
denoised 16-spp frame, interpolated in log-log between the measured spp. The reference's own noise is included in
every measured error; it is reported as the reference's two-half estimate.

--specular-depth D1,D2,...: guides taken after up to D perfectly specular bounces (Progressive.denoise(specular_depth=D)).
For each D, the feature pass at 8 spp is timed and every spp row also reports the denoised error over the pixels whose
first hit is a dirac_delta material (the ray through the pixel's centre), beside the whole frame's."""
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


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return f"nvidia-smi unavailable: {e}"


def delta_first_hit(m, tracer, scene, cam):
    """[H, W] True where the ray through the pixel's centre first hits a dirac_delta material."""
    r = cam.rec
    fwd, left, up = (np.array(v[:3]) for v in (r.forward, r.left, r.up))
    x, y = np.meshgrid(np.arange(cam.width) + 0.5, np.arange(cam.height) + 0.5)
    size = r.sensor_width / cam.width
    d = fwd * r.focal_length + left * (size * (cam.width * 0.5 - x))[..., None] + up * (size * (cam.height * 0.5 - y))[..., None]
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    rays = np.concatenate([np.broadcast_to(np.array(r.eye[:3]), d.shape), d], -1).reshape(-1, 6)
    prim = tracer.intersect(rays)["prim"]
    a = scene.a
    hit = prim != m.NO_PRIM
    out = np.zeros(len(prim), bool)
    out[hit] = a["materials"]["dirac_delta"][a["prim_material"][prim[hit].astype(np.int64)]] != 0
    return out.reshape(cam.height, cam.width)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--ref-spp", type=int, default=1024)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--specular-depth", default="0", help="comma-separated guide depths")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    depths = [int(d) for d in args.specular_depth.split(",")]
    import torch
    m = importlib.import_module("monte-carlo-ray-tracer_b200")
    scene = m.Scene.from_pack(os.path.join(ROOT, "bench_data", "c2_hexagon_room.mcrtpack"))
    cam = scene.cameras()[0].resized(args.width, args.height, 16)
    tracers = {}
    for seed in (S1, S2):
        tracers[seed] = m.PathTracer(scene, precision=m.PRECISION_F64, global_seed=seed)
        tracers[seed].set_option("pool_paths", float(1 << 25))     # as bench.py: 32 Mi paths in flight
    result = {"gpu": gpu_info(), "width": cam.width, "height": cam.height}

    # reference
    ref_prog = m.Progressive(tracers[S2], cam)
    ref_prog.render(64, args.ref_spp)
    ref = ref_prog.frame()
    result["reference"] = {"spp": args.ref_spp, "estimate": ref_prog.error()[0]}

    mask = delta_first_hit(m, tracers[S1], scene, cam)
    result["delta_first_hit_share"] = float(mask.mean())

    def rel(x, where=None):
        where = np.ones(mask.shape, bool) if where is None else where
        return float(np.sqrt(np.sum((x - ref)[where] ** 2) / np.sum(ref[where] ** 2)))

    prog = m.Progressive(tracers[S1], cam)
    rows = []
    for spp in (16, 32, 64):
        pass_spp = spp - prog.samples
        prog.add(pass_spp // 2); prog.add(pass_spp - pass_spp // 2)
        dn, estimate = prog.denoise()
        rows.append({"spp": spp, "noisy": rel(prog.frame()), "noisy_estimate": prog.error()[0], "denoised": rel(dn),
                     "denoised_estimate": estimate, "noisy_delta": rel(prog.frame(), mask)})
        if depths != [0]:
            rows[-1]["by_specular_depth"] = {}
            for d in depths:
                dnd, _ = prog.denoise(specular_depth=d)
                rows[-1]["by_specular_depth"][d] = {"denoised": rel(dnd), "denoised_delta": rel(dnd, mask)}
        print(json.dumps(rows[-1]), flush=True)
    result["quality"] = rows
    # spp at which a noisy render matches denoised 16 spp (log-log interpolation / extrapolation over 16..64)
    s = np.log([r["spp"] for r in rows]); e = np.log([r["noisy"] for r in rows])
    slope, icpt = np.polyfit(s, e, 1)
    result["noisy_spp_matching_denoised_16"] = float(np.exp((np.log(rows[0]["denoised"]) - icpt) / slope))
    result["noisy_error_slope"] = float(slope)

    # feature pass at 8 spp
    f = torch.zeros((cam.height, cam.width, 8), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    feat_ms = []
    for _ in range(3):
        f.zero_(); torch.cuda.synchronize()
        feat_ms.append(tracers[S1].render_features_dev(cam, f.data_ptr(), 0, 8)["gpu_ms_total"])
    result["feature_pass_8spp_ms"] = float(np.median(feat_ms))
    if depths != [0]:
        result["feature_pass_8spp_ms_by_specular_depth"] = {}
        for d in depths:
            ms = []
            for _ in range(3):
                f.zero_(); torch.cuda.synchronize()
                ms.append(tracers[S1].render_features_dev(cam, f.data_ptr(), 0, 8, specular_depth=d)["gpu_ms_total"])
            result["feature_pass_8spp_ms_by_specular_depth"][d] = float(np.median(ms))
        f.zero_(); torch.cuda.synchronize()
        tracers[S1].render_features_dev(cam, f.data_ptr(), 0, 8)   # the denoiser timing below uses the first-hit guides

    # denoiser: CUDA events around the call (the library's stream is synchronised inside the call)
    ptl = tracers[S1]
    out = torch.empty_like(prog.rgb[0])
    params = m.DenoiseParams(m.DENOISE_DEFAULTS["iterations"], 0, m.DENOISE_DEFAULTS["sigma_color"], m.DENOISE_DEFAULTS["sigma_normal"],
                             m.DENOISE_DEFAULTS["sigma_depth"], m.DENOISE_DEFAULTS["sigma_albedo"])

    def call():
        return ptl.denoise_dev(prog.rgb[0].data_ptr(), None, prog.rgb[1].data_ptr(), None, prog.tile_counts, prog.tile, f.data_ptr(),
                               cam.width, cam.height, out.data_ptr(), params)
    for _ in range(3):
        call()
    times = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        times.append((e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3))
    result["denoise_call_ms"] = {"events_median": float(np.median([t[0] for t in times])),
                                 "wall_median": float(np.median([t[1] for t in times]))}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(5):
            call()
        torch.cuda.synchronize()
    kernels = {}
    for ev in p.key_averages():
        if "denoise" in ev.key or "memcpy" in ev.key.lower() or "memset" in ev.key.lower():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            kernels[ev.key[:80]] = {"calls": ev.count, "us_per_call": t / max(ev.count, 1)}
    result["denoise_kernels"] = kernels
    result["gpu_after"] = gpu_info()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as fo:
            json.dump(result, fo, indent=1)
    for t in tracers.values():
        t.close()


if __name__ == "__main__":
    main()
