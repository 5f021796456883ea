#!/usr/bin/env python3
"""Parallel OBJ loader + vertex normals (mcrt_obj_load, mcrt_obj_vertex_normals) against the reference's
Scene::parseOBJ / generateVertexNormals on the reference's own OBJ assets: equality and load time.
Needs the reference checkout. Prints one line per asset."""
import glob
import importlib
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref  # noqa: E402
mcrt = importlib.import_module("monte-carlo-ray-tracer_b200")

if __name__ == "__main__":
    s = ref.RefScene("ior_test.json", dict(width=8, height=8, sqrtspp=1))
    files = sorted(glob.glob("/root/reference/scenes/data/**/*.obj", recursive=True), key=os.path.getsize)
    for f in files[-8:]:
        r = s.parse_obj(f)
        best = None
        for _ in range(3):
            t0 = time.perf_counter(); g = mcrt.load_obj(f); dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        same = all(np.array_equal(r[k], g[k]) for k in ("vertices", "normals", "tri_v", "tri_vt", "tri_vn"))
        msg = (f"{os.path.relpath(f, '/root/reference/scenes/data')}: {os.path.getsize(f) / 1e6:.1f} MB, {len(g['vertices'])} v, {len(g['tri_v'])} f: "
               f"{'IDENTICAL' if same else 'DIFFERENT'}; reference {r['seconds'] * 1e3:.0f} ms, parallel loader {best * 1e3:.0f} ms ({r['seconds'] / best:.1f}x)")
        ok = (g["tri_v"] < len(g["vertices"])).all(axis=1)
        if len(g["tri_v"]) and ok.all():
            n_ref, sec = s.vertex_normals(r["vertices"], r["tri_v"])
            dt = None
            for _ in range(3):
                t0 = time.perf_counter(); n_got = mcrt.vertex_normals(g["vertices"], g["tri_v"]); d1 = time.perf_counter() - t0
                dt = d1 if dt is None else min(dt, d1)
            msg += (f"; vertex normals {'IDENTICAL' if np.array_equal(n_ref, n_got, equal_nan=True) else 'DIFFERENT'}: "
                    f"reference {sec * 1e3:.0f} ms, parallel {dt * 1e3:.0f} ms")
        msg += f"; drop-in bodies (host/obj_adapter.hpp) vs the reference's: {'EQUAL' if s.obj_adapter_check(f) == 1 else 'DIFFERENT'}"
        print(msg, flush=True)
    print(f"host cores: {os.cpu_count()}")
