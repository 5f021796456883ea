"""TEST INFRASTRUCTURE - ctypes binding of tests/light_path_ref.cpp, the CPU restatement of the light-path AOV planes of
mcrt_render_accumulate_aovs_dev. The library is compiled on first use into a temporary directory (never into the
tree), with the flags of oracle/build_oracle.py."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCES = [os.path.join(HERE, "light_path_ref.cpp"), os.path.join(ROOT, "oracle", "mcrt_oracle.cpp"),
           os.path.join(ROOT, "include", "mcrt_abi.h")]
N_PLANES = 8
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for src in SOURCES:
            with open(src, "rb") as f:
                h.update(f.read())
        d = os.path.join(tempfile.gettempdir(), f"mcrt_light_path_{os.getuid()}_{h.hexdigest()[:16]}")
        path = os.path.join(d, "liblight_path.so")
        if not os.path.exists(path):
            os.makedirs(d, exist_ok=True)
            tmp = path + f".{os.getpid()}"
            subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"),
                                   SOURCES[0], "-o", tmp])
            os.replace(tmp, path)
        L = C.CDLL(path)
        L.oracle_scene_create.restype = C.c_void_p
        L.oracle_scene_create.argtypes = [C.c_void_p]
        L.oracle_scene_destroy.argtypes = [C.c_void_p]
        L.oracle_render_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                         C.POINTER(C.c_uint64)]
        L.oracle_render_rows_aovs.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
        _lib = L
    return _lib


def render_rows_aovs(scene, camera, y0, y1, sqrtspp, seed, beauty=False):
    """-> the per-pixel means of each AOV plane of rows [y0, y1), float64 [8, y1 - y0, width, 3], in the order of the
    package's AOV_NAMES; with beauty=True also oracle_render_rows' frame of the same samples [y1 - y0, width, 3].
    scene: the product package's Scene (a container of the flattened arrays); camera: its Camera."""
    L = lib()
    desc = scene.desc()
    h = L.oracle_scene_create(C.addressof(desc))
    try:
        out = np.zeros((N_PLANES, y1 - y0, camera.width, 3))
        L.oracle_render_rows_aovs(h, C.addressof(camera.rec), y0, y1, sqrtspp, seed, out.ctypes.data_as(C.c_void_p))
        if not beauty:
            return out
        frame = np.zeros((y1 - y0, camera.width, 3))
        rays = C.c_uint64()
        L.oracle_render_rows(h, C.addressof(camera.rec), y0, y1, sqrtspp, seed, frame.ctypes.data_as(C.c_void_p), C.byref(rays))
        return out, frame
    finally:
        L.oracle_scene_destroy(h)
