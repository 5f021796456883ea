"""TEST INFRASTRUCTURE - ctypes binding of tests/specular_chain_ref.cpp, the CPU restatement of the guide chains of
mcrt_render_features_chain_dev. The library is compiled on first use into a temporary directory (never into the
tree), with the flags of oracle/build_oracle.py."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCES = [os.path.join(HERE, "specular_chain_ref.cpp"), os.path.join(ROOT, "oracle", "mcrt_oracle.cpp"),
           os.path.join(ROOT, "include", "mcrt_abi.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for src in SOURCES:
            with open(src, "rb") as f:
                h.update(f.read())
        d = os.path.join(tempfile.gettempdir(), f"mcrt_specular_chain_{os.getuid()}_{h.hexdigest()[:16]}")
        path = os.path.join(d, "libspecular_chain.so")
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
        L.oracle_specular_chain.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32,
                                            C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def specular_chain(scene, camera, pixel, sample, seed, max_depth):
    """-> (denoiser guides [n, 8] {T * albedo, shading normal, L + t, 1} of (pixel, sample) pairs, taken at the end of
    each sample's chain of at most max_depth perfectly specular bounces, zeros where the chain misses;
    end [n, 3] {last primitive hit or NO_PRIM, its depth, 1 where the bounce there was rejected or left T at 0}).
    scene: the product package's Scene (a container of the flattened arrays); camera: its Camera."""
    L = lib()
    desc = scene.desc()
    h = L.oracle_scene_create(C.addressof(desc))
    try:
        pixel = np.ascontiguousarray(pixel, dtype=np.uint32); sample = np.ascontiguousarray(sample, dtype=np.uint32)
        out = np.zeros((len(pixel), 8))
        end = np.zeros((len(pixel), 3), dtype=np.uint32)
        L.oracle_specular_chain(h, C.addressof(camera.rec), _p(pixel), _p(sample), len(pixel), seed, int(max_depth), _p(out), _p(end))
    finally:
        L.oracle_scene_destroy(h)
    return out, end
