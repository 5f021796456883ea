"""TEST INFRASTRUCTURE - ctypes binding of tests/pm_lpe_ref.cpp, the CPU restatement of the photon mapper's event
strings: each photon's own events from the restated photon pass, and pmSampleRay's contributions summed per event
string, every photon term under its own. Planes are formed with tests/lpe_ref.py's Strings (Python's re over the same
one-character encoding), independently of the product's compiler. Compiled on first use into a temporary directory."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from lpe_ref import ENCODING, Strings, group_char

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCES = [os.path.join(HERE, "pm_lpe_ref.cpp"), os.path.join(ROOT, "oracle", "mcrt_oracle.cpp"),
           os.path.join(ROOT, "include", "mcrt_abi.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for src in SOURCES:
            with open(src, "rb") as f:
                h.update(f.read())
        d = os.path.join(tempfile.gettempdir(), f"mcrt_pm_lpe_ref_{os.getuid()}_{h.hexdigest()[:16]}")
        path = os.path.join(d, "libpm_lpe_ref.so")
        if not os.path.exists(path):
            os.makedirs(d, exist_ok=True)
            tmp = path + f".{os.getpid()}"
            subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-I",
                                   os.path.join(ROOT, "include"), SOURCES[0], "-o", tmp])
            os.replace(tmp, path)
        L = C.CDLL(path)
        L.oracle_scene_create.restype = C.c_void_p
        L.oracle_scene_create.argtypes = [C.c_void_p]
        L.oracle_scene_destroy.argtypes = [C.c_void_p]
        L.oracle_pm_photon_events.restype = C.c_void_p
        L.oracle_pm_photon_events.argtypes = [C.c_void_p, C.c_uint64, C.c_double, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                              C.POINTER(C.c_uint64)]
        L.oracle_pm_photon_events_get.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_pm_photon_events_free.argtypes = [C.c_void_p]
        L.oracle_pm_lpe_render.restype = C.c_void_p
        L.oracle_pm_lpe_render.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_char_p, C.c_void_p, C.c_uint64, C.c_char_p,
                                           C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                           C.c_uint32, C.c_void_p, C.c_uint32]
        L.oracle_pm_lpe_sizes.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.oracle_pm_lpe_get.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_pm_lpe_free.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class _Scene:
    def __init__(self, scene):
        self.desc = scene.desc()
        self.h = lib().oracle_scene_create(C.addressof(self.desc))

    def __enter__(self):
        return self.h

    def __exit__(self, *a):
        lib().oracle_scene_destroy(self.h)


def photon_events(scene, emissions, caustic_factor, seed, pass_index=0):
    """The restated photon pass with each photon's events -> (maps, mismatched): maps[which] = (photons float32 [n, 8] in
    emission order, emitting light uint32 [n], events [n] strings e1..em in emission order over lpe_ref's encoding);
    mismatched: photons whose second walk differs from the pass's (0 when the walk restates it bit for bit)."""
    L = lib()
    with _Scene(scene) as h:
        n, chars, mism = (C.c_uint64 * 2)(), (C.c_uint64 * 2)(), C.c_uint64()
        handle = L.oracle_pm_photon_events(h, int(emissions), float(caustic_factor), int(pass_index), int(seed), n, chars, C.byref(mism))
        if not handle:
            raise ValueError("the pass's emission indices do not fit 32 bits")
        try:
            maps = []
            for w in range(2):
                ph = np.zeros((n[w], 8), np.float32)
                li = np.zeros(n[w], np.uint32)
                buf = C.create_string_buffer(max(chars[w], 1))
                L.oracle_pm_photon_events_get(handle, w, ph.ctypes.data_as(C.c_void_p), li.ctypes.data_as(C.c_void_p), buf)
                ev = buf.raw[:chars[w]].decode(ENCODING).split("\0")[:n[w]]
                maps.append((ph, li, ev))
        finally:
            L.oracle_pm_photon_events_free(handle)
        return maps, mism.value


def history(events, lights, group_of_light=None):
    """The string a photon adds after x: its events from the last to the first, then its light's character."""
    out = []
    for ev, l in zip(events, lights):
        light = "*" if group_of_light is None else group_char(group_of_light[l])
        out.append(ev[::-1] + light)
    return out


def render_strings(scene, camera, y0, y1, sqrtspp, seed, maps, k, dv, gather_r2=(0.0, 0.0), group_of_light=None):
    """-> lpe_ref.Strings of rows [y0, y1) over maps = ((photons [n, 8], history [n]) caustic, (...) global)."""
    L = lib()
    g = None if group_of_light is None else np.ascontiguousarray(group_of_light, np.uint32)
    n_groups = 0 if g is None or g.size == 0 else int(g.max()) + 1
    ph = [np.ascontiguousarray(m[0], np.float32).reshape(-1, 8) for m in maps]
    hs = [b"".join(s.encode(ENCODING) + b"\0" for s in m[1]) or b"\0" for m in maps]
    r2 = np.ascontiguousarray(gather_r2, np.float64)
    with _Scene(scene) as h:
        handle = L.oracle_pm_lpe_render(h, ph[0].ctypes.data_as(C.c_void_p), len(ph[0]), hs[0], ph[1].ctypes.data_as(C.c_void_p),
                                        len(ph[1]), hs[1], int(k), int(bool(dv)), r2.ctypes.data_as(C.c_void_p),
                                        C.addressof(camera.rec), y0, y1, sqrtspp, int(seed),
                                        None if g is None else g.ctypes.data_as(C.c_void_p), 0 if g is None else g.size)
        try:
            e, n, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
            L.oracle_pm_lpe_sizes(handle, C.byref(e), C.byref(n), C.byref(c))
            pixel = np.zeros(e.value, np.uint32)
            string = np.zeros(e.value, np.uint32)
            value = np.zeros((e.value, 3))
            chars = C.create_string_buffer(max(c.value, 1))
            L.oracle_pm_lpe_get(handle, pixel.ctypes.data_as(C.c_void_p), string.ctypes.data_as(C.c_void_p),
                                value.ctypes.data_as(C.c_void_p), chars)
            strings = chars.raw[:c.value].decode(ENCODING).split("\0")[:n.value]
        finally:
            L.oracle_pm_lpe_free(handle)
    return Strings(strings, pixel.astype(np.int64), string.astype(np.int64), value, y1 - y0, camera.width, n_groups)
