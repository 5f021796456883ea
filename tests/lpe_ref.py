"""TEST INFRASTRUCTURE - ctypes binding of tests/lpe_ref.cpp, the CPU restatement of the event strings of light path
expressions, and a translation of expressions into Python regular expressions over its one-character-per-event
encoding, so that planes are formed without the product's compiler. The library is compiled on first use into a
temporary directory (never into the tree), with the flags of oracle/build_oracle.py."""
import ctypes as C
import hashlib
import os
import re
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCES = [os.path.join(HERE, "lpe_ref.cpp"), os.path.join(ROOT, "oracle", "mcrt_oracle.cpp"),
           os.path.join(ROOT, "include", "mcrt_abi.h")]
# the restatement's characters of the vertex events (tests/lpe_ref.cpp)
VERTEX = {"RD": "a", "RS": "b", "RG": "c", "TS": "d", "TG": "e"}
UNGROUPED = "*"
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for src in SOURCES:
            with open(src, "rb") as f:
                h.update(f.read())
        d = os.path.join(tempfile.gettempdir(), f"mcrt_lpe_ref_{os.getuid()}_{h.hexdigest()[:16]}")
        path = os.path.join(d, "liblpe_ref.so")
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
        L.oracle_lpe_render.restype = C.c_void_p
        L.oracle_lpe_render.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32]
        L.oracle_lpe_sizes.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.oracle_lpe_get.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_lpe_free.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class Strings:
    """The restatement's contributions of rows [y0, y1): strings (list of str), and per (pixel, string) entry its
    pixel (index into the rows' [rows * width]), string index and mean value [3]."""

    def __init__(self, strings, pixel, string, value, rows, width, n_groups):
        self.strings, self.pixel, self.string, self.value = strings, pixel, string, value
        self.rows, self.width, self.n_groups = rows, width, n_groups

    def planes(self, exprs):
        """-> float64 [len(exprs), rows, width, 3]: plane i sums the strings expression i matches (re.fullmatch)."""
        regs = [re.compile(to_regex(e, self.n_groups)) for e in exprs]
        out = np.zeros((len(exprs), self.rows * self.width, 3))
        for i, r in enumerate(regs):
            match = np.array([bool(r.fullmatch(s)) for s in self.strings], bool)
            keep = match[self.string]
            np.add.at(out[i], self.pixel[keep], self.value[keep])
        return out.reshape(len(exprs), self.rows, self.width, 3)

    def beauty(self):
        out = np.zeros((self.rows * self.width, 3))
        np.add.at(out, self.pixel, self.value)
        return out.reshape(self.rows, self.width, 3)


def render_strings(scene, camera, y0, y1, sqrtspp, seed, group_of_light=None):
    """-> Strings of rows [y0, y1). group_of_light: the group of each light (None: every emitter reads '*')."""
    L = lib()
    desc = scene.desc()
    h = L.oracle_scene_create(C.addressof(desc))
    try:
        g = None if group_of_light is None else np.ascontiguousarray(group_of_light, np.uint32)
        n_groups = 0 if g is None or g.size == 0 else int(g.max()) + 1
        handle = L.oracle_lpe_render(h, C.addressof(camera.rec), y0, y1, sqrtspp, seed,
                                     None if g is None else g.ctypes.data_as(C.c_void_p), 0 if g is None else g.size)
        try:
            e, n, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
            L.oracle_lpe_sizes(handle, C.byref(e), C.byref(n), C.byref(c))
            pixel = np.zeros(e.value, np.uint32)
            string = np.zeros(e.value, np.uint32)
            value = np.zeros((e.value, 3))
            chars = C.create_string_buffer(max(c.value, 1))
            L.oracle_lpe_get(handle, pixel.ctypes.data_as(C.c_void_p), string.ctypes.data_as(C.c_void_p),
                             value.ctypes.data_as(C.c_void_p), chars)
            strings = chars.raw[:c.value].decode().split("\0")[:n.value]
        finally:
            L.oracle_lpe_free(handle)
        return Strings(strings, pixel.astype(np.int64), string.astype(np.int64), value, y1 - y0, camera.width, n_groups)
    finally:
        L.oracle_scene_destroy(h)


def render_rows(scene, camera, y0, y1, sqrtspp, seed):
    """oracle_render_rows: the restated reference frame of the same samples [y1 - y0, width, 3]."""
    L = lib()
    desc = scene.desc()
    h = L.oracle_scene_create(C.addressof(desc))
    try:
        frame = np.zeros((y1 - y0, camera.width, 3))
        rays = C.c_uint64()
        L.oracle_render_rows(h, C.addressof(camera.rec), y0, y1, sqrtspp, seed, frame.ctypes.data_as(C.c_void_p), C.byref(rays))
        return frame
    finally:
        L.oracle_scene_destroy(h)


def to_regex(expr, n_groups):
    """The Python regular expression of a light path expression (the grammar of include/mcrt_abi.h) over the
    restatement's encoding with n_groups light groups. L matches every emitter, L'g' those of group g."""
    lights = {chr(ord("0") + g) for g in range(n_groups)} | {UNGROUPED}
    alphabet = {"C", "B"} | set(VERTEX.values()) | lights
    s = "".join(expr.split())
    i = 0

    def event():
        nonlocal i
        ch = s[i]
        i += 1
        if ch in "CB":
            return {ch}
        if ch == ".":
            return set(alphabet)
        if ch in "DGSRT":
            return {k for ev, k in VERTEX.items() if (ch == "D" and ev[1] == "D") or (ch in "GS" and ev[1] == ch)
                    or (ch in "RT" and ev[0] == ch)}
        if ch == "L":
            if i < len(s) and s[i] == "'":
                j = s.index("'", i + 1)
                g = int(s[i + 1:j])
                i = j + 1
                return {chr(ord("0") + g)}
            return set(lights)
        if ch == "<":
            x, y = s[i], s[i + 1]
            assert s[i + 2] == ">", expr
            i += 3
            return {k for ev, k in VERTEX.items() if x in (".", ev[0]) and y in (".", ev[1])}
        raise AssertionError(f"unexpected {ch!r} in {expr!r}")

    def cls(chars):
        return "(?!)" if not chars else "[" + "".join(re.escape(c) for c in sorted(chars)) + "]"

    out = []
    while i < len(s):
        ch = s[i]
        if ch in "()|*+?":
            out.append("(?:" if ch == "(" else ch)
            i += 1
        elif ch == "{":
            j = s.index("}", i)
            out.append(s[i:j + 1])
            i = j + 1
        elif ch == "[":
            i += 1
            neg = s[i] == "^"
            if neg:
                i += 1
            chars = set()
            while s[i] != "]":
                chars |= event()
            i += 1
            out.append(cls(alphabet - chars if neg else chars))
        else:
            out.append(cls(event()))
    return "".join(out)
