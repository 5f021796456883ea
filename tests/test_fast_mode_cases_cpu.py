"""Which float32 kernel instantiations the fast-mode tests (tests/test_gpu_fast_mode.py) reach, without a GPU.

Fast mode runs its own `float` instantiation of every wavefront kernel. `Launch<float>` (csrc/kernels_impl.cuh) picks one
from the scene's primitive class (abi.cu, from prim_type), its material feature set (LITE when no material needs
Oren-Nayar, GGX or conductor Fresnel), the camera's film (default box or a reconstruction filter), the integrator, the
photon k-NN register slots (knnSlotsFor) or the fixed-radius gather, and whether the pass renders a pixel list (adaptive
sampling with retired tiles). `reached` restates that selection; CASES is the table the GPU tests are parametrised over,
and EXPECTED is the list of float branches, written out by hand: a branch added to kernels_impl.cuh without a case here
fails test_cases_reach_every_float_branch instead of going untested."""
import os
from collections import namedtuple

import pytest

from conftest import GOLDEN, golden_cases, load_package

# scene: a golden case, "gen/<name>" (tests/scene_gen.py) or "film_hexagon_room_64" (seed in film_kat.npz)
# film: None (the pack camera's box film) or a name of film_kat.npz's films
# k: photon k-NN neighbours (None: the map's own); gather: fixed-radius gather instead of k-NN
# emit: the photon pass also runs in float32 and its maps are compared; adaptive: one pass with tiles retired
Case = namedtuple("Case", "scene film photon k gather emit adaptive")
Case.__new__.__defaults__ = (None, False, None, False, False, False)

FILMS = ["mitchell", "catmull_rom", "b_spline", "hermite", "gaussian_cached", "lanczos_r3", "lanczos_cached", "box_r1p5",
         "box_default_cached"]
GENERATED = ["gen/mesh", "gen/room", "gen/quadric", "gen/pm"]
PM_K = [32, 33, 64, 65, 128, 129, 256, 257, 673]     # every register-slot class on both sides of its bound, and k > 672

CASES = (
    [Case(c, photon=c.startswith("pm_")) for c in golden_cases()]
    + [Case(c, photon=c == "gen/pm") for c in GENERATED]
    + [Case("film_hexagon_room_64", film=f) for f in FILMS]
    + [Case("pm_hexagon_room_64", photon=True, k=k) for k in PM_K]
    + [Case("metals_64", photon=True, k=k) for k in PM_K]
    + [Case("pm_hexagon_room_64", photon=True, gather=True), Case("metals_64", photon=True, gather=True),
       Case("pm_hexagon_room_64", photon=True, film="mitchell"), Case("pm_hexagon_room_64", photon=True, film="mitchell", gather=True),
       Case("pm_hexagon_room_64", photon=True, emit=True), Case("metals_64", photon=True, emit=True),
       Case("c2_hexagon_room_96", adaptive=True), Case("film_hexagon_room_64", film="mitchell", adaptive=True)]
)


def case_id(c):
    parts = [c.scene] + ([c.film] if c.film else []) + (["photon"] if c.photon and not c.scene.startswith(("pm_", "gen/pm")) else [])
    parts += [f"k{c.k}"] if c.k else []
    parts += [n for n in ("gather", "emit", "adaptive") if getattr(c, n)]
    return "-".join(parts)


# the hand-written list of Launch<float> branches (kernels_impl.cuh); parity-only branches (BVH4 search) are not float's
EXPECTED = sorted([
    "generate<box,list=0>", "generate<filter,list=0>", "generate<box,list=1>", "generate<filter,list=1>",
    "extend<TRI>", "extend<TRI_SPHERE>", "extend<ALL>",
    "shade<path,box,LITE>", "shade<path,box,ALL>", "shade<path,filter,ALL>",
    "shade<photon,box,LITE>", "shade<photon,box,ALL>", "shade<photon,filter,ALL>",
    "gather<box,LITE>", "gather<box,ALL>", "gather<filter,ALL>",
    "knn<0,filter,ALL>",
    "knn<1,box,LITE>", "knn<2,box,LITE>", "knn<4,box,LITE>", "knn<8,box,LITE>", "knn<0,box,LITE>",
    "knn<1,box,ALL>", "knn<2,box,ALL>", "knn<4,box,ALL>", "knn<8,box,ALL>", "knn<0,box,ALL>",
    "shadow<filter,ALL>", "shadow<box,TRI>", "shadow<box,TRI_SPHERE>", "shadow<box,ALL>",
    "emitGenerate", "emitShade",
    "traceUser",
])

MAT_ROUGH_FEATURES = ("rough", "rough_specular", "has_complex_ior")     # SHADE_FEATS_LITE excludes these three


def knn_slots(k):
    """photon.cuh knnSlotsFor: register slots of k_knn, 0 = shared-memory result lists"""
    return 1 if k <= 32 else 2 if k <= 64 else 4 if k <= 128 else 8 if k <= 256 else 0


def is_filtered(film):
    """mcrt_set_film: only the box filter at radius 0.5 (the default) keeps the default film"""
    if not film:
        return False
    f = str(film.get("filter", "box")).lower()
    return not (f == "box" and float(film.get("radius") or 0.5) == 0.5)


def scene_features(mcrt, scene):
    """-> (prims_class, lite) as mcrt_scene_upload derives them (abi.cu) and Launch<R>::shade tests them"""
    types = set(int(t) for t in scene.a["prim_type"])
    pc = "TRI" if types <= {mcrt.PRIM_TRIANGLE} else "TRI_SPHERE" if types <= {mcrt.PRIM_TRIANGLE, mcrt.PRIM_SPHERE} else "ALL"
    mats = scene.a["materials"]
    lite = not any(int(mats[f].any()) for f in MAT_ROUGH_FEATURES)
    return pc, lite


def pack_of(scene):
    # the generated scenes append triangles with the base scene's materials (and one plain emissive copy) to a golden scene
    return {"gen/mesh": "smooth_mesh_64", "gen/room": "c2_hexagon_room_96", "gen/quadric": "quadric_64",
            "gen/pm": "pm_hexagon_room_64"}.get(scene, scene)


def film_of(name):
    import json
    import numpy as np
    return json.loads(str(np.load(os.path.join(GOLDEN, "film_kat.npz"))["films"]))[name] if name else None


def reached(case, prims_class, lite, k_default=50):
    """Launch<float> branches one render of `case` in fast mode takes (plus its closest-hit queries)"""
    film = "filter" if is_filtered(film_of(case.film)) else "box"
    fe = "ALL" if film == "filter" or not lite else "LITE"
    out = {"traceUser", f"generate<{film},list=0>", f"extend<{prims_class}>",
           "shadow<filter,ALL>" if film == "filter" else f"shadow<box,{prims_class}>"}
    if case.adaptive:
        out.add(f"generate<{film},list=1>")
    if not case.photon:
        out.add(f"shade<path,{film},{fe}>")
        return out
    out.add(f"shade<photon,{film},{fe}>")
    if case.gather:
        out.add(f"gather<{film},{fe}>")
    elif film == "filter":
        out.add("knn<0,filter,ALL>")
    else:
        out.add(f"knn<{knn_slots(case.k or k_default)},box,{fe}>")
    if case.emit:
        out |= {"emitGenerate", "emitShade"}
    return out


@pytest.fixture(scope="module")
def features():
    mcrt = load_package()
    cache = {}
    for c in CASES:
        name = pack_of(c.scene)
        if name not in cache:
            cache[name] = scene_features(mcrt, mcrt.Scene.from_pack(os.path.join(GOLDEN, name + ".mcrtpack")))
    return cache


def test_cases_reach_every_float_branch(features):
    got = set()
    for c in CASES:
        got |= reached(c, *features[pack_of(c.scene)])
    assert sorted(got) == EXPECTED, (sorted(set(EXPECTED) - got), sorted(got - set(EXPECTED)))


def test_scene_features_match_the_issue_table(features):
    # the golden scenes' classes, as the packs give them: a changed pack that drops a branch shows up here by name
    assert features["quadric_64"] == ("ALL", False)
    assert features["smooth_mesh_64"] == ("TRI", False)
    for c in ("c2_hexagon_room_96", "film_hexagon_room_64", "hexagon_room_octree_64", "pm_hexagon_room_64", "ior_test_nobvh_64"):
        assert features[c] == ("TRI_SPHERE", True), c
    for c in ("c1_hexagon_diffuse_256", "ggx_64", "metals_64", "oren_nayar_64", "veach_mis_64"):
        assert features[c] == ("TRI_SPHERE", False), c


def test_knn_slot_classes():
    assert [knn_slots(k) for k in PM_K] == [1, 2, 2, 4, 4, 8, 8, 0, 0]
    # photon.cuh knnSharedBytes with KNN_FRONTIER = KNN_HIST_BINS = 256 and 4 warps: k > 672 needs more than the default
    # 48 KB of dynamic shared memory, the launch that raises the kernel's attribute
    def shared_bytes(k):
        return 4 * (((k + 31) // 32 * 32) * 12 + 256 * 12 + 256 * 4)
    assert shared_bytes(672) <= 48 * 1024 < shared_bytes(673)
    assert any(k > 672 for k in PM_K)


def test_case_ids_are_unique():
    ids = [case_id(c) for c in CASES]
    assert len(ids) == len(set(ids))
