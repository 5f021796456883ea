"""Large scenes generated from the golden ones, for the paths the wavefront selects by scene size (DESIGN.md §8): a golden scene
with tens of thousands of seeded triangles appended, its BVH rebuilt by the CPU restatement of BVH::BVH (oracle/port.bvh_build,
pinned to the reference's trees by tests/test_bvh_oracle_cpu.py), so the same scene is available with and without a GPU."""
import os

import numpy as np

from conftest import GOLDEN
from oracle import port

# (base golden scene, appended triangles, seed); each crosses 2048 BVH4 nodes and 4096 primitives
GENERATED = {
    "mesh": ("smooth_mesh_64", 60000, 1),
    "room": ("c2_hexagon_room_96", 60000, 2),
    "quadric": ("quadric_64", 60000, 3),
    "pm": ("pm_hexagon_room_64", 60000, 4),
}
N_DUPLICATES = 512
# where the triangles go when not inside the base scene's bounds: quadric_64's bounds hold its unbounded surfaces' clip boxes, the
# camera sees this part of them
REGION = {"quadric": ((-0.9, -0.15, -3.5), (3.3, 1.5, 5.0))}


def _triangles(rng, lo, hi, n):
    """[n, 3, 3] vertices: clusters of small triangles with empty space between them, strips of triangles that share edges, and
    N_DUPLICATES exact copies of cluster triangles (the last ones); -> (vertices, index of the triangle each copy copies)"""
    ext = hi - lo
    n_strip = n // 5
    n_cluster = n - n_strip - N_DUPLICATES
    # ~300 triangles per cluster around centres spread over the middle of the scene
    n_centres = max(1, n_cluster // 300)
    centres = lo + ext * (0.1 + 0.8 * rng.random((n_centres, 3)))
    c = centres[rng.integers(0, n_centres, n_cluster)] + rng.normal(0, 0.02, (n_cluster, 3)) * ext
    size = 0.004 * ext.max() * rng.uniform(0.5, 2.0, (n_cluster, 1, 1))
    cluster = c[:, None, :] + size * rng.normal(size=(n_cluster, 3, 3))
    # strips of 50: triangle k of a strip is (p_k, p_k+1, p_k+2), so neighbours share an edge exactly
    strips = []
    per = 50
    for _ in range((n_strip + per - 1) // per):
        start = lo + ext * (0.1 + 0.8 * rng.random(3))
        step = rng.normal(size=3); step *= 0.01 * ext.max() / np.linalg.norm(step)
        side = rng.normal(size=3); side -= side.dot(step) / step.dot(step) * step
        side *= 0.01 * ext.max() / np.linalg.norm(side)
        k = np.arange(per + 2)
        pts = start + k[:, None] * step + (k % 2)[:, None] * side + rng.normal(0, 0.002 * ext.max(), (per + 2, 3))
        strips.append(np.stack([pts[:-2], pts[1:-1], pts[2:]], axis=1))
    strip = np.concatenate(strips)[:n_strip]
    src = rng.choice(n_cluster, N_DUPLICATES, replace=False)
    return np.concatenate([cluster, strip, cluster[src]]), src


def generated_scene(mcrt, name):
    base_name, n, seed = GENERATED[name]
    base = mcrt.Scene.from_pack(os.path.join(GOLDEN, base_name + ".mcrtpack"))
    return with_triangles(mcrt, base, n, seed, light=name == "quadric", region=REGION.get(name))


def with_triangles(mcrt, scene, n, seed, light=False, region=None):
    """`scene` with n seeded triangles appended (see _triangles) and the reference's BVH rebuilt over all primitives. The new
    triangles take the scene's non-emissive materials at random (glass and GGX included where the scene has them), a copy another
    material than its original. light: one more
    triangle, emissive, above the others, becomes the scene's only light (for a scene that has none). region: (lo, hi) of the box the
    triangles fill, default the scene's bounds."""
    flat = scene.unbuilt()
    a = dict(flat.a, **flat.extra)
    a["scene_ior"] = np.array([flat.ior])
    rng = np.random.default_rng(seed)
    bounds = np.asarray(scene.extra["scene_bounds"], dtype=np.float64)
    lo, hi = (bounds[:3], bounds[3:]) if region is None else (np.asarray(region[0], np.float64), np.asarray(region[1], np.float64))
    tri, src = _triangles(rng, lo, hi, n)
    mats = a["materials"]
    surface = np.nonzero(mats["emissive"] == 0)[0]
    pick = rng.integers(0, len(surface), len(tri))
    # a copy never shares its original's material: a tie decided unlike the reference's traversal order changes the shading
    pick[-N_DUPLICATES:] = (pick[src] + rng.integers(1, len(surface), N_DUPLICATES)) % len(surface)
    material = surface[pick]
    if light:
        assert scene.n_lights == 0
        plain = (mats["dirac_delta"] == 0) & (mats["rough_specular"] == 0) & (mats["perfect_mirror"] == 0) & (mats["transparency"] == 0)
        lamp = mats[np.nonzero(plain & (mats["emissive"] == 0))[0][0]].copy()
        lamp["emissive"] = 1; lamp["emittance"] = (40.0, 40.0, 40.0); lamp["reflectance"] = (0.0, 0.0, 0.0)
        a["materials"] = mats = np.concatenate([mats, [lamp]])
        c = lo + (hi - lo) * np.array([0.5, 1.0, 0.5])
        r = 0.1 * (hi - lo).max()
        tri = np.concatenate([tri, [[c + (-r, 0, -r), c + (r, 0, -r), c + (0, 0, r)]]])
        material = np.concatenate([material, [len(mats) - 1]])
    v0, v1, v2 = tri[:, 0], tri[:, 1], tri[:, 2]
    # Triangle::Triangle (triangle.cpp): E1, E2, the normal from their cross product, area = |E1 x E2| / 2
    e1, e2 = v1 - v0, v2 - v0
    cross = np.cross(e1, e2)
    length = np.sqrt(np.sum(cross * cross, axis=1))
    assert (length > 0).all()
    n_tri0 = a["tri_vn_index"].size
    n_prim0 = a["prim_type"].size
    for k, v in (("tri_v0", v0), ("tri_v1", v1), ("tri_v2", v2), ("tri_e1", e1), ("tri_e2", e2), ("tri_normal", cross / length[:, None])):
        a[k] = np.concatenate([a[k], v.reshape(-1)])
    m = len(tri)
    a["tri_vn_index"] = np.concatenate([a["tri_vn_index"], np.full(m, -1, a["tri_vn_index"].dtype)])
    a["prim_type"] = np.concatenate([a["prim_type"], np.full(m, mcrt.PRIM_TRIANGLE, a["prim_type"].dtype)])
    a["prim_index"] = np.concatenate([a["prim_index"], (n_tri0 + np.arange(m)).astype(a["prim_index"].dtype)])
    a["prim_material"] = np.concatenate([a["prim_material"], material.astype(a["prim_material"].dtype)])
    a["prim_area"] = np.concatenate([a["prim_area"], 0.5 * length])
    a["prim_original"] = np.arange(n_prim0 + m, dtype=a["prim_original"].dtype)   # unbuilt(): primitives in Scene::surfaces order
    if light:
        a["light_prim"] = np.array([n_prim0 + m - 1], dtype=a["light_prim"].dtype)
        a["light_cdf"] = np.array([1.0])
    lo_all = np.minimum(bounds[:3], tri.reshape(-1, 3).min(axis=0)); hi_all = np.maximum(bounds[3:], tri.reshape(-1, 3).max(axis=0))
    a["scene_bounds"] = np.concatenate([lo_all, hi_all])
    s = mcrt.Scene(a)
    _, bvh_type, bins = (int(v) for v in scene.extra["bvh_params"])
    return s.with_bvh(port.bvh_build(s.prim_bounds(), a["scene_bounds"], bvh_type, bins, mcrt.BvhDesc))
