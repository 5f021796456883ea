"""Scenes whose trees are deep enough to fill the traversal structures of parity and fast mode (DESIGN.md §8), and the rays that fill
them. Seeded; the trees are built by the CPU restatement of BVH::BVH (oracle/port.bvh_build), so the same scenes exist with and
without a GPU.

  nested shells   SHELLS spheres of radius 2^(-SHELL_STEP k) around the origin, each a sparse cloud of PER_SHELL small triangles,
                  inside the hexagon room; the only light is one triangle inside the innermost shell, so shadow rays start at the
                  bottom of the nest. Deep trees: every shell adds levels. A nest of 48 shells at a ratio of 2 fills the order-free
                  stack (40) and bounds the wide stack far above 48, but its heap peaks at 20 (octree) to 28; the heap needs many
                  more far sides of shells pending at once: 512 shells at a ratio of 2^(3/32) (innermost radius 2^-48 again) reach
                  112 on the octree.
  grazing grid    a bumpy floor of GRID x GRID quads in the same room, seen at grazing angles: a ray enters many boxes before its
                  first hit. The best-first heap keeps only boxes entered before the current best hit, and on this floor they are
                  few: its peak stays at 13, far below the nest's.

select_rays() draws candidate rays (out of the nest, into it, grazing over the grid, the room's camera rays) and keeps the ones with
the largest restated peaks (port.PortScene.trace_peaks / trace_fast_peaks)."""
import os

import numpy as np

from conftest import GOLDEN
from oracle import port

BASE = "c2_hexagon_room_96"
SHELLS = 512
SHELL_STEP = 3.0 / 32.0
PER_SHELL = 64
GRID = 192
BUILDERS = {"octree": 0, "binary_sah": 1, "quaternary_sah": 2}


def _append(mcrt, base, tri, light, bvh_type):
    """`base` (a Scene) with the triangles tri [n, 3, 3] appended in its first plain diffuse material and the reference's tree rebuilt by
    `bvh_type`. light: index into tri of the triangle that becomes the scene's only light (the room's lamps stay as unlit surfaces),
    or None."""
    flat = base.unbuilt()
    a = dict(flat.a, **flat.extra)
    a["scene_ior"] = np.array([flat.ior])
    mats = a["materials"].copy()
    plain = (mats["dirac_delta"] == 0) & (mats["rough_specular"] == 0) & (mats["perfect_mirror"] == 0) & (mats["transparency"] == 0)
    diffuse = int(np.nonzero(plain & (mats["emissive"] == 0))[0][0])
    material = np.full(len(tri), diffuse)
    if light is not None:
        lamp = mats[diffuse].copy()
        lamp["emissive"] = 1; lamp["emittance"] = (1e4, 1e4, 1e4); lamp["reflectance"] = (0.0, 0.0, 0.0)
        mats["emissive"] = 0
        mats = np.concatenate([mats, [lamp]])
        material[light] = len(mats) - 1
    a["materials"] = mats
    v0, v1, v2 = tri[:, 0], tri[:, 1], tri[:, 2]
    e1, e2 = v1 - v0, v2 - v0
    cross = np.cross(e1, e2)
    length = np.sqrt(np.sum(cross * cross, axis=1))
    assert (length > 0).all()
    n_tri0, n_prim0, m = a["tri_vn_index"].size, a["prim_type"].size, len(tri)
    for k, v in (("tri_v0", v0), ("tri_v1", v1), ("tri_v2", v2), ("tri_e1", e1), ("tri_e2", e2), ("tri_normal", cross / length[:, None])):
        a[k] = np.concatenate([a[k], v.reshape(-1)])
    a["tri_vn_index"] = np.concatenate([a["tri_vn_index"], np.full(m, -1, a["tri_vn_index"].dtype)])
    a["prim_type"] = np.concatenate([a["prim_type"], np.full(m, mcrt.PRIM_TRIANGLE, a["prim_type"].dtype)])
    a["prim_index"] = np.concatenate([a["prim_index"], (n_tri0 + np.arange(m)).astype(a["prim_index"].dtype)])
    a["prim_material"] = np.concatenate([a["prim_material"], material.astype(a["prim_material"].dtype)])
    a["prim_area"] = np.concatenate([a["prim_area"], 0.5 * length])
    a["prim_original"] = np.arange(n_prim0 + m, dtype=a["prim_original"].dtype)
    if light is not None:
        a["light_prim"] = np.array([n_prim0 + light], dtype=a["light_prim"].dtype)
        a["light_cdf"] = np.array([1.0])
    bounds = np.asarray(base.extra["scene_bounds"], dtype=np.float64)
    a["scene_bounds"] = np.concatenate([np.minimum(bounds[:3], tri.reshape(-1, 3).min(axis=0)), np.maximum(bounds[3:], tri.reshape(-1, 3).max(axis=0))])
    s = mcrt.Scene(a)
    bins = int(base.extra["bvh_params"][2])
    return s.with_bvh(port.bvh_build(s.prim_bounds(), a["scene_bounds"], bvh_type, bins, mcrt.BvhDesc))


def _small_triangles(centre, size, rng):
    """one triangle of circumradius `size` per centre, in a random plane through it"""
    n = len(centre)
    a = rng.normal(size=(n, 3)); a /= np.linalg.norm(a, axis=1, keepdims=True)
    b = np.cross(a, rng.normal(size=(n, 3))); b /= np.linalg.norm(b, axis=1, keepdims=True)
    ang = rng.uniform(0, 2 * np.pi, (n, 1)) + np.array([0.0, 2 * np.pi / 3, 4 * np.pi / 3])
    return centre[:, None, :] + size[:, None, None] * (np.cos(ang)[..., None] * a[:, None, :] + np.sin(ang)[..., None] * b[:, None, :])


def base_scene(mcrt):
    return mcrt.Scene.from_pack(os.path.join(GOLDEN, BASE + ".mcrtpack"))


def nested_shells(mcrt, builder, shells=SHELLS, seed=11):
    """-> Scene: shell k (k < shells) holds PER_SHELL triangles of circumradius 0.02 r_k centred on the sphere of radius
    r_k = 2^(-SHELL_STEP k); the light is the last triangle, at 0.37 r_(shells-1) from the origin."""
    rng = np.random.default_rng(seed)
    radius = np.repeat(2.0 ** (-SHELL_STEP * np.arange(shells)), PER_SHELL)
    d = rng.normal(size=(len(radius), 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    tri = _small_triangles(d * radius[:, None], 0.02 * radius, rng)
    inner = 2.0 ** (-SHELL_STEP * (shells - 1))
    lamp = _small_triangles(np.array([[0.3 * inner, 0.1 * inner, -0.2 * inner]]), np.array([0.1 * inner]), rng)
    return _append(mcrt, base_scene(mcrt), np.concatenate([tri, lamp]), len(tri), BUILDERS[builder])


def grazing_grid(mcrt, builder, n=GRID, seed=12):
    """-> Scene: an n x n grid of quads (two triangles each) over x in [-1.5, 11.5], z in [-5, 5] at height -4 plus a seeded bump of up to
    0.02 per vertex, so that the boxes have height and a grazing ray enters many of them"""
    rng = np.random.default_rng(seed)
    x = np.linspace(-1.5, 11.5, n + 1); z = np.linspace(-5.0, 5.0, n + 1)
    X, Z = np.meshgrid(x, z, indexing="ij")
    Y = -4.0 + 0.02 * rng.random(X.shape)
    P = np.stack([X, Y, Z], axis=-1)
    p00, p10, p01, p11 = P[:-1, :-1].reshape(-1, 3), P[1:, :-1].reshape(-1, 3), P[:-1, 1:].reshape(-1, 3), P[1:, 1:].reshape(-1, 3)
    tri = np.concatenate([np.stack([p00, p10, p11], axis=1), np.stack([p00, p11, p01], axis=1)])
    return _append(mcrt, base_scene(mcrt), tri, None, BUILDERS[builder])


def scene_scale(scene):
    """ctx->scene_scale as mcrt_scene_upload computes it (float)"""
    return float(np.float32(np.abs(scene.a["node_bounds"][:6]).max()))


def wide_stack_bound(scene):
    """The most entries fast mode's depth-first stack (traverseWide, intersect.cuh) can hold on this tree: the largest sum of
    (children - 1) over the inner nodes of one root-to-leaf path of the reference's tree."""
    count, nxt = scene.a["node_prim_count"], scene.a["node_next_sibling"]
    best = np.zeros(len(count), dtype=np.int64)
    for node in range(len(count) - 1, -1, -1):      # children follow their parent: node + 1, then next_sibling
        if count[node]:
            continue
        child, k, deepest = node + 1, 0, 0
        while child != 0:
            k += 1; deepest = max(deepest, best[child]); child = int(nxt[child])
        best[node] = k - 1 + deepest
    return int(best[0])


def _unit(v):
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def candidate_rays(mcrt, scene, kind, n, seed):
    """n seeded rays [n, 6]. kind: "out" (from points near the origin at every shell's scale, outwards), "in" (from the room towards
    points near the origin), "graze" (over the grid at 0.05 to 3 degrees), "camera" (the room camera's rays)."""
    rng = np.random.default_rng(seed)
    if kind == "out":
        o = _unit(rng.normal(size=(n, 3))) * (2.0 ** -rng.uniform(0, SHELLS * SHELL_STEP, (n, 1)))
        return np.concatenate([o, _unit(rng.normal(size=(n, 3)))], axis=1)
    if kind == "in":
        o = np.array([5.0, 0.0, 0.0]) + rng.uniform(-1, 1, (n, 3)) * (2.5, 4.0, 5.0)
        target = _unit(rng.normal(size=(n, 3))) * (2.0 ** -rng.uniform(0, SHELLS * SHELL_STEP, (n, 1)))
        return np.concatenate([o, _unit(target - o)], axis=1)
    if kind == "graze":
        o = np.stack([rng.uniform(-1.4, 0.0, n), -4.0 + rng.uniform(0.021, 0.2, n), rng.uniform(-4.9, 4.9, n)], axis=1)
        elev = np.radians(rng.uniform(0.05, 3.0, n)); az = rng.uniform(-0.6, 0.6, n)
        d = np.stack([np.cos(elev) * np.cos(az), -np.sin(elev), np.cos(elev) * np.sin(az)], axis=1)
        return np.concatenate([o, d], axis=1)
    assert kind == "camera"
    cam = scene.cameras()[0]
    ps = port.PortScene(scene)
    try:
        pixel = rng.integers(0, cam.width * cam.height, n).astype(np.uint32)
        _, rays = ps.sample_pixels(cam, pixel, np.zeros(n, np.uint32), 7)
    finally:
        ps.close()
    return rays


def select_rays(mcrt, scene, kinds, n=20000, keep=256, seed=5):
    """Candidates of every kind, then the `keep` rays with the largest order-free stack peaks and the `keep` with the largest replay
    heap peaks. -> dict(rays, heap_peak, stack_peak, flagged, ref) over the kept rays"""
    rays = np.concatenate([candidate_rays(mcrt, scene, k, n, seed + i) for i, k in enumerate(kinds)])
    ps = port.PortScene(scene)
    try:
        ref, heap = ps.trace_peaks(rays)
        _, flagged, stack = ps.trace_fast_peaks(mcrt.bvh4_host(scene), scene_scale(scene), rays)
    finally:
        ps.close()
    pick = np.unique(np.concatenate([np.argsort(-stack.astype(np.int64), kind="stable")[:keep],
                                     np.argsort(-heap.astype(np.int64), kind="stable")[:keep]]))
    return dict(rays=rays[pick], heap_peak=heap[pick], stack_peak=stack[pick], flagged=flagged[pick], ref=ref[pick])
