"""The generated large scenes of tests/scene_gen.py on the CPU: they are well-formed, they are big enough for the auto settings to
select dynamic fetch, whole reference leaves in the BVH4 and source-primitive ray-sort keys, and on them the restated order-free search
(oracle_trace_fast) and occlusion query (oracle_trace_visible) answer every ray they do not flag as the reference-order traversal does.
The golden scenes are all below those thresholds; tests/test_gpu_schedules.py renders these scenes on the device."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import port
from scene_gen import GENERATED, N_DUPLICATES, generated_scene
from test_abi_cpu import check_scene_is_consistent
from test_fast_search_cpu import check_occlusion_query, check_unflagged_answers, search_rays

BVH4_DYNAMIC_FETCH_NODES = 2048     # abi.cu: dynamic_fetch auto
BIG_SCENE_PRIMS = 4096              # abi.cu: whole reference leaves (buildBvh4) and sort_prim_key auto


@pytest.fixture(scope="module")
def scenes(mcrt):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = generated_scene(mcrt, name)
        return cache[name]
    return get


def camera_rays(ps, scene, n, seed):
    cam = scene.cameras()[0]
    rng = np.random.default_rng(seed)
    pixel = rng.integers(0, cam.width * cam.height, n).astype(np.uint32)
    sample = rng.integers(0, cam.sqrtspp ** 2, n).astype(np.uint32)
    return ps.sample_pixels(cam, pixel, sample, 0x12345678)[1]


def duplicate_prims(mcrt, scene):
    """Primitives (in BVH order) that are triangles with exactly the same vertices as another primitive."""
    a = scene.a
    tri = np.nonzero(a["prim_type"] == mcrt.PRIM_TRIANGLE)[0]
    idx = a["prim_index"][tri]
    verts = np.concatenate([a[k].reshape(-1, 3)[idx] for k in ("tri_v0", "tri_v1", "tri_v2")], axis=1)
    _, inverse, counts = np.unique(verts, axis=0, return_inverse=True, return_counts=True)
    return tri[counts[inverse.reshape(-1)] > 1]


@pytest.mark.parametrize("name", sorted(GENERATED))
def test_generated_scene_is_consistent(name, mcrt, scenes):
    scene = scenes(name)
    base = mcrt.Scene.from_pack(os.path.join(GOLDEN, GENERATED[name][0] + ".mcrtpack"))
    check_scene_is_consistent(mcrt, scene)
    a = scene.a
    assert scene.n_prims >= BIG_SCENE_PRIMS
    nodes = mcrt.bvh4_host(scene)
    assert len(nodes) >= BVH4_DYNAMIC_FETCH_NODES, len(nodes)
    # the base scene's primitives are all there, in the BVH's order
    assert sorted(scene.extra["prim_original"].tolist()) == list(range(scene.n_prims))
    types = set(np.unique(a["prim_type"]).tolist())
    expected = {"mesh": {mcrt.PRIM_TRIANGLE}, "room": {mcrt.PRIM_TRIANGLE, mcrt.PRIM_SPHERE}, "pm": {mcrt.PRIM_TRIANGLE, mcrt.PRIM_SPHERE},
                "quadric": {mcrt.PRIM_TRIANGLE, mcrt.PRIM_QUADRIC}}[name]
    assert types == expected                                                    # PRIMS_TRI, PRIMS_TRI_SPHERE, PRIMS_ALL on the device
    dup = duplicate_prims(mcrt, scene)
    assert len(dup) == 2 * N_DUPLICATES
    v0 = a["tri_v0"].reshape(-1, 3)[a["prim_index"][dup]]
    order = np.lexsort(v0.T)                                                    # copies side by side
    pairs = dup[order].reshape(-1, 2)
    assert (a["prim_material"][pairs[:, 0]] != a["prim_material"][pairs[:, 1]]).all()
    # the appended triangles use the base scene's glass and GGX materials where it has them
    m = a["materials"][a["prim_material"]]
    bm = base.a["materials"]
    assert (m["transparency"] > 0).sum() > 1000 or not (bm["transparency"] > 0).any()
    assert (m["rough_specular"] > 0).sum() > 1000 or not (bm["rough_specular"] > 0).any()
    if name == "quadric":
        assert base.n_lights == 0 and scene.n_lights == 1 and np.array_equal(a["light_cdf"], [1.0])
    else:
        assert scene.n_lights == base.n_lights
    if name == "pm":
        assert scene.photon_maps() is not None


@pytest.mark.parametrize("name", sorted(GENERATED))
def test_unflagged_answers_equal_reference_order(name, mcrt, scenes):
    scene = scenes(name)
    g = np.load(os.path.join(GOLDEN, GENERATED[name][0] + ".npz"))
    ps = port.PortScene(scene)
    try:
        base = np.concatenate([camera_rays(ps, scene, 4096, 7), g["tr_rays"]])
        rays = search_rays(mcrt, ps, base, np.random.default_rng(3))
        # shared strip edges and duplicates are flagged more often than in the golden scenes, but still rarely
        check_unflagged_answers(mcrt, ps, mcrt.bvh4_host(scene), rays)
    finally:
        ps.close()


@pytest.mark.parametrize("name", sorted(GENERATED))
def test_rays_hitting_duplicates_are_flagged(name, mcrt, scenes):
    """A ray whose closest hit is one of two copies of a triangle has a tie the search cannot order: it must go to the replay."""
    scene = scenes(name)
    a = scene.a
    dup = duplicate_prims(mcrt, scene)
    rng = np.random.default_rng(13)
    idx = a["prim_index"][dup]
    v0, e1, e2 = (a[k].reshape(-1, 3)[idx] for k in ("tri_v0", "tri_e1", "tri_e2"))
    nrm = np.cross(e1, e2)
    area = np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm /= area
    rays = []
    for _ in range(4):
        u = rng.uniform(0.1, 0.4, (len(dup), 2))
        target = v0 + u[:, :1] * e1 + u[:, 1:] * e2
        off = 0.05 * np.sqrt(area)
        rays += [np.concatenate([target + off * nrm, -nrm], 1), np.concatenate([target - off * nrm, nrm], 1)]
    rays = np.concatenate(rays)
    ps = port.PortScene(scene)
    try:
        ref = ps.trace(rays)
        fast, flagged, _, _ = ps.trace_fast(mcrt.bvh4_host(scene), float(np.float32(np.abs(a["node_bounds"][:6]).max())), rays)
    finally:
        ps.close()
    hit_dup = np.isin(ref["prim"], dup)
    assert hit_dup.mean() > 0.9
    assert flagged[hit_dup].all()


@pytest.mark.parametrize("name", sorted(GENERATED))
def test_occlusion_query_equals_closest_hit_comparison(name, mcrt, scenes):
    scene = scenes(name)
    g = np.load(os.path.join(GOLDEN, GENERATED[name][0] + ".npz"))
    ps = port.PortScene(scene)
    try:
        base = np.concatenate([camera_rays(ps, scene, 4096, 8), g["tr_rays"]])
        check_occlusion_query(mcrt, ps, mcrt.bvh4_host(scene), base, np.random.default_rng(21), n=20000)
    finally:
        ps.close()
