"""CPU-side checks (no GPU): the C-ABI library loads and exports every symbol include/mcrt_abi.h
declares, scene packs parse, compute calls fail loudly without a device (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, golden_cases


def test_library_exports_every_declared_symbol(mcrt):
    header = open(os.path.join(ROOT, "include", "mcrt_abi.h")).read()
    declared = set(re.findall(r"\b(mcrt_[a-z_0-9]+)\s*\(", header))
    assert declared == set(mcrt.ABI_SYMBOLS)
    L = mcrt.lib()
    for sym in declared:
        assert hasattr(L, sym), sym
    assert L.mcrt_abi_version() == 1


def test_struct_layouts_match_header(mcrt):
    assert C.sizeof(mcrt.MaterialRec) == 26 * 8 + 8 * 4
    assert C.sizeof(mcrt.CameraRec) == 12 * 8 + 4 * 8 + 16
    assert C.sizeof(mcrt.HitRec) == 32
    assert mcrt.HIT_DTYPE.itemsize == 32


@pytest.mark.parametrize("cid", golden_cases())
def test_scene_pack_is_consistent(cid, mcrt):
    check_scene_is_consistent(mcrt, mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack")))


def check_scene_is_consistent(mcrt, scene):
    a = scene.a
    n = scene.n_prims
    assert n > 0 and a["prim_index"].size == n and a["prim_material"].size == n and a["prim_area"].size == n
    assert a["prim_material"].max() < a["materials"].size
    tri = a["prim_type"] == mcrt.PRIM_TRIANGLE
    assert tri.sum() == a["tri_vn_index"].size
    if scene.n_nodes:
        leaves = a["node_prim_count"] > 0
        # every primitive belongs to exactly one leaf
        cover = np.zeros(n, dtype=int)
        for f, c in zip(a["node_first_prim"][leaves], a["node_prim_count"][leaves]):
            cover[f:f + c] += 1
        assert np.all(cover == 1)
    if scene.n_lights:
        assert np.all(np.diff(a["light_cdf"]) >= 0) and abs(a["light_cdf"][-1] - 1.0) < 1e-12
        assert np.all(a["materials"]["emissive"][a["prim_material"][a["light_prim"]]] == 1)
    cam = scene.cameras()[0]
    assert cam.width > 0 and cam.height > 0


def test_no_cpu_fallback(mcrt):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "c1_hexagon_diffuse_256.mcrtpack"))
    with pytest.raises(mcrt.McrtError):
        mcrt.PathTracer(scene)


def test_shard_rows_partition(mcrt):
    for h in (1, 7, 54, 1080, 2160):
        for n in (1, 2, 3, 4, 8):
            blocks = [mcrt.shard_rows(h, r, n) for r in range(n)]
            assert blocks[0][0] == 0 and blocks[-1][1] == h
            assert all(blocks[i][1] == blocks[i + 1][0] for i in range(n - 1))
            sizes = [b - a for a, b in blocks]
            assert max(sizes) - min(sizes) <= 1


def test_python_mirror_is_complete(mcrt):
    # the helpers the GPU tests and tools call must exist (catches an accidentally dropped function on CPU)
    for name in ("Scene", "Camera", "PathTracer", "PhotonMapper", "read_pack", "bvh_build", "build_photon_octree", "load_obj",
                 "vertex_normals", "shard_rows", "ImageParams", "FILM_FILTERS", "BVH_TYPES"):
        assert hasattr(mcrt, name), name
    for name in ("render_rows", "render_rows_dev", "render_rows_strided_dev", "sampleRay", "intersect", "tonemap", "tonemap_dev",
                 "set_film", "set_option", "sampler_stream"):
        assert hasattr(mcrt.Integrator, name), name
    for name in ("prim_bounds", "reordered", "unbuilt", "with_bvh", "cameras", "photon_maps"):
        assert hasattr(mcrt.Scene, name), name


def test_scene_reorder_round_trip(mcrt):
    """Scene.unbuilt() / with_bvh(): taking a packed scene back to Scene::surfaces order and re-attaching
    the tree it was built with must give back the packed arrays (the host-side half of mcrt_bvh_build)."""
    import os
    import numpy as np
    from conftest import GOLDEN
    for cid in ("c2_hexagon_room_96", "quadric_64", "veach_mis_64"):
        scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
        flat = scene.unbuilt()
        assert flat.n_nodes == 0 and np.array_equal(flat.extra["prim_original"], np.arange(flat.n_prims))
        # boxes follow the primitives through the permutation
        assert np.array_equal(flat.prim_bounds()[scene.extra["prim_original"]], scene.prim_bounds())
        tree = {k: scene.a[k] for k in ("node_bounds", "node_first_prim", "node_prim_count", "node_next_sibling")}
        tree["prim_order"] = scene.extra["prim_original"]
        back = flat.with_bvh(tree)
        for k in mcrt.Scene._ARRAYS:
            assert np.array_equal(back.a[k], scene.a[k]), (cid, k)
        # every leaf box contains the boxes of its primitives; the root box is Scene::BB()
        b = scene.prim_bounds()
        nb = scene.a["node_bounds"].reshape(-1, 6)
        for n in np.nonzero(scene.a["node_prim_count"])[0]:
            f, c = int(scene.a["node_first_prim"][n]), int(scene.a["node_prim_count"][n])
            assert (b[f:f + c, :3] >= nb[n, :3]).all() and (b[f:f + c, 3:] <= nb[n, 3:]).all()
        assert np.array_equal(nb[0], scene.extra["scene_bounds"])
