"""The order-free search over the BVH4 with spatial splits (option bvh4_split, on by default below 4096 primitives) against the same
search over the tree without them and against the reference-order replay: bit-equal closest hits, the same paths, equal frames."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases

CASES = [c for c in golden_cases() if c != "ior_test_nobvh_64"]


def _rays(mcrt, pt, base, rng, n=100_000):
    h = pt.intersect(base)
    ok = h["prim"] != mcrt.NO_PRIM
    pts = base[ok, :3] + base[ok, 3:] * h["t"][ok, None]
    a = pts[rng.integers(0, len(pts), n)]
    d = pts[rng.integers(0, len(pts), n)] + rng.normal(0, 1e-3, (n, 3)) - a
    nrm = np.linalg.norm(d, axis=1, keepdims=True)
    keep = nrm[:, 0] > 1e-9
    d2 = rng.normal(size=(n, 3)); d2 /= np.linalg.norm(d2, axis=1, keepdims=True)
    return np.concatenate([base, np.concatenate([a[keep], d[keep] / nrm[keep]], 1), np.concatenate([a + 1e-9 * d2, d2], 1)])


@pytest.mark.gpu
@pytest.mark.parametrize("cid", CASES)
def test_intersect_split_equals_unsplit_and_reference_order(cid, mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    pt = mcrt.PathTracer(scene, device=0, precision=mcrt.PRECISION_F64, global_seed=int(g["seed"]))
    try:
        rays = _rays(mcrt, pt, g["tr_rays"], np.random.default_rng(17))
        split = pt.intersect(rays)
        pt.set_option("exact_traversal", 1)
        exact = pt.intersect(rays)
        pt.set_option("exact_traversal", 0)
        pt.set_option("bvh4_split", 0)
        pt.upload_scene()
        unsplit = pt.intersect(rays)
        for f in ("prim", "t", "u", "v", "interpolate"):
            assert np.array_equal(split[f], unsplit[f]), f
            assert np.array_equal(split[f], exact[f]), f
    finally:
        pt.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "c1_hexagon_diffuse_256", "veach_mis_64", "smooth_mesh_64", "quadric_64"])
def test_render_split_equals_unsplit(cid, mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    cam = scene.cameras()[0]
    out = []
    for split in (1, 0):
        pt = mcrt.PathTracer(scene, device=0, precision=mcrt.PRECISION_F64, global_seed=int(g["seed"]))
        try:
            pt.set_option("bvh4_split", split)
            pt.upload_scene()
            img = pt.render_rows(cam)
            out.append((img, pt.last_stats))
        finally:
            pt.close()
    (a, sa), (b, sb) = out
    assert (sa["extension_rays"], sa["shadow_rays"]) == (sb["extension_rays"], sb["shadow_rays"])
    assert np.allclose(a, b, rtol=1e-12, atol=0.0)
