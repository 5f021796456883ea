"""CPU checks of the denoiser guides taken after perfectly specular bounces: the restatement's chain
(tests/specular_chain_ref.cpp, which the GPU tests hold mcrt_render_features_chain_dev to) against the first-hit guides of
oracle/denoise_ref.py and against the rule that a chain ends on the first non-delta material."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases
from oracle import denoise_ref as dr
import specular_chain_ref as scr

W, H, SPP = 20, 12, 2


def setup(mcrt, cid):
    from oracle import port
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    cam = scene.cameras()[0].resized(W, H)
    n = cam.width * cam.height
    pixel = np.repeat(np.arange(n, dtype=np.uint32), SPP)
    sample = np.tile(np.arange(SPP, dtype=np.uint32), n)
    return port.PortScene(scene), scene, cam, pixel, sample, int(g["seed"])


def delta_prims(scene, prims, no_prim):
    """True where the primitive's material is dirac_delta (False for misses)."""
    a = scene.a
    hit = prims != no_prim
    out = np.zeros(len(prims), bool)
    out[hit] = a["materials"]["dirac_delta"][a["prim_material"][prims[hit].astype(np.int64)]] != 0
    return out


@pytest.mark.parametrize("cid", golden_cases())
def test_depth_0_is_the_first_hit_guide(cid, mcrt):
    ps, scene, cam, pixel, sample, seed = setup(mcrt, cid)
    try:
        _, rays = ps.sample_pixels(cam, pixel, sample, seed)
        hits = ps.trace(rays)
        got, end = scr.specular_chain(scene, cam, pixel, sample, seed, 0)
    finally:
        ps.close()
    want = dr.hit_features(scene, rays, hits, mcrt.PRIM_TRIANGLE, mcrt.PRIM_SPHERE, mcrt.NO_PRIM)
    assert np.array_equal(got[:, 7], want[:, 7])
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
    assert np.array_equal(end[:, 0], hits["prim"]) and not end[:, 1].any() and not end[:, 2].any()


@pytest.mark.parametrize("cid", golden_cases())
def test_chains_end_on_a_non_delta_material(cid, mcrt):
    ps, scene, cam, pixel, sample, seed = setup(mcrt, cid)
    D = mcrt.FEATURES_MAX_SPECULAR_DEPTH
    try:
        got, end = scr.specular_chain(scene, cam, pixel, sample, seed, D)
    finally:
        ps.close()
    prim, depth, terminated = end[:, 0], end[:, 1], end[:, 2] != 0
    hit = prim != mcrt.NO_PRIM
    assert np.array_equal(got[:, 7], hit.astype(np.float64))
    assert (depth <= D).all()
    free = hit & (depth < D) & ~terminated
    assert not delta_prims(scene, prim[free], mcrt.NO_PRIM).any()
    # a chain only ever stops early on a delta material when its bounce was rejected
    assert delta_prims(scene, prim[hit & terminated], mcrt.NO_PRIM).all()
    # the guide's depth is a path length: at least the first hit's distance
    assert (got[hit, 6] > 0).all()
    # the normal is a unit vector; the weighted albedo stays finite and non-negative
    np.testing.assert_allclose(np.linalg.norm(got[hit, 3:6], axis=1), 1.0, rtol=1e-9)
    assert np.isfinite(got).all() and (got[:, 0:3] >= 0).all()


@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "ior_test_nobvh_64", "smooth_mesh_64", "quadric_64"])
def test_depth_1_moves_only_the_delta_first_hits(cid, mcrt):
    ps, scene, cam, pixel, sample, seed = setup(mcrt, cid)
    try:
        _, rays = ps.sample_pixels(cam, pixel, sample, seed)
        first = ps.trace(rays)["prim"]
        g0, _ = scr.specular_chain(scene, cam, pixel, sample, seed, 0)
        g1, _ = scr.specular_chain(scene, cam, pixel, sample, seed, 1)
    finally:
        ps.close()
    delta = delta_prims(scene, first, mcrt.NO_PRIM)
    assert np.array_equal(g1[~delta], g0[~delta])
    assert delta.any(), "the scene has delta materials in view"
    differs = (g1[delta] != g0[delta]).any(axis=1)
    assert differs.mean() > 0.5
