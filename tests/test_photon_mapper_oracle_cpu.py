"""CPU tests (no GPU) of the photon-mapper restatement (oracle/mcrt_oracle.cpp: photonPass, pmSampleRay) against the
reference's outputs in pm_hexagon_room_64 (2 triangle lights, smooth glass, a mirror, Lambertian walls; k = 50,
caustic_factor 10, 200 photons per leaf, direct_visualization off):
    emission       the pack's maps from the pack's photon-pass parameters: every octree array and every photon record
                   equal bit for bit, photon order inside the leaves included (the pack was made by a single-threaded
                   reference pass; its leaves hold their photons in reverse emission order)
    sampleRay      ps_rgb and the frame at |d| <= 1e-12 max(1, |ref|) on the pack's maps (Photon::dir calls glibc's
                   sinf / cosf on both sides), Scene::intersect calls and shadow rays equal
    k-NN           the brute-force search returns the reference's distances and photon positions
    components     the four terms of every sample add up to its radiance
tests/test_gpu_photon_mapper.py then holds the device to this restatement on every lit golden scene and material case."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import port

CID = "pm_hexagon_room_64"
TOL = 1e-12
NAMES = ("caustic", "global")


@pytest.fixture(scope="module")
def pack(mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, CID + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, CID + ".npz"))
    ps = port.PortScene(scene)
    pm = ps.photon_mapper(scene.photon_maps())
    yield scene, g, ps, pm
    pm.close()
    ps.close()


def test_emission_equals_reference_maps(mcrt, pack):
    scene, g, ps, _ = pack
    params = scene.extra["photon_emit_params"]
    ref = scene.photon_maps()
    caustic, glob, lights, total, _ = ps.photon_pass(int(params[0]), float(params[1]), int(params[2]), params[3:9], int(g["seed"]))
    assert total == int(params[0] * params[1])
    for which, got in enumerate((caustic, glob)):
        for key in ("octant_bounds", "octant_start", "octant_count", "octant_next", "octant_leaf", "photons"):
            assert got[key].dtype == ref[which][key].dtype and np.array_equal(got[key], ref[which][key]), (NAMES[which], key)
        assert len(lights[which]) == len(got["photons"]) // 8
        assert np.array_equal(np.unique(lights[which]), np.arange(scene.n_lights)), NAMES[which]


def test_sample_ray(pack):
    _, g, _, pm = pack
    rgb, comp, counts = pm.sample_rays(g["ps_rays"], g["ps_pixel"], g["ps_sample"], int(g["seed"]))
    err = np.abs(rgb - g["ps_rgb"]) / np.maximum(1.0, np.abs(g["ps_rgb"]))
    assert err.max() <= TOL, f"worst {err.max():.3e}"
    assert counts["knn_ties"] == 0
    assert np.abs(comp.sum(axis=1) - rgb).max() <= TOL * max(1.0, np.abs(rgb).max())


def test_image(pack):
    scene, g, _, pm = pack
    cam = scene.cameras()[0]
    img, comp, counts = pm.render_rows(cam, 0, cam.height, cam.sqrtspp, int(g["seed"]))
    assert np.abs(img - g["image"]).max() <= TOL * max(1.0, np.abs(g["image"]).max())
    assert counts["rays"] == int(g["total_rays"]) and counts["shadow_rays"] == int(g["shadow_rays"])
    assert counts["knn_ties"] == 0
    assert np.abs(comp.sum(axis=0) - img).max() <= TOL * max(1.0, np.abs(img).max())


def test_knn_matches_reference(mcrt, pack):
    scene, g, _, pm = pack
    assert pm.k == int(g["knn_k"])
    maps = scene.photon_maps()
    for which, name in enumerate(NAMES):
        idx, d2, cnt, ties = pm.knn(which, g["knn_points"])
        assert ties == 0
        assert np.array_equal(cnt, g[f"knn_{name}_count"])
        for q in range(len(cnt)):
            n = int(cnt[q])
            assert np.array_equal(d2[q, :n], g[f"knn_{name}_d2"][q, :n]), (name, q)
            pos = maps[which]["photons"].reshape(-1, 8)[idx[q, :n], 3:6]
            assert np.array_equal(pos, g[f"knn_{name}_pos"][q, :n]), (name, q)


def test_knn_reports_ties(mcrt, pack):
    """Coincident photons at the k-th distance: which of them the reference takes follows its octree walk, so the brute-force
    search reports the tie instead of picking one silently."""
    _, _, ps, _ = pack
    ph = np.zeros((6, 8), np.float32)
    ph[:, 0:3] = 1.0
    ph[:, 3:6] = [[0, 0, 0], [1, 0, 0], [1, 0, 0], [0, 2, 0], [0, 0, 3], [0, 3, 0]]
    empty = {"photons": np.zeros(0, np.float32)}
    for k, want in ((1, 0), (2, 1), (3, 0), (4, 0), (5, 1), (6, 0), (9, 0)):
        pm = ps.photon_mapper(({"photons": ph.ravel()}, empty, k, 0))
        try:
            idx, d2, cnt, ties = pm.knn(0, np.zeros((1, 3)))
            assert ties == want, k
            assert cnt[0] == min(k, 6) and np.all(np.diff(d2[0, :cnt[0]]) >= 0)
            _, _, cnt, ties = pm.knn(1, np.zeros((1, 3)))
            assert cnt[0] == 0 and ties == 0
        finally:
            pm.close()


def test_components_split_the_radiance(pack):
    """The four terms add up to every sample's radiance; with direct_visualization on, every path ends in the global
    estimate at its first non-delta vertex, so no next-event estimate and no MIS-weighted emission is left."""
    scene, g, ps, pm = pack
    caustic, glob, k, _ = scene.photon_maps()
    for dv in (False, True):
        m = pm if not dv else ps.photon_mapper((caustic, glob, k, 1))
        try:
            rgb, comp, counts = m.sample_rays(g["ps_rays"], g["ps_pixel"], g["ps_sample"], int(g["seed"]))
        finally:
            if dv:
                m.close()
        assert np.abs(comp.sum(axis=1) - rgb).max() <= TOL * max(1.0, np.abs(rgb).max())
        assert (comp >= 0).all()
        for c in range(4):
            assert comp[:, c].max() > 0 or (dv and c == 1), (dv, c)
        if dv:
            assert not comp[:, 1].any() and counts["shadow_rays"] == 0
