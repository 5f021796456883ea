"""CPU tests (no GPU) of the restatement's progressive photon mapping (oracle/mcrt_oracle.cpp: photonPass with a pass
index, gatherBrute and photonEstimate with a gather radius), pinned to what tests/test_photon_mapper_oracle_cpu.py already
pins to the reference's pm_hexagon_room_64:
    pass index     pass 0 is the reference's photon pass bit for bit; passes 0..P-1 of E emissions are the pieces of the one
                   pass of P * E emissions (emission indices, positions and directions equal, flux P times as large); a pass
                   whose emission indices do not fit 32 bits is refused at the pass the device refuses
    gather         the brute-force fixed-radius search equals test_ppm_cpu.gather_reference
    estimate       gathering within the k-th nearest photon's distance gives the k-NN estimate, which is the reference's: the
                   one thing that ties the fixed-radius estimate to the reference-pinned one
    components     in gather mode the four terms still add up to each sample's radiance
tests/test_gpu_ppm_oracle.py then holds the device's passes and gather estimates to this restatement."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import port
from test_ppm_cpu import emission_counts, gather_reference, union_passes

CID = "pm_hexagon_room_64"
TOL = 1e-12
NAMES = ("caustic", "global")
MAP_KEYS = ("octant_bounds", "octant_start", "octant_count", "octant_next", "octant_leaf", "photons")


@pytest.fixture(scope="module")
def pack(mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, CID + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, CID + ".npz"))
    ps = port.PortScene(scene)
    pm = ps.photon_mapper(scene.photon_maps())
    yield scene, g, ps, pm
    pm.close()
    ps.close()


def params_of(scene):
    p = scene.extra["photon_emit_params"]
    return int(p[0]), float(p[1]), int(p[2]), p[3:9]


def emission_index(paths):
    return (paths & np.uint64(0xFFFFFFFF)).astype(np.int64)


# ---------------------------------------------------------------------------------------------- pass index
def test_pass_zero_is_the_reference_pass(pack):
    scene, g, ps, _ = pack
    emissions, cf, leaf, bounds = params_of(scene)
    ref = scene.photon_maps()
    default = ps.photon_pass(emissions, cf, leaf, bounds, int(g["seed"]))
    zero = ps.photon_pass(emissions, cf, leaf, bounds, int(g["seed"]), pass_index=0)
    n = emission_counts(scene, emissions, cf)
    assert zero[3] == default[3] == n.sum()
    for which in (0, 1):
        for key in MAP_KEYS:
            assert np.array_equal(zero[which][key], ref[which][key]), (NAMES[which], key)
            assert np.array_equal(default[which][key], zero[which][key]), (NAMES[which], key)
        assert np.array_equal(zero[4][which], default[4][which]) and np.array_equal(zero[2][which], default[2][which])
        assert (emission_index(zero[4][which]) < n[zero[2][which]]).all()


def test_passes_are_pieces_of_one_long_pass(pack):
    """Pass i of E emissions draws light l's emissions at [i n_l, (i + 1) n_l) with the flux of an E-emission map, so the
    union of passes 0..P-1 holds the photons of the one P * E pass: the same paths (light and emission index), at the same
    positions and directions, with P times the flux (rtol 2e-7, test_gpu_ppm's bar: the flux differs by rounding)."""
    scene, g, ps, _ = pack
    _, cf, leaf, bounds = params_of(scene)
    P = 3
    E = union_passes(scene, cf, P, range(2000, 2200))
    n = emission_counts(scene, E, cf)
    passes = [ps.photon_pass(E, cf, leaf, bounds, int(g["seed"]), pass_index=i) for i in range(P)]
    long = ps.photon_pass(P * E, cf, leaf, bounds, int(g["seed"]))
    for which in (0, 1):
        for i, p in enumerate(passes):
            idx = emission_index(p[4][which])
            lo = i * n[p[2][which]]
            assert ((idx >= lo) & (idx < lo + n[p[2][which]])).all(), (NAMES[which], i)
        union = np.concatenate([np.asarray(p[which]["photons"], np.float32).reshape(-1, 8) for p in passes])
        tags = np.concatenate([p[4][which] for p in passes])
        one = np.asarray(long[which]["photons"], np.float32).reshape(-1, 8)
        assert len(union) == len(one) > 0
        # key: path, then position and direction bits; each path stores at most one photon per vertex
        ku = np.column_stack([tags.view(np.uint32).reshape(-1, 2), union[:, 3:8].view(np.uint32)])
        ko = np.column_stack([long[4][which].view(np.uint32).reshape(-1, 2), one[:, 3:8].view(np.uint32)])
        ou, oo = np.lexsort(ku.T[::-1]), np.lexsort(ko.T[::-1])
        assert np.array_equal(ku[ou], ko[oo]), f"{NAMES[which]}: paths, positions or directions differ"
        np.testing.assert_allclose(union[ou, 0:3], P * one[oo, 0:3].astype(np.float64), rtol=2e-7, atol=0)


def test_pass_index_overflow_is_refused(pack):
    """The last pass whose emission indices fit 32 bits is the one test_gpu_ppm's test_pass_index_overflow_is_refused
    emits on the device; the next one is refused on both sides."""
    scene, g, ps, _ = pack
    _, cf, leaf, bounds = params_of(scene)
    n = emission_counts(scene, 4000, cf)
    last_ok = (1 << 32) // int(n.max()) - 1
    with pytest.raises(ValueError, match="32 bits"):
        ps.photon_pass(4000, cf, leaf, bounds, int(g["seed"]), pass_index=last_ok + 1)
    with pytest.raises(ValueError):
        ps.photon_pass(4000, cf, leaf, bounds, int(g["seed"]), pass_index=1 << 32)
    caustic, glob, lights, total, paths = ps.photon_pass(4000, cf, leaf, bounds, int(g["seed"]), pass_index=last_ok)
    assert total == n.sum() and len(caustic["photons"]) and len(glob["photons"])
    for which in (0, 1):
        idx = emission_index(paths[which])
        lo = last_ok * n[lights[which]]
        assert ((idx >= lo) & (idx < lo + n[lights[which]])).all()
        assert idx.max() >= 0xFFFFFFFF - 2 * int(n.max())   # the light with the most emissions reaches just below 2^32


# ---------------------------------------------------------------------------------------------- gather search
def test_gather_matches_brute_force_reference(pack):
    """test_gpu_ppm's test_gather_matches_brute_force on the reference's maps: jittered, uniform and on-the-sphere points"""
    scene, _, _, pm = pack
    rng = np.random.default_rng(11)
    lo, hi = scene.extra["scene_bounds"][:3], scene.extra["scene_bounds"][3:]
    for which, m in enumerate(scene.photon_maps()[:2]):
        pos = np.asarray(m["photons"], np.float32).reshape(-1, 8)[:, 3:6].astype(np.float64)
        pick = rng.choice(len(pos), 300, replace=False)
        jitter = pos[pick] + rng.normal(0.0, 0.05, (300, 3))
        uniform = rng.uniform(lo, hi, (300, 3))
        for radius in (1e-7, 0.05, 0.3125, 1.0, 4.0):
            on = pos[pick[:50]] + [0.6 * radius, 0.8 * radius, 0.0] if radius == 0.3125 else pos[pick[:50]] + [radius, 0.0, 0.0]
            pts = np.concatenate([jitter, uniform, on])
            cnt, f, c = pm.gather(which, pts, radius)
            rc, rf, rcone = gather_reference(m["photons"], pts, radius)
            assert np.array_equal(cnt, rc), (NAMES[which], radius)
            np.testing.assert_allclose(f, rf, rtol=TOL, atol=0)
            np.testing.assert_allclose(c, rcone, rtol=TOL, atol=1e-300)
            if radius in (0.3125, 1.0):
                assert (rc[600:] >= 1).all()
        assert (pm.gather(which, uniform, 1e-7)[0] == 0).all()


# ---------------------------------------------------------------------------------------------- estimate
def test_gather_at_the_kth_distance_is_the_knn_estimate(pack):
    """At the first vertex of the golden camera samples: where the k-th nearest photon's distance2 d2_k is a square in
    float64 (sqrt(d2_k)^2 == d2_k) and no photon left out shares it, the gather within r = sqrt(d2_k) takes exactly the k
    nearest photons and normalises with r^2 = d2_k, so it must give the k-NN estimate (which test_photon_mapper_oracle_cpu
    pins to the reference) to 1e-12."""
    _, g, _, pm = pack
    rays, pixel, sample, seed = g["ps_rays"], g["ps_pixel"], g["ps_sample"], int(g["seed"])
    for which in (0, 1):
        knn_est, pos, ran = pm.first_estimate(which, rays, pixel, sample, seed, 0.0)
        q = np.nonzero(ran)[0]
        _, d2, cnt, _ = pm.knn(which, pos[q])
        assert (cnt == pm.k).all()
        kth = d2[:, pm.k - 1]
        r = np.sqrt(kth)
        ok = r * r == kth
        # no photon beyond the k nearest at the same distance: gather at d2_k would take it too
        for j in np.nonzero(ok)[0]:
            n_at, _, _ = pm.gather(which, pos[q[j]], r[j])
            ok[j] = n_at[0] == pm.k
        use = q[ok]
        assert len(use) >= 0.3 * len(q) and len(use) >= 100, (NAMES[which], len(use), len(q))
        got, pos2, ran2 = pm.first_estimate(which, rays[use], pixel[use], sample[use], seed, r[ok])
        assert ran2.all() and np.array_equal(pos2, pos[use])
        assert (knn_est[use] > 0).any(axis=1).mean() > 0.5
        err = np.abs(got - knn_est[use]) / np.maximum(np.abs(knn_est[use]), 1e-300)
        assert err.max() <= TOL, (NAMES[which], float(err.max()))
        # a radius just short of d2_k drops the k-th photon: the estimate changes
        short, _, _ = pm.first_estimate(which, rays[use[:50]], pixel[use[:50]], sample[use[:50]], seed, np.nextafter(r[ok][:50], 0))
        assert not np.array_equal(short, got[:50])


def test_gather_mode_components_and_counts(pack):
    """With gather radii set, every sample's four terms still add up to its radiance; the estimate differs from the k-NN
    one; every query counts, those that take no photon too, and a fixed radius has no ties. (0, 0) restores k-NN."""
    _, g, ps, pm = pack
    rays, pixel, sample, seed = g["ps_rays"], g["ps_pixel"], g["ps_sample"], int(g["seed"])
    knn_rgb, _, knn_counts = pm.sample_rays(rays, pixel, sample, seed)
    assert knn_counts["empty_queries"] == 0 and knn_counts["photons"] == pm.k * knn_counts["knn_queries"]
    seen = {}
    for rc, rg in ((0.4, 0.6), (0.004, 0.006), (0.2, 20.0)):
        pm.gather_radius(rc, rg)
        try:
            rgb, comp, counts = pm.sample_rays(rays, pixel, sample, seed)
        finally:
            pm.gather_radius(0, 0)
        assert np.abs(comp.sum(axis=1) - rgb).max() <= TOL * max(1.0, np.abs(rgb).max())
        assert (comp >= 0).all() and np.isfinite(rgb).all()
        assert counts["knn_ties"] == 0 and counts["knn_queries"] == knn_counts["knn_queries"]
        assert counts["rays"] == knn_counts["rays"] and counts["shadow_rays"] == knn_counts["shadow_rays"]
        assert not np.allclose(rgb, knn_rgb, rtol=1e-6)
        seen[rc] = counts
    assert seen[0.004]["empty_queries"] > 0.5 * seen[0.004]["knn_queries"]
    assert seen[0.4]["empty_queries"] < seen[0.004]["empty_queries"]
    assert seen[0.2]["photons"] > seen[0.4]["photons"]
    again, _, counts = pm.sample_rays(rays, pixel, sample, seed)
    assert np.array_equal(again, knn_rgb) and counts == knn_counts
    for bad in ((0.5, 0.0), (-1.0, 1.0), (float("inf"), 1.0), (float("nan"), 1.0), (1e200, 1.0)):
        with pytest.raises(ValueError):
            pm.gather_radius(*bad)
