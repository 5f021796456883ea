"""Progressive photon mapping on pm_hexagon_room_64: one photon map per pass (mcrt_photon_emit_pass), the
fixed-radius gather (k_gather, mcrt_photon_gather_search) against a float64 brute force and against the k-NN
search, the k-NN mode left as it was, and ProgressivePhotonMapping's resume, convergence and inherited machinery."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_ppm_cpu import emission_counts, gather_reference, union_passes

pytestmark = pytest.mark.gpu

CID = "pm_hexagon_room_64"


@pytest.fixture(scope="module")
def setup(mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, CID + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, CID + ".npz"))
    ep = scene.extra["photon_emit_params"]
    return scene, int(g["seed"]), float(ep[1]), int(ep[2])


@pytest.fixture(scope="module")
def pm(mcrt, setup):
    scene, seed, _, _ = setup
    p = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=seed)
    yield p
    p.close()


def host_maps(pm):
    caustic, glob, _, _ = pm._maps
    return caustic, glob


def rows(photons, cols=slice(0, 8)):
    """Photon records as sortable rows of their float32 bit patterns."""
    return np.ascontiguousarray(np.asarray(photons, np.float32).reshape(-1, 8)[:, cols]).view(np.uint32)


def sort_rows(r):
    return r[np.lexsort(r.T[::-1])]


def leaf_sorted(m):
    """The photons with each leaf's range sorted: the order inside a leaf follows the emission's atomics."""
    ph = np.asarray(m["photons"], np.float32).reshape(-1, 8).copy()
    for s, c, leaf in zip(m["octant_start"], m["octant_count"], m["octant_leaf"]):
        if leaf:
            ph[int(s):int(s + c)] = ph[int(s):int(s + c)][np.lexsort(rows(ph[int(s):int(s + c)]).T[::-1])]
    return ph


def rel_rmse(a, b):
    return float(np.sqrt(np.mean((a - b) ** 2)) / np.sqrt(np.mean(b ** 2)))


def down4(img):
    h, w = img.shape[0] // 4 * 4, img.shape[1] // 4 * 4
    return img[:h, :w].reshape(h // 4, 4, w // 4, 4, 3).mean(axis=(1, 3))


# ---------------------------------------------------------------------------------------------- 1. pass 0
def test_pass_zero_is_the_photon_pass(pm, setup):
    _, _, cf, leaf = setup
    pm.emit(4000, cf, leaf)
    a = host_maps(pm)
    n = pm.emit_pass(0, 4000, cf, leaf)
    b = host_maps(pm)
    assert n == tuple(len(m["photons"]) // 8 for m in a)
    for ma, mb in zip(a, b):
        for key in ("octant_bounds", "octant_start", "octant_count", "octant_next", "octant_leaf"):
            assert np.array_equal(ma[key], mb[key]), key
        assert np.array_equal(leaf_sorted(ma), leaf_sorted(mb))


# ---------------------------------------------------------------------------------------------- 2. union of passes
def test_passes_are_pieces_of_one_long_pass(mcrt, pm, setup):
    scene, _, cf, leaf = setup
    P = 3
    E = union_passes(scene, cf, P, range(2000, 2200))
    passes = []
    for i in range(P):
        pm.emit_pass(i, E, cf, leaf)
        passes.append(host_maps(pm))
    pm.emit(P * E, cf, leaf)
    long = host_maps(pm)
    for which in (0, 1):
        union = np.concatenate([np.asarray(p[which]["photons"], np.float32).reshape(-1, 8) for p in passes])
        one = np.asarray(long[which]["photons"], np.float32).reshape(-1, 8)
        assert len(union) == len(one) > 0
        ku, ko = rows(union, slice(3, 8)), rows(one, slice(3, 8))
        ou, oo = np.lexsort(ku.T[::-1]), np.lexsort(ko.T[::-1])
        assert np.array_equal(ku[ou], ko[oo]), f"map {which}: positions / directions differ"
        np.testing.assert_allclose(union[ou, 0:3], P * one[oo, 0:3].astype(np.float64), rtol=2e-7, atol=0)
        for i in range(P):
            for j in range(i + 1, P):
                a, b = (sort_rows(rows(p[which]["photons"])) for p in (passes[i], passes[j]))
                assert a.shape != b.shape or not np.array_equal(a, b), f"map {which}: passes {i} and {j} are equal"


def test_pass_index_overflow_is_refused(mcrt, pm, setup):
    scene, _, cf, leaf = setup
    n_max = int(emission_counts(scene, 4000, cf).max())
    last_ok = (1 << 32) // n_max - 1   # its last emission index is (last_ok + 1) * n_max - 1 < 2^32
    with pytest.raises(mcrt.McrtError):
        pm.emit_pass(last_ok + 1, 4000, cf, leaf)
    nc, ng = pm.emit_pass(last_ok, 4000, cf, leaf)
    assert nc > 0 and ng > 0


# ---------------------------------------------------------------------------------------------- 3. brute force
def test_gather_matches_brute_force(pm, setup):
    scene, _, cf, leaf = setup
    pm.emit_pass(1, 4000, cf, leaf)
    rng = np.random.default_rng(11)
    lo, hi = scene.extra["scene_bounds"][:3], scene.extra["scene_bounds"][3:]
    for which, m in enumerate(host_maps(pm)):
        pos = np.asarray(m["photons"], np.float32).reshape(-1, 8)[:, 3:6].astype(np.float64)
        pick = rng.choice(len(pos), 300, replace=False)
        jitter = pos[pick] + rng.normal(0.0, 0.05, (300, 3))
        uniform = rng.uniform(lo, hi, (300, 3))
        for radius in (1e-7, 0.05, 0.3125, 1.0, 4.0):
            # points exactly on the sphere around a photon: d^2 = (3/5 r)^2 + (4/5 r)^2 = r^2 in float64 for these radii
            on = pos[pick[:50]] + [0.6 * radius, 0.8 * radius, 0.0] if radius == 0.3125 else pos[pick[:50]] + [radius, 0.0, 0.0]
            pts = np.concatenate([jitter, uniform, on])
            cnt, f, c = pm.gather(which, pts, radius)
            rc, rf, rcone = gather_reference(m["photons"], pts, radius)
            assert np.array_equal(cnt, rc), (which, radius)
            np.testing.assert_allclose(f, rf, rtol=1e-12, atol=0)
            np.testing.assert_allclose(c, rcone, rtol=1e-12, atol=1e-300)
            if radius == 1e-7:
                assert (cnt[300:600] == 0).all()
            if radius == 4.0:
                assert cnt.max() > 4 * leaf   # spans several leaves
            if radius in (0.3125, 1.0):
                assert (rc[600:] >= 1).all()


# ---------------------------------------------------------------------------------------------- 4. against k-NN
def test_gather_agrees_with_knn(pm, setup):
    _, _, cf, leaf = setup
    pm.emit_pass(2, 4000, cf, leaf)
    rng = np.random.default_rng(12)
    k = pm.k_nearest
    for which, m in enumerate(host_maps(pm)):
        ph = np.asarray(m["photons"], np.float32).reshape(-1, 8)
        pts = ph[rng.choice(len(ph), 64, replace=False), 3:6].astype(np.float64) + rng.normal(0.0, 0.02, (64, 3))
        idx, d2, cnt = pm.knn(which, pts)
        used = 0
        for q in range(len(pts)):
            r2 = d2[q, :cnt[q]].max()
            cands = [r for r in (np.sqrt(r2), np.nextafter(np.sqrt(r2), 0), np.nextafter(np.sqrt(r2), np.inf)) if r * r == r2]
            if not cands:
                continue
            n, f, _ = pm.gather(which, pts[q:q + 1], cands[0])
            assert n[0] == k
            np.testing.assert_allclose(f[0], ph[idx[q], 0:3].astype(np.float64).sum(0), rtol=1e-12)
            used += 1
        assert used >= 16


# ---------------------------------------------------------------------------------------------- 5. k-NN untouched
def test_knn_mode_is_untouched(mcrt, pm, setup):
    scene, _, cf, leaf = setup
    cam = scene.cameras()[0]
    pm.emit(4000, cf, leaf)
    before = pm.render_rows(cam, sqrtspp=2)
    pm.gather_radius(0.5, 0.5)
    gathered = pm.render_rows(cam, sqrtspp=2)
    pm.gather_radius(0, 0)
    after = pm.render_rows(cam, sqrtspp=2)
    # not bit for bit: the float64 film takes its additions through atomics, so two renders of the same k-NN frame
    # differ in the last bits too; the bar is the repeatability one of the other render tests
    np.testing.assert_allclose(after, before, rtol=1e-12, atol=1e-14)
    assert not np.array_equal(before, gathered) and np.isfinite(gathered).all()
    for bad in ((0.5, 0.0), (-1.0, 1.0), (float("inf"), 1.0), (float("nan"), 1.0)):
        with pytest.raises(mcrt.McrtError):
            pm.gather_radius(*bad)


# ---------------------------------------------------------------------------------------------- 6. resume
def test_resume_equals_an_uninterrupted_run(mcrt, setup, tmp_path):
    scene, seed, cf, leaf = setup
    cam = scene.cameras()[0]
    kw = dict(max_photons_per_octree_leaf=leaf, alpha=0.7)

    def mapper(s=seed):
        return mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=s)

    pm1 = mapper()
    run = mcrt.ProgressivePhotonMapping(pm1, cam, 2000, cf, **kw)
    for _ in range(6):
        run.add(2)
    pm2 = mapper()
    first = mcrt.ProgressivePhotonMapping(pm2, cam, 2000, cf, **kw)
    for _ in range(3):
        first.add(2)
    path = str(tmp_path / "ppm.npz")
    first.save(path)
    pm3 = mapper()
    resumed = mcrt.ProgressivePhotonMapping.load(path, pm3, cam, 2000, cf, **kw)
    assert resumed.radius == run.radius and resumed.passes == 3
    for _ in range(3):
        resumed.add(2)
    np.testing.assert_allclose(resumed.frame(), run.frame(), rtol=1e-12, atol=1e-14)
    assert resumed.error()[0] == pytest.approx(run.error()[0], rel=1e-9)

    for what, args, kwargs, m in (("ppm_alpha", (2000, cf), dict(kw, alpha=0.5), pm3),
                                  ("ppm_emissions", (2001, cf), kw, pm3),
                                  ("ppm_radius", (2000, cf), dict(kw, radius=(0.3, 0.4)), pm3),
                                  ("seed", (2000, cf), kw, None)):
        other = m if m is not None else mapper(seed + 1)
        with pytest.raises(mcrt.McrtError, match=what):
            mcrt.ProgressivePhotonMapping.load(path, other, cam, *args, **kwargs)
        if m is None:
            other.close()
    for p in (pm1, pm2, pm3):
        p.close()


# ---------------------------------------------------------------------------------------------- 7. convergence
def test_no_path_escapes_the_scene(mcrt, pm, setup):
    """The photon mapper adds no sky (photon-mapper.cpp:292-295) and the path tracer does, so their images can only
    agree where no path escapes. Rays in every direction from the camera, and from points just off the lit surfaces,
    must all hit. A surface point is taken 1e-4 from a photon's position along the direction the photon arrived from,
    so it lies on the photon's own path, inside the room; at the photon's position itself, float32 rounding can put it
    behind the surface (0.07 % of such rays then leave through the wall they start in)."""
    scene, _, cf, leaf = setup
    pm.emit(4000, cf, leaf)
    rng = np.random.default_rng(13)
    eye = np.asarray(scene.cameras()[0].rec.eye, np.float64)
    allph = np.concatenate([np.asarray(m["photons"], np.float32).reshape(-1, 8) for m in host_maps(pm)])
    ph = allph[rng.choice(len(allph), 16384)]
    phi, theta = ph[:, 6].astype(np.float64), ph[:, 7].astype(np.float64)
    back = np.stack([np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.cos(theta)], axis=1)
    origins = np.concatenate([np.repeat(eye[None], 8192, 0), ph[:, 3:6].astype(np.float64) + 1e-4 * back])
    d = rng.normal(size=(len(origins), 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    hits = pm.intersect(np.concatenate([origins, d], axis=1))
    assert (hits["prim"] != mcrt.NO_PRIM).all()


def test_progressive_photon_mapping_converges(mcrt, setup, capsys):
    """Relative RMSE against the path tracer at 4096 spp (another seed) over the 4x4-downsampled frame; the scene is
    closed (test above), so both integrators estimate the same image. Measured on the H100, 4 / 16 / 64 passes of
    16 spp with 4000 emissions each:
      automatic radii (caustic 0.918, global 0.987)  0.0122 / 0.0068 / 0.0050
      half of them                                   0.0101 / 0.0036 / 0.0026
      a quarter of them                              0.0100 / 0.0029 / 0.0022
    and the fixed-map photon mapper (one 4000-emission map, k = 50, 1024 spp) 0.0026 (0.0025 at 4096 spp). The error
    falls strictly with the passes at every radius. At 64 passes the automatic radii stay 1.9x above the fixed map;
    the gap shrinks as the initial radius does, so it is the radius's bias, and a quarter of the automatic radii
    meets the fixed map's error within 64 passes."""
    scene, seed, cf, leaf = setup
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=mcrt.PRECISION_F64, global_seed=seed + 7)
    ref = down4(pt.render_rows(cam, sqrtspp=64))   # 4096 spp
    pt.close()
    fixed = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=seed)
    fixed.emit(4000, cf, leaf, 50)
    e_fixed = rel_rmse(down4(fixed.render_rows(cam, sqrtspp=32)), ref)   # 1024 spp
    fixed.close()
    errs, auto = {}, None
    for scale in (1.0, 0.5, 0.25):
        pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=seed)
        radius = None if auto is None else (scale * auto[0], scale * auto[1])
        run = mcrt.ProgressivePhotonMapping(pm, cam, 4000, cf, leaf, radius=radius)
        auto = auto or run.radius
        errs[scale] = {}
        for n in range(1, 65):
            run.add(16)
            if n in (4, 16, 64):
                errs[scale][n] = rel_rmse(down4(run.frame()), ref)
        pm.close()
    with capsys.disabled():
        print(f"\nppm convergence: automatic radii {auto}, rel RMSE by radius scale {errs}, fixed map {e_fixed:.4f}")
    for e in errs.values():
        assert e[4] > e[16] > e[64]
    assert errs[1.0][64] > errs[0.5][64] > errs[0.25][64]
    assert errs[0.25][64] < e_fixed


# ---------------------------------------------------------------------------------------------- 8. inherited machinery
def test_adaptive_denoise_and_fast_mode(mcrt, setup, capsys):
    scene, seed, cf, leaf = setup
    cam = scene.cameras()[0]
    pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=seed)
    run = mcrt.ProgressivePhotonMapping(pm, cam, 2000, cf, leaf, tile=16)
    run.render_adaptive(4, 64, target_error=0.02, min_samples=8)
    assert run.stop_reason in ("target", "no active tile", "max_samples")
    out, err = run.denoise()
    assert np.isfinite(out).all() and np.isfinite(err)

    frames = {}
    for prec in (mcrt.PRECISION_F64, mcrt.PRECISION_F32):
        p = mcrt.PhotonMapper(scene, precision=prec, global_seed=seed)
        r = mcrt.ProgressivePhotonMapping(p, cam, 2000, cf, leaf, radius=run.radius)
        for _ in range(8):
            r.add(8)
        frames[prec] = r.frame()
        p.close()
    pm.close()
    d = rel_rmse(down4(frames[mcrt.PRECISION_F32]), down4(frames[mcrt.PRECISION_F64]))
    with capsys.disabled():
        print(f"\nppm fast vs parity: rel RMSE {d:.4f}, adaptive stop {run.stop_reason}, denoised error {err:.4f}")
    assert d < 1e-3   # measured 1e-4 on the H100: float32 paths, the same maps' structure and the same radii


def test_initial_radius_of_maps_smaller_than_k(mcrt, setup):
    """With fewer photons than k_nearest_photons in a map, the k-NN search returns all of them and pads the rest; the
    initial radius is then the median distance to the farthest photon, not the padding."""
    scene, seed, cf, leaf = setup
    pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=seed)
    run = mcrt.ProgressivePhotonMapping(pm, scene.cameras()[0], 10, cf, leaf, k_nearest_photons=50)
    maps = host_maps(pm)
    assert 0 < len(maps[0]["photons"]) // 8 < 50 and 0 < len(maps[1]["photons"]) // 8 < 50
    for which, m in enumerate(maps):
        pos = np.asarray(m["photons"], np.float32).reshape(-1, 8)[:, 3:6].astype(np.float64)
        d = pos[:, None, :] - pos[None, :, :]
        far = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]).max(axis=1)
        assert run.radius[which] == pytest.approx(float(np.median(np.sqrt(far))), rel=1e-12)
    run.add(2)
    assert np.isfinite(run.frame()).all() and run.frame().max() > 0
    pm.close()
