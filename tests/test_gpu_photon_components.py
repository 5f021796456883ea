"""Photon-mapper components (mcrt_render_accumulate_photon_components_dev, Progressive(components=True)): every deposit of
the photon mapper lands in the plane of the estimator that made it - emission, direct light, caustic map, global map.

The oracles are exact, built from the product alone:
- no estimate is split, so the planes add up to the one-plane sums of the same samples at rtol 1e-12 in both precisions:
  every deposit value is the one-plane kernel's (float32 included), only the order of the float64 film additions differs;
- a photon estimate is linear in photon flux, and zeroing a map's flux moves no photon, so the k-NN sets and gather sets
  stay the same: the render with the caustic (global) map's flux zeroed is every plane but the caustic (global) one;
- the sampler draws each purpose from its own dimensions (DIM_LIGHT, sampler.cuh), so a scene with an empty light list
  (emitters still emit, but next-event estimation and its MIS partner are gone) traces the same paths and queries: its
  render is emission + caustic + global, and with both maps zeroed the emission plane alone."""
import ctypes as C

import numpy as np
import pytest

from scene_gen import generated_scene
from test_gpu_photon_light_groups import emit_params, gather_radius_of, load, render_beauty, torch_zeros

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-12, 1e-14
STATS = ("paths", "extension_rays", "shadow_rays", "knn_queries")
ERR_INVALID, ERR_UNSUPPORTED, ERR_NO_PHOTONS = -1, -4, -5
EMISSION, DIRECT, CAUSTIC, GLOBAL = range(4)
NP = 4
SPP = 4


def same_stats(a, b, keys=STATS):
    for k in keys:
        assert a[k] == b[k], (k, a[k], b[k])


def render_components(pm, cam, spp=SPP, active=None, tile=16):
    planes = torch_zeros((NP, cam.height, cam.width, 3))
    st = pm.render_accumulate_components_dev(cam, planes.data_ptr(), 0, spp, tile=tile, active=active)
    return planes.cpu().numpy(), st


def mapper(mcrt, scene, seed, maps, precision=0, k=50, dv=False):
    """maps: "pack" (the reference's CPU pass, mcrt_photon_upload), "emit" (mcrt_photon_emit) or "built"
    (mcrt_photon_build_dev, the sharded pass on one GPU)."""
    if maps == "pack":
        return mcrt.PhotonMapper(scene, precision=precision, global_seed=seed)
    ep = emit_params(scene, k=k, dv=dv)
    pm = mcrt.PhotonMapper(scene, precision=precision, global_seed=seed, emit=ep)
    if maps == "built":
        pm.emit_sharded(0, 1, ep["emissions"], ep["caustic_factor"], ep["max_photons_per_octree_leaf"], k, dv)
    return pm


def flux_scaled(maps, caustic, glob):
    """The maps (caustic, global, k, dv) with every photon's flux multiplied by caustic / glob; positions, directions and
    the octrees unchanged."""
    out = []
    for m, s in zip(maps[:2], (caustic, glob)):
        m = dict(m)
        ph = np.asarray(m["photons"], np.float32).reshape(-1, 8).copy()
        ph[:, 0:3] *= np.float32(s)
        m["photons"] = ph.reshape(-1)
        out.append(m)
    return (out[0], out[1]) + tuple(maps[2:])


def without_lights(mcrt, scene):
    """`scene` with an empty light list: emissive materials still emit when a ray hits them, but nothing samples them."""
    a = dict(scene.a, **scene.extra)
    a["scene_ior"] = np.array([scene.ior])
    a["light_prim"] = np.zeros(0, np.asarray(scene.a["light_prim"]).dtype)
    a["light_cdf"] = np.zeros(0, np.asarray(scene.a["light_cdf"]).dtype)
    s = mcrt.Scene(a)
    assert s.n_lights == 0
    return s


def check_planes(planes, beauty, st, st0, dv):
    same_stats(st, st0)
    assert st0["knn_queries"] > 0
    assert (planes >= 0).all()
    np.testing.assert_allclose(planes.sum(axis=0), beauty, rtol=RTOL, atol=ATOL * SPP)
    assert planes[GLOBAL].any()
    if dv:
        # the first non-delta vertex queries both maps and the path ends: no next-event estimation, no MIS hit
        assert not planes[DIRECT].any() and st["shadow_rays"] == 0
    else:
        assert planes[DIRECT].any() and st["shadow_rays"] > 0


# ---------------------------------------------------------------------------------------------- 1. planes sum to the beauty
CASES = [  # cid, precision, maps, k (None: fixed-radius gather), direct_visualization, active-tile mask, pool_paths
    ("pm_hexagon_room_64", 0, "pack", None, None, False, None),
    ("pm_hexagon_room_64", 1, "pack", None, None, True, None),
    ("pm_hexagon_room_64", 0, "emit", 20, False, False, None),
    ("pm_hexagon_room_64", 0, "emit", 50, True, False, None),
    ("pm_hexagon_room_64", 0, "emit", 100, False, True, None),
    ("pm_hexagon_room_64", 0, "emit", 200, False, False, None),
    ("pm_hexagon_room_64", 0, "emit", 300, True, False, None),
    ("pm_hexagon_room_64", 0, "emit", 700, False, False, None),
    ("pm_hexagon_room_64", 0, "emit", "gather", False, True, None),
    ("pm_hexagon_room_64", 1, "emit", 50, False, False, None),
    ("pm_hexagon_room_64", 1, "emit", 700, True, False, None),
    ("pm_hexagon_room_64", 1, "emit", "gather", False, False, None),
    ("pm_hexagon_room_64", 0, "built", 50, False, False, None),
    ("pm_hexagon_room_64", 1, "built", "gather", True, False, None),
    ("veach_mis_64", 0, "emit", 50, False, False, 4096),
    ("veach_mis_64", 1, "emit", "gather", False, False, 4096),
    ("ggx_64", 0, "emit", 50, False, False, None),
    ("ggx_64", 1, "emit", "gather", True, False, None),
    ("metals_64", 0, "emit", "gather", False, True, None),
    ("metals_64", 1, "built", 100, False, False, None),
]


@pytest.mark.parametrize("cid,precision,maps,k,dv,masked,pool", CASES)
def test_planes_sum_to_beauty(cid, precision, maps, k, dv, masked, pool, mcrt):
    scene, seed = load(mcrt, cid)
    gather = k == "gather"
    pm = mapper(mcrt, scene, seed, maps, precision, 50 if gather else k, dv)
    try:
        cam = scene.cameras()[0]
        if gather:
            pm.gather_radius(*gather_radius_of(pm))
        if pool:
            pm.set_option("pool_paths", float(pool))
        active = None
        if masked:
            active = np.zeros(mcrt.tile_grid(cam.height, cam.width, 16), bool)
            active[::2, 1::2] = True
            active[-1, 0] = True
        planes, st = render_components(pm, cam, active=active)
        beauty, st0 = render_beauty(pm, cam, SPP, active)
        check_planes(planes, beauty, st, st0, bool(pm._maps[3]))
    finally:
        pm.close()


def test_planes_sum_to_beauty_generated(mcrt):
    """The generated photon-mapping scene (60 044 primitives): dynamic fetch and primitive sort keys."""
    scene = generated_scene(mcrt, "pm")
    _, seed = load(mcrt, "pm_hexagon_room_64")
    pm = mcrt.PhotonMapper(scene, global_seed=seed)   # the base scene's maps from the pack
    try:
        cam = scene.cameras()[0].resized(96, 54, 8)
        planes, st = render_components(pm, cam)
        beauty, st0 = render_beauty(pm, cam, SPP)
        check_planes(planes, beauty, st, st0, bool(pm._maps[3]))
    finally:
        pm.close()


# ---------------------------------------------------------------------------------------------- 2. exact oracle per plane
@pytest.mark.parametrize("cid", ["pm_hexagon_room_64", "veach_mis_64"])
@pytest.mark.parametrize("gather", [False, True])
def test_each_plane_against_a_modified_render(cid, gather, mcrt):
    scene, seed = load(mcrt, cid)
    pm = mapper(mcrt, scene, seed, "emit")
    dark = without_lights(mcrt, scene)
    others = []
    try:
        cam = scene.cameras()[0]
        radius = gather_radius_of(pm) if gather else None
        if gather:
            pm.gather_radius(*radius)
        planes, st = render_components(pm, cam)
        assert planes[DIRECT].any() and planes[GLOBAL].any() and st["shadow_rays"] > 0
        # every plane the scene can fill is filled, so a deposit routed to a neighbouring plane fails a row below: both
        # cameras see an emitter, and pm_hexagon_room's glass fills the caustic map (veach_mis has no delta surface)
        assert planes[EMISSION].any()
        if cid == "pm_hexagon_room_64":
            assert pm.n_photons[0] > 0 and planes[CAUSTIC].any()
        elif pm.n_photons[0] == 0:
            assert not planes[CAUSTIC].any()
        maps = pm._maps

        def render(sc, caustic, glob):
            other = mcrt.PhotonMapper(sc, global_seed=seed, photon_maps=flux_scaled(maps, caustic, glob))
            others.append(other)
            if gather:
                other.gather_radius(*radius)
            return render_beauty(other, cam, SPP)

        rows = [  # (scene, caustic flux, global flux) -> the planes it must equal
            ((scene, 0.0, 1.0), (EMISSION, DIRECT, GLOBAL)),
            ((scene, 1.0, 0.0), (EMISSION, DIRECT, CAUSTIC)),
            ((dark, 1.0, 1.0), (EMISSION, CAUSTIC, GLOBAL)),
            ((dark, 0.0, 0.0), (EMISSION,)),
        ]
        for args, keep in rows:
            beauty, sb = render(*args)
            if args[0] is scene:
                same_stats(st, sb)
            else:
                assert sb["shadow_rays"] == 0
                same_stats(st, sb, ("paths", "extension_rays", "knn_queries"))
            np.testing.assert_allclose(planes[list(keep)].sum(axis=0), beauty, rtol=RTOL, atol=ATOL * SPP, err_msg=str(keep))
    finally:
        for o in others:
            o.close()
        pm.close()


# ---------------------------------------------------------------------------------------------- 3. progressive
def test_progressive_with_components(mcrt, tmp_path):
    scene, seed = load(mcrt, "pm_hexagon_room_64")
    cam = scene.cameras()[0]
    pm = mcrt.PhotonMapper(scene, global_seed=seed)
    no_caustics = mcrt.PhotonMapper(scene, global_seed=seed, photon_maps=flux_scaled(pm._maps, 0.0, 1.0))
    try:
        prog = mcrt.Progressive(pm, cam, components=True)
        plain = mcrt.Progressive(pm, cam)
        ref = mcrt.Progressive(no_caustics, cam)
        for s in (1, 3, 2):
            for p in (prog, plain, ref):
                p.add(s)
        assert prog.rgb[0].shape == (NP, cam.height, cam.width, 3)
        np.testing.assert_allclose(prog.frame(), plain.frame(), rtol=RTOL, atol=ATOL)
        (e, t), (e0, t0) = prog.error(), plain.error()
        assert np.isclose(e, e0, rtol=RTOL, atol=0) and np.allclose(t, t0, rtol=RTOL, atol=ATOL)
        assert prog.stats == plain.stats
        frames, errors = prog.component_frames()
        assert frames.shape == (NP, cam.height, cam.width, 3) and errors.shape == (NP,)
        assert np.isfinite(errors).all() and (errors >= 0).all()
        np.testing.assert_allclose(frames.sum(0), plain.frame(), rtol=1e-11, atol=ATOL)
        # the caustics removed: the render whose caustic map carries no flux
        np.testing.assert_allclose(prog.relight([1, 1, 0, 1])[0], ref.frame(), rtol=RTOL, atol=ATOL)
        den, den_err = prog.denoise()
        ref_den, ref_den_err = plain.denoise()
        assert np.allclose(den, ref_den, rtol=1e-9, atol=1e-12) and np.isclose(den_err, ref_den_err, rtol=1e-9)
        den_w, _ = prog.denoise(weights=[1, 1, 0, 1])
        assert np.allclose(den_w, ref.denoise()[0], rtol=1e-9, atol=1e-12)
        # checkpoints: the planes come back; a component checkpoint and a plain one refuse each other
        path, path0 = str(tmp_path / "components.npz"), str(tmp_path / "plain.npz")
        prog.save(path)
        plain.save(path0)
        back = mcrt.Progressive.load(path, pm, cam, components=True)
        for h in (0, 1):
            assert np.array_equal(back.rgb[h].cpu().numpy(), prog.rgb[h].cpu().numpy())
        back.add(2)
        prog.add(2)
        np.testing.assert_allclose(back.frame(), prog.frame(), rtol=RTOL, atol=ATOL)
        with pytest.raises(mcrt.McrtError, match="components"):
            mcrt.Progressive.load(path, pm, cam)
        with pytest.raises(mcrt.McrtError, match="components"):
            mcrt.Progressive.load(path0, pm, cam, components=True)
        with pytest.raises(mcrt.McrtError):
            plain.component_frames()
        with pytest.raises(mcrt.McrtError):
            prog.aov_frames()
    finally:
        no_caustics.close()
        pm.close()


def test_adaptive_retires_the_same_tiles(mcrt):
    scene, seed = load(mcrt, "pm_hexagon_room_64")
    cam = scene.cameras()[0]
    pm = mcrt.PhotonMapper(scene, global_seed=seed)
    try:
        first = mcrt.Progressive(pm, cam, tile=16)
        first.add(2)
        first.add(2)
        target = 0.5 * first.error()[0]
        runs = []
        for components in (True, False):
            prog = mcrt.Progressive(pm, cam, tile=16, components=components)
            frame = prog.render_adaptive(2, 32, target, min_samples=4)
            runs.append((prog, frame))
        (a, fa), (b, fb) = runs
        assert len(a.history) == len(b.history) > 1 and a.stop_reason == b.stop_reason
        assert any(h["retired"].any() for h in a.history)
        for ha, hb in zip(a.history, b.history):
            assert np.array_equal(ha["retired"], hb["retired"]) and np.array_equal(ha["tile_counts"], hb["tile_counts"])
        np.testing.assert_allclose(fa, fb, rtol=RTOL, atol=ATOL)
        np.testing.assert_allclose(a.component_frames()[0].sum(0), fb, rtol=1e-11, atol=ATOL)
    finally:
        pm.close()


def test_progressive_photon_mapping_with_components(mcrt, tmp_path):
    scene, seed = load(mcrt, "pm_hexagon_room_64")
    ep = emit_params(scene)
    cam = scene.cameras()[0]
    args = (cam, 4000, ep["caustic_factor"], ep["max_photons_per_octree_leaf"])
    mappers = [mcrt.PhotonMapper(scene, global_seed=seed) for _ in range(4)]
    try:
        plain = mcrt.ProgressivePhotonMapping(mappers[0], *args, radius=0.2)
        comp = mcrt.ProgressivePhotonMapping(mappers[1], *args, radius=0.2, components=True)
        for _ in range(3):
            plain.add(2)
            comp.add(2)
        np.testing.assert_allclose(comp.frame(), plain.frame(), rtol=RTOL, atol=ATOL)
        assert np.isclose(comp.error()[0], plain.error()[0], rtol=RTOL, atol=0)
        frames, errors = comp.component_frames()
        assert np.isfinite(errors).all() and frames[GLOBAL].any()
        np.testing.assert_allclose(comp.relight(np.ones(NP))[0], plain.frame(), rtol=RTOL, atol=ATOL)

        path_c, path_p = str(tmp_path / "components.npz"), str(tmp_path / "plain.npz")
        comp.save(path_c)
        plain.save(path_p)
        resumed = mcrt.ProgressivePhotonMapping.load(path_c, mappers[2], *args, radius=0.2, components=True)
        assert resumed.passes == comp.passes
        resumed.add(2)
        comp.add(2)
        np.testing.assert_allclose(resumed.frame(), comp.frame(), rtol=RTOL, atol=ATOL)
        with pytest.raises(mcrt.McrtError, match="components"):
            mcrt.ProgressivePhotonMapping.load(path_c, mappers[3], *args, radius=0.2)
        with pytest.raises(mcrt.McrtError, match="components"):
            mcrt.ProgressivePhotonMapping.load(path_p, mappers[3], *args, radius=0.2, components=True)
        with pytest.raises(mcrt.McrtError):
            mcrt.ProgressivePhotonMapping(mappers[3], *args, radius=0.2, components=True, aovs=True)
    finally:
        for m in mappers:
            m.close()


# ---------------------------------------------------------------------------------------------- 4. refusals
def raw_call(mcrt, ig, cam, planes_ptr, n_planes, integrator_kind=1):
    return mcrt.lib().mcrt_render_accumulate_photon_components_dev(ig.ctx, C.byref(cam.rec), 0, 1, cam.height, 16, None, 0, 1,
                                                                   ig.global_seed, integrator_kind, 0, C.c_void_p(planes_ptr),
                                                                   n_planes, None)


def test_refusals_leave_the_sums_untouched(mcrt):
    scene, seed = load(mcrt, "pm_hexagon_room_64")
    cam = scene.cameras()[0]
    sums = torch_zeros((NP + 1, cam.height, cam.width, 3), 7.0)
    pm = mapper(mcrt, scene, seed, "emit")
    pt = mcrt.PathTracer(scene, global_seed=seed)
    try:
        L = mcrt.lib()
        assert raw_call(mcrt, pm, cam, sums.data_ptr(), NP, integrator_kind=0) == ERR_UNSUPPORTED   # path tracer
        for kind in (2, -1, 0x7FFFFFFF):                                                             # no such integrator
            assert raw_call(mcrt, pm, cam, sums.data_ptr(), NP, integrator_kind=kind) == ERR_INVALID
        assert raw_call(mcrt, pm, cam, sums.data_ptr(), NP - 1) == ERR_INVALID                       # n_planes != 4
        assert raw_call(mcrt, pm, cam, sums.data_ptr(), NP + 1) == ERR_INVALID
        assert raw_call(mcrt, pm, cam, None, NP) == ERR_INVALID                                      # null planes
        # no photon maps: what the one-plane photon render returns
        one = L.mcrt_render_accumulate_dev(pt.ctx, C.byref(cam.rec), 0, 1, cam.height, 0, 1, seed, 1, 0,
                                           C.c_void_p(sums.data_ptr()), None, None)
        assert one == ERR_NO_PHOTONS and raw_call(mcrt, pt, cam, sums.data_ptr(), NP) == ERR_NO_PHOTONS
        film = mcrt.FilmRec(mcrt.FILM_FILTERS["mitchell-netravali"], 0, 0.0)
        assert L.mcrt_set_film(pm.ctx, C.byref(film)) == 0
        assert raw_call(mcrt, pm, cam, sums.data_ptr(), NP) == ERR_UNSUPPORTED                       # reconstruction filter
        assert L.mcrt_set_film(pm.ctx, None) == 0
        assert bool((sums == 7.0).all())
        # Python
        ids = np.arange(scene.n_lights, dtype=np.uint32)
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive(pt, cam, components=True)
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive(pm, cam, light_groups=ids, components=True)
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive(pm, cam, aovs=True, components=True)
        filtered = scene.cameras()[0]
        filtered.film = {"filter": "mitchell-netravali"}
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive(pm, filtered, components=True)
        with pytest.raises(mcrt.McrtError):
            pm.render_accumulate_aovs_dev(cam, sums.data_ptr(), 0, 1)
        assert bool((sums == 7.0).all())
    finally:
        pt.close()
        pm.close()


def test_one_plane_render_after_components(mcrt):
    """A component render leaves no state behind: the next one-plane render is the one it would have been."""
    scene, seed = load(mcrt, "pm_hexagon_room_64")
    cam = scene.cameras()[0]
    pm = mcrt.PhotonMapper(scene, global_seed=seed)
    try:
        before, st0 = render_beauty(pm, cam, SPP)
        render_components(pm, cam)
        sums = torch_zeros((2, cam.height, cam.width, 3))   # room for a second plane the render must not touch
        st = pm.render_accumulate_dev(cam, sums.data_ptr(), None, 0, SPP)
        out = sums.cpu().numpy()
    finally:
        pm.close()
    np.testing.assert_allclose(out[0], before, rtol=RTOL, atol=ATOL * SPP)
    assert not out[1].any()
    same_stats(st, st0)
