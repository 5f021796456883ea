"""Light groups for the photon mapper: maps emitted on the device record which light emitted each photon
(mcrt_photon_download_lights), and k_knn / k_gather split their estimates by the photon's light group.

The oracles are exact. Every photon comes from exactly one light, and the estimate is linear in photon flux, so:
- a light's photons in the map are, as a multiset of 32-byte records, the photons of its emission work items emitted alone;
- the planes add up to the one-plane sums of the same samples (float64: rtol 1e-12, the same additions in another order);
- plane g plus the sky's plane is the render of the scene with every light outside g dark, on the same octree with the
  flux of every photon outside g set to 0 (so the k-NN sets, paths and rays stay the same);
- relighting with power-of-two weights (exact on float32 flux and float64 emittance) is the render with scaled emittance
  and scaled photon flux on the same octree."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_ppm_cpu import emission_counts

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-12, 1e-14
STATS = ("paths", "extension_rays", "shadow_rays", "knn_queries")
ERR_INVALID, ERR_UNSUPPORTED, ERR_NO_PHOTONS = -1, -4, -5
EMISSIONS = 20000


def torch_zeros(shape, fill=0.0):
    import torch
    t = torch.full(shape, fill, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()   # the library renders on its own stream
    return t


def load(mcrt, cid):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    return scene, int(np.load(os.path.join(GOLDEN, cid + ".npz"))["seed"])


def emit_params(scene, k=50, dv=False, emissions=EMISSIONS):
    """The pack's photon-pass parameters where it has them (caustic factor, leaf size), else 4 and 100."""
    ep = scene.extra.get("photon_emit_params")
    cf, leaf = (float(ep[1]), int(ep[2])) if ep is not None else (4.0, 100)
    return dict(emissions=emissions, caustic_factor=cf, max_photons_per_octree_leaf=leaf, k_nearest_photons=k,
                direct_visualization=dv)


def emitted(mcrt, cid, precision=0, **kw):
    scene, seed = load(mcrt, cid)
    return scene, mcrt.PhotonMapper(scene, precision=precision, global_seed=seed, emit=emit_params(scene, **kw))


def per_light(scene):
    return np.arange(scene.n_lights, dtype=np.uint32)


def groups_of(mcrt, scene, how):
    return mcrt.light_groups_by_emittance(scene)[0] if how == "emittance" else per_light(scene)


def with_emittance_rgb(mcrt, scene, scale):
    """`scene` with light l's material emittance multiplied by scale[l] (RGB; flags, light list and CDF unchanged)."""
    a = dict(scene.a, **scene.extra)
    a["scene_ior"] = np.array([scene.ior])
    rows = np.asarray(scene.a["prim_material"], np.int64)[np.asarray(scene.a["light_prim"], np.int64)]
    assert len(np.unique(rows)) == len(rows), "every light needs its own material row"
    mats = scene.a["materials"].copy()
    for l, m in enumerate(rows):
        mats[m]["emittance"] = mats[m]["emittance"] * np.asarray(scale[l], np.float64)
    a["materials"] = mats
    return mcrt.Scene(a)


def scaled_maps(pm, group_of_photon_scale):
    """The current maps with each photon's flux multiplied by group_of_photon_scale(light indices) -> [n, 3] float32."""
    caustic, glob, k, dv = pm._maps
    out = []
    for which, m in enumerate((caustic, glob)):
        m = dict(m)
        ph = np.asarray(m["photons"], np.float32).reshape(-1, 8).copy()
        ph[:, 0:3] *= group_of_photon_scale(pm.photon_lights(which)).astype(np.float32)
        m["photons"] = ph.reshape(-1)
        out.append(m)
    return (out[0], out[1], k, dv)


def render_planes(pm, cam, ids, spp, active=None, tile=16):
    n_planes = int(np.max(ids)) + 2
    pm.set_light_groups(ids, n_planes - 1)
    planes = torch_zeros((n_planes, cam.height, cam.width, 3))
    st = pm.render_accumulate_groups_dev(cam, planes.data_ptr(), n_planes, 0, spp, tile=tile, active=active)
    return planes.cpu().numpy(), st


def render_beauty(ig, cam, spp, active=None, tile=16):
    sums = torch_zeros((cam.height, cam.width, 3))
    if active is None:
        st = ig.render_accumulate_dev(cam, sums.data_ptr(), None, 0, spp)
    else:
        st = ig.render_accumulate_tiles_dev(cam, sums.data_ptr(), None, 0, spp, tile, active)
    return sums.cpu().numpy(), st


def same_stats(a, b):
    for k in STATS:
        assert a[k] == b[k], (k, a[k], b[k])


def rows32(ph):
    r = np.ascontiguousarray(np.asarray(ph, np.float32).reshape(-1, 8)).view(np.uint32)
    return r[np.lexsort(r.T[::-1])]


# ---------------------------------------------------------------------------------------------- 1. attribution
@pytest.mark.parametrize("cid,precision,dv", [("pm_hexagon_room_64", 0, False), ("pm_hexagon_room_64", 1, True),
                                              ("veach_mis_64", 0, True), ("veach_mis_64", 1, False),
                                              ("ggx_64", 0, False), ("metals_64", 1, True)])
def test_each_light_owns_the_photons_of_its_emissions(cid, precision, dv, mcrt):
    import torch
    from importlib import import_module
    mdist = import_module(mcrt.__name__ + ".distributed")
    scene, pm = emitted(mcrt, cid, precision, dv=dv)
    try:
        assert pm.has_photon_lights
        ep = emit_params(scene, dv=dv)
        maps = pm._maps
        lights = [pm.photon_lights(w) for w in (0, 1)]
        for w in (0, 1):
            assert lights[w].shape == (maps[w]["photons"].size // 8,)
            assert (lights[w] < scene.n_lights).all()
        counts = emission_counts(scene, ep["emissions"], ep["caustic_factor"])
        offsets = np.concatenate([[0], np.cumsum(counts)])
        p = pm._emit_params(ep["emissions"], ep["caustic_factor"], ep["max_photons_per_octree_leaf"], ep["k_nearest_photons"],
                            dv, None)
        for l in range(scene.n_lights):
            ptr = [C.c_void_p(), C.c_void_p()]; n = [C.c_uint64(), C.c_uint64()]
            assert mcrt.lib().mcrt_photon_emit_range(pm.ctx, C.byref(p), precision, int(offsets[l]), int(counts[l]),
                                                     C.byref(ptr[0]), C.byref(n[0]), C.byref(ptr[1]), C.byref(n[1]),
                                                     C.byref(mcrt.Stats())) == 0
            for w in (0, 1):
                alone = mdist.device_view(ptr[w].value, n[w].value * 8, torch.float32, torch.device("cuda")).cpu().numpy()
                mine = np.asarray(maps[w]["photons"], np.float32).reshape(-1, 8)[lights[w] == l]
                assert np.array_equal(rows32(mine), rows32(alone)), (l, w)
    finally:
        pm.close()


# ---------------------------------------------------------------------------------------------- 2. planes sum to the beauty
# float32 estimate: per query the planes regroup the same non-negative float32 terms. A float32 sum of n non-negative terms
# is within (n - 1) u of the exact sum (u = 2^-24), the warp's tree adds 5 levels, the scale and weight products a few
# roundings: each side is within (k + 8) u of the exact deposit, so the two within 2 (k + 8) u; non-negative deposits keep
# that bound relative per pixel.
def f32_rtol(k):
    return 2.0 * (k + 8) * 2.0 ** -24


CASES = [  # cid, precision, how, k (None: fixed-radius gather), active-tile mask, pool_paths
    ("pm_hexagon_room_64", 0, "per_light", 20, False, None),
    ("pm_hexagon_room_64", 0, "per_light", 50, False, None),
    ("pm_hexagon_room_64", 0, "per_light", 100, True, None),
    ("pm_hexagon_room_64", 0, "per_light", 200, False, None),
    ("pm_hexagon_room_64", 0, "per_light", 300, False, None),
    ("pm_hexagon_room_64", 0, "per_light", 700, False, None),
    ("pm_hexagon_room_64", 0, "per_light", None, True, None),
    ("pm_hexagon_room_64", 1, "per_light", 50, False, None),
    ("pm_hexagon_room_64", 1, "per_light", None, False, None),
    ("veach_mis_64", 0, "emittance", 50, False, None),
    ("veach_mis_64", 0, "per_light", 50, False, 4096),
    ("veach_mis_64", 1, "per_light", None, False, None),
    ("ggx_64", 0, "per_light", 50, False, None),
    ("ggx_64", 0, "emittance", None, False, None),
    ("metals_64", 0, "per_light", 100, True, None),
    ("metals_64", 1, "per_light", 50, False, None),
]


def gather_radius_of(pm):
    """A fixed gather radius of about the 50th-nearest-photon distance: the median over 256 photons of each map."""
    radii = []
    for which in (0, 1):
        pos = np.asarray(pm._maps[which]["photons"], np.float32).reshape(-1, 8)[:, 3:6].astype(np.float64)
        if len(pos) == 0:
            radii.append(None)
            continue
        _, d2, cnt = pm.knn(which, pos[:: max(1, len(pos) // 256)])
        radii.append(float(np.median(np.sqrt(np.where(np.arange(d2.shape[1])[None] < cnt[:, None], d2, 0).max(axis=1)))))
    return (radii[1] if radii[0] is None else radii[0], radii[1])


def max_gathered(pm):
    """A bound on the photons one fixed-radius query sums: a query that finds a photon within r lies within r of it, so
    its ball lies in that photon's ball of 2r; the most photons any photon's 2r-ball holds bound every query."""
    n = 1
    for which, r in enumerate(pm.gather_radii):
        pos = np.asarray(pm._maps[which]["photons"], np.float32).reshape(-1, 8)[:, 3:6].astype(np.float64)
        if len(pos):
            n = max(n, int(pm.gather(which, pos, 2.0 * r)[0].max()))
    return n


@pytest.mark.parametrize("cid,precision,how,k,masked,pool", CASES)
def test_planes_sum_to_beauty(cid, precision, how, k, masked, pool, mcrt):
    scene, pm = emitted(mcrt, cid, precision, k=k or 50)
    try:
        cam = scene.cameras()[0]
        if k is None:
            pm.gather_radius(*gather_radius_of(pm))
        if pool:
            pm.set_option("pool_paths", float(pool))
        ids = groups_of(mcrt, scene, how)
        active = None
        if masked:
            active = np.zeros(mcrt.tile_grid(cam.height, cam.width, 16), bool)
            active[::2, 1::2] = True
            active[-1, 0] = True
        spp = 4
        planes, sp = render_planes(pm, cam, ids, spp, active)
        beauty, sb = render_beauty(pm, cam, spp, active)
        same_stats(sp, sb)
        assert sb["knn_queries"] > 0
        assert (planes >= 0).all()
        assert not planes[-1].any()            # the photon mapper adds no sky
        rtol = RTOL if precision == 0 else f32_rtol(k or max_gathered(pm))
        np.testing.assert_allclose(planes.sum(axis=0), beauty, rtol=rtol, atol=ATOL * spp)
        if masked:
            assert planes.any() and beauty.any()
    finally:
        pm.close()


# ---------------------------------------------------------------------------------------------- 3. exact oracle per group
@pytest.mark.parametrize("how,gather", [("per_light", False), ("emittance", False), ("per_light", True)])
def test_plane_is_scene_with_other_groups_dark(how, gather, mcrt):
    cid = "veach_mis_64"
    scene, pm = emitted(mcrt, cid)
    others = []
    try:
        cam = scene.cameras()[0]
        radius = gather_radius_of(pm) if gather else None
        if gather:
            pm.gather_radius(*radius)
        ids = groups_of(mcrt, scene, how)
        spp = 4
        planes, sp = render_planes(pm, cam, ids, spp)
        for g in range(int(ids.max()) + 1):
            on = (ids == g).astype(np.float64)
            dark = with_emittance_rgb(mcrt, scene, np.repeat(on[:, None], 3, axis=1))
            maps = scaled_maps(pm, lambda li: np.repeat(on[li][:, None], 3, axis=1))
            other = mcrt.PhotonMapper(dark, global_seed=pm.global_seed, photon_maps=maps)
            others.append(other)
            if gather:
                other.gather_radius(*radius)
            beauty, sb = render_beauty(other, cam, spp)
            same_stats(sp, sb)
            np.testing.assert_allclose(planes[g] + planes[-1], beauty, rtol=RTOL, atol=ATOL * spp)
    finally:
        for o in others:
            o.close()
        pm.close()


# ---------------------------------------------------------------------------------------------- 4. relight
def pow2_weights(n_planes):
    w = np.array([[2.0, 1.0, 0.5], [0.25, 4.0, 1.0], [1.0, 0.5, 8.0], [0.125, 2.0, 2.0]])
    return np.concatenate([w[np.arange(n_planes - 1) % len(w)], [[1.0, 1.0, 1.0]]])


def test_relight_one_shot_progressive(mcrt):
    scene, pm = emitted(mcrt, "veach_mis_64")
    other = None
    try:
        cam = scene.cameras()[0]
        ids = per_light(scene)
        w = pow2_weights(len(ids) + 1)
        prog = mcrt.Progressive(pm, cam, light_groups=ids)
        prog.add(4)
        relit = prog.relight(w)[0]
        scaled = with_emittance_rgb(mcrt, scene, w[ids])
        other = mcrt.PhotonMapper(scaled, global_seed=pm.global_seed, photon_maps=scaled_maps(pm, lambda li: w[ids[li]]))
        ref = mcrt.Progressive(other, cam)
        ref.add(4)
        np.testing.assert_allclose(relit, ref.frame(), rtol=RTOL, atol=ATOL)
    finally:
        if other is not None:
            other.close()
        pm.close()


def test_relight_progressive_photon_mapping(mcrt):
    import torch
    scene, seed = load(mcrt, "veach_mis_64")
    ep = emit_params(scene)
    pm = mcrt.PhotonMapper(scene, global_seed=seed, emit=ep)
    others = []
    try:
        cam = scene.cameras()[0]
        ids = per_light(scene)
        w = pow2_weights(len(ids) + 1)
        scaled = with_emittance_rgb(mcrt, scene, w[ids])
        ppm = mcrt.ProgressivePhotonMapping(pm, cam, EMISSIONS, ep["caustic_factor"], ep["max_photons_per_octree_leaf"],
                                            light_groups=ids)
        halves = [torch_zeros((cam.height, cam.width, 3)) for _ in range(2)]
        for i in range(2):
            ppm.add(2)
            # the same pass on the same octree: the pass's map, flux scaled by group
            other = mcrt.PhotonMapper(scaled, global_seed=seed, photon_maps=scaled_maps(pm, lambda li: w[ids[li]]))
            others.append(other)
            other.gather_radius(*ppm.pass_radii(i))
            other.render_accumulate_dev(cam, halves[i % 2].data_ptr(), None, 2 * i, 2)
        ref = (halves[0] + halves[1]).cpu().numpy() / 4.0
        np.testing.assert_allclose(ppm.relight(w)[0], np.maximum(ref, 0.0), rtol=RTOL, atol=ATOL)
    finally:
        for o in others:
            o.close()
        pm.close()


# ---------------------------------------------------------------------------------------------- 5. progressive photon mapping
def test_progressive_photon_mapping_with_groups(mcrt, tmp_path):
    scene, seed = load(mcrt, "pm_hexagon_room_64")
    ep = emit_params(scene)
    cam = scene.cameras()[0]
    ids = per_light(scene)
    args = (cam, 4000, ep["caustic_factor"], ep["max_photons_per_octree_leaf"])
    mappers = [mcrt.PhotonMapper(scene, global_seed=seed) for _ in range(4)]
    try:
        plain = mcrt.ProgressivePhotonMapping(mappers[0], *args, radius=0.2)
        grouped = mcrt.ProgressivePhotonMapping(mappers[1], *args, radius=0.2, light_groups=ids)
        for _ in range(3):
            plain.add(2)
            grouped.add(2)
        np.testing.assert_allclose(grouped.frame(), plain.frame(), rtol=RTOL, atol=ATOL)
        assert grouped.error()[0] == pytest.approx(plain.error()[0], rel=1e-9)
        np.testing.assert_allclose(grouped.relight(np.ones(len(ids) + 1))[0], plain.frame(), rtol=RTOL, atol=ATOL)
        target = 0.5 * plain.error()[0]
        plain.render_adaptive(2, 12, target, min_samples=4)
        grouped.render_adaptive(2, 12, target, min_samples=4)
        assert np.array_equal(plain.active, grouped.active)
        assert np.array_equal(plain.tile_counts, grouped.tile_counts)
        np.testing.assert_allclose(grouped.frame(), plain.frame(), rtol=RTOL, atol=ATOL)

        path_g, path_p = str(tmp_path / "grouped.npz"), str(tmp_path / "plain.npz")
        grouped.save(path_g)
        plain.save(path_p)
        resumed = mcrt.ProgressivePhotonMapping.load(path_g, mappers[2], *args, radius=0.2, light_groups=ids)
        assert resumed.passes == grouped.passes
        resumed.add(2)
        grouped.add(2)
        np.testing.assert_allclose(resumed.frame(), grouped.frame(), rtol=RTOL, atol=ATOL)
        with pytest.raises(mcrt.McrtError, match="light groups"):
            mcrt.ProgressivePhotonMapping.load(path_g, mappers[3], *args, radius=0.2)
        with pytest.raises(mcrt.McrtError, match="light groups"):
            mcrt.ProgressivePhotonMapping.load(path_p, mappers[3], *args, radius=0.2, light_groups=ids)
    finally:
        for m in mappers:
            m.close()


def test_progressive_checkpoint_digests_photon_lights(mcrt, tmp_path):
    scene, pm = emitted(mcrt, "veach_mis_64")
    others = []
    try:
        cam = scene.cameras()[0]
        ids = per_light(scene)
        prog = mcrt.Progressive(pm, cam, light_groups=ids)
        prog.add(2)
        path = str(tmp_path / "groups.npz")
        prog.save(path)
        resumed = mcrt.Progressive.load(path, pm, cam, light_groups=ids)
        resumed.add(2)
        prog.add(2)
        np.testing.assert_allclose(resumed.frame(), prog.frame(), rtol=RTOL, atol=ATOL)
        # the same photons attributed to other lights: a map of this light set with the lights' index swapped cannot
        # be told apart by the records alone, so the digest must hold the indices. Here: the same records uploaded
        # (no indices) are refused for groups altogether.
        other = mcrt.PhotonMapper(scene, global_seed=pm.global_seed, photon_maps=pm._maps)
        others.append(other)
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive.load(path, other, cam, light_groups=ids)
        ident = prog._photon_identity()["photon_digest"]
        plain = mcrt.Progressive(pm, cam)._photon_identity()["photon_digest"]
        assert ident != plain
    finally:
        for o in others:
            o.close()
        pm.close()


# ---------------------------------------------------------------------------------------------- 6. refusals
def raw_groups_call(mcrt, ig, cam, sums, n_planes):
    return mcrt.lib().mcrt_render_accumulate_groups_dev(ig.ctx, C.byref(cam.rec), 0, 1, cam.height, 16, None, 0, 1,
                                                        ig.global_seed, 1, 0, C.c_void_p(sums.data_ptr()), n_planes, None)


def set_table(mcrt, ig, ids, n_groups):
    ids = np.ascontiguousarray(ids, np.uint32)
    return mcrt.lib().mcrt_set_light_groups(ig.ctx, ids.ctypes.data_as(C.c_void_p), ids.size, n_groups)


def refused_everywhere(mcrt, ig, cam, ids, sums):
    """ABI refusal and McrtError from every Python entry point, the sums untouched."""
    assert set_table(mcrt, ig, ids, int(ids.max()) + 1) == 0
    assert raw_groups_call(mcrt, ig, cam, sums, int(ids.max()) + 2) == ERR_UNSUPPORTED
    out = np.zeros(1, np.uint32)
    # host maps (no device-built map at all) or device-built maps without indices
    assert mcrt.lib().mcrt_photon_download_lights(ig.ctx, 0, out.ctypes.data_as(C.c_void_p), 1) in (ERR_UNSUPPORTED, ERR_NO_PHOTONS)
    with pytest.raises(mcrt.McrtError):
        ig.set_light_groups(ids)
    with pytest.raises(mcrt.McrtError):
        ig.render_accumulate_groups_dev(cam, sums.data_ptr(), int(ids.max()) + 2, 0, 1)
    with pytest.raises(mcrt.McrtError):
        mcrt.Progressive(ig, cam, light_groups=ids)
    with pytest.raises(mcrt.McrtError):
        ig.photon_lights(0)
    assert not ig.has_photon_lights
    assert bool((sums == 7.0).all())


def test_maps_without_light_indices_are_refused(mcrt):
    scene, seed = load(mcrt, "pm_hexagon_room_64")
    cam = scene.cameras()[0]
    ids = per_light(scene)
    sums = torch_zeros((len(ids) + 1, cam.height, cam.width, 3), 7.0)
    mappers = []
    try:
        pack = mcrt.PhotonMapper(scene, global_seed=seed)               # the reference's CPU pass, from the pack
        mappers.append(pack)
        refused_everywhere(mcrt, pack, cam, ids, sums)
        em = mcrt.PhotonMapper(scene, global_seed=seed, emit=emit_params(scene))
        mappers.append(em)
        uploaded = mcrt.PhotonMapper(scene, global_seed=seed, photon_maps=em._maps)   # mcrt_photon_upload of emitted maps
        mappers.append(uploaded)
        refused_everywhere(mcrt, uploaded, cam, ids, sums)
        ep = emit_params(scene)
        em.emit_sharded(0, 1, ep["emissions"], ep["caustic_factor"], ep["max_photons_per_octree_leaf"])   # mcrt_photon_build_dev
        refused_everywhere(mcrt, em, cam, ids, sums)
        em.emit(**ep)                                                    # emitted again: accepted
        assert em.has_photon_lights
        assert set_table(mcrt, em, ids, len(ids)) == 0
        assert raw_groups_call(mcrt, em, cam, sums, len(ids)) == ERR_INVALID        # n_planes != n_groups + 1
        film = mcrt.FilmRec(mcrt.FILM_FILTERS["mitchell-netravali"], 0, 0.0)
        assert mcrt.lib().mcrt_set_film(em.ctx, C.byref(film)) == 0
        assert raw_groups_call(mcrt, em, cam, sums, len(ids) + 1) == ERR_UNSUPPORTED  # reconstruction filter
        assert mcrt.lib().mcrt_set_film(em.ctx, None) == 0
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive(em, cam, aovs=True)
        with pytest.raises(mcrt.McrtError):
            mcrt.ProgressivePhotonMapping(em, cam, 2000, ep["caustic_factor"], aovs=True)
        with pytest.raises(mcrt.McrtError):
            em.render_accumulate_aovs_dev(cam, sums.data_ptr(), 0, 1)
        em.upload_scene()                                                # another scene's light list
        assert not em.has_photon_lights or mcrt.lib().mcrt_photon_download_lights(em.ctx, 0, None, 0) == ERR_UNSUPPORTED
        assert bool((sums == 7.0).all())
    finally:
        for m in mappers:
            m.close()
