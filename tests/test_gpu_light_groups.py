"""Light groups (mcrt_set_light_groups, mcrt_render_accumulate_groups_dev, mcrt_light_groups_combine_dev and Progressive's
light_groups): every contribution lands in the plane of the light it comes from, or in the sky's plane.

The oracle is exact. Each light of the golden scenes has its own material row, and k_shade queues the shadow ray of a sampled
light whatever its emittance, so the scene with every light outside group g switched dark (material emittance 0, emissive flag,
light list and CDF kept) traces the same paths and rays as the full scene and renders exactly plane g plus the sky's plane (the
sky stays lit); with every light dark it renders the sky's plane. The planes are compared
with those renders at the bar of the progressive tests (rtol 1e-12, atol 1e-14: the same float64 additions in another order), and
on two scenes with the CPU restatement of the reference's sampleRay."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases
from scene_gen import generated_scene

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-12, 1e-14
PATH_CASES = [c for c in golden_cases() if not c.startswith("pm_")]
STATS = ("paths", "extension_rays", "shadow_rays")
ERR_INVALID, ERR_NO_SCENE, ERR_UNSUPPORTED = -1, -3, -4


def torch_zeros(shape, fill=0.0):
    import torch
    t = torch.full(shape, fill, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()   # the library renders on its own stream
    return t


def load(mcrt, cid):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    return scene, int(np.load(os.path.join(GOLDEN, cid + ".npz"))["seed"])


def per_light(scene):
    return np.arange(scene.n_lights, dtype=np.uint32)


def with_emittance(mcrt, scene, scale):
    """`scene` with light l's material emittance multiplied by scale[l] (flags, light list and CDF unchanged)."""
    a = dict(scene.a, **scene.extra)
    a["scene_ior"] = np.array([scene.ior])
    rows = np.asarray(scene.a["prim_material"], np.int64)[np.asarray(scene.a["light_prim"], np.int64)]
    assert len(np.unique(rows)) == len(rows), "every light needs its own material row"
    mats = scene.a["materials"].copy()
    for l, m in enumerate(rows):
        mats[m]["emittance"] = mats[m]["emittance"] * float(scale[l])
    a["materials"] = mats
    return mcrt.Scene(a)


def dark_except(mcrt, scene, ids, g):
    return with_emittance(mcrt, scene, (np.asarray(ids) == g).astype(np.float64))


def render_planes(mcrt, pt, cam, ids, n_groups=None, precision=None, spp=None):
    n_groups = (int(np.max(ids)) + 1 if len(ids) else 0) if n_groups is None else n_groups
    spp = cam.sqrtspp ** 2 if spp is None else spp
    pt.set_light_groups(ids, n_groups)
    planes = torch_zeros((n_groups + 1, cam.height, cam.width, 3))
    st = pt.render_accumulate_groups_dev(cam, planes.data_ptr(), n_groups + 1, 0, spp, precision=precision)
    return planes.cpu().numpy() / spp, st


def render_beauty(pt, cam, precision=None, spp=None):
    spp = cam.sqrtspp ** 2 if spp is None else spp
    sums = torch_zeros((cam.height, cam.width, 3))
    st = pt.render_accumulate_dev(cam, sums.data_ptr(), None, 0, spp, precision=precision)
    return sums.cpu().numpy() / spp, st


def same_stats(a, b):
    for k in STATS:
        assert a[k] == b[k], (k, a[k], b[k])


# ---------------------------------------------------------------------------------------------- 1. planes sum to the beauty frame
@pytest.mark.parametrize("grouping", ["emittance", "per_light"])
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("cid", PATH_CASES)
def test_planes_sum_to_beauty(cid, precision, grouping, mcrt):
    scene, seed = load(mcrt, cid)
    ids = mcrt.light_groups_by_emittance(scene)[0] if grouping == "emittance" else per_light(scene)
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=precision, global_seed=seed)
    try:
        planes, st = render_planes(mcrt, pt, cam, ids)
        beauty, st0 = render_beauty(pt, cam)
    finally:
        pt.close()
    assert planes.shape[0] == (int(ids.max()) + 2 if len(ids) else 1)
    total = mcrt.light_groups_combine(planes, np.ones(planes.shape[0]))
    assert np.allclose(total, beauty, rtol=RTOL, atol=ATOL), np.abs(total - beauty).max()
    same_stats(st, st0)


@pytest.mark.parametrize("name", ["room", "mesh"])
def test_planes_sum_to_beauty_generated(name, mcrt):
    """Dynamic fetch and primitive sort keys (scenes past 2048 BVH4 nodes and 4096 primitives), one group per light."""
    scene = generated_scene(mcrt, name)
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=0, global_seed=7)
    try:
        planes, st = render_planes(mcrt, pt, cam, per_light(scene))
        beauty, st0 = render_beauty(pt, cam)
    finally:
        pt.close()
    total = mcrt.light_groups_combine(planes, np.ones(planes.shape[0]))
    assert np.allclose(total, beauty, rtol=RTOL, atol=ATOL), np.abs(total - beauty).max()
    same_stats(st, st0)


@pytest.mark.parametrize("precision", [0, 1])
def test_planes_sum_to_beauty_saturated_pool(precision, mcrt):
    """A 4096-path pool: camera work waits for room in every iteration."""
    scene, seed = load(mcrt, "veach_mis_64")
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=precision, global_seed=seed)
    try:
        pt.set_option("pool_paths", 4096)
        planes, st = render_planes(mcrt, pt, cam, per_light(scene))
        beauty, st0 = render_beauty(pt, cam)
    finally:
        pt.close()
    total = mcrt.light_groups_combine(planes, np.ones(planes.shape[0]))
    assert np.allclose(total, beauty, rtol=RTOL, atol=ATOL), np.abs(total - beauty).max()
    same_stats(st, st0)


# ---------------------------------------------------------------------------------------------- 2. plane g = the scene lit by group g only
def lit_by(planes, g):
    """What the scene with only group g's lights lit renders: plane g and the sky's (g = the sky's plane: that plane alone)."""
    return planes[g] + planes[-1] if g < planes.shape[0] - 1 else planes[-1]


def split_ids(mcrt, scene, how):
    if how == "emittance":
        return mcrt.light_groups_by_emittance(scene)[0]
    if how == "per_light":
        return per_light(scene)
    return (np.arange(scene.n_lights) >= scene.n_lights // 2).astype(np.uint32)   # two halves of the light list


@pytest.mark.parametrize("cid,how", [("veach_mis_64", "emittance"), ("ggx_64", "emittance"), ("c2_hexagon_room_96", "per_light"),
                                     ("smooth_mesh_64", "halves")])
def test_plane_is_scene_with_other_lights_dark(cid, how, mcrt):
    scene, seed = load(mcrt, cid)
    cam = scene.cameras()[0]
    ids = split_ids(mcrt, scene, how)
    n_groups = int(ids.max()) + 1
    assert n_groups >= 2
    pt = mcrt.PathTracer(scene, precision=0, global_seed=seed)
    try:
        planes, st = render_planes(mcrt, pt, cam, ids)
    finally:
        pt.close()
    for g in range(n_groups + 1):
        # g == n_groups: the sky plane against the scene with every light dark
        dark = mcrt.PathTracer(dark_except(mcrt, scene, ids, g), precision=0, global_seed=seed)
        try:
            ref, st_ref = render_beauty(dark, cam)
        finally:
            dark.close()
        lit = lit_by(planes, g)
        assert np.allclose(lit, ref, rtol=RTOL, atol=ATOL), (g, np.abs(lit - ref).max())
        same_stats(st, st_ref)
    assert planes[:n_groups].max() > 0


def test_sky_plane_of_lightless_scene_is_the_frame(mcrt):
    scene, seed = load(mcrt, "oren_nayar_64")
    assert scene.n_lights == 0
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=0, global_seed=seed)
    try:
        planes, st = render_planes(mcrt, pt, cam, mcrt.light_groups_by_emittance(scene)[0])
        beauty, st0 = render_beauty(pt, cam)
    finally:
        pt.close()
    assert planes.shape[0] == 1
    assert np.allclose(planes[0], beauty, rtol=RTOL, atol=ATOL)
    same_stats(st, st0)


# ---------------------------------------------------------------------------------------------- 3. against the CPU restatement
@pytest.mark.parametrize("cid", ["veach_mis_64", "ggx_64"])
def test_planes_match_cpu_restatement(cid, mcrt):
    from oracle import port
    scene, seed = load(mcrt, cid)
    cam = scene.cameras()[0]
    ids = mcrt.light_groups_by_emittance(scene)[0]
    pt = mcrt.PathTracer(scene, precision=0, global_seed=seed)
    try:
        planes, _ = render_planes(mcrt, pt, cam, ids)
    finally:
        pt.close()
    for g in range(planes.shape[0]):
        ref, _ = port.PortScene(dark_except(mcrt, scene, ids, g)).render_rows(cam, 0, cam.height, cam.sqrtspp, seed)
        rmse = float(np.sqrt(np.mean((lit_by(planes, g) - ref) ** 2)))
        assert rmse / max(float(np.abs(ref).mean()), 1e-300) < 1e-9, (g, rmse)


# ---------------------------------------------------------------------------------------------- 4. relighting
def test_combine_is_bit_equal_to_numpy(mcrt):
    import torch
    scene, seed = load(mcrt, "ggx_64")
    pt = mcrt.PathTracer(scene, global_seed=seed)
    rng = np.random.default_rng(5)
    try:
        for n_planes, n_values in ((1, 3), (3, 64 * 48 * 3), (7, 3 * 100003)):
            planes = rng.normal(size=(n_planes, n_values)) * 10.0 ** rng.integers(-3, 4, (n_planes, 1))
            w = rng.normal(size=(n_planes, 3))
            dev = torch.from_numpy(planes).cuda()
            out = torch_zeros((n_values,), np.nan)
            pt.light_groups_combine_dev(dev.data_ptr(), n_planes, n_values, w, out.data_ptr())
            got = out.cpu().numpy()
            want = mcrt.light_groups_combine(planes.reshape(n_planes, -1, 3), w).reshape(-1)
            assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    finally:
        pt.close()


def progressive_passes(mcrt, pt, cam, passes, **kw):
    prog = mcrt.Progressive(pt, cam, **kw)
    for s in passes:
        prog.add(s)
    return prog


@pytest.mark.parametrize("cid", ["veach_mis_64", "ggx_64"])
def test_relight_equals_scaled_scene(cid, mcrt):
    scene, seed = load(mcrt, cid)
    cam = scene.cameras()[0].resized(64, 48, 4)
    ids = mcrt.light_groups_by_emittance(scene)[0]
    n_groups = int(ids.max()) + 1
    w_group = np.linspace(0.25, 3.0, n_groups)
    weights = np.concatenate([w_group, [1.0]])   # the sky keeps weight 1
    passes = (3, 5, 8)
    pt = mcrt.PathTracer(scene, global_seed=seed)
    try:
        prog = progressive_passes(mcrt, pt, cam, passes, light_groups=ids)
        frame, err, tiles = prog.relight(weights)
        den, den_err = prog.denoise(weights=weights)
    finally:
        pt.close()
    scaled = mcrt.PathTracer(with_emittance(mcrt, scene, w_group[ids]), global_seed=seed)
    try:
        ref = progressive_passes(mcrt, scaled, cam, passes)
        ref_frame = ref.frame()
        ref_err, ref_tiles = ref.error()
        ref_den, ref_den_err = ref.denoise()
    finally:
        scaled.close()
    assert np.allclose(frame, ref_frame, rtol=RTOL, atol=ATOL), np.abs(frame - ref_frame).max()
    assert np.isclose(err, ref_err, rtol=1e-9) and np.allclose(tiles, ref_tiles, rtol=1e-9, atol=1e-12)
    assert np.allclose(den, ref_den, rtol=1e-9, atol=1e-12), np.abs(den - ref_den).max()
    assert np.isclose(den_err, ref_den_err, rtol=1e-9)


# ---------------------------------------------------------------------------------------------- 5. Progressive integration
def test_progressive_with_groups_matches_groupless(mcrt, tmp_path):
    scene, seed = load(mcrt, "veach_mis_64")
    cam = scene.cameras()[0]
    ids = mcrt.light_groups_by_emittance(scene)[0]
    pt = mcrt.PathTracer(scene, global_seed=seed)
    try:
        prog = progressive_passes(mcrt, pt, cam, (1, 3), light_groups=ids)
        plain = progressive_passes(mcrt, pt, cam, (1, 3))
        assert np.allclose(prog.frame(), plain.frame(), rtol=RTOL, atol=ATOL)
        (e, t), (e0, t0) = prog.error(), plain.error()
        assert np.isclose(e, e0, rtol=1e-9) and np.allclose(t, t0, rtol=1e-9, atol=1e-12)
        groups = prog.group_frames()
        assert groups.shape == (4, cam.height, cam.width, 3)
        assert np.allclose(groups.sum(0), plain.frame(), rtol=1e-11, atol=ATOL)
        assert prog.stats == plain.stats
        # checkpoints: the planes come back; a groups checkpoint and a groupless one refuse each other
        path, path0 = str(tmp_path / "groups.npz"), str(tmp_path / "plain.npz")
        prog.save(path)
        plain.save(path0)
        back = mcrt.Progressive.load(path, pt, cam, light_groups=ids)
        for h in (0, 1):
            assert np.array_equal(back.rgb[h].cpu().numpy(), prog.rgb[h].cpu().numpy())
        back.add(2)
        prog.add(2)
        assert np.allclose(back.frame(), prog.frame(), rtol=RTOL, atol=ATOL)
        with pytest.raises(mcrt.McrtError, match="light groups"):
            mcrt.Progressive.load(path, pt, cam)
        with pytest.raises(mcrt.McrtError, match="light groups"):
            mcrt.Progressive.load(path0, pt, cam, light_groups=ids)
        with pytest.raises(mcrt.McrtError, match="light_groups"):
            mcrt.Progressive.load(path, pt, cam, light_groups=per_light(scene)[::-1].copy())
    finally:
        pt.close()


def test_adaptive_retires_the_same_tiles(mcrt):
    scene, seed = load(mcrt, "c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54, 8)
    ids = per_light(scene)
    pt = mcrt.PathTracer(scene, global_seed=seed)
    try:
        runs = []
        for groups in (ids, None):
            prog = mcrt.Progressive(pt, cam, tile=16, light_groups=groups)
            frame = prog.render_adaptive(4, 64, 0.05, min_samples=8)
            runs.append((prog, frame))
    finally:
        pt.close()
    (a, fa), (b, fb) = runs
    assert len(a.history) == len(b.history) > 1 and a.stop_reason == b.stop_reason
    assert any(h["retired"].any() for h in a.history)
    for ha, hb in zip(a.history, b.history):
        assert np.array_equal(ha["retired"], hb["retired"]) and np.array_equal(ha["tile_counts"], hb["tile_counts"])
    assert np.allclose(fa, fb, rtol=RTOL, atol=ATOL)


# ---------------------------------------------------------------------------------------------- 6. refusals
def raw_groups_call(mcrt, pt, cam, sums, n_planes, integrator_kind=0, active=None):
    mask = np.ascontiguousarray(active, np.uint8) if active is not None else None
    return mcrt.lib().mcrt_render_accumulate_groups_dev(pt.ctx, C.byref(cam.rec), 0, 1, cam.height, 16,
                                                        mask.ctypes.data_as(C.c_void_p) if mask is not None else None, 0, 1,
                                                        pt.global_seed, integrator_kind, 0, C.c_void_p(sums.data_ptr()), n_planes, None)


def set_table(mcrt, pt, ids, n_lights, n_groups):
    ids = np.ascontiguousarray(ids, np.uint32)
    return mcrt.lib().mcrt_set_light_groups(pt.ctx, ids.ctypes.data_as(C.c_void_p), n_lights, n_groups)


def test_refusals_leave_the_sums_untouched(mcrt):
    scene, seed = load(mcrt, "veach_mis_64")
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, global_seed=seed)
    sums = torch_zeros((4, cam.height, cam.width, 3), 7.0)
    try:
        L = mcrt.lib()
        assert raw_groups_call(mcrt, pt, cam, sums, 4) == ERR_INVALID          # no table yet
        assert set_table(mcrt, pt, [0, 1, 3], 3, 3) == ERR_INVALID             # id >= n_groups
        assert set_table(mcrt, pt, [0, 1], 2, 3) == ERR_INVALID                # wrong n_lights
        assert raw_groups_call(mcrt, pt, cam, sums, 4) == ERR_INVALID          # the refused tables set nothing
        assert set_table(mcrt, pt, [0, 1, 2], 3, 3) == 0
        assert raw_groups_call(mcrt, pt, cam, sums, 3) == ERR_INVALID          # n_planes != n_groups + 1
        assert raw_groups_call(mcrt, pt, cam, sums, 4, integrator_kind=1) == ERR_UNSUPPORTED   # photon mapper
        film = mcrt.FilmRec(mcrt.FILM_FILTERS["mitchell-netravali"], 0, 0.0)
        assert L.mcrt_set_film(pt.ctx, C.byref(film)) == 0
        assert raw_groups_call(mcrt, pt, cam, sums, 4) == ERR_UNSUPPORTED      # reconstruction filter
        assert L.mcrt_set_film(pt.ctx, None) == 0
        pt.upload_scene()
        assert raw_groups_call(mcrt, pt, cam, sums, 4) == ERR_INVALID          # a new upload clears the table
        assert bool((sums == 7.0).all())
        assert set_table(mcrt, pt, [0, 1, 2], 3, 3) == 0
        assert L.mcrt_set_light_groups(pt.ctx, None, 0, 0) == 0                # clearing
        assert raw_groups_call(mcrt, pt, cam, sums, 4) == ERR_INVALID
        assert bool((sums == 7.0).all())
    finally:
        pt.close()


def test_photon_mapper_has_no_groups(mcrt):
    scene, seed = load(mcrt, "pm_hexagon_room_64")
    cam = scene.cameras()[0]
    pm = mcrt.PhotonMapper(scene, global_seed=seed)
    sums = torch_zeros((2, cam.height, cam.width, 3), 7.0)
    try:
        with pytest.raises(mcrt.McrtError):
            pm.set_light_groups([0, 0])
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive(pm, cam, light_groups=[0, 0])
        assert set_table(mcrt, pm, [0, 0], 2, 1) == 0
        assert raw_groups_call(mcrt, pm, cam, sums, 2, integrator_kind=1) == ERR_UNSUPPORTED
        with pytest.raises(mcrt.McrtError):
            pm.render_accumulate_groups_dev(cam, sums.data_ptr(), 2, 0, 1)
        assert bool((sums == 7.0).all())
    finally:
        pm.close()


def test_table_before_any_upload(mcrt):
    ctx = C.c_void_p()
    assert mcrt.lib().mcrt_init(0, C.byref(ctx)) == 0
    try:
        ids = np.zeros(1, np.uint32)
        assert mcrt.lib().mcrt_set_light_groups(ctx, ids.ctypes.data_as(C.c_void_p), 1, 1) == ERR_NO_SCENE
    finally:
        mcrt.lib().mcrt_destroy(ctx)


def test_one_plane_entry_points_ignore_the_table(mcrt):
    scene, seed = load(mcrt, "ggx_64")
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, global_seed=seed)
    spp = cam.sqrtspp ** 2
    try:
        before, st0 = render_beauty(pt, cam)
        pt.set_light_groups(per_light(scene))
        sums = torch_zeros((2, cam.height, cam.width, 3))   # room for a second plane the render must not touch
        st = pt.render_accumulate_dev(cam, sums.data_ptr(), None, 0, spp)
        out = sums.cpu().numpy()
    finally:
        pt.close()
    assert np.allclose(out[0] / spp, before, rtol=RTOL, atol=ATOL)
    assert not out[1].any()
    same_stats(st, st0)
