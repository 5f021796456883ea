"""Light path expressions (mcrt_render_accumulate_lpe_dev and Progressive's lpes): each plane holds the contributions
whose event string its expression matches.

The AOV planes, the light-group planes and the beauty frame are each a handful of expressions, so the LPE render is first
held to those three existing renders: every deposit is the existing kernels' value, and only the order of the float64
film additions differs (rtol 1e-12, equal ray counts). New expressions are then held to identities between planes that
partition the same contributions another way and to the CPU restatement of each contribution's event string
(tests/lpe_ref.cpp) at the parity bar, and the dead-state rule to an unchanged plane with fewer rays."""
import ctypes as C

import numpy as np
import pytest

from conftest import golden_cases
from scene_gen import generated_scene
from test_aovs_cpu import load_case
from test_gpu_aovs import ATOL, BAND_RULE, DIRECT_FLOOR, RTOL, bias_ratio, render_aovs, render_beauty, same_stats, torch_zeros
from test_gpu_fast_mode import BIAS_FLOOR

pytestmark = pytest.mark.gpu

PATH_CASES = [c for c in golden_cases() if not c.startswith("pm_")]
NEW_GROUND = ["C<RD>L'0'", "C.{2}[LB]", "C.{3,}[LB]", "C[^S]*L", "C<RD>S+L", "C(<RS>|<TS>)+B"]
NEW_CASES = ["ior_test_nobvh_64", "metals_64", "ggx_64", "c2_hexagon_room_96", "glass_room"]
ERR_INVALID, ERR_UNSUPPORTED = -1, -4


def render_lpe(pt, cam, n, precision=None, spp=None, active=None, tile=0):
    spp = cam.sqrtspp ** 2 if spp is None else spp
    planes = torch_zeros((n, cam.height, cam.width, 3))
    st = pt.render_accumulate_lpe_dev(cam, planes.data_ptr(), n, 0, spp, tile=tile, active=active, precision=precision)
    return planes.cpu().numpy() / spp, st


def render_groups(pt, cam, n, precision=None, spp=None, active=None, tile=0):
    spp = cam.sqrtspp ** 2 if spp is None else spp
    planes = torch_zeros((n, cam.height, cam.width, 3))
    st = pt.render_accumulate_groups_dev(cam, planes.data_ptr(), n, 0, spp, tile=tile, active=active, precision=precision)
    return planes.cpu().numpy() / spp, st


def close(a, b):
    assert np.allclose(a, b, rtol=RTOL, atol=ATOL), np.abs(a - b).max()


def existing_equivalents(mcrt, pt, scene, cam, precision=None, active=None, tile=0):
    """The LPE render of the AOV, light-group and beauty expressions against those three renders."""
    ids, emittance = mcrt.light_groups_by_emittance(scene)
    n_groups = len(emittance)
    exprs = list(mcrt.AOV_LPES) + [f"C.*L'{g}'" for g in range(n_groups)] + ["C.*B", "C.*"]
    pt.set_light_groups(ids, n_groups)
    pt.set_light_path_expressions(exprs)
    planes, st = render_lpe(pt, cam, len(exprs), precision, active=active, tile=tile)
    aovs, st_a = render_aovs(pt, cam, precision, active=active, tile=tile)
    groups, st_g = render_groups(pt, cam, n_groups + 1, precision, active=active, tile=tile)
    beauty, st_b = render_beauty(pt, cam, precision, active=active, tile=tile)
    close(planes[:8], aovs)
    same_stats(st, st_a)
    close(planes[8:9 + n_groups], groups)
    close(planes[-1], beauty)
    same_stats(st, st_g)
    same_stats(st, st_b)
    return planes


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("cid", PATH_CASES + ["glass_room"])
def test_equal_to_aovs_groups_and_beauty(cid, precision, mcrt):
    scene, seed = load_case(mcrt, cid)
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=precision, global_seed=seed)
    try:
        existing_equivalents(mcrt, pt, scene, cam)
    finally:
        pt.close()


def test_equal_on_generated_room(mcrt):
    """Dynamic fetch and primitive sort keys (a scene past 2048 BVH4 nodes and 4096 primitives)."""
    scene = generated_scene(mcrt, "room")
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=0, global_seed=7)
    try:
        existing_equivalents(mcrt, pt, scene, cam)
    finally:
        pt.close()


@pytest.mark.parametrize("precision", [0, 1])
def test_equal_with_saturated_pool(precision, mcrt):
    scene, seed = load_case(mcrt, "c2_hexagon_room_96")
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=precision, global_seed=seed)
    try:
        pt.set_option("pool_paths", 4096)
        existing_equivalents(mcrt, pt, scene, cam)
    finally:
        pt.close()


@pytest.mark.parametrize("precision", [0, 1])
def test_equal_with_active_tiles(precision, mcrt):
    scene, seed = load_case(mcrt, "c2_hexagon_room_96")
    cam = scene.cameras()[0]
    tile = 16
    active = np.zeros(mcrt.tile_grid(cam.height, cam.width, tile), bool)
    active.flat[::3] = True
    pt = mcrt.PathTracer(scene, precision=precision, global_seed=seed)
    try:
        planes = existing_equivalents(mcrt, pt, scene, cam, active=active, tile=tile)
    finally:
        pt.close()
    inactive = ~np.kron(active, np.ones((tile, tile), bool))[:cam.height, :cam.width]
    assert not planes[:, inactive].any()


# ---------------------------------------------------------------------------------------------- new expressions
# NEW_GROUND, then planes that split the same contributions another way: by the number of vertices (C[LB], C.[LB] with
# C.{2}[LB] and C.{3,}[LB] partition every string), and the diffuse direct light by source (with C<RD>L'0')
SPLITS = ["C[LB]", "C.[LB]", "C<RD>L'1'", "C<RD>B", "C.*"]


def two_groups(scene):
    return np.arange(scene.n_lights, dtype=np.uint32) % 2


@pytest.mark.parametrize("cid", NEW_CASES)
def test_new_expressions_split_consistently(cid, mcrt):
    scene, seed = load_case(mcrt, cid)
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=0, global_seed=seed)
    try:
        pt.set_light_groups(two_groups(scene), 2)
        pt.set_light_path_expressions(NEW_GROUND + SPLITS)
        planes, _ = render_lpe(pt, cam, len(NEW_GROUND) + len(SPLITS))
        aovs, _ = render_aovs(pt, cam)
    finally:
        pt.close()
    p = dict(zip(NEW_GROUND + SPLITS, planes))
    assert np.isfinite(planes).all() and (planes >= 0).all()
    close(p["C[LB]"] + p["C.[LB]"] + p["C.{2}[LB]"] + p["C.{3,}[LB]"], p["C.*"])
    close(p["C<RD>L'0'"] + p["C<RD>L'1'"] + p["C<RD>B"], aovs[2])   # diffuse_direct
    close(p["C[LB]"], aovs[0] + aovs[1])
    assert p["C.{2}[LB]"].any() and p["C.{3,}[LB]"].any() and p["C[^S]*L"].any()
    # a subset never exceeds its superset: C<RD>S+L and C<RD>L'0' are inside C.*
    assert (p["C<RD>S+L"] <= p["C.*"] * (1 + 1e-12) + ATOL).all()


# Every vertex event on its own, at any depth and at a deep one: a wrong smooth / rough or reflect / refract label, or an
# event stated at the wrong vertex, moves light between these planes
EVENTS = ["C.*<RS>.*", "C.*<RG>.*", "C.*<TS>.*", "C.*<TG>.*", "C..<RD>.*", "C...<.G>.*"]


@pytest.mark.parametrize("cid", NEW_CASES)
def test_planes_match_cpu_restatement(cid, mcrt):
    """Parity planes against tests/lpe_ref.cpp (the restated reference's contributions per event string, matched by
    Python's re) at the parity bar, relative RMSE 1e-9; the C2-band rule of DESIGN.md §8 for the glass room only, as in
    tests/test_gpu_aovs.py."""
    import lpe_ref
    scene, seed = load_case(mcrt, cid)
    cam = scene.cameras()[0]
    ids = two_groups(scene)
    exprs = NEW_GROUND + EVENTS
    pt = mcrt.PathTracer(scene, precision=0, global_seed=seed)
    try:
        pt.set_light_groups(ids, 2)
        pt.set_light_path_expressions(exprs)
        planes, _ = render_lpe(pt, cam, len(exprs))
    finally:
        pt.close()
    ref = lpe_ref.render_strings(scene, cam, 0, cam.height, cam.sqrtspp, seed, ids).planes(exprs)
    keep = np.ones((cam.height, cam.width), bool)
    if cid in BAND_RULE:
        d = np.abs(planes - ref).max(axis=(0, 3))
        out = d > 1e-9 * max(1.0, np.abs(ref).max())
        print(f"{cid}: {int(out.sum())} of {out.size} pixels differ from the restatement")
        assert out.sum() <= out.size // 1000
        keep = ~out
    for k, e in enumerate(exprs):
        a, b = planes[k][keep], ref[k][keep]
        if not b.any():
            assert not a.any(), (e, np.abs(a).max())
            continue
        rel = float(np.sqrt(np.mean((a - b) ** 2))) / float(np.abs(b).mean())
        print(f"{cid} {e}: mean {b.mean():.3e}, relative RMSE {rel:.2e}")
        assert rel < 1e-9, (e, rel)


@pytest.mark.parametrize("cid", NEW_CASES)
def test_fast_mode_new_planes_agree_with_parity(cid, mcrt):
    scene, seed = load_case(mcrt, cid)
    cam = scene.cameras()[0]
    cam = cam.resized(cam.width, cam.height, 8)
    pt = mcrt.PathTracer(scene, precision=0, global_seed=seed)
    try:
        pt.set_light_groups(two_groups(scene), 2)
        pt.set_light_path_expressions(NEW_GROUND)
        a, _ = render_lpe(pt, cam, len(NEW_GROUND), precision=0)
        b, _ = render_lpe(pt, cam, len(NEW_GROUND), precision=1)
    finally:
        pt.close()
    assert np.isfinite(b).all()
    # Planes made mostly of next-event light at one vertex depth take the AOV tests' direct-plane floor: their low
    # variance resolves fast mode's next-event offset bias, as the direct AOV planes' does. Measured on one H100 at 8x8
    # spp: C.{2}[LB] (light sampled at the second vertex) on ior_test_nobvh_64 at 1.5 times the frame-bias bar.
    next_event = {"C<RD>L'0'", "C.{2}[LB]", "C[^S]*L"}
    over = []
    for k, e in enumerate(NEW_GROUND):
        if not a[k].any() and not b[k].any():
            continue
        z, ratio = bias_ratio(b[k] - a[k], a[k], DIRECT_FLOOR if e in next_event else BIAS_FLOOR)
        print(f"{cid} {e}: mean f64 {a[k].mean():.3e} f32 {b[k].mean():.3e}, bias z {np.round(z, 2).tolist()}, "
              f"bias/bar {ratio.max():.2f}")
        if not (ratio <= 1.0).all():
            over.append((e, ratio))
    assert not over, over


# ---------------------------------------------------------------------------------------------- dead paths
def test_dead_paths_end_early(mcrt):
    scene, seed = load_case(mcrt, "c2_hexagon_room_96")
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=0, global_seed=seed)
    try:
        pt.set_light_path_expressions(["C<RD>L"])
        alone, st = render_lpe(pt, cam, 1)
        pt.set_light_path_expressions(["C<RD>L", "C.*"])
        both, st_all = render_lpe(pt, cam, 2)
    finally:
        pt.close()
    close(alone[0], both[0])
    assert alone[0].any()
    assert st["paths"] == st_all["paths"]
    assert st["extension_rays"] < st_all["extension_rays"] and st["shadow_rays"] < st_all["shadow_rays"]
    print(f"C<RD>L alone: {st['extension_rays']} extension / {st['shadow_rays']} shadow rays, with C.*: "
          f"{st_all['extension_rays']} / {st_all['shadow_rays']}")


# ---------------------------------------------------------------------------------------------- Progressive
LPES = ["C<RD>L'0'", "C.{3,}[LB]", "C[^S]*L"]


def test_progressive_with_lpes(mcrt, tmp_path):
    scene, seed = load_case(mcrt, "c2_hexagon_room_96")
    cam = scene.cameras()[0]
    ids = two_groups(scene)
    pt = mcrt.PathTracer(scene, global_seed=seed)
    try:
        prog = mcrt.Progressive(pt, cam, lpes=LPES, light_groups=ids)
        plain = mcrt.Progressive(pt, cam)
        for s in (1, 3):
            prog.add(s)
            plain.add(s)
        assert np.allclose(prog.frame(), plain.frame(), rtol=RTOL, atol=ATOL)
        (e, t), (e0, t0) = prog.error(), plain.error()
        assert np.isclose(e, e0, rtol=1e-9) and np.allclose(t, t0, rtol=1e-9, atol=1e-12)
        assert prog.stats == plain.stats
        frames, errors = prog.lpe_frames()
        assert frames.shape == (len(LPES), cam.height, cam.width, 3) and errors.shape == (len(LPES),)
        assert np.isfinite(errors).all() and (errors >= 0).all()
        # relight: one weight per expression, the beauty plane left out
        frame, err, tiles = prog.relight([1.0, 0.0, 0.0])
        assert np.allclose(frame, frames[0], rtol=1e-9, atol=1e-12)
        frame2, _, _ = prog.relight([0.0, 2.0, 1.0])
        assert np.allclose(frame2, 2 * frames[1] + frames[2], rtol=1e-9, atol=1e-12)
        with pytest.raises(mcrt.McrtError):
            prog.relight(np.ones(len(LPES) + 1))
        den, den_err = prog.denoise()
        ref_den, ref_den_err = plain.denoise()
        assert np.allclose(den, ref_den, rtol=1e-9, atol=1e-12) and np.isclose(den_err, ref_den_err, rtol=1e-9)
        prog.denoise(weights=[1.0, 1.0, 0.0])
        # checkpoints: expressions and groups are part of the identity
        path, path0 = str(tmp_path / "lpe.npz"), str(tmp_path / "plain.npz")
        prog.save(path)
        plain.save(path0)
        back = mcrt.Progressive.load(path, pt, cam, light_groups=ids, lpes=LPES)
        for h in (0, 1):
            assert np.array_equal(back.rgb[h].cpu().numpy(), prog.rgb[h].cpu().numpy())
        back.add(2)
        prog.add(2)
        assert np.allclose(back.frame(), prog.frame(), rtol=RTOL, atol=ATOL)
        assert np.allclose(back.lpe_frames()[0], prog.lpe_frames()[0], rtol=RTOL, atol=ATOL)
        with pytest.raises(mcrt.McrtError, match="light path expressions"):
            mcrt.Progressive.load(path, pt, cam)
        with pytest.raises(mcrt.McrtError, match="light path expressions"):
            mcrt.Progressive.load(path0, pt, cam, light_groups=ids, lpes=LPES)
        with pytest.raises(mcrt.McrtError, match="lpes"):
            mcrt.Progressive.load(path, pt, cam, light_groups=ids, lpes=LPES[:2] + ["C.*B"])
        with pytest.raises(mcrt.McrtError, match="lpe_groups"):
            mcrt.Progressive.load(path, pt, cam, light_groups=1 - ids, lpes=LPES)
        with pytest.raises(mcrt.McrtError):
            plain.lpe_frames()
    finally:
        pt.close()


def test_adaptive_retires_the_same_tiles(mcrt):
    scene, seed = load_case(mcrt, "c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54, 8)
    pt = mcrt.PathTracer(scene, global_seed=seed)
    try:
        runs = []
        for lpes in (LPES, None):
            prog = mcrt.Progressive(pt, cam, tile=16, lpes=lpes, light_groups=two_groups(scene) if lpes else None)
            frame = prog.render_adaptive(4, 64, 0.05, min_samples=8)
            runs.append((prog, frame))
        (a, fa), (b, fb) = runs
        assert len(a.history) == len(b.history) > 1 and a.stop_reason == b.stop_reason
        assert any(h["retired"].any() for h in a.history)
        for ha, hb in zip(a.history, b.history):
            assert np.array_equal(ha["retired"], hb["retired"]) and np.array_equal(ha["tile_counts"], hb["tile_counts"])
        assert np.allclose(fa, fb, rtol=RTOL, atol=ATOL)
    finally:
        pt.close()


# ---------------------------------------------------------------------------------------------- refusals
def raw_lpe_call(mcrt, pt, cam, sums_ptr, n_planes, integrator_kind=0):
    return mcrt.lib().mcrt_render_accumulate_lpe_dev(pt.ctx, C.byref(cam.rec), 0, 1, cam.height, 16, None, 0, 1,
                                                     pt.global_seed, integrator_kind, 0, C.c_void_p(sums_ptr), n_planes, None)


def test_refusals_leave_the_sums_untouched(mcrt):
    scene, seed = load_case(mcrt, "ggx_64")
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, global_seed=seed)
    sums = torch_zeros((4, cam.height, cam.width, 3), 7.0)
    exprs = ["C<RD>L", "C.*"]
    try:
        L = mcrt.lib()
        assert raw_lpe_call(mcrt, pt, cam, sums.data_ptr(), 2) == ERR_INVALID                 # no table
        pt.set_light_path_expressions(exprs)
        assert raw_lpe_call(mcrt, pt, cam, sums.data_ptr(), 1) == ERR_INVALID                 # n_planes != 2
        assert raw_lpe_call(mcrt, pt, cam, sums.data_ptr(), 3) == ERR_INVALID
        assert raw_lpe_call(mcrt, pt, cam, None, 2) == ERR_INVALID                            # null planes
        assert raw_lpe_call(mcrt, pt, cam, sums.data_ptr(), 2, integrator_kind=1) == ERR_UNSUPPORTED   # photon mapper
        film = mcrt.FilmRec(mcrt.FILM_FILTERS["mitchell-netravali"], 0, 0.0)
        assert L.mcrt_set_film(pt.ctx, C.byref(film)) == 0
        assert raw_lpe_call(mcrt, pt, cam, sums.data_ptr(), 2) == ERR_UNSUPPORTED             # reconstruction filter
        assert L.mcrt_set_film(pt.ctx, None) == 0
        pt.set_light_groups(np.zeros(scene.n_lights, np.uint32), 1)                          # clears the LPE table
        assert raw_lpe_call(mcrt, pt, cam, sums.data_ptr(), 2) == ERR_INVALID
        pt.set_light_path_expressions(exprs)
        pt.upload_scene()                                                                     # so does a scene upload
        assert raw_lpe_call(mcrt, pt, cam, sums.data_ptr(), 2) == ERR_INVALID
        pt.set_light_path_expressions(exprs)
        pt.set_light_path_expressions(None)                                                   # and clearing it
        assert raw_lpe_call(mcrt, pt, cam, sums.data_ptr(), 2) == ERR_INVALID
        assert bool((sums == 7.0).all())
        # compiler refusals reach the caller with the compiler's reason
        with pytest.raises(mcrt.McrtError, match="offset 3"):
            pt.set_light_path_expressions(["C<RX>L"])
        with pytest.raises(mcrt.McrtError, match="no group table"):
            pt.set_light_path_expressions(["CL'0'"])
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive(pt, cam, lpes=exprs, aovs=True)
        # Progressive adds the beauty plane: 31 expressions of its caller at most
        with pytest.raises(mcrt.McrtError, match="32 expressions, at most 31"):
            mcrt.Progressive(pt, cam, lpes=["C.*"] * 32)
        mcrt.Progressive(pt, cam, lpes=["C.*"] * 31)
        # labels need the groups they name: without light_groups, Progressive does not resolve them against the
        # integrator's current table
        pt.set_light_groups(np.zeros(scene.n_lights, np.uint32), 1)
        with pytest.raises(mcrt.McrtError, match="no group table"):
            mcrt.Progressive(pt, cam, lpes=["C.*L'0'"])
        mcrt.Progressive(pt, cam, lpes=["C.*L'0'"], light_groups=np.zeros(scene.n_lights, np.uint32))
        filtered = scene.cameras()[0]
        filtered.film = {"filter": "mitchell-netravali"}
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive(pt, filtered, lpes=exprs)
    finally:
        pt.close()


def test_photon_mapper_has_no_lpes(mcrt):
    scene, seed = load_case(mcrt, "pm_hexagon_room_64")
    cam = scene.cameras()[0]
    pm = mcrt.PhotonMapper(scene, global_seed=seed)
    sums = torch_zeros((2, cam.height, cam.width, 3), 7.0)
    try:
        with pytest.raises(mcrt.McrtError):
            mcrt.Progressive(pm, cam, lpes=["C.*"])
        pm.set_light_path_expressions(["C.*L", "C.*"])
        assert raw_lpe_call(mcrt, pm, cam, sums.data_ptr(), 2, integrator_kind=1) == ERR_UNSUPPORTED
        assert bool((sums == 7.0).all())
    finally:
        pm.close()


def test_table_changes_no_other_entry_point(mcrt):
    scene, seed = load_case(mcrt, "ggx_64")
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, global_seed=seed)
    try:
        ids, emittance = mcrt.light_groups_by_emittance(scene)
        n_groups = len(emittance)
        pt.set_light_groups(ids, n_groups)
        before, st0 = render_beauty(pt, cam)
        aovs0, sa0 = render_aovs(pt, cam)
        groups0, sg0 = render_groups(pt, cam, n_groups + 1)
        pt.set_light_path_expressions(["C<RD>L'0'", "C.*B"])
        render_lpe(pt, cam, 2)
        after, st = render_beauty(pt, cam)
        aovs, sa = render_aovs(pt, cam)
        groups, sg = render_groups(pt, cam, n_groups + 1)
    finally:
        pt.close()
    close(after, before)
    close(aovs, aovs0)
    close(groups, groups0)
    same_stats(st, st0)
    same_stats(sa, sa0)
    same_stats(sg, sg0)
