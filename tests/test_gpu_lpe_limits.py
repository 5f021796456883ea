"""Light path expressions on the device at the limits of include/mcrt_abi.h: the tables of tests/test_lpe_limits_cpu.py,
which reach forward and reverse DFA states past 127 (the 8-bit state fields of k_shade, k_emit_shade and KnnQuery), an
accept mask with all 32 bits set (ALL32, whose photon runs are keyed by 0xFFFFFFFF), 64 labels (71 symbols) and
Progressive's beauty plane on bit 31 (P31).

- the path tracer: float64 planes against the CPU restatement (tests/lpe_ref.cpp) at relative RMSE 1e-9, float32 planes
  against float64 at the fast-mode bars, and the identities: every ALL32 plane is the one-plane render, each LABELS
  plane is its light-group plane, and C.* is the beauty under every table;
- the photon mapper, k-NN and fixed-radius gather: each photon's state is the reverse table over its restated events,
  planes match the restatement (tests/pm_lpe_ref.cpp) at 1e-9, and ALL32 planes are the one-plane render;
- Progressive and ProgressivePhotonMapping with 31 expressions behave as without them."""
import numpy as np
import pytest

from test_aovs_cpu import load_case
from test_gpu_aovs import ATOL, BAND_RULE, DIRECT_FLOOR, RTOL, bias_ratio, render_beauty, same_stats, torch_zeros
from test_gpu_fast_mode import BIAS_FLOOR
from test_gpu_lpe import close, render_groups, render_lpe
from test_gpu_photon_light_groups import emit_params, f32_rtol, gather_radius_of, max_gathered
from test_gpu_photon_light_groups import render_beauty as pm_render_beauty
from test_gpu_photon_mapper import allowance, camera_of, frame_error
from test_gpu_pm_lpe import REF_SEED, reverse_walk, restated_for_device, set_table
from test_gpu_pm_lpe import same_stats as pm_same_stats
from test_lpe_limits_cpu import ALL32, GLASS_ROOM, HEAD, LABEL_GROUPS, LABELS, N_LABEL_GROUPS, P31, TAIL, label_ids

pytestmark = pytest.mark.gpu

TABLES = {"TAIL": TAIL, "HEAD": HEAD, "LABELS": LABELS}
# (table, case): TAIL on three golden scenes and on the glass room, where paths keep TAIL states past 127 between vertices;
# HEAD on ior_test_nobvh_64 (states past 127 through two smooth transmissions); LABELS on the scene with 320 lights
PATH_CASES = [("TAIL", "smooth_mesh_64"), ("LABELS", "smooth_mesh_64"), ("TAIL", "ior_test_nobvh_64"), ("TAIL", "ggx_64"),
              ("TAIL", GLASS_ROOM), ("HEAD", "ior_test_nobvh_64")]


def set_pt_table(pt, scene, table):
    if table == "LABELS":
        pt.set_light_groups(label_ids(scene), N_LABEL_GROUPS)
    else:
        pt.set_light_groups(None)
    pt.set_light_path_expressions(TABLES[table])


# ---------------------------------------------------------------------------------------------- path tracer
@pytest.mark.parametrize("table,cid", PATH_CASES)
def test_path_planes_match_cpu_restatement(table, cid, mcrt):
    """test_gpu_lpe's restatement test at the limit tables"""
    import lpe_ref
    scene, seed = load_case(mcrt, cid)
    cam = scene.cameras()[0]
    exprs = TABLES[table]
    pt = mcrt.PathTracer(scene, precision=0, global_seed=seed)
    try:
        set_pt_table(pt, scene, table)
        planes, _ = render_lpe(pt, cam, len(exprs))
    finally:
        pt.close()
    ids = label_ids(scene) if table == "LABELS" else None
    ref = lpe_ref.render_strings(scene, cam, 0, cam.height, cam.sqrtspp, seed, ids).planes(exprs)
    keep = np.ones((cam.height, cam.width), bool)
    if cid in BAND_RULE:
        d = np.abs(planes - ref).max(axis=(0, 3))
        out = d > 1e-9 * max(1.0, np.abs(ref).max())
        print(f"{cid}: {int(out.sum())} of {out.size} pixels differ from the restatement")
        assert out.sum() <= out.size // 1000
        keep = ~out
    reached = 0
    for k, e in enumerate(exprs):
        a, b = planes[k][keep], ref[k][keep]
        if not b.any():
            assert not a.any(), (e, np.abs(a).max())
            continue
        reached += 1
        rel = float(np.sqrt(np.mean((a - b) ** 2))) / float(np.abs(b).mean())
        assert rel < 1e-9, (e, rel)
    print(f"{table} {cid}: {reached} of {len(exprs)} planes nonzero")
    assert reached > len(exprs) // 2


@pytest.mark.parametrize("table,cid", PATH_CASES)
def test_fast_mode_limit_planes_agree_with_parity(table, cid, mcrt):
    """test_fast_mode_new_planes_agree_with_parity's bars: the direct-plane floor for the planes made mostly of the light
    at one vertex class (TAIL's and HEAD's event planes) or of one group's light (LABELS), the frame's for C.*"""
    scene, seed = load_case(mcrt, cid)
    cam = scene.cameras()[0]
    cam = cam.resized(cam.width, cam.height, 8)
    exprs = TABLES[table]
    pt = mcrt.PathTracer(scene, precision=0, global_seed=seed)
    try:
        set_pt_table(pt, scene, table)
        a, _ = render_lpe(pt, cam, len(exprs), precision=0)
        b, _ = render_lpe(pt, cam, len(exprs), precision=1)
    finally:
        pt.close()
    assert np.isfinite(b).all()
    over = []
    for k, e in enumerate(exprs):
        if not a[k].any() and not b[k].any():
            continue
        _, ratio = bias_ratio(b[k] - a[k], a[k], BIAS_FLOOR if e == "C.*" else DIRECT_FLOOR)
        if not (ratio <= 1.0).all():
            over.append((e, ratio))
    assert not over, over


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("cid", ["smooth_mesh_64", GLASS_ROOM])
def test_path_identities_at_the_limits(cid, precision, mcrt):
    """Every ALL32 plane is the one-plane render; C.* is the beauty under TAIL, HEAD and P31 + C.*; on smooth_mesh_64,
    each LABELS plane is its group's plane of render_accumulate_groups_dev, the union of the 64 labels their sum."""
    scene, seed = load_case(mcrt, cid)
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, precision=precision, global_seed=seed)
    try:
        beauty, st0 = render_beauty(pt, cam)
        pt.set_light_path_expressions(ALL32)
        planes, st = render_lpe(pt, cam, len(ALL32))
        same_stats(st, st0)
        for p in planes:
            close(p, beauty)
        for exprs in (TAIL, HEAD, P31 + ["C.*"]):
            pt.set_light_path_expressions(exprs)
            planes, st = render_lpe(pt, cam, len(exprs))
            close(planes[-1], beauty)
            same_stats(st, st0)
        if scene.n_lights >= N_LABEL_GROUPS:
            ids = label_ids(scene)
            pt.set_light_groups(ids, N_LABEL_GROUPS)
            groups, st_g = render_groups(pt, cam, N_LABEL_GROUPS + 1)
            pt.set_light_path_expressions(LABELS)
            planes, st = render_lpe(pt, cam, len(LABELS))
            same_stats(st, st_g)
            for i, g in enumerate(LABEL_GROUPS):
                close(planes[i], groups[g])
                assert groups[g].any()
            close(planes[-1], groups[:-1].sum(axis=0))
    finally:
        pt.close()


# ---------------------------------------------------------------------------------------------- photon mapper
def pm_params(scene, cid):
    """the photon-pass parameters of the restatement tests: k 100, caustic factor 1, 20000 emissions"""
    return dict(emissions=20000, caustic_factor=1.0, max_photons_per_octree_leaf=200, k_nearest_photons=100,
                direct_visualization=False, scene_bounds=scene.extra["scene_bounds"])


def pm_ids(scene, table):
    return label_ids(scene) if table == "LABELS" else None


@pytest.mark.parametrize("table,cid", [("TAIL", GLASS_ROOM), ("TAIL", "pm_hexagon_room_64"), ("HEAD", "pm_hexagon_room_64")])
def test_photon_states_follow_the_restated_events(table, cid, mcrt):
    """test_gpu_pm_lpe's check at the limit tables: every paired photon's state is the reverse table over its restated
    events; on the glass room some are past 127"""
    scene, _ = load_case(mcrt, cid)
    ep = pm_params(scene, cid)
    exprs = TABLES[table]
    pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=REF_SEED, emit=ep)
    try:
        set_table(pm, exprs)
        pm.emit_again()
        t = mcrt.lpe_compile_photon(exprs, 0)
        events, allowed, unpaired = restated_for_device(mcrt, pm, scene, ep)
        assert unpaired <= allowed * 8, (unpaired, allowed)
        checked, high = 0, 0
        for which in (0, 1):
            states = pm.photon_lpe_states(which)
            for i, ev in enumerate(events[which]):
                if ev is None:
                    continue
                assert states[i] == reverse_walk(mcrt, t, mcrt.LPE_SYM_L, ev), (which, i, ev, states[i])
                checked += 1
                high += 128 <= states[i] < mcrt.LPE_DEAD
        print(f"{table} {cid}: {checked} photons checked, {high} past state 127")
        assert checked > 0
        if cid == GLASS_ROOM:
            assert high > 0
    finally:
        pm.close()


# The glass room is left out here: its photon-mapped one-plane frame already departs from the restatement by up to ~2e-6
# (rough glass, libm's last bits), far above this bar; its photon states are held to the restatement above
@pytest.mark.parametrize("table,cid,radius", [("TAIL", "pm_hexagon_room_64", False), ("HEAD", "pm_hexagon_room_64", False),
                                              ("HEAD", "pm_hexagon_room_64", True), ("LABELS", "smooth_mesh_64", False)])
def test_photon_planes_match_the_restatement(table, cid, radius, mcrt):
    """test_gpu_pm_lpe's restatement test at the limit tables: HEAD's queries on pm_hexagon_room_64 keep states past 127
    (C<TS><TS><RD>), LABELS has 71 symbols"""
    import pm_lpe_ref
    from oracle import port
    scene, _ = load_case(mcrt, cid)
    ep = pm_params(scene, cid)
    exprs = TABLES[table]
    ids = pm_ids(scene, table)
    pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=REF_SEED, emit=ep)
    try:
        cam, y0, y1 = camera_of(scene, cid)
        spp = cam.sqrtspp ** 2
        r2 = (0.0, 0.0)
        if radius:
            rc, rg = gather_radius_of(pm)
            pm.gather_radius(rc, rg)
            r2 = (rc * rc, rg * rg)
        set_table(pm, exprs, ids)
        pm.emit_again()
        planes = torch_zeros((len(exprs), y1 - y0, cam.width, 3))
        pm.render_accumulate_lpe_dev(cam, planes.data_ptr(), len(exprs), 0, spp, y_first=y0, n_rows=y1 - y0)
        got = planes.cpu().numpy() / spp
        events, _, _ = restated_for_device(mcrt, pm, scene, ep)
        maps = []
        for which in (0, 1):
            hist = pm_lpe_ref.history(["?" if e is None else e for e in events[which]], pm.photon_lights(which), ids)
            maps.append((pm._maps[which]["photons"].reshape(-1, 8), hist))
        st = pm_lpe_ref.render_strings(scene, cam, y0, y1, cam.sqrtspp, REF_SEED, maps, ep["k_nearest_photons"],
                                       ep["direct_visualization"], r2, ids)
        ref = st.planes(exprs)
        ps = port.PortScene(scene)
        rpm = ps.photon_mapper(pm._maps)
        try:
            if radius:
                rpm.gather_radius(*np.sqrt(r2))
            _, _, counts = rpm.render_rows(cam, y0, y1, cam.sqrtspp, REF_SEED)
        finally:
            rpm.close()
            ps.close()
        allowed = allowance(scene, (y1 - y0) * cam.width * spp) + counts["knn_ties"]
        for i, e in enumerate(exprs):
            rel, out = frame_error(got[i], ref[i], spp)
            assert rel < 1e-9 and out <= allowed, (e, rel, out, allowed)
        assert any(got[i].any() for i in range(len(exprs) - 1))
    finally:
        pm.close()


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("k", [50, None])
def test_photon_all32_planes_are_the_one_plane_render(k, precision, mcrt):
    """Every photon term's mask is 0xFFFFFFFF: each of the 32 planes is the one-plane render, with its query count"""
    scene, seed = load_case(mcrt, "pm_hexagon_room_64")
    cam = scene.cameras()[0]
    pm = mcrt.PhotonMapper(scene, precision=precision, global_seed=seed, emit=emit_params(scene, k=k or 50))
    try:
        if k is None:
            pm.gather_radius(*gather_radius_of(pm))
        spp = 4
        beauty, st0 = pm_render_beauty(pm, cam, spp)
        set_table(pm, ALL32)
        pm.emit_again()
        planes = torch_zeros((len(ALL32), cam.height, cam.width, 3))
        st = pm.render_accumulate_lpe_dev(cam, planes.data_ptr(), len(ALL32), 0, spp, tile=16)
        planes = planes.cpu().numpy()
        pm_same_stats(st, st0)
        assert st0["knn_queries"] > 0 and beauty.any()
        rtol = 1e-12 if precision == 0 else f32_rtol(max_gathered(pm) if k is None else k)
        for p in planes:
            np.testing.assert_allclose(p, beauty, rtol=rtol, atol=1e-14 * spp)
    finally:
        pm.close()


# ---------------------------------------------------------------------------------------------- Progressive with P31
def test_progressive_with_31_expressions(mcrt, tmp_path):
    """The beauty plane on bit 31 drives frame, error, denoise and the checkpoints as the plain frame does; relight with
    31 weights is the weighted sum of lpe_frames"""
    scene, seed = load_case(mcrt, "c2_hexagon_room_96")
    cam = scene.cameras()[0]
    pt = mcrt.PathTracer(scene, global_seed=seed)
    try:
        prog = mcrt.Progressive(pt, cam, lpes=P31)
        plain = mcrt.Progressive(pt, cam)
        for s in (1, 3):
            prog.add(s)
            plain.add(s)
        assert np.allclose(prog.frame(), plain.frame(), rtol=RTOL, atol=ATOL)
        (e, t), (e0, t0) = prog.error(), plain.error()
        assert np.isclose(e, e0, rtol=1e-9) and np.allclose(t, t0, rtol=1e-9, atol=1e-12)
        assert prog.stats == plain.stats
        frames, errors = prog.lpe_frames()
        assert frames.shape == (len(P31), cam.height, cam.width, 3) and np.isfinite(errors).all()
        w = 2.0 ** -np.arange(len(P31))
        np.testing.assert_allclose(prog.relight(w)[0], np.maximum(np.tensordot(w, frames, 1), 0.0), rtol=1e-9, atol=1e-12)
        den, den_err = prog.denoise()
        ref_den, ref_den_err = plain.denoise()
        assert np.allclose(den, ref_den, rtol=1e-9, atol=1e-12) and np.isclose(den_err, ref_den_err, rtol=1e-9)
        path = str(tmp_path / "p31.npz")
        prog.save(path)
        back = mcrt.Progressive.load(path, pt, cam, lpes=P31)
        back.add(2)
        prog.add(2)
        plain.add(2)
        assert np.allclose(back.frame(), prog.frame(), rtol=RTOL, atol=ATOL)
        assert np.allclose(back.frame(), plain.frame(), rtol=RTOL, atol=ATOL)
        assert np.allclose(back.lpe_frames()[0], prog.lpe_frames()[0], rtol=RTOL, atol=ATOL)
    finally:
        pt.close()


def test_adaptive_with_31_expressions_retires_the_same_tiles(mcrt):
    scene, seed = load_case(mcrt, "c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54, 8)
    pt = mcrt.PathTracer(scene, global_seed=seed)
    try:
        runs = []
        for lpes in (P31, None):
            prog = mcrt.Progressive(pt, cam, tile=16, lpes=lpes)
            runs.append((prog, prog.render_adaptive(4, 64, 0.05, min_samples=8)))
        (a, fa), (b, fb) = runs
        assert len(a.history) == len(b.history) > 1 and a.stop_reason == b.stop_reason
        assert any(h["retired"].any() for h in a.history)
        for ha, hb in zip(a.history, b.history):
            assert np.array_equal(ha["retired"], hb["retired"]) and np.array_equal(ha["tile_counts"], hb["tile_counts"])
        assert np.allclose(fa, fb, rtol=RTOL, atol=ATOL)
    finally:
        pt.close()


def test_progressive_photon_mapping_with_31_expressions(mcrt):
    scene, seed = load_case(mcrt, "pm_hexagon_room_64")
    ep = emit_params(scene)
    cam = scene.cameras()[0]
    args = (cam, 4000, ep["caustic_factor"], ep["max_photons_per_octree_leaf"])
    mappers = [mcrt.PhotonMapper(scene, global_seed=seed) for _ in range(2)]
    try:
        plain = mcrt.ProgressivePhotonMapping(mappers[0], *args, radius=0.2)
        split = mcrt.ProgressivePhotonMapping(mappers[1], *args, radius=0.2, lpes=P31)
        for _ in range(3):
            plain.add(2)
            split.add(2)
        np.testing.assert_allclose(split.frame(), plain.frame(), rtol=1e-12, atol=1e-14)
        assert split.error()[0] == pytest.approx(plain.error()[0], rel=1e-9)
        frames, _ = split.lpe_frames()
        assert frames.shape[0] == len(P31) and any(f.any() for f in frames)
    finally:
        for m in mappers:
            m.close()
