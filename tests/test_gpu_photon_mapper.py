"""The photon mapper on the device against the scalar float64 restatement (oracle/mcrt_oracle.cpp: photonPass,
pmSampleRay), which tests/test_photon_mapper_oracle_cpu.py pins to the reference's pm_hexagon_room_64 (run on an H100).

Cases: every golden scene with a light and every MATERIAL_CASES entry whose scene has one (the `lit` and `nested`
geometries), each under one point of a small cross-product of photon-pass parameters: direct_visualization off / on,
caustic_factor 1 / 10, 200 / 8 photons per leaf, and k in {1, 33, 100, 256} (1, 2, 4 and 8 register slots of the warp
search) and {96, 257} (the shared-memory search: ceil(k / 32) = 3 and 9). The scenes without a light are refused.

    a. emission      PhotonMapper(emit=...) at float64 against the restated photon pass: photon records (with the light
                     that emitted each) equal as multisets - flux and position exact, polar angles within 2.4e-7 pi (CUDA
                     vs glibc atan2), at least 99.9 % of the records identical - the bars of test_gpu_parity's
                     check_emitted_maps
    b. estimates     the device's emitted maps fed to the restatement, so that (a) and (b) fail independently: sampleRay on
                     16384 camera samples per sample at |d| <= 1e-6 max(1, |ref|) (test_gpu_parity's photon-mapped bar:
                     Photon::dir takes glibc's sinf / cosf in the restatement, double sin / cos rounded to float on the
                     device); the frame and the four component planes at relative RMSE < 1e-6
    c. CPU maps      the restatement's maps uploaded through photon_maps= (mcrt_photon_upload) on three cases, at (b)'s bars

The one allowance is test_gpu_materials' OUTLIERS: in scenes with glass a path can orbit inside it, where glibc's and
CUDA's sincos part ways, so up to 1 in 1000 photon records, samples or frame samples may differ; elsewhere none may.
A query whose k-th distance is shared by a photon left out (the restatement reports these) may also differ. The module
prints each case's counts."""
import collections
import time

import numpy as np
import pytest

from material_gen import golden_scene
from oracle import port
from test_gpu_materials import case_scene, has_glass
from test_gpu_photon_light_groups import torch_zeros
from test_material_cases_cpu import MATERIAL_CASES, mat_case_id

pytestmark = pytest.mark.gpu

SEED = 0x12345678
N_SAMPLES = 16384
TOL = 1e-6
OUTLIERS = 1e-3
ANGLE_TOL = 2.4e-7 * np.pi
EMISSION_PATHS = 20000     # emissions * caustic_factor: seconds of brute-force k-NN per case on the CPU

GOLDEN_LIT = ["c1_hexagon_diffuse_256", "c2_hexagon_room_96", "hexagon_room_octree_64", "ggx_64", "metals_64", "veach_mis_64",
              "smooth_mesh_64", "ior_test_nobvh_64", "pm_hexagon_room_64"]
UNLIT = ["oren_nayar_64", "quadric_64"] + [c for c in MATERIAL_CASES if c.geometry == "sky"]
LIT_MATERIAL = [c for c in MATERIAL_CASES if c.geometry != "sky"]
CASES = GOLDEN_LIT + LIT_MATERIAL

# (direct_visualization, caustic_factor, max_photons_per_octree_leaf, k): each value of each parameter in several cases
PARAMS = [(False, 10.0, 200, 100), (True, 1.0, 8, 33), (False, 1.0, 200, 256), (True, 10.0, 8, 257), (False, 10.0, 8, 1),
          (True, 1.0, 200, 96)]
CPU_MAP_CASES = ["c1_hexagon_diffuse_256", "ggx_64", LIT_MATERIAL[0]]


def case_id(case):
    return case if isinstance(case, str) else mat_case_id(case)


def params_of(case):
    dv, cf, leaf, k = PARAMS[CASES.index(case) % len(PARAMS)]
    return dict(emissions=int(EMISSION_PATHS / cf), caustic_factor=cf, max_photons_per_octree_leaf=leaf, k_nearest_photons=k,
                direct_visualization=dv)


def scene_of(mcrt, case):
    return golden_scene(mcrt, case) if isinstance(case, str) else case_scene(mcrt, case)


def camera_of(scene, case):
    """-> (camera, y0, y1): c1_hexagon_diffuse_256 at a band of its 256 x 256 frame, the rest at 64 x 48, 4 spp"""
    cam = scene.cameras()[0]
    if case == "c1_hexagon_diffuse_256":
        return cam.resized(cam.width, cam.height, 1), 112, 144
    cam = cam.resized(64, 48, 2)
    return cam, 0, cam.height


REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\nphoton mapper:")
        for k in sorted(REPORT):
            print(f"  {k:64s} {REPORT[k]}")


@pytest.fixture(scope="module")
def held(mcrt):
    """one case at a time: (device PhotonMapper emitted at float64, restatement scene, scene, emit params, restated pass)"""
    state = {}

    def close():
        for o in state.get("objs", ()):
            o.close()
        state.clear()

    def get(case):
        if state.get("case") != case:
            close()
            scene = scene_of(mcrt, case)
            ep = dict(params_of(case), scene_bounds=scene.extra["scene_bounds"])
            t = time.time()
            pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=SEED, emit=ep)
            ps = port.PortScene(scene)
            restated = ps.photon_pass(ep["emissions"], ep["caustic_factor"], ep["max_photons_per_octree_leaf"], ep["scene_bounds"], SEED)
            state.update(case=case, objs=(pm, ps), scene=scene, ep=ep, restated=restated, t=time.time() - t)
        return state["objs"][0], state["objs"][1], state["scene"], state["ep"], state["restated"]
    yield get
    close()


def pos_tolerance(scene):
    """|d| of a photon coordinate between the two sides: the float64 round-off of o + t d in a scene of this size. Where a
    coordinate is itself round-off (a hit on a plane through 0), libm's last bit in the sampled direction (CUDA's and glibc's
    sin / cos differ in it) moves that residue by ~1e-15, which float32 keeps."""
    return 64.0 * np.finfo(np.float64).eps * float(np.abs(scene.extra["scene_bounds"]).max())


def match_records(got, got_lights, ref, ref_lights, pos_tol):
    """Pairs each device photon with an unused restated one of equal flux and light, polar angles within ANGLE_TOL and
    every position coordinate within pos_tol -> (pairs [m, 2], unmatched device indices, unmatched restated indices)"""
    from scipy.spatial import cKDTree
    a, b = np.asarray(got, np.float32).reshape(-1, 8), np.asarray(ref, np.float32).reshape(-1, 8)
    pairs, used = [], np.zeros(len(b), bool)
    if len(a) and len(b):
        near = cKDTree(b[:, 3:6].astype(np.float64)).query_ball_point(a[:, 3:6].astype(np.float64), r=pos_tol, p=np.inf)
        for i, cand in enumerate(near):
            for j in sorted(cand):
                if not used[j] and got_lights[i] == ref_lights[j] and np.array_equal(a[i, :3], b[j, :3]) \
                        and np.abs(a[i, 6:].astype(np.float64) - b[j, 6:]).max() <= ANGLE_TOL:
                    used[j] = True
                    pairs.append((i, j))
                    break
    pairs = np.array(pairs, np.int64).reshape(-1, 2)
    got_off = np.setdiff1d(np.arange(len(a)), pairs[:, 0])
    return pairs, got_off, np.nonzero(~used)[0]


def allowance(scene, n):
    return int(OUTLIERS * n) if has_glass(scene) else 0


# ------------------------------------------------------------------------------------------------------- a. emission
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_emission_matches_restatement(case, mcrt, held):
    """Photon records as multisets. Flux and light are exact; polar angles within ANGLE_TOL and identical in 99.9 % of the
    records; positions within pos_tolerance (exact, but where the coordinate is the round-off residue of a hit on a plane
    through 0). In scenes with glass a path orbiting inside it may part ways (test_gpu_materials' OUTLIERS): at most 1 in
    1000 emission paths may leave records on either side that the other lacks."""
    pm, _, scene, _, restated = held(case)
    assert pm.has_photon_lights
    check_emission(pm, scene, restated, f"a {case_id(case)}")


def check_emission(pm, scene, restated, tag, report=REPORT, angles_by_path=False):
    """test_emission_matches_restatement's bars for the device's current maps against a restated photon pass.
    angles_by_path: in scenes with glass, a matched record whose angles differ counts its path against the allowance of
    paths parting ways, instead of against the 99.9 % of identical records"""
    caustic, glob, lights, total, paths = restated
    pos_tol = pos_tolerance(scene)
    notes, paths_off = [], set()
    extra = 0
    for which, ref_map in enumerate((caustic, glob)):
        got_ph = pm._maps[which]["photons"].reshape(-1, 8)
        ref_ph = ref_map["photons"].reshape(-1, 8)
        pairs, got_off, ref_off = match_records(got_ph, pm.photon_lights(which), ref_ph, lights[which], pos_tol)
        a, b = got_ph[pairs[:, 0]], ref_ph[pairs[:, 1]]
        moved = a[:, 3:6] != b[:, 3:6]
        residue = int(moved.any(axis=1).sum())
        assert np.all(np.abs(b[:, 3:6][moved]) <= pos_tol), "a position moved where its coordinate is not round-off"
        same_angles = np.all(a[:, 6:] == b[:, 6:], axis=1)
        paths_off.update(paths[which][ref_off].tolist())
        extra += len(got_off)
        notes.append(f"{('caustic', 'global')[which]} {len(got_ph)}/{len(ref_ph)} unmatched {len(got_off)}/{len(ref_off)} "
                     f"residue positions {residue} angles differ {int((~same_angles).sum())}")
        if angles_by_path and has_glass(scene):
            paths_off.update(paths[which][pairs[~same_angles, 1]].tolist())
        else:
            assert same_angles.mean() >= 0.999 if len(pairs) else True, notes[-1]
    # the longest trail of records one restated path left: a path that parts ways on the device leaves one of similar length
    longest = max([int(np.unique(p, return_counts=True)[1].max()) for p in paths if len(p)] or [0])
    allowed = allowance(scene, total)
    report[tag] = (f"{total} emissions, paths parting {len(paths_off)} (allowed {allowed}), " + "; ".join(notes))
    assert len(paths_off) <= allowed, report[tag]
    assert extra <= allowed * max(2 * longest, 1), report[tag]


# ------------------------------------------------------------------------------------------------------- b. estimates
def device_maps_restated(pm, ps):
    return ps.photon_mapper(pm._maps)


def compare_samples(pm, rpm, scene, case, tag, report=REPORT):
    """-> (camera rays, pixel, sample, the device's radiance, the restatement's counts)"""
    cam, _, _ = camera_of(scene, case)
    rng = np.random.default_rng(5)
    pixel = rng.integers(0, cam.width * cam.height, N_SAMPLES).astype(np.uint32)
    sample = rng.integers(0, 256, N_SAMPLES).astype(np.uint32)
    ref, comp, rays, counts = rpm.sample_pixels(cam, pixel, sample, SEED)
    assert np.abs(comp.sum(axis=1) - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
    got = pm.sampleRay(rays, pixel, sample)
    bad = (np.abs(got - ref) / np.maximum(1.0, np.abs(ref)) > TOL).any(axis=1)
    key = f"{tag} samples {case_id(case)}"
    report[key] = (f"{int(bad.sum())} of {N_SAMPLES} outliers, knn ties {counts['knn_ties']}, queries {counts['knn_queries']}, "
                   f"mean {ref.mean():.3e}")
    assert np.isfinite(got).all()
    assert bad.sum() <= allowance(scene, N_SAMPLES) + counts["knn_ties"], report[key]
    return rays, pixel, sample, got, counts


def frame_error(img, ref, spp):
    """-> (relative RMSE over the pixels that agree, number of pixels that do not): a sample that parts ways in glass
    moves its pixel by its whole radiance, which the allowance counts instead of the RMSE"""
    out = np.abs(img - ref).max(axis=-1) > TOL * max(1.0, np.abs(ref).max())
    fixed = np.where(out[..., None], ref, img)
    return float(np.sqrt(np.mean((fixed - ref) ** 2))) / max(1.0, float(np.abs(ref).mean())), int(out.sum())


def compare_frames(pm, rpm, scene, case, tag, report=REPORT):
    """-> the restatement's counts"""
    cam, y0, y1 = camera_of(scene, case)
    spp = cam.sqrtspp ** 2
    ref, ref_comp, counts = rpm.render_rows(cam, y0, y1, cam.sqrtspp, SEED)
    img = pm.render_rows(cam, y0, y1)
    st = pm.last_stats
    planes = torch_zeros((4, y1 - y0, cam.width, 3))
    pm.render_accumulate_components_dev(cam, planes.data_ptr(), 0, spp, y_first=y0, n_rows=y1 - y0)
    comp = planes.cpu().numpy() / spp
    allowed = allowance(scene, (y1 - y0) * cam.width * spp) + counts["knn_ties"]
    rel, out = frame_error(img, ref, spp)
    notes = [f"frame rel rmse {rel:.1e} outlier pixels {out}"]
    assert st["paths"] == (y1 - y0) * cam.width * spp
    assert rel < TOL and out <= allowed, notes[0]
    for c, name in enumerate(("emission", "direct", "caustic", "global")):
        rel_c, out_c = frame_error(comp[c], ref_comp[c], spp)
        notes.append(f"{name} {rel_c:.1e}/{out_c}")
        assert rel_c < TOL and out_c <= allowed, (name, notes)
    if not out:
        # the restatement counts every Scene::intersect call; the device skips shadow rays whose BSDF value is zero
        assert st["extension_rays"] == counts["rays"] - counts["shadow_rays"] and st["shadow_rays"] <= counts["shadow_rays"]
        assert st["knn_queries"] == counts["knn_queries"]
    report[f"{tag} frame {case_id(case)}"] = ", ".join(notes) + f", knn ties {counts['knn_ties']}"
    return counts


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_samples_on_device_maps(case, mcrt, held):
    pm, ps, scene, _, _ = held(case)
    rpm = device_maps_restated(pm, ps)
    try:
        compare_samples(pm, rpm, scene, case, "b")
    finally:
        rpm.close()


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_frame_and_components_on_device_maps(case, mcrt, held):
    pm, ps, scene, _, _ = held(case)
    rpm = device_maps_restated(pm, ps)
    t = time.time()
    try:
        compare_frames(pm, rpm, scene, case, "b")
    finally:
        rpm.close()
    REPORT[f"b frame {case_id(case)}"] += f" ({time.time() - t:.1f} s)"


# ------------------------------------------------------------------------------------------------------- c. CPU maps
@pytest.mark.parametrize("case", CPU_MAP_CASES, ids=[case_id(c) for c in CPU_MAP_CASES])
def test_device_renders_restated_maps(case, mcrt, held):
    """mcrt_photon_upload: the restatement's own maps on the device"""
    _, ps, scene, ep, (caustic, glob, _, _, _) = held(case)
    maps = (caustic, glob, ep["k_nearest_photons"], int(ep["direct_visualization"]))
    pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=SEED, photon_maps=maps)
    rpm = ps.photon_mapper(maps)
    try:
        assert not pm.has_photon_lights
        compare_samples(pm, rpm, scene, case, "c")
        compare_frames(pm, rpm, scene, case, "c")
    finally:
        rpm.close()
        pm.close()


def test_emit_refuses_scenes_without_lights(mcrt):
    for case in UNLIT:
        scene = golden_scene(mcrt, case) if isinstance(case, str) else case_scene(mcrt, case)
        assert scene.n_lights == 0
        pm = None
        with pytest.raises(mcrt.McrtError, match="no emissive surfaces"):
            pm = mcrt.PhotonMapper(scene, global_seed=SEED, emit=dict(emissions=1000, caustic_factor=1.0,
                                                                       scene_bounds=scene.extra["scene_bounds"]))
        assert pm is None
