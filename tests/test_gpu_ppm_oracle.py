"""Progressive photon mapping on the device against the scalar float64 restatement (oracle/mcrt_oracle.cpp: photonPass
with a pass index, photonEstimate with a fixed gather radius), which tests/test_ppm_oracle_cpu.py pins to the k-NN
estimate that tests/test_photon_mapper_oracle_cpu.py pins to the reference (run on an H100).

Cases, photon-pass parameters and bars are test_gpu_photon_mapper.py's (CASES, params_of, camera_of, TOL, OUTLIERS),
each case at photon passes 1 and 5 and, on three cases, at the last pass whose emission indices fit 32 bits (indices
just below 2^32). Each case gathers in one radius regime, rotated over the cases:
    auto    the initial radii ProgressivePhotonMapping picks from the case's pass-0 maps
    small   0.02 x auto: most queries find no photon, so most estimates deposit nothing
    whole   caustic 0.5 x auto, global just above the scene bounds' diagonal: every global query takes every photon, by
            the whole-octant branch of the gather; the caustic one walks the octree through the gather stack

    a. emission   emit_pass(i) at float64 against the restated pass i, at test_emission_matches_restatement's bars
    b. samples    the device's pass-i maps fed to the restatement, both sides gathering at the regime's radii: sampleRay
                  on 16384 camera samples at |d| <= 1e-6 max(1, |ref|); the device must have gathered (its values differ
                  from its k-NN values on the same samples)
    c. frames     the frame and the four component planes at relative RMSE < 1e-6; rays, shadow rays and queries equal
    d. driver     ProgressivePhotonMapping for 3 passes of 1 spp: its frame and component frames against the mean of the
                  restatement's samples, pass i's on pass i's maps at the radii of ppm_radii(r1, alpha, i + 1)

A fixed radius has no ties at a k-th distance, so the one allowance is test_gpu_materials' OUTLIERS in scenes with glass.
The module prints each case's counts: outliers, queries, queries that took no photon, photons per query."""
import time

import numpy as np
import pytest

from oracle import port
from test_gpu_materials import has_glass
from test_gpu_photon_mapper import (CASES, LIT_MATERIAL, N_SAMPLES, SEED, TOL, allowance, camera_of, case_id, check_emission,
                                    compare_frames, compare_samples, frame_error, params_of, scene_of)
from test_ppm_cpu import emission_counts

pytestmark = pytest.mark.gpu

REGIMES = ("whole", "auto", "small")   # rotated with the cases: "whole" falls on caustic factor 10, the smaller global maps
LAST_PASS_CASES = ["ggx_64", "ior_test_nobvh_64", "veach_mis_64"]
PASSES = [(c, i) for c in CASES for i in (1, 5)] + [(c, "last") for c in LAST_PASS_CASES]
DRIVER_CASES = ["pm_hexagon_room_64", "ggx_64", LIT_MATERIAL[2]]   # k >= 2: see held
DRIVER_PASSES = 3


def regime_of(case):
    return REGIMES[CASES.index(case) % len(REGIMES)]


def pass_id(p):
    return f"{case_id(p[0])}-pass{p[1]}"


def last_pass(scene, ep):
    """test_gpu_ppm's last_ok: the last pass whose emission indices (pass + 1) * n_l - 1 fit 32 bits for every light"""
    return (1 << 32) // int(emission_counts(scene, ep["emissions"], ep["caustic_factor"]).max()) - 1


def bounds_diagonal(scene):
    b = np.asarray(scene.extra["scene_bounds"], np.float64)
    return float(np.linalg.norm(b[3:] - b[:3]))


REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\nprogressive photon mapping:")
        for k in sorted(REPORT):
            print(f"  {k:72s} {REPORT[k]}")


@pytest.fixture(scope="module")
def held(mcrt):
    """one (case, pass) at a time -> dict: pm (device PhotonMapper at float64 holding pass i's maps), ps (restatement
    scene), scene, ep (emit params), pass_index, radii (the regime's (caustic, global)), restated() (the restated pass)"""
    state, auto = {}, {}

    def close():
        for o in state.get("objs", ()):
            o.close()
        state.clear()

    def get(case, which_pass):
        if state.get("key") != (case, which_pass):
            close()
            scene = scene_of(mcrt, case)
            ep = dict(params_of(case), scene_bounds=scene.extra["scene_bounds"])
            pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=SEED, emit=ep)
            if case not in auto:
                cam, _, _ = camera_of(scene, case)
                # the driver measures the k-th distance at photon positions, where the nearest photon is the photon
                # itself: with k = 1 its radius is 0, which it refuses; those cases take the 2nd nearest
                run = mcrt.ProgressivePhotonMapping(pm, cam, ep["emissions"], ep["caustic_factor"], ep["max_photons_per_octree_leaf"],
                                                    k_nearest_photons=max(2, ep["k_nearest_photons"]))
                auto[case] = run.radius
                del run
            rc, rg = auto[case]
            regime = regime_of(case)
            radii = {"auto": (rc, rg), "small": (0.02 * rc, 0.02 * rg), "whole": (0.5 * rc, 1.001 * bounds_diagonal(scene))}[regime]
            i = last_pass(scene, ep) if which_pass == "last" else which_pass
            pm.emit_pass(i, **ep)
            ps = port.PortScene(scene)
            state.update(key=(case, which_pass), objs=(pm, ps), pm=pm, ps=ps, scene=scene, ep=ep, pass_index=i, regime=regime,
                         radii=radii, auto=auto[case],
                         restated=lambda: ps.photon_pass(ep["emissions"], ep["caustic_factor"], ep["max_photons_per_octree_leaf"],
                                                         ep["scene_bounds"], SEED, pass_index=i))
        return state
    yield get
    close()


def check_regime(st):
    """the regime does what it claims on these maps"""
    maps = st["pm"]._maps
    rc, rg = st["radii"]
    if len(maps[0]["photons"]):
        assert rc != rg, "the caustic and the global radius must differ, or a swap of the two goes unseen"
    if st["regime"] == "whole":
        b = np.asarray(st["scene"].extra["scene_bounds"], np.float64)
        pos = np.asarray(maps[1]["photons"], np.float32).reshape(-1, 8)[:, 3:6].astype(np.float64)
        slack = 1e-9 * bounds_diagonal(st["scene"])   # photons on a bounding plane carry round-off
        assert (pos >= b[:3] - slack).all() and (pos <= b[3:] + slack).all() and rg > 1.0005 * bounds_diagonal(st["scene"])


def counts_note(counts):
    q = max(counts["knn_queries"], 1)
    return (f"queries {counts['knn_queries']}, empty {counts['empty_queries']} ({counts['empty_queries'] / q:.0%}), "
            f"photons/query {counts['photons'] / q:.1f}")


# ------------------------------------------------------------------------------------------------------- a. emission
@pytest.mark.parametrize("case,which_pass", PASSES, ids=[pass_id(p) for p in PASSES])
def test_pass_emission_matches_restatement(case, which_pass, held):
    st = held(case, which_pass)
    assert st["pm"].has_photon_lights
    restated = st["restated"]()
    n = emission_counts(st["scene"], st["ep"]["emissions"], st["ep"]["caustic_factor"])
    for which in (0, 1):
        idx = (restated[4][which] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        lo = st["pass_index"] * n[restated[2][which]]
        assert ((idx >= lo) & (idx < lo + n[restated[2][which]])).all()
    # passes after the first send other paths into the glass orbits where CUDA's and glibc's sincos part ways (test_gpu_materials'
    # OUTLIERS); a record such a path leaves may still match within ANGLE_TOL, so it counts as that path parting ways
    check_emission(st["pm"], st["scene"], restated, f"a {pass_id((case, which_pass))}", REPORT, angles_by_path=True)


# ------------------------------------------------------------------------------------------------------- b. samples
@pytest.mark.parametrize("case,which_pass", PASSES, ids=[pass_id(p) for p in PASSES])
def test_gather_samples_match_restatement(case, which_pass, held):
    st = held(case, which_pass)
    pm, scene = st["pm"], st["scene"]
    check_regime(st)
    rpm = st["ps"].photon_mapper(pm._maps)
    tag = f"b {st['regime']} pass {which_pass}"
    try:
        pm.gather_radius(*st["radii"])
        rpm.gather_radius(*st["radii"])
        rays, pixel, sample, got, counts = compare_samples(pm, rpm, scene, case, tag, REPORT)
        assert pm.gather_radii == st["radii"] and pm.last_stats["knn_queries"] > 0
        assert counts["knn_ties"] == 0 and counts["knn_queries"] > 0
        pm.gather_radius(0, 0)
        knn = pm.sampleRay(rays, pixel, sample)
    finally:
        pm.gather_radius(0, 0)
        rpm.close()
    changed = int((np.abs(knn - got) > TOL * np.maximum(1.0, np.abs(knn))).any(axis=1).sum())
    REPORT[f"{tag} samples {case_id(case)}"] += f", {counts_note(counts)}, {changed} of {N_SAMPLES} differ from k-NN"
    assert changed > 0, "the device did not gather"
    if st["regime"] == "small":
        assert counts["empty_queries"] > 0.5 * counts["knn_queries"]


# ------------------------------------------------------------------------------------------------------- c. frames
@pytest.mark.parametrize("case,which_pass", PASSES, ids=[pass_id(p) for p in PASSES])
def test_gather_frame_and_components_match_restatement(case, which_pass, held):
    st = held(case, which_pass)
    pm = st["pm"]
    rpm = st["ps"].photon_mapper(pm._maps)
    tag = f"c {st['regime']} pass {which_pass}"
    t = time.time()
    try:
        pm.gather_radius(*st["radii"])
        rpm.gather_radius(*st["radii"])
        counts = compare_frames(pm, rpm, st["scene"], case, tag, REPORT)
    finally:
        pm.gather_radius(0, 0)
        rpm.close()
    assert counts["knn_ties"] == 0
    REPORT[f"{tag} frame {case_id(case)}"] += f", {counts_note(counts)} ({time.time() - t:.1f} s)"


# ------------------------------------------------------------------------------------------------------- d. driver
@pytest.mark.parametrize("case", DRIVER_CASES, ids=[case_id(c) for c in DRIVER_CASES])
def test_driver_equals_the_restated_passes(case, mcrt):
    """ProgressivePhotonMapping end to end: pass i emits map i and gathers samples [i, i + 1) of every pixel at the radii
    ppm_radii(r1, alpha, i + 1)[-1] (Knaus & Zwicker's schedule, computed here from the initial radii r1); the frame is
    the equal-weight mean of the passes' samples."""
    scene = scene_of(mcrt, case)
    ep = params_of(case)
    cam = scene.cameras()[0].resized(32, 24, 1)
    n = cam.width * cam.height
    pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=SEED,
                           emit=dict(ep, scene_bounds=scene.extra["scene_bounds"]))
    ps = port.PortScene(scene)
    try:
        run = mcrt.ProgressivePhotonMapping(pm, cam, ep["emissions"], ep["caustic_factor"], ep["max_photons_per_octree_leaf"],
                                            k_nearest_photons=ep["k_nearest_photons"], components=True)
        maps = []
        for _ in range(DRIVER_PASSES):
            run.add(1)
            maps.append(pm._maps)
        frame, (planes, _) = run.frame(), run.component_frames()
        rgb_sum, comp_sum, notes = np.zeros((n, 3)), np.zeros((n, 4, 3)), []
        pixel = np.arange(n, dtype=np.uint32)
        for i, m in enumerate(maps):
            radii = tuple(float(mcrt.ppm_radii(r, run.alpha, i + 1)[-1]) for r in run.radius)
            rpm = ps.photon_mapper(m)
            try:
                rpm.gather_radius(*radii)
                rgb, comp, _, counts = rpm.sample_pixels(cam, pixel, np.full(n, i, np.uint32), SEED)
            finally:
                rpm.close()
            assert counts["knn_ties"] == 0
            rgb_sum += rgb
            comp_sum += comp
            notes.append(f"pass {i} radii ({radii[0]:.4f}, {radii[1]:.4f}) {counts_note(counts)}")
        ref = (rgb_sum / DRIVER_PASSES).reshape(cam.height, cam.width, 3)
        ref_planes = (comp_sum / DRIVER_PASSES).transpose(1, 0, 2).reshape(4, cam.height, cam.width, 3)
        allowed = allowance(scene, n * DRIVER_PASSES)
        rel, out = frame_error(frame, ref, DRIVER_PASSES)
        notes.insert(0, f"frame rel rmse {rel:.1e} outlier pixels {out}")
        for c, name in enumerate(("emission", "direct", "caustic", "global")):
            rel_c, out_c = frame_error(planes[c], ref_planes[c], DRIVER_PASSES)
            notes.insert(c + 1, f"{name} {rel_c:.1e}/{out_c}")
            assert rel_c < TOL and out_c <= allowed, (name, notes)
        REPORT[f"d driver {case_id(case)}"] = ", ".join(notes)
        assert rel < TOL and out <= allowed, notes
        assert has_glass(scene) or out == 0
    finally:
        ps.close()
        pm.close()
