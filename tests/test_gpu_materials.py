"""The BSDF branches no golden scene reaches (rough glass, partial transparency, smooth conductors, coated Oren-Nayar,
conductors and interfaces at scene IOR != 1), on the device against two kinds of oracle (run on an H100):
    restatement      the scalar float64 restatement (oracle/mcrt_oracle.cpp) on the same scene: per sample
                     |d| <= 1e-9 max(1, |ref|), frames at relative RMSE < 1e-9 (tests/test_gpu_parity.py's bars)
    closed forms     numpy float64 Fresnel and sky, independent of both implementations: a mirror, a smooth conductor and a
                     coated dielectric lit by the sky alone, and a green-channel white furnace
and fast mode (float32) against float64 with tests/test_gpu_fast_mode.py's paired bars. The cases and the branches they
reach are the table of tests/test_material_cases_cpu.py; the materials come from tests/material_gen.py."""
import os

import numpy as np
import pytest

from material_gen import (GEOMETRY, GOLD, METAL_NEG, TINT, coated, conductor, glass, golden_scene, lambert, material,
                          material_set, mirror, single_sphere, with_materials)
from oracle import port
from test_gpu_fast_mode import BIAS_SE, agree_mask, paired_bias
from test_material_cases_cpu import MATERIAL_CASES, case_rows, mat_case_id

pytestmark = pytest.mark.gpu

SEED = 0x12345678
F32, F64 = 1, 0
N_SAMPLES = 16384
SAMPLE_TOL = 1e-9          # per-sample and frame bars of tests/test_gpu_parity.py
OUTLIERS = 1e-3            # restatement outliers allowed where a path can orbit inside glass (glibc vs CUDA sincos)


def case_scene(mcrt, case):
    rows = case_rows(mcrt, case)
    base = golden_scene(mcrt, GEOMETRY[case.geometry])
    return with_materials(mcrt, base, rows, scene_ior=case.ior, flip_dirac=case.flip, fill=case.geometry != "nested")


def has_glass(scene):
    return bool((scene.a["materials"]["transparency"] > 0).any())


REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\nmaterials:")
        for k in sorted(REPORT):
            print(f"  {k:56s} {REPORT[k]}")


@pytest.fixture(scope="module")
def held(mcrt):
    """one case's (integrator, restatement, scene) at a time: each integrator holds a full path pool"""
    state = {}

    def get(case):
        if state.get("case") != case:
            for o in state.get("objs", ()):
                o.close()
            scene = case_scene(mcrt, case)
            state["case"] = case
            state["objs"] = (mcrt.PathTracer(scene, global_seed=SEED), port.PortScene(scene))
            state["scene"] = scene
        return state["objs"][0], state["objs"][1], state["scene"]
    yield get
    for o in state.get("objs", ()):
        o.close()


def camera_samples(ps, scene, n=N_SAMPLES, seed=5):
    cam = scene.cameras()[0]
    rng = np.random.default_rng(seed)
    pixel = rng.integers(0, cam.width * cam.height, n).astype(np.uint32)
    sample = rng.integers(0, 256, n).astype(np.uint32)
    _, rays = ps.sample_pixels(cam, pixel, sample, SEED)
    return rays, pixel, sample


def first_hit_labels(mcrt, pt, scene, case, rays):
    """first-hit material label of each ray ('miss', 'other' for the geometry's own materials)"""
    names = {}
    rows = material_set(mcrt, case.mats)
    mats = scene.a["materials"]
    for i in range(len(mats)):
        for label, r in rows:
            if mats[i]["ior"] == r["ior"] and mats[i]["a"][0] == r["a"][0] and mats[i]["transparency"] == r["transparency"] \
                    and np.array_equal(mats[i]["reflectance"], r["reflectance"]) and mats[i]["roughness"] == r["roughness"] \
                    and mats[i]["has_complex_ior"] == r["has_complex_ior"] and mats[i]["perfect_mirror"] == r["perfect_mirror"] \
                    and np.array_equal(mats[i]["complex_ior_real"], r["complex_ior_real"]):
                names[i] = label
                break
    prim = pt.intersect(rays)["prim"]
    return np.array(["miss" if p == mcrt.NO_PRIM else names.get(int(scene.a["prim_material"][p]), "other") for p in prim])


# ------------------------------------------------------------------------------------------------------------- 1. restatement
@pytest.mark.parametrize("case", MATERIAL_CASES, ids=[mat_case_id(c) for c in MATERIAL_CASES])
def test_samples_match_restatement(case, mcrt, held):
    pt, ps, scene = held(case)
    rays, pixel, sample = camera_samples(ps, scene)
    ref = ps.sample_rays(rays, pixel, sample, SEED)
    got = pt.sampleRay(rays, pixel, sample)
    bad = (np.abs(got - ref) / np.maximum(1.0, np.abs(ref)) > SAMPLE_TOL).any(axis=1)
    labels = first_hit_labels(mcrt, pt, scene, case, rays)
    REPORT[f"restatement samples {mat_case_id(case)}"] = (f"{int(bad.sum())} of {len(rays)} outliers "
                                                          f"{sorted(set(labels[bad].tolist()))}")
    # the only allowance: a path orbiting inside glass, where glibc's and CUDA's sincos part ways after a diffuse bounce
    allowed = int(OUTLIERS * len(rays)) if has_glass(scene) else 0
    assert bad.sum() <= allowed, (REPORT[f"restatement samples {mat_case_id(case)}"], np.argwhere(bad)[:5].ravel().tolist())
    assert np.isfinite(got).all()


@pytest.mark.parametrize("case", MATERIAL_CASES, ids=[mat_case_id(c) for c in MATERIAL_CASES])
def test_frame_matches_restatement(case, mcrt, held):
    pt, ps, scene = held(case)
    cam = scene.cameras()[0].resized(64, 48, 4)
    img = pt.render_rows(cam)
    st = pt.last_stats
    ref, rays = ps.render_rows(cam, 0, cam.height, cam.sqrtspp, SEED)
    out = np.abs(img - ref).max(axis=2) > SAMPLE_TOL * max(1.0, np.abs(ref).max())
    fixed = np.where(out[..., None], ref, img)
    rel = float(np.sqrt(np.mean((fixed - ref) ** 2))) / max(1.0, float(np.abs(ref).mean()))
    REPORT[f"restatement frame {mat_case_id(case)}"] = (f"rel rmse {rel:.2e}, outlier pixels {int(out.sum())}, ext {st['extension_rays']} "
                                                        f"shadow {st['shadow_rays']} restatement rays {rays}")
    # the per-sample allowance: at most 1 in 1000 of the frame's samples may part ways (measured: at most 34 of 49 152, all in
    # the scenes with glass, and at most 2 in one pixel)
    spp = cam.sqrtspp ** 2
    allowed = int(OUTLIERS * out.size * spp) if has_glass(scene) else 0
    assert rel < SAMPLE_TOL, REPORT[f"restatement frame {mat_case_id(case)}"]
    parted = 0
    for y, x in np.argwhere(out):
        pixel = np.full(spp, y * cam.width + x, np.uint32)
        sample = np.arange(spp, dtype=np.uint32)
        _, r = ps.sample_pixels(cam, pixel, sample, SEED)
        want = ps.sample_rays(r, pixel, sample, SEED)
        err = (np.abs(pt.sampleRay(r, pixel, sample) - want) / np.maximum(1.0, np.abs(want))).max(axis=1)
        assert (err > SAMPLE_TOL).any(), (y, x)          # an outlier pixel is explained by the samples that part ways
        parted += int((err > SAMPLE_TOL).sum())
    REPORT[f"restatement frame {mat_case_id(case)}"] += f", samples parting {parted}"
    assert parted <= allowed, REPORT[f"restatement frame {mat_case_id(case)}"]
    assert st["paths"] == cam.width * cam.height * cam.sqrtspp ** 2 and st["ior_stack_overflows"] == 0
    # the restatement counts every Scene::intersect call; the device skips shadow rays whose BSDF value is already zero
    if not out.any():
        if scene.n_lights == 0:
            assert st["extension_rays"] == rays and st["shadow_rays"] == 0
        else:
            assert st["extension_rays"] + st["shadow_rays"] <= rays and st["extension_rays"] < rays


# ------------------------------------------------------------------------------------------------------------- 2. closed forms
COS = [1.0, 0.9, 0.5, 0.1, 1e-3, 1e-6]
NORMAL = np.array([0.3, 0.8, 0.52]) / np.linalg.norm([0.3, 0.8, 0.52])
# Relative bar of the closed forms. The device's position is o + t d rounded, its normal that position over the radius,
# so cos carries an absolute error of a few 1e-16 from the hit point and the sky adds the libm asin (<= 2 ulp): 1e-9
# holds with six orders to spare. At cos = 1e-6 the sphere solve forms the discriminant cos^2 = 1e-12 from terms of size
# |o - centre|^2 ~ 2, so it carries an absolute error of ~4.4e-16, relative 4.4e-4; t moves by cos * 2.2e-4 = 2.2e-10 and
# cos with it. |dF/dcos| <= 8 for every interface here and the reflected direction moves by 2 dcos, which the sky turns into
# at most 0.2 dcos relative: 2e-9 in all, so the bar there is 1e-8.
TOL = {c: 1e-9 for c in COS}
TOL[1e-6] = 1e-8


def rays_at_incidence(cos_list):
    """rays hitting the unit sphere at the origin at NORMAL with incidence cos, from 1 away -> (rays [n, 6], d [n, 3])"""
    t = np.cross(NORMAL, [1.0, 0.0, 0.0]); t /= np.linalg.norm(t)
    out, dirs = [], []
    for c in cos_list:
        s = np.sqrt(max(0.0, 1.0 - c * c))
        d = -c * NORMAL + s * t
        d /= np.linalg.norm(d)
        out.append(np.concatenate([NORMAL - d, d])); dirs.append(d)
    return np.array(out), np.array(dirs)


def sky(d):
    """Scene::skyColor: orange below, blue above, 0.5 green everywhere"""
    fy = (1.0 + np.arcsin(d[..., 1]) / np.pi) / 2.0
    return np.stack([1.0 - fy, np.full_like(fy, 0.5), fy], axis=-1)


def fresnel_dielectric(n1, n2, c):
    """unpolarised Fresnel reflectance from the Snell form"""
    st = n1 / n2 * np.sqrt(max(0.0, 1.0 - c * c))
    if st >= 1.0:
        return 1.0
    ct = np.sqrt(1.0 - st * st)
    rs = (n1 * c - n2 * ct) / (n1 * c + n2 * ct)
    rp = (n2 * c - n1 * ct) / (n2 * c + n1 * ct)
    return 0.5 * (rs * rs + rp * rp)


def fresnel_conductor(n1, eta, k, c):
    """unpolarised Fresnel reflectance of a conductor of complex IOR eta + i k under a medium of IOR n1, complex arithmetic"""
    e = (np.asarray(eta) + 1j * np.asarray(k)) / n1
    s2 = 1.0 - c * c
    w = np.sqrt(e * e - s2)
    rs = (c - w) / (c + w)
    rp = (e * e * c - w) / (e * e * c + w)
    return 0.5 * (np.abs(rs) ** 2 + np.abs(rp) ** 2)


def reflected(d):
    return d + 2.0 * np.sum(-d * NORMAL, axis=1, keepdims=True) * NORMAL


def sphere_tracer(mcrt, row, scene_ior):
    return mcrt.PathTracer(single_sphere(mcrt, row, scene_ior), global_seed=SEED)


SPEC = np.array([0.9, 1.0, 0.95])
DELTA_CASES = [("mirror", 1.0, None), ("mirror", 1.33, None), ("conductor_neg", 1.0, METAL_NEG), ("conductor_neg", 1.33, METAL_NEG),
               ("conductor_gold", 1.0, GOLD), ("conductor_gold", 1.33, GOLD)]


@pytest.mark.parametrize("label,scene_ior,ior", DELTA_CASES, ids=[f"{l}-ior{n:g}" for l, n, _ in DELTA_CASES])
def test_closed_form_delta_reflection(label, scene_ior, ior, mcrt):
    """perfect mirror: L = spec * sky(reflect(d, n)); smooth conductor: L = spec * F_conductor(n1, eta, k, cos) * sky(reflect),
    for every sample (a hit at depth 0 takes no roulette, and the reflected ray leaves to the sky)"""
    row = mirror(mcrt, spec=tuple(SPEC)) if ior is None else conductor(mcrt, ior, spec=tuple(SPEC))
    pt = sphere_tracer(mcrt, row, scene_ior)
    try:
        rays, d = rays_at_incidence(COS)
        reps = 64
        got = pt.sampleRay(np.repeat(rays, reps, axis=0), np.zeros(len(rays) * reps, np.uint32),
                           np.tile(np.arange(reps, dtype=np.uint32), len(rays))).reshape(len(rays), reps, 3)
    finally:
        pt.close()
    worst = 0.0
    for i, c in enumerate(COS):
        want = SPEC * sky(reflected(d[i:i + 1]))[0]
        if ior is not None:
            want = want * fresnel_conductor(scene_ior, ior["complex_ior_real"], ior["complex_ior_imag"], c)
        err = np.abs(got[i] - want).max() / np.abs(want).max()
        worst = max(worst, err / TOL[c])
        assert err <= TOL[c], (label, scene_ior, c, got[i][0], want, err)
    REPORT[f"closed form {label} ior {scene_ior:g}"] = f"worst error / bar {worst:.2e}"


COAT_CASES = [(1.0, 1.5), (1.33, 1.5), (1.33, 1.0), (1.0, 2.4)]


@pytest.mark.parametrize("scene_ior,ior", COAT_CASES, ids=[f"ior{n:g}-in{m:g}" for n, m in COAT_CASES])
def test_closed_form_coated_dielectric(scene_ior, ior, mcrt):
    """a smooth coat over black diffuse (reflectance 0, T = 0): every sample is spec * sky(reflect) or 0, and over 4096 sample
    indices of one ray the reflected fraction is F_dielectric(n1, n2, cos) within a 5 sigma binomial bound; exactly 1 where
    F = 1 (an IOR 1.0 sphere in a scene of IOR 1.33 reflects totally from outside below cos = 0.659)"""
    row = material(mcrt, reflectance=(0.0, 0.0, 0.0), specular_reflectance=tuple(SPEC), ior=ior)
    pt = sphere_tracer(mcrt, row, scene_ior)
    n = 4096
    try:
        rays, d = rays_at_incidence(COS)
        got = pt.sampleRay(np.repeat(rays, n, axis=0), np.zeros(len(rays) * n, np.uint32),
                           np.tile(np.arange(n, dtype=np.uint32), len(rays))).reshape(len(rays), n, 3)
    finally:
        pt.close()
    fractions = []
    for i, c in enumerate(COS):
        want = SPEC * sky(reflected(d[i:i + 1]))[0]
        is_ref = np.abs(got[i] - want).max(axis=1) <= TOL[c] * np.abs(want).max()
        is_zero = np.all(got[i] == 0.0, axis=1)
        assert np.all(is_ref | is_zero), (c, got[i][~(is_ref | is_zero)][:3], want)
        F = fresnel_dielectric(scene_ior, ior, c)
        frac = float(is_ref.mean())
        fractions.append(f"{c:g}: {frac:.4f}/{F:.4f}")
        if F == 1.0:
            assert frac == 1.0, (c, frac)
        else:
            assert abs(frac - F) <= 5.0 * np.sqrt(F * (1.0 - F) / n) + 1.0 / n, (c, frac, F)
    REPORT[f"closed form coat ior {scene_ior:g} in {ior:g}"] = ", ".join(fractions)


# ------------------------------------------------------------------------------------------------------------- 3. white furnace
def on_sky_spheres(mcrt, rows):
    """oren_nayar_64's materials: rows in turn on its 8 spheres, Lambert on its floor (material 4). A transparent floor would
    send paths into the space below it, a medium of the glass's IOR, and keep their (n1/n2)^2 radiance compression."""
    out = [rows[i % len(rows)] for i in range(8)]
    return out[:4] + [lambert(mcrt)] + out[4:]


def furnace_scene(mcrt, name):
    """-> (scene, exact): every green weight is 1 where exact, else only energy must not be gained"""
    sky_scene = golden_scene(mcrt, GEOMETRY["sky"])
    nested = golden_scene(mcrt, GEOMETRY["nested"])

    def on_sky(rows, **kw):
        return with_materials(mcrt, sky_scene, on_sky_spheres(mcrt, rows), lights=False, **kw)
    if name == "lambert":
        return on_sky([lambert(mcrt)]), True
    if name == "glass_T1":
        return on_sky([glass(mcrt), lambert(mcrt)]), True
    if name == "coat_lambert":
        return on_sky([coated(mcrt, 0.0), lambert(mcrt)]), True
    if name == "nested":
        rows = [r for _, r in material_set(mcrt, "nested_smooth")] + [lambert(mcrt)] * 3
        return with_materials(mcrt, nested, rows, lights=False), True
    if name == "index_matched":
        return on_sky([glass(mcrt, ior=1.33), glass(mcrt, ior=1.33, T=0.5)], scene_ior=1.33), True
    if name == "rough_glass":
        return on_sky([glass(mcrt, sr=0.3), glass(mcrt, sr=0.05, T=0.4), lambert(mcrt)]), False
    if name == "rough_conductor":
        return on_sky([conductor(mcrt, GOLD, sr=0.4, spec=TINT), conductor(mcrt, METAL_NEG, sr=0.1, spec=TINT), lambert(mcrt)]), False
    if name == "nested_rough":
        rows = [r for _, r in material_set(mcrt, "nested")] + [lambert(mcrt)] * 3
        return with_materials(mcrt, nested, rows, lights=False), False
    raise KeyError(name)


OFF_COMPRESSION = 3e-4


# the interfaces where a compression can be kept: (IOR outside, IOR inside) of a sphere. oren_nayar_64's spheres sit on its
# floor in the scene's medium; ior_test_nobvh_64's outer sphere holds the next one
COMPRESSION_PAIRS = {"glass_T1": [(1.0, 1.5)], "nested": [(1.0, 1.4), (1.4, 1.3)]}


def compression_of(g, pairs, tol):
    """g = 0.5 0.95^-k (n_out / n_in)^2 for some whole k and one interface (n_out, n_in) of the scene"""
    for na, nb in pairs:
        x = g / (na / nb) ** 2
        k = np.rint(np.log(x / 0.5) / np.log(1.0 / 0.95))
        if abs(x - 0.5 * 0.95 ** -k) <= tol * x:
            return True
    return False


FURNACE = ["lambert", "glass_T1", "coat_lambert", "nested", "index_matched",
           "rough_glass", "rough_conductor", "nested_rough"]


@pytest.mark.parametrize("name", FURNACE)
def test_green_white_furnace(name, mcrt):
    """The sky is 0.5 green in every direction. With green reflectance, specular reflectance and transmittance 1 every lobe's
    green weight is 1 and refraction scaling cancels on exit, so a sample's green is 0 or 0.5 * 0.95^-k after k roulette
    survivals (rel 1e-12 in float64, 1e-5 (1 + k) in float32), and the mean is 0.5 within 5 SE. Rough glass and rough
    conductors lose energy to shadowing: their mean may not exceed 0.5 + 5 SE. Glass at 0 < T < 1 traps light (see
    test_partial_transparency_furnace). Independent of the restatement."""
    scene, exact = furnace_scene(mcrt, name)
    pt = mcrt.PathTracer(scene, global_seed=SEED)
    ps = port.PortScene(scene)
    try:
        rays, pixel, sample = camera_samples(ps, scene, n=65536, seed=7)
        res = {}
        for prec, tol in ((F64, 1e-12), (F32, 1e-5)):
            g = pt.sampleRay(rays, pixel, sample, precision=prec)[:, 1]
            assert np.isfinite(g).all()
            mean, se = float(g.mean()), float(g.std(ddof=1) / np.sqrt(len(g)))
            nz = g != 0.0
            k = np.rint(np.log(np.where(nz, g, 0.5) / 0.5) / np.log(1.0 / 0.95))
            rel = np.abs(g - 0.5 * 0.95 ** -k) / np.where(nz, g, 1.0)
            res[prec] = (mean, se, float(np.where(nz, rel / (1.0 + np.abs(k)), 0.0).max()), float(nz.mean()), int(k.max()))
            if exact:
                bar = tol * (1.0 + np.abs(k) * (prec == F32))
                off = nz & ~(rel <= bar)
                # A path whose IOR bookkeeping parts from the geometry keeps one interface's (n1/n2)^2 radiance compression:
                # a diffuse bounce off the floor where a glass sphere touches it, outside the sphere but still "in glass", or
                # a grazing entry into a nested sphere whose chord is shorter than the ray offset. Both sides of parity do
                # this (it is the reference's behaviour); measured 4 (smooth glass) and 1 (nested) of 65536 samples.
                assert off.sum() <= OFF_COMPRESSION * len(g), (name, prec, int(off.sum()))
                assert all(compression_of(g[i], COMPRESSION_PAIRS.get(name, []), bar[i]) for i in np.nonzero(off)[0]), (name, prec, g[off][:5])
                assert abs(mean - 0.5) <= BIAS_SE * se, (name, prec, mean, se)
            else:
                assert mean <= 0.5 + BIAS_SE * se, (name, prec, mean, se)
        REPORT[f"furnace {name}"] = "; ".join(f"{'f64' if p == F64 else 'f32'} mean {m:.5f} se {s:.1e} max rel/(1+k) {r:.1e} "
                                              f"nonzero {z:.3f} kmax {km}" for p, (m, s, r, z, km) in res.items())
    finally:
        ps.close()
        pt.close()


@pytest.mark.parametrize("T,ior", [(0.3, 1.5), (0.7, 1.5), (0.3, 1.1)], ids=["T0.3-ior1.5", "T0.7-ior1.5", "T0.3-ior1.1"])
def test_partial_transparency_furnace(T, ior, mcrt):
    """Smooth glass at 0 < T < 1 on a lone sphere under the sky, rays at fixed incidence. Light that enters refracts to an
    angle below the critical one and would leave; a diffuse bounce at the inner surface (probability (1 - R)(1 - T),
    interaction.cpp's selectType) sends it into a cosine-weighted direction, and a sphere keeps a chord's incidence angle at
    every reflection, so a direction beyond the critical angle (a fraction 1 - 1/n^2 of them) is reflected totally for ever
    and only roulette ends it. With q = 1/n^2 the escape probability after entering is E = T + (1 - T) q T / (1 - q (1 - T))
    and the expected green 0.5 (1 - (1 - F(cos)) T (1 - E)). Each sample is 0 or on the 0.5 0.95^-k grid, or, for a
    trapped orbit that leaves the sphere without refracting (at most 15 % of the samples at grazing incidence), on that grid
    times (1/n)^2; the float64 on-grid samples' mean is the closed form within 5 SE."""
    pt = sphere_tracer(mcrt, glass(mcrt, T=T, ior=ior), 1.0)
    n = 32768
    cos = [1.0, 0.9, 0.5, 0.1]
    try:
        rays, _ = rays_at_incidence(cos)
        out = {prec: pt.sampleRay(np.repeat(rays, n, axis=0), np.zeros(len(cos) * n, np.uint32),
                                  np.tile(np.arange(n, dtype=np.uint32), len(cos)), precision=prec)[:, 1].reshape(len(cos), n)
               for prec in (F64, F32)}
    finally:
        pt.close()
    q = 1.0 / ior ** 2
    escape = T + (1.0 - T) * q * T / (1.0 - q * (1.0 - T))
    zs = []
    for prec, tol in ((F64, 1e-12), (F32, 1e-5)):
        for i, c in enumerate(cos):
            g = out[prec][i]
            assert np.isfinite(g).all()
            nz = g != 0.0
            k = np.rint(np.log(np.where(nz, g, 0.5) / 0.5) / np.log(1.0 / 0.95))
            bar = tol * (1.0 + np.abs(k) * (prec == F32))
            on = nz & (np.abs(g - 0.5 * 0.95 ** -k) <= bar * g)
            off = nz & ~on
            assert all(compression_of(g[j], [(1.0, ior)], bar[j]) for j in np.nonzero(off)[0]), (T, ior, c, prec, g[off][:5])
            assert off.mean() <= 0.15, (T, ior, c, prec, off.mean())
            if prec == F32:
                continue      # float32's trapped orbits leave the sphere at another rate (the grid check above holds)
            adj = np.where(on, g, 0.0)
            want = 0.5 * (1.0 - (1.0 - fresnel_dielectric(1.0, ior, c)) * T * (1.0 - escape))
            z = (adj.mean() - want) / (adj.std(ddof=1) / np.sqrt(n))
            zs.append(round(float(z), 2))
            assert abs(z) <= BIAS_SE, (T, ior, c, prec, adj.mean(), want)
    REPORT[f"furnace partial T {T:g} ior {ior:g}"] = f"z of the on-grid mean against the closed form {zs}"


# ------------------------------------------------------------------------------------------------------------- 4. fast mode
from test_gpu_fast_mode import AGREE, AGREE_CASE, AGREE_GROUP, AGREE_SPECULAR     # noqa: E402

# per case (overall, specular groups, other groups), as test_gpu_fast_mode's AGREE_CASE. The smooth nested spheres take
# ior_test_nobvh_64's own exception (measured 0.703, dielectric 0.592); with rough glass inside them paths part sooner
# still (measured 0.612, outer sphere 0.465; the paired bias stays at 0.19 of its bar). Rough glass at an index-matched interface passes
# straight through, where the half vector of ggxTransmission is the round-off of n1 wo + n2 wi in either precision, so the
# two draw unrelated weights there: measured matched_rough 0.810, the rest of that case >= 0.87, and 0.941 for the lights,
# which reach the scene through those spheres
FAST_BARS = {"nested": (0.55, 0.40, AGREE_GROUP), "nested_smooth": AGREE_CASE["ior_test_nobvh_64"],
             "index_matched": (AGREE, 0.75, 0.90)}
GROUP_MIN = 500


def specular_label(scene, mcrt, case, label):
    """a first-hit group of glass, mirror or conductor (test_gpu_fast_mode's SPECULAR_GROUPS)"""
    for name, r in material_set(mcrt, case.mats):
        if name == label:
            return bool(r["transparency"] > 0 or r["perfect_mirror"] or r["has_complex_ior"])
    return False




@pytest.mark.parametrize("case", MATERIAL_CASES, ids=[mat_case_id(c) for c in MATERIAL_CASES])
def test_fast_mode_matches_float64(case, mcrt, held):
    """PRECISION_F32 against float64 sample by sample: every sample finite, no paired bias beyond 5 SE + 1e-5 mean|f64| per
    channel, and test_gpu_fast_mode's agreement bars per case and per first-hit material group"""
    pt, ps, scene = held(case)
    rays, pixel, sample = camera_samples(ps, scene)
    a = pt.sampleRay(rays, pixel, sample, precision=F64)
    b = pt.sampleRay(rays, pixel, sample, precision=F32)
    assert np.isfinite(b).all(), f"{int((~np.isfinite(b)).any(axis=1).sum())} non-finite float32 samples"
    ok = agree_mask(b, a)
    labels = first_hit_labels(mcrt, pt, scene, case, rays)
    groups = {g: float(ok[labels == g].mean()) for g in np.unique(labels) if (labels == g).sum() >= GROUP_MIN}
    z, ratio = paired_bias(b - a, a)
    REPORT[f"fast {mat_case_id(case)}"] = (f"agree {ok.mean():.4f}, bias z {np.round(z, 2).tolist()}, bias/bar {ratio.max():.2f}, groups "
                                           + ", ".join(f"{g} {f:.3f}" for g, f in sorted(groups.items())))
    assert ratio.max() <= 1.0, REPORT[f"fast {mat_case_id(case)}"]
    agree_bar, specular_bar, group_bar = FAST_BARS.get(case.mats, (AGREE, AGREE_SPECULAR, AGREE_GROUP))
    assert ok.mean() >= agree_bar, REPORT[f"fast {mat_case_id(case)}"]
    for g, f in groups.items():
        assert f >= (specular_bar if specular_label(scene, mcrt, case, g) else group_bar), (g, REPORT[f"fast {mat_case_id(case)}"])
