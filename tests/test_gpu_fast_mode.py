"""Fast mode (PRECISION_F32) against the float64 path, sample by sample (run on an H100).

Parity mode is pinned to the reference (tests/test_gpu_parity.py), so it is the high-precision reference here. At the same
global seed, sample s of pixel p draws the same sampler dimensions in both precisions: most samples make the same decisions
and differ only by float32 round-off, and the rest diverge where a float32 decision flips (an edge, a grazing hit, a
Russian-roulette or BSDF-lobe choice within round-off of its threshold). So the comparison is paired:
    closest hit         same primitive for >= 0.999 of the rays, every other ray explained (boundary, tie, duplicate, grazing);
                        |dt| <= C_T * 2^-24 * (scene_scale + t) / max(|cos|, COS_FLOOR) where the primitives agree
    per-sample radiance all finite; |f32 - f64| <= 1e-3 * max(|f64|, 0.1 mean|f64|) for >= AGREE of the samples and for
                        >= AGREE_GROUP of each first-hit material group; per channel |mean D| <= 5 SE(D) + 1e-5 mean|f64|
    frames              the same paired-bias bar over per-pixel D, equal paths, ray counts within the divergence rate
A bias that a 1 % frame-mean test cannot see (a lobe scaled by 1.01, an offset that does not follow the scene's scale)
moves mean D by many standard errors, because D is zero for almost every sample. The cases are the table of
tests/test_fast_mode_cases_cpu.py, which reaches every float branch of Launch<float>. Measured values are next to each
bar (H100 80GB HBM3, 700 W)."""
import contextlib
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import port
from scene_gen import generated_scene
from test_fast_mode_cases_cpu import CASES, Case, case_id, film_of, pack_of
from test_gpu_parity import photon_emit_args

pytestmark = pytest.mark.gpu

F64_TOL = 1e-3          # per-sample agreement: relative to max(|f64|, 0.1 mean|f64|)
AGREE = 0.95            # fraction of agreeing samples per case (measured 0.966 c2 ... 0.9999 oren_nayar_64)
AGREE_GROUP = 0.95      # per first-hit material group of >= GROUP_MIN samples (measured >= 0.9855, c1 diffuse), except:
AGREE_SPECULAR = 0.85   # glass, mirrors and near-specular metal (GGX alpha <= 0.1): specular chains over curved surfaces
                        # magnify float32 position error bounce by bounce until the path takes another branch (measured
                        # dielectric 0.903-0.951, mirror 0.928-0.95, metals_64 conductor 0.897)
SPECULAR_GROUPS = ("dielectric", "mirror", "conductor")
# (case, specular groups, other groups); translate_64x: see test_transformed_scene. Nested dielectrics (glass inside
# glass, no BVH): most paths bounce between interfaces, measured 0.686 / dielectric 0.561
AGREE_CASE = {"ior_test_nobvh_64": (0.60, 0.50, AGREE_GROUP), "translate_64x": (0.20, 0.18, 0.18)}
GROUP_MIN = 500
BIAS_SE = 5.0           # paired bias: |mean D| <= BIAS_SE * SE(D) + BIAS_FLOOR * mean|f64|
BIAS_FLOOR = 1e-5
HIT_AGREE = 0.999
C_T = 48.0              # closest-hit |dt| constant: measured max 23.5 (c1), 11.5 (c2, veach_mis), <= 3.1 elsewhere
COS_FLOOR = 1e-2
GRAZING = 0.02          # |cos| below which a differing primitive is a grazing hit
EDGE = 1e-4             # float32-sized onTriangleBoundary epsilon (bvh4.cuh uses 1e-9 for float64)
RAY_RATE = 0.02         # extension / shadow ray counts of a frame agree to this fraction (measured max 8.7e-3, ior_test_nobvh)
# share of a float32 map's photons with a float64 photon within 1e-4 scene_scale carrying its flux to 1e-4, per (scene, map).
# Every photon of pm_hexagon_room_64's caustic map, and many of its global map, crossed glass balls (the specular chains of
# AGREE_SPECULAR): measured 0.628 and 0.832. metals_64 has no caustic map; its global map measured 1.0
EMIT_MATCHED = {("pm_hexagon_room_64", 0): 0.55, ("pm_hexagon_room_64", 1): 0.75, ("metals_64", 1): 0.99}
REPEATS = 16            # sample indices per golden ps_ray
F32, F64 = 1, 0


# ------------------------------------------------------------------------------------------------------------- helpers
def scene_scale(scene):
    """mcrt_scene_upload's scene_scale: largest |coordinate| of the root box, or of the primitives without a BVH"""
    a = scene.a
    if scene.n_nodes:
        return float(np.abs(a["node_bounds"][:6]).max())
    m = 0.0
    for k in ("tri_v0", "tri_v1", "tri_v2", "quadric_bounds"):
        if a[k].size:
            v = np.abs(a[k]); m = max(m, float(v[v < 1e300].max()))
    s = a["sphere_origin_radius"].reshape(-1, 4)
    if len(s):
        m = max(m, float((np.abs(s[:, :3]).max(axis=1) + s[:, 3]).max()))
    return m or 1.0


def load_scene(mcrt, name):
    if name.startswith("gen/"):
        return generated_scene(mcrt, name[4:])
    return mcrt.Scene.from_pack(os.path.join(GOLDEN, name + ".mcrtpack"))


def golden_of(name):
    base = pack_of(name)
    if base == "film_hexagon_room_64":
        return np.load(os.path.join(GOLDEN, "film_kat.npz"))
    return np.load(os.path.join(GOLDEN, base + ".npz"))


def emission_args(scene):
    """the pack's photon pass, or for a scene without maps the pm scene's emission count and factor over its own bounds"""
    if "photon_emit_params" in scene.extra:
        return photon_emit_args(scene)
    return dict(emissions=4000, caustic_factor=10.0, max_photons_per_octree_leaf=200, k_nearest_photons=50,
                direct_visualization=False, scene_bounds=scene.extra["scene_bounds"])


@pytest.fixture(scope="module")
def tracer(mcrt):
    """The float64 integrator of one scene at a time (each holds a full path pool); photon mappers carry a map emitted in
    float64 (the pack's photon pass for pm scenes). Scenes are kept, so a generated scene's BVH is built once."""
    scenes, held = {}, {}

    def get(name, photon=False):
        key = (name, photon)
        if key not in held:
            for pt, _, _ in held.values():
                pt.close()
            held.clear()
            if name not in scenes:
                scenes[name] = load_scene(mcrt, name)
            scene, g = scenes[name], golden_of(name)
            if photon:
                pt = mcrt.PhotonMapper(scene, global_seed=int(g["seed"]), emit=emission_args(scene))
                pt.f64_maps = pt._maps
            else:
                pt = mcrt.PathTracer(scene, global_seed=int(g["seed"]))
            held[key] = (pt, scene, g)
        return held[key]
    yield get
    for pt, _, _ in held.values():
        pt.close()


@contextlib.contextmanager
def ray_eps_scale(pt, value):
    pt.set_option("ray_eps_scale", value)
    try:
        yield
    finally:
        pt.set_option("ray_eps_scale", 1e-5)      # mcrt_ctx default


def paired_bias(d, ref):
    """-> (per-channel |mean D| / SE, bar ratio <= 1 passes): D = f32 - f64 over pairs (samples or pixels), [n, 3]"""
    d = d.reshape(-1, 3)
    n = len(d)
    mean = d.mean(axis=0)
    se = d.std(axis=0, ddof=1) / np.sqrt(n)
    floor = BIAS_FLOOR * np.abs(ref.reshape(-1, 3)).mean(axis=0)
    z = np.abs(mean) / np.maximum(se, 1e-300)
    ratio = np.abs(mean) / (BIAS_SE * se + floor)
    return z, ratio


def agree_mask(a, b):
    """per sample: |a - b| <= F64_TOL * max(|b|, 0.1 mean|b|) in every channel (b the float64 value)"""
    scale = np.maximum(np.abs(b).max(axis=1), 0.1 * np.abs(b).mean())
    return (np.abs(a - b).max(axis=1) <= F64_TOL * np.maximum(scale, 1e-300))


def material_class(mats, m):
    """diffuse, oren_nayar, ggx, conductor, dielectric, mirror or emissive"""
    r = mats[m]
    if r["emissive"]:
        return "emissive"
    if r["dirac_delta"] and r["perfect_mirror"]:
        return "mirror"
    if r["transparency"] > 0:
        return "dielectric"
    if r["has_complex_ior"]:
        return "conductor"
    if r["rough_specular"]:
        return "ggx"
    if r["rough"]:
        return "oren_nayar"
    return "diffuse"


REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if REPORT:
        print("\nfast vs parity:")
        for k in sorted(REPORT):
            print(f"  {k:48s} {REPORT[k]}")


# ------------------------------------------------------------------------------------------------------------- 2. closest hit
def hit_geometry(scene, prim, rays, t):
    """-> (|cos| between ray and geometric normal, triangle barycentrics (u, v) or NaN) at o + t d on primitive `prim`"""
    a = scene.a
    n = len(prim)
    cos = np.full(n, np.nan); u = np.full(n, np.nan); v = np.full(n, np.nan)
    o, d = rays[:, :3], rays[:, 3:]
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    p = o + d * t[:, None]
    ptype, pidx = a["prim_type"][prim], a["prim_index"][prim]
    tri = ptype == 0
    if tri.any():
        i = pidx[tri]
        v0 = a["tri_v0"].reshape(-1, 3)[i]; e1 = a["tri_e1"].reshape(-1, 3)[i]; e2 = a["tri_e2"].reshape(-1, 3)[i]
        nrm = a["tri_normal"].reshape(-1, 3)[i]
        cos[tri] = np.abs(np.sum(nrm * d[tri], axis=1))
        pv = np.cross(d[tri], e2); det = np.sum(e1 * pv, axis=1)
        tv = o[tri] - v0
        uu = np.sum(tv * pv, axis=1) / det
        vv = np.sum(d[tri] * np.cross(tv, e1), axis=1) / det
        u[tri], v[tri] = uu, vv
    sph = ptype == 1
    if sph.any():
        s = a["sphere_origin_radius"].reshape(-1, 4)[pidx[sph]]
        nrm = (p[sph] - s[:, :3]) / s[:, 3:4]
        cos[sph] = np.abs(np.sum(nrm * d[sph], axis=1)) / np.linalg.norm(nrm, axis=1)
    quad = ptype == 2
    if quad.any():
        Q = a["quadric_Q"].reshape(-1, 4, 4)[pidx[quad]].transpose(0, 2, 1)
        X = np.concatenate([p[quad], np.ones((quad.sum(), 1))], axis=1)
        grad = np.einsum("nij,nj->ni", Q + Q.transpose(0, 2, 1), X)[:, :3]
        cos[quad] = np.abs(np.sum(grad * d[quad], axis=1)) / np.maximum(np.linalg.norm(grad, axis=1), 1e-300)
    return cos, u, v


def dt_bound(scale, t, cos):
    return C_T * 2.0 ** -24 * (scale + t) / np.maximum(cos, COS_FLOOR)


def duplicate_triangles(scene, p, q):
    """p and q are triangles with the same three vertices (the generated scenes' exact copies)"""
    a = scene.a
    out = np.zeros(len(p), bool)
    ok = (a["prim_type"][p] == 0) & (a["prim_type"][q] == 0)
    if ok.any():
        def verts(x):
            i = a["prim_index"][x]
            return np.sort(np.stack([a[k].reshape(-1, 3)[i] for k in ("tri_v0", "tri_v1", "tri_v2")], axis=1), axis=1)
        out[ok] = np.all(verts(p[ok]) == verts(q[ok]), axis=(1, 2))
    return out


def check_closest_hit(mcrt, pt, scene, rays, label):
    h64 = pt.intersect(rays, precision=F64)
    h32 = pt.intersect(rays, precision=F32)
    scale = scene_scale(scene)
    same = h64["prim"] == h32["prim"]
    agree = float(same.mean())
    # a differing primitive: geometry at the float64 hit (or at the float32 hit where float64 missed)
    diff = np.nonzero(~same)[0]
    use64 = h64["prim"][diff] != mcrt.NO_PRIM
    prim = np.where(use64, h64["prim"][diff], h32["prim"][diff])
    t = np.where(use64, h64["t"][diff], h32["t"][diff])
    cos, u, v = hit_geometry(scene, prim, rays[diff], t)
    e = EDGE * np.maximum(1.0, t / scale)
    edge = (u < e) | (v < e) | (u + v > 1 - e)
    both = use64 & (h32["prim"][diff] != mcrt.NO_PRIM)
    tie = both & (np.abs(h32["t"][diff] - h64["t"][diff]) <= dt_bound(scale, h64["t"][diff], cos))
    dup = both & duplicate_triangles(scene, np.where(both, h64["prim"][diff], 0), np.where(both, h32["prim"][diff], 0))
    grazing = cos < GRAZING
    unexplained = ~(edge | tie | dup | grazing)
    # where the primitives agree: float32 round-off of t, relative to the scene's scale and the hit's slope
    hit = same & (h64["prim"] != mcrt.NO_PRIM)
    cos_s, _, _ = hit_geometry(scene, h64["prim"][hit], rays[hit], h64["t"][hit])
    dt = np.abs(h32["t"][hit] - h64["t"][hit])
    c = C_T * dt / dt_bound(scale, h64["t"][hit], cos_s)
    REPORT[f"hit {label}"] = (f"agree {agree:.5f}, differ {len(diff)} (edge {int(edge.sum())} tie {int(tie.sum())} dup {int(dup.sum())} "
                              f"grazing {int(grazing.sum())} unexplained {int(unexplained.sum())}), dt constant max {c.max():.2f} "
                              f"p99.9 {np.quantile(c, 0.999):.2f}")
    assert agree >= HIT_AGREE, REPORT[f"hit {label}"]
    assert not unexplained.any(), (REPORT[f"hit {label}"], diff[unexplained][:5].tolist(), cos[unexplained][:5].tolist())
    assert c.max() <= C_T, REPORT[f"hit {label}"]


@pytest.mark.parametrize("name", sorted({c.scene for c in CASES}))
def test_closest_hit(name, mcrt, tracer):
    pt, scene, g = tracer(name)
    rays = g["tr_rays"] if "tr_rays" in g.files else np.load(os.path.join(GOLDEN, "c2_hexagon_room_96.npz"))["tr_rays"]
    check_closest_hit(mcrt, pt, scene, rays, name)


# ------------------------------------------------------------------------------------------------------------- 3. per-sample radiance
def paired_samples(g):
    n = len(g["ps_rays"])
    rays = np.tile(g["ps_rays"], (REPEATS, 1))
    pixel = np.tile(g["ps_pixel"], REPEATS).astype(np.uint32)
    sample = (np.tile(g["ps_sample"], REPEATS) + np.repeat(np.arange(REPEATS), n) * 4096).astype(np.uint32)
    return rays, pixel, sample


def check_samples(mcrt, pt, scene, g, label, case_name=None):
    """-> (agreement, worst group, bias/bar ratio per channel)"""
    agree_bar, specular_bar, group_bar = AGREE_CASE.get(case_name, (AGREE, AGREE_SPECULAR, AGREE_GROUP))
    rays, pixel, sample = paired_samples(g)
    a = pt.sampleRay(rays, pixel, sample, precision=F64)
    b = pt.sampleRay(rays, pixel, sample, precision=F32)
    assert np.isfinite(b).all(), f"{int((~np.isfinite(b)).any(axis=1).sum())} non-finite float32 samples"
    ok = agree_mask(b, a)
    first = pt.intersect(rays[:len(g["ps_rays"])], precision=F64)["prim"]
    mats = scene.a["materials"]
    cls = np.array(["miss" if p == mcrt.NO_PRIM else material_class(mats, scene.a["prim_material"][p]) for p in first])
    cls = np.tile(cls, REPEATS)
    groups = {c: float(ok[cls == c].mean()) for c in np.unique(cls) if (cls == c).sum() >= GROUP_MIN}
    worst = min(groups.items(), key=lambda kv: kv[1])
    z, ratio = paired_bias(b - a, a)
    REPORT[f"samples {label}"] = (f"agree {ok.mean():.4f}, worst group {worst[0]} {worst[1]:.4f}, bias z {np.round(z, 2).tolist()}, "
                                  f"bias/bar {ratio.max():.2f}")
    assert ok.mean() >= agree_bar, REPORT[f"samples {label}"]
    for c, f in groups.items():
        assert f >= (specular_bar if c in SPECULAR_GROUPS else group_bar), (c, REPORT[f"samples {label}"])
    return ok.mean(), worst, ratio


SAMPLE_CASES = [c for c in CASES if c.film is None and c.k is None and not c.gather and not c.emit and not c.adaptive]


@pytest.mark.parametrize("case", SAMPLE_CASES, ids=[case_id(c) for c in SAMPLE_CASES])
def test_sample_radiance(case, mcrt, tracer):
    pt, scene, g = tracer(case.scene, case.photon)
    _, _, ratio = check_samples(mcrt, pt, scene, g, case_id(case), pack_of(case.scene))
    assert ratio.max() <= 1.0, REPORT[f"samples {case_id(case)}"]


# ------------------------------------------------------------------------------------------------------------- 4. frames
def camera_of(scene, case):
    cam = scene.cameras()[0]
    if case.scene.startswith("gen/"):
        cam = cam.resized(96, 54)
    cam = cam.resized(cam.width, cam.height, 8)
    cam.film = film_of(case.film)
    return cam


def check_frames(pt, cam, label, bar=True):
    """-> bias/bar ratio of the float32 frame against the float64 frame (asserted <= 1 when bar)"""
    a = pt.render_rows(cam, precision=F64); sa = pt.last_stats
    b = pt.render_rows(cam, precision=F32); sb = pt.last_stats
    assert np.isfinite(b).all(), f"{int((~np.isfinite(b)).any(axis=2).sum())} non-finite float32 pixels"
    z, ratio = paired_bias(b - a, a)
    rate = [abs(sb[k] - sa[k]) / max(1, sa[k]) for k in ("extension_rays", "shadow_rays")]
    REPORT[f"frame {label}"] = (f"bias z {np.round(z, 2).tolist()}, bias/bar {ratio.max():.2f}, ray count rate ext {rate[0]:.2e} "
                                f"shadow {rate[1]:.2e}, mean rel {abs(b.mean() - a.mean()) / a.mean():.2e}")
    if bar:
        assert sa["paths"] == sb["paths"] == cam.width * cam.height * cam.sqrtspp ** 2
        assert sa["ior_stack_overflows"] == 0 and sb["ior_stack_overflows"] == 0
        assert max(rate) <= RAY_RATE, REPORT[f"frame {label}"]
        assert ratio.max() <= 1.0, REPORT[f"frame {label}"]
    return ratio.max()


FRAME_CASES = [c for c in CASES if not c.emit and not c.adaptive]


@pytest.mark.parametrize("case", FRAME_CASES, ids=[case_id(c) for c in FRAME_CASES])
def test_frame(case, mcrt, tracer):
    pt, scene, g = tracer(case.scene, case.photon)
    cam = camera_of(scene, case)
    if case.photon:
        # one float64 map, rendered by both precisions: the float32 query and shade side alone
        c, gl, k, dv = pt.f64_maps
        pt._maps = (c, gl, case.k or k, dv)
        pt.upload_photons()
        pt.gather_radius(*(gather_radii(pt) if case.gather else (0.0, 0.0)))
    try:
        check_frames(pt, cam, case_id(case))
    finally:
        if case.photon:
            pt.gather_radius(0.0, 0.0)
            cam.film = None
            pt.set_film(cam)


def gather_radii(pm):
    """the median distance to the k-th nearest photon of each map at the photons themselves (ProgressivePhotonMapping's rule)"""
    out = []
    for which in (0, 1):
        ph = pm._maps[which]["photons"].reshape(-1, 8)[::17, 3:6].astype(np.float64)
        if len(ph) == 0:
            out.append(0.0)
            continue
        _, d2, _ = pm.knn(which, ph)
        out.append(float(np.sqrt(np.median(np.where(np.isfinite(d2), d2, 0.0).max(axis=1)))))
    # a map without photons (metals_64 has no caustic paths) still needs a positive radius
    return [r if r > 0 else max(out) for r in out]


ADAPTIVE_CASES = [c for c in CASES if c.adaptive]


@pytest.mark.parametrize("case", ADAPTIVE_CASES, ids=[case_id(c) for c in ADAPTIVE_CASES])
def test_adaptive_pass(case, mcrt, tracer):
    """generate's pixel-list form: one pass over all tiles, every other tile retired, one more pass"""
    _, scene, g = tracer(case.scene)
    cam = camera_of(scene, case)
    frames, stats = [], []
    for prec in (F64, F32):
        pt = mcrt.PathTracer(scene, precision=prec, global_seed=int(g["seed"]))
        try:
            prog = mcrt.Progressive(pt, cam, tile=8)
            prog.add(16)
            mask = np.zeros(prog.active.shape, bool); mask.flat[::2] = True
            prog.retire(mask)
            prog.add(16)
            frames.append(prog.frame()); stats.append(dict(prog.stats))
        finally:
            pt.close()
    a, b = frames
    assert np.isfinite(b).all()
    z, ratio = paired_bias(b - a, a)
    rate = abs(stats[1]["extension_rays"] - stats[0]["extension_rays"]) / stats[0]["extension_rays"]
    REPORT[f"adaptive {case_id(case)}"] = f"bias z {np.round(z, 2).tolist()}, bias/bar {ratio.max():.2f}, ext rate {rate:.2e}"
    assert stats[0]["paths"] == stats[1]["paths"]
    assert rate <= RAY_RATE and ratio.max() <= 1.0, REPORT[f"adaptive {case_id(case)}"]


# ------------------------------------------------------------------------------------------------------------- 5. photon emission
EMIT_CASES = [c for c in CASES if c.emit]


@pytest.mark.parametrize("case", EMIT_CASES, ids=[case_id(c) for c in EMIT_CASES])
def test_photon_emission(case, mcrt, tracer):
    from scipy.spatial import cKDTree
    pm, scene, g = tracer(case.scene, True)
    args = emission_args(scene)
    n64 = pm.emit(**args, precision=F64); m64 = pm._maps
    n32 = pm.emit(**args, precision=F32); m32 = pm._maps
    scale = scene_scale(scene)
    try:
        for which in (0, 1):
            p64 = m64[which]["photons"].reshape(-1, 8).astype(np.float64)
            p32 = m32[which]["photons"].reshape(-1, 8).astype(np.float64)
            rate = abs(n32[which] - n64[which]) / max(1, n64[which])
            if n64[which] == 0:
                assert n32[which] == 0
                continue
            d, j = cKDTree(p64[:, 3:6]).query(p32[:, 3:6])
            flux_ok = np.all(np.abs(p32[:, :3] - p64[j, :3]) <= 1e-4 * np.maximum(np.abs(p64[j, :3]), 1e-30), axis=1)
            matched = (d <= 1e-4 * scale) & flux_ok
            # total flux: the unmatched photons are the divergent ones; their spread is the noise of the difference
            diff = p32[:, :3].sum(axis=0) - p64[:, :3].sum(axis=0)
            un32, un64 = p32[~matched, :3], np.delete(p64, j[matched], axis=0)[:, :3]
            se = np.sqrt((un32 ** 2).sum(axis=0) + (un64 ** 2).sum(axis=0))
            ratio = np.abs(diff) / (BIAS_SE * se + BIAS_FLOOR * np.abs(p64[:, :3]).sum(axis=0))
            REPORT[f"emit {case_id(case)} map {which}"] = (f"photons {n64[which]} / {n32[which]} (rate {rate:.2e}), matched "
                                                          f"{matched.mean():.5f}, flux bias/bar {ratio.max():.2f}")
            assert rate <= RAY_RATE and matched.mean() >= EMIT_MATCHED[(case.scene, which)] and ratio.max() <= 1.0, REPORT[f"emit {case_id(case)} map {which}"]
    finally:
        pm._maps = pm.f64_maps
        pm.upload_photons()


# ------------------------------------------------------------------------------------------------------------- 6. float-specific edges
def transformed(mcrt, scene, s=1.0, shift=(0.0, 0.0, 0.0)):
    """scene with every point p -> s p + shift (triangles and spheres) and its camera, the BVH rebuilt by oracle/port.bvh_build"""
    flat = scene.unbuilt()
    a = dict(flat.a, **flat.extra)
    a["scene_ior"] = np.array([flat.ior])
    shift = np.asarray(shift, np.float64)
    tri = [(a[k].reshape(-1, 3) * s + shift) for k in ("tri_v0", "tri_v1", "tri_v2")]
    a["tri_v0"], a["tri_v1"], a["tri_v2"] = (t.reshape(-1) for t in tri)
    a["tri_e1"] = (tri[1] - tri[0]).reshape(-1); a["tri_e2"] = (tri[2] - tri[0]).reshape(-1)
    sph = a["sphere_origin_radius"].reshape(-1, 4).copy()
    sph[:, :3] = sph[:, :3] * s + shift; sph[:, 3] *= s
    a["sphere_origin_radius"] = sph.reshape(-1)
    a["prim_area"] = a["prim_area"] * s * s
    b = np.asarray(a["scene_bounds"], np.float64)
    a["scene_bounds"] = np.concatenate([b[:3] * s + shift, b[3:] * s + shift])
    cam = a["camera_f64"].copy()
    cam[0:3] = cam[0:3] * s + shift
    cam[15] = cam[15] * s if cam[15] > 0 else cam[15]      # focus distance
    a["camera_f64"] = cam
    out = mcrt.Scene(a)
    _, bvh_type, bins = (int(v) for v in scene.extra["bvh_params"])
    return out.with_bvh(port.bvh_build(out.prim_bounds(), a["scene_bounds"], bvh_type, bins, mcrt.BvhDesc))


def transformed_rays(rays, s=1.0, shift=(0.0, 0.0, 0.0)):
    r = rays.copy()
    r[:, :3] = r[:, :3] * s + np.asarray(shift)
    return r


EDGE_CASES = [("scale_2^-10", 2.0 ** -10, 0.0), ("scale_2^10", 2.0 ** 10, 0.0), ("translate_64x", 1.0, 63.0)]


@pytest.mark.parametrize("label,s,shift", EDGE_CASES, ids=[e[0] for e in EDGE_CASES])
def test_transformed_scene(label, s, shift, mcrt):
    """c2 (triangles and spheres) scaled by a power of two, exact in both precisions, or moved by 63 times its scale along x,
    which makes scene_scale and with it the fast mode's ray offset follow the translation. Closest hits, the paired bias of
    the samples and the frame must meet the same bars as the untransformed scene (measured bias/bar 0.33 and 0.58).

    The per-sample agreement bar is loosened for the translation only, to 0.20 of the samples and 0.18 of every material
    group (measured 0.245, worst group dielectric 0.228). Two effects, neither of them a bias: the fast mode's offset is
    1e-5 x scene_scale = 8.3e-3 here, 64 times c2's, and moves every next-event distance, and with it the 1/r^2 of the light
    pdf, by about 1e-3 relative, the size of the agreement tolerance (the float64 path offsets by 1e-9); and float32 positions
    carry 64 times the absolute error, so specular chains part sooner."""
    base = mcrt.Scene.from_pack(os.path.join(GOLDEN, "c2_hexagon_room_96.mcrtpack"))
    g = dict(np.load(os.path.join(GOLDEN, "c2_hexagon_room_96.npz")))
    vec = np.array([shift * scene_scale(base), 0.0, 0.0])
    scene = transformed(mcrt, base, s, vec)
    g["tr_rays"] = transformed_rays(g["tr_rays"], s, vec)
    g["ps_rays"] = transformed_rays(g["ps_rays"], s, vec)
    pt = mcrt.PathTracer(scene, global_seed=int(g["seed"]))
    try:
        check_closest_hit(mcrt, pt, scene, g["tr_rays"], label)
        _, _, ratio = check_samples(mcrt, pt, scene, g, label, label if label in AGREE_CASE else "c2_hexagon_room_96")
        assert ratio.max() <= 1.0, REPORT[f"samples {label}"]
        check_frames(pt, scene.cameras()[0].resized(96, 54, 8), label)
    finally:
        pt.close()


def test_wrong_ray_offset_fails_the_bias_bar(mcrt, tracer):
    """The paired-bias bar has teeth: quadric_64 with a ray offset of 1e-9 x scene_scale (self-intersection acne on the
    quadrics in float32) must fail it, in the per-sample and in the frame comparison."""
    pt, scene, g = tracer("quadric_64")
    with ray_eps_scale(pt, 1e-9):
        rays, pixel, sample = paired_samples(g)
        a = pt.sampleRay(rays, pixel, sample, precision=F64)
        b = pt.sampleRay(rays, pixel, sample, precision=F32)
        _, ratio = paired_bias(b - a, a)
        frame_ratio = check_frames(pt, camera_of(scene, Case("quadric_64")), "quadric_64 eps 1e-9", bar=False)
    REPORT["negative control quadric_64 eps 1e-9"] = f"samples bias/bar {ratio.max():.2f}, frame bias/bar {frame_ratio:.2f}"
    assert ratio.max() > 1.0 and frame_ratio > 1.0, REPORT["negative control quadric_64 eps 1e-9"]
    # and the restored default passes
    _, _, ratio = check_samples(mcrt, pt, scene, g, "quadric_64 restored", "quadric_64")
    assert ratio.max() <= 1.0
