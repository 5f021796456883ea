"""Progressive photon mapping without a GPU: the radius schedule (ppm_radii), a numpy restatement of the emission
plan's per-light counts (emissionPlan in csrc/abi.cu), and the float64 brute-force fixed-radius gather that
test_gpu_ppm.py holds the kernels to."""
import os

import numpy as np
import pytest

from conftest import GOLDEN


def emission_counts(scene, emissions, caustic_factor):
    """emissionPlan's emissions per light, in its float64 expression order: photon_emissions = (size_t)(emissions *
    caustic_factor); light l's share is compAdd(emittance * area) over the sum of all lights'; n_l = (size_t)(photon_emissions
    * share)."""
    a = scene.a
    prims = a["light_prim"].astype(np.int64)
    flux = [a["materials"]["emittance"][a["prim_material"][p]] * a["prim_area"][p] for p in prims]
    add = [0.0 + f[0] + f[1] + f[2] for f in flux]
    total = 0.0
    for x in add:
        total += x
    photon_emissions = int(float(emissions) * float(caustic_factor))
    return np.array([int(float(photon_emissions) * (x / total)) for x in add], np.int64)


def union_passes(scene, caustic_factor, passes, candidates):
    """The first emission count E of `candidates` whose per-light counts for passes * E emissions are exactly `passes`
    times those for E: then passes 0..passes-1 of E emissions cover the emission indices of one pass of passes * E."""
    for e in candidates:
        one, many = emission_counts(scene, e, caustic_factor), emission_counts(scene, passes * e, caustic_factor)
        if (one > 0).all() and np.array_equal(many, passes * one):
            return int(e)
    raise AssertionError("no emission count in the candidates splits into equal passes")


def gather_reference(photons, points, radius):
    """Brute-force fixed-radius gather in float64 -> (count [n], flux_sum [n, 3], cone_sum [n, 3]). The distance is
    the kernel's: the float32 position widened, dx = px - x, (dx*dx + dy*dy) + dz*dz, accepted when <= radius^2; the
    cone weight is max(0, 1 - sqrt(d2 * (1 / radius^2)))."""
    ph = np.asarray(photons, np.float32).reshape(-1, 8)
    pos, flux = ph[:, 3:6].astype(np.float64), ph[:, 0:3].astype(np.float64)
    points = np.asarray(points, np.float64).reshape(-1, 3)
    r2 = float(radius) * float(radius)
    inv = 1.0 / r2
    count = np.zeros(len(points), np.uint32)
    fsum, csum = np.zeros((len(points), 3)), np.zeros((len(points), 3))
    for s in range(0, len(points), 256):
        p = points[s:s + 256]
        dx = p[:, None, 0] - pos[None, :, 0]
        dy = p[:, None, 1] - pos[None, :, 1]
        dz = p[:, None, 2] - pos[None, :, 2]
        d2 = dx * dx + dy * dy + dz * dz
        inside = d2 <= r2
        w = np.where(inside, np.maximum(0.0, 1.0 - np.sqrt(d2 * inv)), 0.0)
        count[s:s + 256] = inside.sum(1)
        fsum[s:s + 256] = inside.astype(np.float64) @ flux
        csum[s:s + 256] = w @ flux
    return count, fsum, csum


@pytest.fixture(scope="module")
def pm_scene(mcrt):
    return mcrt.Scene.from_pack(os.path.join(GOLDEN, "pm_hexagon_room_64.mcrtpack"))


# ---------------------------------------------------------------------------------------------- radius schedule
@pytest.mark.parametrize("alpha", [0.1, 0.5, 2 / 3, 0.9])
def test_ppm_radii_follow_the_schedule(mcrt, alpha):
    r1 = 0.37
    r = mcrt.ppm_radii(r1, alpha, 200)
    assert r.shape == (200,) and r[0] == r1
    i = np.arange(1, 200, dtype=np.float64)
    np.testing.assert_allclose(r[1:] ** 2 / r[:-1] ** 2, (i + alpha) / (i + 1.0), rtol=1e-12)
    assert (np.diff(r) < 0).all()


def test_ppm_radii_refuse_bad_arguments(mcrt):
    for alpha in (0.0, 1.0, -0.5, 1.5, float("nan")):
        with pytest.raises(mcrt.McrtError):
            mcrt.ppm_radii(1.0, alpha, 4)
    for r1 in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(mcrt.McrtError):
            mcrt.ppm_radii(r1, 0.5, 4)
    assert mcrt.ppm_radii(2.5, 0.5, 1).tolist() == [2.5]


# ---------------------------------------------------------------------------------------------- emission plan
def test_emission_counts_restate_the_plan(pm_scene):
    params = pm_scene.extra["photon_emit_params"]
    counts = emission_counts(pm_scene, params[0], params[1])
    photon_emissions = int(params[0] * params[1])
    assert len(counts) == pm_scene.a["light_prim"].size and (counts > 0).all()
    # each light's count is rounded down, so together they fall short of the total by less than one per light
    assert photon_emissions - len(counts) < counts.sum() <= photon_emissions


def test_union_passes_split_exactly(pm_scene):
    cf = float(pm_scene.extra["photon_emit_params"][1])
    e = union_passes(pm_scene, cf, 3, range(1000, 1100))
    assert np.array_equal(emission_counts(pm_scene, 3 * e, cf), 3 * emission_counts(pm_scene, e, cf))


# ---------------------------------------------------------------------------------------------- brute-force gather
def test_gather_reference_matches_a_plain_loop():
    rng = np.random.default_rng(5)
    ph = np.zeros((300, 8), np.float32)
    ph[:, 0:3] = rng.uniform(0, 1, (300, 3))
    ph[:, 3:6] = rng.uniform(-1, 1, (300, 3))
    pts = np.concatenate([rng.uniform(-1.2, 1.2, (40, 3)), ph[:10, 3:6].astype(np.float64) + [0.1875, 0.25, 0.0]])
    radius = 0.3125   # the last 10 points lie exactly on this sphere around photons 0..9
    count, fsum, csum = gather_reference(ph, pts, radius)
    for q, p in enumerate(pts):
        n, f, c = 0, np.zeros(3), np.zeros(3)
        for x in ph:
            d = [p[0] - float(x[3]), p[1] - float(x[4]), p[2] - float(x[5])]
            d2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2]
            if d2 <= radius * radius:
                n += 1
                f += x[0:3].astype(np.float64)
                c += x[0:3].astype(np.float64) * max(0.0, 1.0 - np.sqrt(d2 * (1.0 / (radius * radius))))
        assert count[q] == n
        np.testing.assert_allclose(fsum[q], f, rtol=1e-13, atol=0)
        np.testing.assert_allclose(csum[q], c, rtol=1e-12, atol=1e-300)
    assert (count[40:] >= 1).all()   # the boundary photon itself is inside: the test is inclusive
