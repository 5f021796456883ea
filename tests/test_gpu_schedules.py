"""The wavefront's schedules and size-selected paths against the reference (run on an H100).

The golden scenes are small: under the default settings they never fill the path pool, never reach the dynamic-fetch search and
never take primitive-keyed ray sorting. Here every golden case is rendered under each schedule option (a pool of 1024 paths that is
refilled every iteration, dynamic fetch forced on, sorting off or changed, one CTA per SM, polling every iteration or every 64) to the
bars of tests/test_gpu_parity.py; the photon pass, a reconstruction filter, progressive passes and the C2 benchmark band run through a
saturated pool; and the generated scenes of tests/scene_gen.py, which cross the size thresholds, are rendered with the auto settings
against the CPU restatement and against the same frame with each size-selected path turned off.

Tolerances are those of test_gpu_parity.py. A schedule changes which paths share a launch and in which order the float64 film sums are
added, nothing on a path, so a frame under any schedule equals the default frame to 1e-12 relative, with equal ray counts."""
import contextlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases
from oracle import port
from scene_gen import GENERATED, generated_scene
from test_gpu_big_scenes import check_c2_benchmark_rows
from test_gpu_parity import check_emitted_maps, photon_emit_args

pytestmark = pytest.mark.gpu

DEFAULTS = dict(dynamic_fetch=-1, pool_paths=1 << 23, sort_rays=1, sort_shade=0, sort_shade_class=1, sort_prim_key=-1,
                blocks_per_sm=16, poll_interval=4, exact_traversal=0)      # mcrt_ctx (abi.cu)
SCHEDULES = [dict(dynamic_fetch=1), dict(pool_paths=1024), dict(pool_paths=1024, dynamic_fetch=1), dict(sort_rays=0), dict(sort_shade=1),
             dict(sort_shade_class=0), dict(blocks_per_sm=1), dict(poll_interval=1), dict(poll_interval=64)]
SATURATED = dict(pool_paths=1024, dynamic_fetch=1)


def schedule_id(opts):
    return ",".join(f"{k}={v}" for k, v in opts.items())


@contextlib.contextmanager
def options(pt, **opts):
    for k, v in opts.items():
        pt.set_option(k, v)
    try:
        yield
    finally:
        for k in opts:
            pt.set_option(k, DEFAULTS[k])


def rel_rmse(img, ref):
    return float(np.sqrt(np.mean((img - ref) ** 2))) / max(1.0, float(np.abs(ref).mean()))


def equal_frames(a, b):
    """Same paths, film sums added in another order."""
    return np.abs(a - b).max() <= 1e-12 * max(1.0, np.abs(b).max())


@pytest.fixture(scope="module")
def golden_tracer(mcrt):
    """One golden case's tracer at a time, with its frame's shadow-ray count under the default settings."""
    held = {}

    def get(cid):
        if cid not in held:
            for pt, _, _, _ in held.values():
                pt.close()
            held.clear()
            scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
            g = np.load(os.path.join(GOLDEN, cid + ".npz"))
            cls = mcrt.PhotonMapper if scene.photon_maps() is not None else mcrt.PathTracer
            pt = cls(scene, precision=mcrt.PRECISION_F64, global_seed=int(g["seed"]))
            pt.render_rows(scene.cameras()[0])
            held[cid] = (pt, scene, g, pt.last_stats["shadow_rays"])
        return held[cid]
    yield get
    for pt, _, _, _ in held.values():
        pt.close()


# ------------------------------------------------------------------------------------------- a. golden scenes, every schedule
@pytest.mark.parametrize("cid,opts", [(c, o) for c in golden_cases() for o in SCHEDULES],
                         ids=[f"{c}-{schedule_id(o)}" for c in golden_cases() for o in SCHEDULES])
def test_golden_case_under_schedule(cid, opts, mcrt, golden_tracer):
    pt, scene, g, default_shadow = golden_tracer(cid)
    cam = scene.cameras()[0]
    with options(pt, **opts):
        img = pt.render_rows(cam)
        st = pt.last_stats
        rgb = pt.sampleRay(g["ps_rays"], g["ps_pixel"], g["ps_sample"])     # 4096 user rays, more than a pool of 1024
    tol = 1e-6 if cid.startswith("pm_") else 1e-9
    assert rel_rmse(img, g["image"]) < tol
    assert st["paths"] == cam.width * cam.height * cam.sqrtspp ** 2
    assert st["extension_rays"] == int(g["total_rays"]) - int(g["shadow_rays"])
    assert st["shadow_rays"] == default_shadow
    err = np.abs(rgb - g["ps_rgb"]) / np.maximum(1.0, np.abs(g["ps_rgb"]))
    assert err.max() <= tol, f"{int((err > tol).sum())} samples differ, worst {err.max():.3e}"


# ------------------------------------------------------------------------------------------- b. other entry points, saturated
def test_photon_emission_through_a_saturated_pool(mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "pm_hexagon_room_64.mcrtpack"))
    g = np.load(os.path.join(GOLDEN, "pm_hexagon_room_64.npz"))
    pm = mcrt.PhotonMapper(scene, global_seed=int(g["seed"]))
    try:
        with options(pm, **SATURATED):
            pm.emit(**photon_emit_args(scene))
            check_emitted_maps(mcrt, pm, scene, g)
    finally:
        pm.close()


def test_filtered_film_through_a_saturated_pool(mcrt):
    k = np.load(os.path.join(GOLDEN, "film_kat.npz"))
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "film_hexagon_room_64.mcrtpack"))
    cam = scene.cameras()[0]
    cam.film = json.loads(str(k["films"]))["mitchell"]
    pt = mcrt.PathTracer(scene, precision=mcrt.PRECISION_F64, global_seed=int(k["seed"]))
    try:
        with options(pt, **SATURATED):
            img = pt.render_rows(cam)
    finally:
        pt.close()
    ref = k["image_mitchell"]
    assert rel_rmse(img, ref) < 1e-9
    assert np.abs(img - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max())


def test_progressive_passes_through_a_saturated_pool(mcrt, golden_tracer):
    pt, scene, g, _ = golden_tracer("c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54, 4)
    with options(pt, **SATURATED):
        one = pt.render_rows(cam)
        st = pt.last_stats
        prog = mcrt.Progressive(pt, cam)
        for s in (1, 2, 13):
            prog.add(s)
        img = prog.frame()
    assert np.allclose(img, one, rtol=1e-12, atol=1e-14), np.abs(img - one).max()
    assert prog.stats["paths"] == st["paths"] and prog.stats["extension_rays"] == st["extension_rays"]


# ------------------------------------------------------------------------------------------- c. the benchmark band, saturated
def test_c2_benchmark_rows_through_a_saturated_pool(mcrt):
    """1.97 M paths through a pool of 2^18: about 8 refills, each appending new paths behind the survivors."""
    st = check_c2_benchmark_rows(mcrt, pool_paths=1 << 18)
    assert st["paths"] > 7 * (1 << 18)


# ------------------------------------------------------------------------------------------- d. buffer resizes
def test_pool_resizes_between_renders(mcrt):
    """Changing pool_paths between renders reallocates the wave and sort buffers (and the photon mapper's k-NN queue)."""
    for cid in ("c2_hexagon_room_96", "pm_hexagon_room_64"):
        scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
        g = np.load(os.path.join(GOLDEN, cid + ".npz"))
        cls = mcrt.PhotonMapper if scene.photon_maps() is not None else mcrt.PathTracer
        pt = cls(scene, precision=mcrt.PRECISION_F64, global_seed=int(g["seed"]))
        try:
            frames = []
            for pool in (1024, DEFAULTS["pool_paths"], 4096):
                pt.set_option("pool_paths", pool)
                frames.append((pt.render_rows(scene.cameras()[0]), pt.last_stats))
        finally:
            pt.close()
        first, st0 = frames[0]
        for img, st in frames[1:]:
            assert equal_frames(img, first), cid
            assert (st["extension_rays"], st["shadow_rays"], st["paths"]) == (st0["extension_rays"], st0["shadow_rays"], st0["paths"]), cid


# ------------------------------------------------------------------------------------------- e. generated scenes, auto settings
VARIANTS = [dict(dynamic_fetch=0), dict(exact_traversal=1), dict(sort_prim_key=0), dict(pool_paths=4096)]


def generated_camera(scene):
    return scene.cameras()[0].resized(96, 54, 8)     # 331 776 paths: 81 refills of a pool of 4096


def outlier_pixels(img, ref):
    d = np.abs(img - ref).max(axis=2)
    return d > 1e-9 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("name", ["mesh", "room", "quadric"])
def test_generated_scene_matches_restatement(name, mcrt):
    """Auto settings on a scene past every size threshold: dynamic fetch, whole reference leaves, primitive sort keys. The CPU
    restatement calls glibc's sincos where the device calls CUDA's, so a path trapped in a total-internal-reflection orbit can
    diverge (DESIGN.md §8, test_c2_benchmark_rows_match_reference): at most 1 pixel in 1000 may differ, and in such a pixel at most
    one sample."""
    scene = generated_scene(mcrt, name)
    g = np.load(os.path.join(GOLDEN, GENERATED[name][0] + ".npz"))
    seed = int(g["seed"])
    cam = generated_camera(scene)
    spp = cam.sqrtspp ** 2
    pt = mcrt.PathTracer(scene, precision=mcrt.PRECISION_F64, global_seed=seed)
    ps = port.PortScene(scene)
    try:
        img = pt.render_rows(cam)
        st = pt.last_stats
        ref, _ = ps.render_rows(cam, 0, cam.height, cam.sqrtspp, seed)
        out = outlier_pixels(img, ref)
        print(f"{name}: {scene.n_prims} prims, {len(mcrt.bvh4_host(scene))} BVH4 nodes, {st['replayed_rays']} replayed rays, "
              f"{int(out.sum())} outlier pixels of {out.size}")
        assert out.sum() <= out.size // 1000
        assert rel_rmse(np.where(out[..., None], ref, img), ref) < 1e-9
        for y, x in np.argwhere(out):
            pixel = np.full(spp, y * cam.width + x, np.uint32)
            sample = np.arange(spp, dtype=np.uint32)
            _, rays = ps.sample_pixels(cam, pixel, sample, seed)
            err = np.abs(pt.sampleRay(rays, pixel, sample) - ps.sample_rays(rays, pixel, sample, seed)).max(axis=1)
            assert (err > 1e-9).sum() <= 1, (y, x, int((err > 1e-9).sum()))

        # camera rays through sampleRay
        rng = np.random.default_rng(17)
        n = 8192
        pixel = rng.integers(0, cam.width * cam.height, n).astype(np.uint32)
        sample = rng.integers(0, spp, n).astype(np.uint32)
        _, rays = ps.sample_pixels(cam, pixel, sample, seed)
        rgb_ref = ps.sample_rays(rays, pixel, sample, seed)
        rgb = pt.sampleRay(rays, pixel, sample)
        bad = (np.abs(rgb - rgb_ref) / np.maximum(1.0, np.abs(rgb_ref)) > 1e-9).any(axis=1)
        print(f"{name}: {int(bad.sum())} of {n} sampleRay outliers")
        assert bad.sum() <= n // 1000

        # each size-selected path off, or the pool saturated: the same frame
        for opts in VARIANTS:
            with options(pt, **opts):
                other = pt.render_rows(cam)
                sto = pt.last_stats
            assert equal_frames(other, img), opts
            assert (sto["extension_rays"], sto["shadow_rays"]) == (st["extension_rays"], st["shadow_rays"]), opts
        assert st["replayed_rays"] > 0                       # the duplicates and shared edges reach the replay
    finally:
        ps.close()
        pt.close()


def sorted_rows(a):
    return a[np.lexsort(a.T[::-1])]


def test_generated_photon_mapped_scene(mcrt):
    """The photon pass and the photon-mapped render on a scene past the thresholds: with the auto settings (dynamic fetch), with
    dynamic fetch off and with every ray in the reference's order, the same photon maps and frames."""
    scene = generated_scene(mcrt, "pm")
    g = np.load(os.path.join(GOLDEN, "pm_hexagon_room_64.npz"))
    cam = generated_camera(scene)
    pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=int(g["seed"]))
    try:
        runs = []
        for opts in (dict(), dict(dynamic_fetch=0), dict(exact_traversal=1)):
            with options(pm, **opts):
                n = pm.emit(**photon_emit_args(scene))
                maps = [sorted_rows(pm._maps[w]["photons"].reshape(-1, 8).view(np.uint32)) for w in (0, 1)]
                img = pm.render_rows(cam)
                runs.append((n, maps, img, pm.last_stats))
        n0, maps0, img0, st0 = runs[-1]
        assert n0[0] > 0 and n0[1] > 0
        for n, maps, img, st in runs[:-1]:
            assert n == n0
            assert all(np.array_equal(m, m0) for m, m0 in zip(maps, maps0))
            assert equal_frames(img, img0)
            assert (st["extension_rays"], st["shadow_rays"]) == (st0["extension_rays"], st0["shadow_rays"])
    finally:
        pm.close()
