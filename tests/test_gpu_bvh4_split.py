"""The order-free search over the BVH4 with spatial splits (option bvh4_split, on by default below 4096 primitives) against the same
search over the tree without them and against the reference-order replay: bit-equal closest hits, the same paths, equal frames.

On the scenes of tests/split_scene_gen.py, which split spheres and lights, the device's replay count is pinned to the restatement's flag
count (port.PortScene.trace_fast with the tree's refs): that holds only if the device walks the split tree and applies the restated
duplicate rule, whereas final answers alone would not notice a rule that flags too much."""
import os

import numpy as np
import pytest

import split_scene_gen as sg
from conftest import GOLDEN, golden_cases
from oracle import port
from test_gpu_materials import OUTLIERS, has_glass
from test_gpu_parity import photon_emit_args
from test_gpu_schedules import equal_frames, outlier_pixels, rel_rmse, sorted_rows

pytestmark = pytest.mark.gpu

CASES = [c for c in golden_cases() if c != "ior_test_nobvh_64"]
HIT_FIELDS = ("prim", "t", "u", "v", "interpolate")


def _rays(mcrt, pt, base, rng, n=100_000):
    h = pt.intersect(base)
    ok = h["prim"] != mcrt.NO_PRIM
    pts = base[ok, :3] + base[ok, 3:] * h["t"][ok, None]
    a = pts[rng.integers(0, len(pts), n)]
    d = pts[rng.integers(0, len(pts), n)] + rng.normal(0, 1e-3, (n, 3)) - a
    nrm = np.linalg.norm(d, axis=1, keepdims=True)
    keep = nrm[:, 0] > 1e-9
    d2 = rng.normal(size=(n, 3)); d2 /= np.linalg.norm(d2, axis=1, keepdims=True)
    return np.concatenate([base, np.concatenate([a[keep], d[keep] / nrm[keep]], 1), np.concatenate([a + 1e-9 * d2, d2], 1)])


@pytest.mark.parametrize("cid", CASES)
def test_intersect_split_equals_unsplit_and_reference_order(cid, mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    pt = mcrt.PathTracer(scene, device=0, precision=mcrt.PRECISION_F64, global_seed=int(g["seed"]))
    try:
        rays = _rays(mcrt, pt, g["tr_rays"], np.random.default_rng(17))
        split = pt.intersect(rays)
        pt.set_option("exact_traversal", 1)
        exact = pt.intersect(rays)
        pt.set_option("exact_traversal", 0)
        pt.set_option("bvh4_split", 0)
        pt.upload_scene()
        unsplit = pt.intersect(rays)
        for f in HIT_FIELDS:
            assert np.array_equal(split[f], unsplit[f]), f
            assert np.array_equal(split[f], exact[f]), f
    finally:
        pt.close()


@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "c1_hexagon_diffuse_256", "veach_mis_64", "smooth_mesh_64", "quadric_64"])
def test_render_split_equals_unsplit(cid, mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    cam = scene.cameras()[0]
    out = []
    for split in (1, 0):
        pt = mcrt.PathTracer(scene, device=0, precision=mcrt.PRECISION_F64, global_seed=int(g["seed"]))
        try:
            pt.set_option("bvh4_split", split)
            pt.upload_scene()
            img = pt.render_rows(cam)
            out.append((img, pt.last_stats))
        finally:
            pt.close()
    (a, sa), (b, sb) = out
    assert (sa["extension_rays"], sa["shadow_rays"]) == (sb["extension_rays"], sb["shadow_rays"])
    assert np.allclose(a, b, rtol=1e-12, atol=0.0)


# ------------------------------------------------------------------------------------------- scenes that split spheres and lights
SEED = 0x2468ACE


@pytest.fixture(scope="module")
def held(mcrt):
    """per generated scene: (tracer, scene, nodes, refs, search rays + adversarial rays, restated flags, reference-order hits)"""
    cache = {}

    def get(cid):
        if cid not in cache:
            scene = sg.split_scene(mcrt, cid)
            nodes, refs = mcrt.bvh4_split_host(scene)
            ps = port.PortScene(scene)
            try:
                base = sg.camera_rays(mcrt, scene)
                ref0 = ps.trace(base)
                ok = ref0["prim"] != mcrt.NO_PRIM
                surface = base[ok, :3] + base[ok, 3:] * ref0["t"][ok, None]
                rng = np.random.default_rng(23)
                a = surface[rng.integers(0, len(surface), 30000)]
                b = surface[rng.integers(0, len(surface), 30000)] - a
                keep = np.linalg.norm(b, axis=1) > 1e-9 * sg.scene_scale(scene)
                seg = np.concatenate([a[keep], b[keep] / np.linalg.norm(b[keep], axis=1, keepdims=True)], 1)
                adv, _ = sg.adversarial_rays(mcrt, scene, nodes, refs, surface, np.random.default_rng(9))
                rays = np.concatenate([base, seg, adv])
                ref = ps.trace(rays)
                _, flagged, _, _ = ps.trace_fast(nodes, sg.scene_scale(scene), rays, refs)
            finally:
                ps.close()
            pt = mcrt.PathTracer(scene, device=0, precision=mcrt.PRECISION_F64, global_seed=SEED)
            cache[cid] = (pt, scene, rays, flagged, ref)
        return cache[cid]
    yield get
    for v in cache.values():
        v[0].close()


@pytest.mark.parametrize("cid", sg.SCENES)
def test_intersect_on_split_scenes_replays_the_restated_flags(cid, mcrt, held):
    """Camera rays, rays between surfaces and rays at the cut lines and silhouettes: the split tree's answers are bit-equal to the
    reference's order (exact_traversal=1), to the tree without splits and to the restatement, and the device replays exactly the
    rays the restated search flags."""
    pt, scene, rays, flagged, ref = held(cid)
    try:
        split = pt.intersect(rays)
        replayed = pt.last_stats["replayed_rays"]
        pt.set_option("exact_traversal", 1)
        exact = pt.intersect(rays)
        pt.set_option("exact_traversal", 0)
        pt.set_option("bvh4_split", 0)
        pt.upload_scene()
        unsplit = pt.intersect(rays)
    finally:
        pt.set_option("exact_traversal", 0)
        pt.set_option("bvh4_split", -1)
        pt.upload_scene()
    print(f"{cid}: {len(rays)} rays, {replayed} replayed, {int(flagged.sum())} flagged by the restatement")
    for f in HIT_FIELDS:
        assert np.array_equal(split[f], exact[f]), f
        assert np.array_equal(split[f], unsplit[f]), f
        assert np.array_equal(split[f], ref[f]), f
    assert replayed == int(flagged.sum()) and replayed > 0


RENDER_SCENES = ["clutter", "sphere_light", "far"]


@pytest.mark.parametrize("cid", RENDER_SCENES)
def test_render_on_split_scenes(cid, mcrt, held):
    """Split, unsplit and exact frames agree to 1e-12 with the same ray counts, under dynamic fetch either way and a pool of 1024
    paths; the frame matches the restatement's (test_gpu_schedules' outlier rule); sampleRay on the adversarial rays matches
    the restatement's sample by sample."""
    pt, scene, rays, _, _ = held(cid)
    cam = scene.cameras()[0].resized(96, 54, 4)
    frames = []
    try:
        for opts in (dict(), dict(dynamic_fetch=0), dict(dynamic_fetch=1), dict(pool_paths=1024), dict(bvh4_split=0),
                     dict(bvh4_split=0, dynamic_fetch=1), dict(exact_traversal=1)):
            for k, v in opts.items():
                pt.set_option(k, v)
            if "bvh4_split" in opts:
                pt.upload_scene()
            frames.append((opts, pt.render_rows(cam), pt.last_stats))
            for k in opts:
                pt.set_option(k, dict(bvh4_split=-1, dynamic_fetch=-1, pool_paths=1 << 23, exact_traversal=0)[k])
            if "bvh4_split" in opts:
                pt.upload_scene()
    finally:
        pt.set_option("bvh4_split", -1)
    _, img, st = frames[0]
    assert st["shadow_rays"] > 0 and img.max() > 0
    # the restated render over the split tree flags none of its 35 000-39 000 intersect calls (test_bvh4_split_cpu): a duplicate rule
    # that mistakes a second reference of the best hit or of a shadow ray's target for a competitor replays most rays instead
    assert st["replayed_rays"] <= 0.01 * (st["extension_rays"] + st["shadow_rays"]), st["replayed_rays"]
    for opts, other, sto in frames[1:]:
        assert equal_frames(other, img), opts
        assert (sto["extension_rays"], sto["shadow_rays"]) == (st["extension_rays"], st["shadow_rays"]), opts

    ps = port.PortScene(scene)
    try:
        ref, _ = ps.render_rows(cam, 0, cam.height, cam.sqrtspp, SEED)
        out = outlier_pixels(img, ref)
        print(f"{cid}: {st['replayed_rays']} replayed rays, {int(out.sum())} outlier pixels of {out.size}")
        assert out.sum() <= out.size // 1000
        assert rel_rmse(np.where(out[..., None], ref, img), ref) < 1e-9
        n = 8192
        sel = rays[-n:]
        pixel = np.arange(n, dtype=np.uint32); sample = np.zeros(n, np.uint32)
        got = pt.sampleRay(sel, pixel, sample)
        want = ps.sample_rays(sel, pixel, sample, SEED)
    finally:
        ps.close()
    err = (np.abs(got - want) / np.maximum(1.0, np.abs(want))).max(axis=1)
    allowed = int(OUTLIERS * n) if has_glass(scene) else 0
    assert (err > 1e-9).sum() <= allowed, (int((err > 1e-9).sum()), float(err.max()))


def test_photon_emission_from_a_split_light(mcrt):
    """pm_hexagon_room_64 with the clutter and a long thin light cut into several references: the photon maps emitted over the split
    tree and over the tree without splits are equal as sorted rows, and so are the ray counts."""
    scene = sg.split_scene(mcrt, "pm_split")
    pm = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64, global_seed=SEED)
    try:
        runs = []
        for split in (1, 0):
            pm.set_option("bvh4_split", split)
            pm.upload_scene()
            n = pm.emit(**photon_emit_args(scene))
            runs.append((n, [sorted_rows(pm._maps[w]["photons"].reshape(-1, 8).view(np.uint32)) for w in (0, 1)]))
    finally:
        pm.close()
    (n1, maps1), (n0, maps0) = runs
    assert n1 == n0 and n0[0] + n0[1] > 0
    assert all(np.array_equal(a, b) for a, b in zip(maps1, maps0))
