"""CPU test of the algorithm behind the product's parity-mode closest hit (csrc/bvh4.cuh): an order-free search over a 4-wide
float-box BVH whose answer is FINAL unless it flags the ray as ambiguous (two candidates within delta), in which case the product
replays the ray in the reference's visiting order. oracle_trace_fast restates the search on the CPU - same float32 slab arithmetic,
margins and pruning limit, over the very nodes the product builds (mcrt_bvh4_host) - and oracle_trace is the reference-order
traversal pinned to the reference's golden hits (tests/test_oracle_cpu.py). The claim under test: every answer the search does not
flag equals the reference-order answer bit for bit, flags are rare, and misses agree."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases
from oracle import port

CASES = [c for c in golden_cases() if c != "ior_test_nobvh_64" and not c.startswith("pm_")]


def search_rays(mcrt, ps, base, rng, n=20000):
    """base rays, segments from surface to surface, rays leaving surfaces and axis-parallel rays (the last 600)."""
    ref0 = ps.trace(base)
    ok = ref0["prim"] != mcrt.NO_PRIM
    pts = base[ok, :3] + base[ok, 3:] * ref0["t"][ok, None]
    a = pts[rng.integers(0, len(pts), n)]
    b = pts[rng.integers(0, len(pts), n)] + rng.normal(0, 1e-3, (n, 3))
    d = b - a
    nrm = np.linalg.norm(d, axis=1, keepdims=True)
    keep = nrm[:, 0] > 1e-9
    seg = np.concatenate([a[keep], d[keep] / nrm[keep]], axis=1)              # start exactly on surfaces, aim at surfaces
    d2 = rng.normal(size=(n, 3)); d2 /= np.linalg.norm(d2, axis=1, keepdims=True)
    leave = np.concatenate([a + 1e-9 * d2, d2], axis=1)                        # leave surfaces in random directions
    axis = np.zeros((600, 6)); axis[:, :3] = pts[rng.integers(0, len(pts), 600)] + rng.normal(0, 0.3, (600, 3))
    axis[np.arange(600), 3 + np.arange(600) % 3] = np.where(np.arange(600) % 2, 1.0, -1.0)   # axis-parallel rays: 1/d = inf in the reference
    return np.concatenate([base, seg, leave, axis], axis=0)


def check_unflagged_answers(mcrt, ps, nodes, rays, max_flagged=0.02):
    """Every answer of the order-free search that is not flagged equals the reference-order answer; rays with a zero direction
    component (the last 600 of search_rays) are always flagged, other flags are rare and never on a miss. -> (reference hits, flags)"""
    scene = ps.scene
    scale = float(np.float32(np.abs(scene.a["node_bounds"][:6]).max()))      # ctx->scene_scale (float) as mcrt_scene_upload computes it
    ref = ps.trace(rays)
    fast, flagged, box, prim = ps.trace_fast(nodes, scale, rays)
    final = ~flagged
    for f in ("prim", "t", "u", "v", "interpolate"):
        assert np.array_equal(fast[f][final], ref[f][final]), (f, int((fast[f][final] != ref[f][final]).sum()))
    generic = np.ones(len(rays), dtype=bool); generic[-600:] = False          # rays with a zero direction component always go to the replay
    assert flagged[~generic].all()
    assert flagged[generic].mean() < max_flagged, flagged[generic].mean()
    assert not flagged[generic & (ref["prim"] == mcrt.NO_PRIM)].any()          # a generic miss is never ambiguous
    assert box > 0 and prim > 0
    return ref, flagged


@pytest.mark.parametrize("max_leaf", [0xFFFFFFFF, 0])
@pytest.mark.parametrize("cid", CASES)
def test_unflagged_answers_equal_reference_order(cid, max_leaf, mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    ps = port.PortScene(scene)
    try:
        rays = search_rays(mcrt, ps, g["tr_rays"], np.random.default_rng(3))
        check_unflagged_answers(mcrt, ps, mcrt.bvh4_host(scene, max_leaf), rays)
    finally:
        ps.close()


def test_coincident_geometry_is_flagged(mcrt):
    """Two copies of the same triangle: equal t, the winner depends on the visiting order - the search must hand such rays to the replay."""
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "c2_hexagon_room_96.mcrtpack"))
    a = dict(scene.a); a.update(scene.extra); a["scene_ior"] = scene.ior
    tri = int(np.nonzero(a["prim_type"] == 0)[0][0])           # an ordered primitive that is a triangle
    idx = int(a["prim_index"][tri])
    # overwrite another triangle's geometry with this one's (same node layout, boxes of the tree still contain... only if equal): use the
    # neighbour in the same leaf when there is one, else skip
    leaf = next((i for i in range(len(a["node_first_prim"])) if a["node_prim_count"][i] >= 2 and
                 all(a["prim_type"][a["node_first_prim"][i] + k] == 0 for k in range(2))), None)
    if leaf is None:
        pytest.skip("no leaf with two triangles in the fixture")
    p0, p1 = int(a["node_first_prim"][leaf]), int(a["node_first_prim"][leaf]) + 1
    i0, i1 = int(a["prim_index"][p0]), int(a["prim_index"][p1])
    for k in ("tri_v0", "tri_v1", "tri_v2", "tri_e1", "tri_e2", "tri_normal"):
        arr = a[k].reshape(-1, 3).copy(); arr[i1] = arr[i0]; a[k] = arr.reshape(-1)
    dup = mcrt.Scene(a)
    ps = port.PortScene(dup)
    try:
        nodes = mcrt.bvh4_host(dup, 0)
        v0 = dup.a["tri_v0"].reshape(-1, 3)[i0]; e1 = dup.a["tri_e1"].reshape(-1, 3)[i0]; e2 = dup.a["tri_e2"].reshape(-1, 3)[i0]
        target = v0 + 0.3 * e1 + 0.3 * e2
        nrm = np.cross(e1, e2); nrm /= np.linalg.norm(nrm)
        rays = np.array([np.concatenate([target + 0.5 * nrm, -nrm]), np.concatenate([target - 0.5 * nrm, nrm])])
        ref = ps.trace(rays)
        fast, flagged, _, _ = ps.trace_fast(nodes, float(np.float32(np.abs(dup.a["node_bounds"][:6]).max())), rays)
        hit_dup = np.isin(ref["prim"], (p0, p1))
        assert hit_dup.any()
        assert flagged[hit_dup].all()            # ties go to the replay, whichever copy the search saw first
    finally:
        ps.close()


@pytest.mark.parametrize("cid", ["v3_spaceship", "v5_lego_bulldozer"])
def test_big_scene_unflagged_answers_equal_reference_order(cid, mcrt):
    """The same claim on the 457 k-triangle spaceship and the 2 M-triangle bulldozer (coincident faces in the model: ~1 % of rays that
    start on its surfaces are flagged)."""
    from conftest import ROOT
    pack = os.path.join(ROOT, "bench_data", cid + ".mcrtpack.xz")
    if not os.path.exists(pack):
        pytest.skip(f"{pack} not present (git-ignored, regenerable: tools/validate_big.py make)")
    scene = mcrt.Scene.from_pack(pack)
    g = np.load(os.path.join(GOLDEN, "big", cid + ".npz"))
    ps = port.PortScene(scene)
    try:
        nodes = mcrt.bvh4_host(scene)
        scale = float(np.float32(np.abs(scene.a["node_bounds"][:6]).max()))
        rng = np.random.default_rng(8)
        base = g["tr_rays"]
        ref0 = ps.trace(base)
        assert np.array_equal(ref0["prim"], g["tr_prim"])            # the reference-order restatement against the reference itself
        ok = ref0["prim"] != mcrt.NO_PRIM
        pts = base[ok, :3] + base[ok, 3:] * ref0["t"][ok, None]
        n = 60000
        a = pts[rng.integers(0, len(pts), n)]
        d2 = rng.normal(size=(n, 3)); d2 /= np.linalg.norm(d2, axis=1, keepdims=True)
        rays = np.concatenate([base, np.concatenate([a + 1e-9 * d2, d2], axis=1)], axis=0)
        ref = ps.trace(rays)
        fast, flagged, _, _ = ps.trace_fast(nodes, scale, rays)
        final = ~flagged
        for f in ("prim", "t", "u", "v"):
            assert np.array_equal(fast[f][final], ref[f][final]), f
        assert flagged.mean() < 0.03
    finally:
        ps.close()


@pytest.mark.parametrize("cid", ["c1_hexagon_diffuse_256", "c2_hexagon_room_96", "veach_mis_64", "smooth_mesh_64"])
def test_occlusion_query_equals_closest_hit_comparison(cid, mcrt):
    """Shadow rays (integrator.cpp:68-86: visible iff the closest hit is that very light primitive): the product tests the light
    directly and searches only for something in front of it. Restated on the CPU: verdict 'visible' <=> the reference-order closest
    hit is the light, with the same t; 'not visible' <=> it is something else; ties are handed to the replay."""
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    ps = port.PortScene(scene)
    try:
        check_occlusion_query(mcrt, ps, mcrt.bvh4_host(scene), g["tr_rays"], np.random.default_rng(21))
    finally:
        ps.close()


def check_occlusion_query(mcrt, ps, nodes, base, rng, n=30000):
    """Rays from surface points (where `base` rays hit) to points on random lights: the occlusion query's verdict against the
    reference-order closest hit. -> verdicts"""
    scene = ps.scene
    scale = float(np.float32(np.abs(scene.a["node_bounds"][:6]).max()))
    ref0 = ps.trace(base)
    ok = ref0["prim"] != mcrt.NO_PRIM
    pts = base[ok, :3] + base[ok, 3:] * ref0["t"][ok, None]
    lights = scene.a["light_prim"]
    assert len(lights) > 0
    tgt = lights[rng.integers(0, len(lights), n)].astype(np.uint32)
    # a point on each target light: triangle lights by barycentric sampling, sphere lights through their centre
    a = scene.a
    lp = np.zeros((n, 3))
    for j in range(n):
        t, idx = int(a["prim_type"][tgt[j]]), int(a["prim_index"][tgt[j]])
        if t == 0:
            u, v = rng.uniform(0, 1, 2); su = np.sqrt(u)
            lp[j] = ((1 - su) * a["tri_v0"].reshape(-1, 3)[idx] + (1 - v) * su * a["tri_v1"].reshape(-1, 3)[idx] + v * su * a["tri_v2"].reshape(-1, 3)[idx])
        else:
            lp[j] = a["sphere_origin_radius"].reshape(-1, 4)[idx][:3]
    o = pts[rng.integers(0, len(pts), n)]
    d = lp - o
    nrm = np.linalg.norm(d, axis=1, keepdims=True)
    keep = nrm[:, 0] > 1e-9
    rays = np.concatenate([o[keep], d[keep] / nrm[keep]], axis=1)
    tgt = tgt[keep]
    ref = ps.trace(rays)
    verdict, t = ps.trace_visible(nodes, scale, rays, tgt)
    vis, occ = verdict == 0, verdict == 1
    assert np.array_equal(ref["prim"][vis], tgt[vis]) and np.array_equal(ref["t"][vis], t[vis])
    assert (ref["prim"][occ] != tgt[occ]).all()
    assert vis.sum() > 100 and occ.sum() > 100 and (verdict == 2).mean() < 0.02
    return verdict


def _unit(v):
    n = np.linalg.norm(v, axis=1, keepdims=True)
    return v / np.where(n > 0, n, 1)


def degenerate_ray_families(scene, n=20000, seed=5):
    """Seven families of rays that run exactly along planes, through vertices and along edges of the scene's triangles."""
    a = scene.a
    rng = np.random.default_rng(seed)
    tri = np.nonzero(a["prim_type"] == 0)[0]
    idx = a["prim_index"][tri]
    v0, v1, v2 = (a[k].reshape(-1, 3)[idx] for k in ("tri_v0", "tri_v1", "tri_v2"))
    nrm = _unit(np.cross(v1 - v0, v2 - v0))
    nt = len(tri)
    vs = np.stack([v0, v1, v2], 1)
    fam = []
    i, j = rng.integers(0, nt, n), rng.integers(0, nt, n)
    o, t = vs[i, rng.integers(0, 3, n)], vs[j, rng.integers(0, 3, n)]
    ok = np.linalg.norm(t - o, axis=1) > 1e-9
    fam.append(np.concatenate([o[ok], _unit((t - o)[ok])], 1))                                            # vertex to vertex
    i = rng.integers(0, nt, n); u = rng.uniform(0, 1, (n, 2)); su = np.sqrt(u[:, :1])
    p = (1 - su) * v0[i] + (1 - u[:, 1:]) * su * v1[i] + u[:, 1:] * su * v2[i]
    e = _unit(v1[i] - v0[i]); f = np.cross(nrm[i], e); ang = rng.uniform(0, 2 * np.pi, (n, 1))
    fam.append(np.concatenate([p, _unit(np.cos(ang) * e + np.sin(ang) * f)], 1))                           # inside a triangle's plane
    fam.append(np.concatenate([p + 1e-9 * nrm[i], -nrm[i]], 1))                                           # straight back into the surface
    d = nrm[i].copy(); d[:, 0] += 1e-20
    fam.append(np.concatenate([p + 1e-9 * nrm[i], _unit(d)], 1))                                          # denormal-size direction component
    far = _unit(rng.normal(size=(n, 3))) * 1e6; t = vs[rng.integers(0, nt, n), rng.integers(0, 3, n)]
    fam.append(np.concatenate([far, _unit(t - far)], 1))                                                   # from 1e6 away at vertices
    m_ = 3 * (n // 10)
    o = vs[rng.integers(0, nt, m_), rng.integers(0, 3, m_)].copy(); d = np.zeros((m_, 3))
    d[np.arange(m_), np.arange(m_) % 3] = np.where(np.arange(m_) % 2, 1.0, -1.0)
    fam.append(np.concatenate([o, d], 1))                                                                  # axis-parallel from vertex coordinates
    fam.append(np.concatenate([v0[i] + 1e-12 * nrm[i] - 3 * _unit(v1[i] - v0[i]), _unit(v1[i] - v0[i])], 1))   # grazing along an edge
    rays = np.concatenate(fam, 0)
    return rays[np.isfinite(rays).all(1)]


@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "c1_hexagon_diffuse_256", "smooth_mesh_64", "veach_mis_64", "hexagon_room_octree_64"])
def test_degenerate_rays_are_flagged_not_answered_differently(cid, mcrt):
    """Rays built to run exactly along box planes, through vertices and along edges, where the reference's float64 slab test decides by
    rounding (or by NaN: 0 * inf for a zero direction component) whether a box - and with it a primitive the ray does touch - is reached at
    all. The search's conservative boxes never miss such a primitive, so there its answer CAN differ from the reference's; it therefore
    hands these rays to the replay: a direction component of (nearly) zero, or a winner hit within 1e-9 (scaled with distance) of its
    triangle's boundary. Seven adversarial families, 250 k rays per scene: no unflagged answer may differ."""
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    a = scene.a
    ps = port.PortScene(scene)
    try:
        rays = degenerate_ray_families(scene)
        ref = ps.trace(rays)
        scale = float(np.float32(np.abs(a["node_bounds"][:6]).max()))
        for max_leaf in (0xFFFFFFFF, 0):
            fast, flagged, _, _ = ps.trace_fast(mcrt.bvh4_host(scene, max_leaf), scale, rays)
            final = ~flagged
            for f_ in ("prim", "t", "u", "v"):
                assert np.array_equal(fast[f_][final], ref[f_][final]), (cid, max_leaf, f_, int((fast[f_][final] != ref[f_][final]).sum()))
            assert final.sum() > 10000          # the generic members of the families are still answered by the search
    finally:
        ps.close()


@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "quadric_64", "metals_64"])
def test_curved_primitives_and_near_degenerate_directions(cid, mcrt):
    """Sphere tangents (impact parameter r (1 +- 0, 1e-12, 1e-7)), rays through / from sphere centres and surfaces, rays from exact hit
    points with zero offset, direction components of 2e-12 .. 1e-9 (just above the replay rule), near-tangent leaving rays: every answer the
    search does not flag equals the reference-order answer."""
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    a = scene.a
    ps = port.PortScene(scene)
    try:
        rng = np.random.default_rng(9)
        n = 6000
        base = g["tr_rays"]
        ref0 = ps.trace(base)
        ok = ref0["prim"] != mcrt.NO_PRIM
        pts = base[ok, :3] + base[ok, 3:] * ref0["t"][ok, None]
        fam = []
        sph = a["sphere_origin_radius"].reshape(-1, 4)
        if len(sph):
            i = rng.integers(0, len(sph), n); c, r = sph[i, :3], sph[i, 3:4]
            dirn = _unit(rng.normal(size=(n, 3)))
            perp = _unit(np.cross(dirn, rng.normal(size=(n, 3))))
            for eps in (0.0, 1e-12, -1e-12, 1e-7, -1e-7):
                fam.append(np.concatenate([c + perp * r * (1 + eps) - dirn * 5.0, dirn], 1))
            fam.append(np.concatenate([c - dirn * 3.0, dirn], 1))
            fam.append(np.concatenate([c + dirn * r, _unit(rng.normal(size=(n, 3)))], 1))
            fam.append(np.concatenate([c, dirn], 1))
        d = _unit(rng.normal(size=(n, 3))); k = rng.integers(0, 3, n)
        d[np.arange(n), k] = rng.choice([1e-9, 2e-12, 1e-11, -3e-12, 1e-10], n)
        fam.append(np.concatenate([pts[rng.integers(0, len(pts), n)] + rng.normal(0, 1e-3, (n, 3)), _unit(d)], 1))
        fam.append(np.concatenate([pts[rng.integers(0, len(pts), n)], _unit(rng.normal(size=(n, 3)))], 1))
        rays = np.concatenate(fam, 0)
        ref = ps.trace(rays)
        scale = float(np.float32(np.abs(a["node_bounds"][:6]).max()))
        fast, flagged, _, _ = ps.trace_fast(mcrt.bvh4_host(scene), scale, rays)
        final = ~flagged
        for f_ in ("prim", "t", "u", "v"):
            assert np.array_equal(fast[f_][final], ref[f_][final]), (cid, f_)
        assert final.mean() > 0.9
    finally:
        ps.close()


@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "smooth_mesh_64", "veach_mis_64", "quadric_64"])
def test_every_intersect_call_of_a_render_agrees(cid, mcrt):
    """A whole render by the restated path tracer with EVERY Scene::intersect call - camera, bounce and shadow rays, the rays a renderer
    actually generates - also answered by the restated search: no unflagged answer differs, flags are a handful, and the image is the
    reference's."""
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    cam = scene.cameras()[0]
    ps = port.PortScene(scene)
    try:
        scale = float(np.float32(np.abs(scene.a["node_bounds"][:6]).max()))
        img, calls, flagged, mismatches = ps.render_rows_checked(mcrt.bvh4_host(scene), scale, cam, 0, cam.height, cam.sqrtspp, int(g["seed"]))
        assert calls == int(g["total_rays"]) and mismatches == 0 and flagged <= calls // 1000
        assert np.array_equal(img, g["image"])
    finally:
        ps.close()
