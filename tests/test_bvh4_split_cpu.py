"""CPU tests of the order-free search's BVH4 with spatial splits (buildBvh4Split in csrc/abi.cu, option bvh4_split; mcrt_bvh4_split_host
exposes it without a CUDA call). A leaf's (first, count) index a reference array that maps each reference to its ordered primitive; a
primitive cut by a spatial split has several references, each with a box clipped to its part of the primitive.

The restatement (port.PortScene.trace_fast / trace_visible with the tree's `refs`) runs the device's rules in the device's visiting
order: a leaf index goes through refs to the ordered primitive, a repeat of the best primitive (same t, same primitive) is not its
competitor, and the occlusion query skips every reference of its target. Every unflagged answer must equal the reference-order answer.

Besides the golden scenes, which barely split, the scenes of tests/split_scene_gen.py cut spheres and lights. On them the rays aimed at
the cut lines (where a split primitive meets the faces of its references' boxes) and at split spheres' silhouettes near the cuts test
coverage where clipped boxes meet."""
import os

import numpy as np
import pytest

import split_scene_gen as sg
from conftest import GOLDEN, golden_cases
from oracle import port
from test_fast_search_cpu import search_rays, degenerate_ray_families

GOLDEN_CASES = [c for c in golden_cases() if c != "ior_test_nobvh_64" and not c.startswith("pm_")]
CASES = GOLDEN_CASES + sg.SCENES
# flag rates of generic rays measured on the split scenes with the restated duplicate rule: 0 of 44 000 on every one (a restatement
# without the rule, over Scene.reordered(refs), flags 12-15 % of them and 31-36 % of those that hit a sphere)
MAX_FLAGGED = 0.02
# adversarial rays are aimed at triangle edges (a cut line ends on the triangle's boundary) and graze spheres: 6-9 % are flagged
MAX_FLAGGED_ADVERSARIAL = 0.15


@pytest.fixture(scope="module")
def scenes(mcrt):
    held = {}

    def get(cid):
        if cid not in held:
            if cid in sg.SCENES:
                scene = sg.split_scene(mcrt, cid)
                base = sg.camera_rays(mcrt, scene)
            else:
                scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
                base = np.load(os.path.join(GOLDEN, cid + ".npz"))["tr_rays"]
            nodes, refs = mcrt.bvh4_split_host(scene)
            held[cid] = (scene, base, nodes, refs)
        return held[cid]
    return get


def _scale(scene):
    return sg.scene_scale(scene)


def _leaves(nodes):
    """-> list of (node, slot, first, count) of every leaf reference"""
    out = []
    for i, n in enumerate(nodes):
        for c in range(4):
            ch = int(n["child"][c])
            if ch & 0x80000000:
                out.append((i, c, (ch >> 8) & 0x7FFFFF, ch & 0xFF))
    return out


def _surface_points(mcrt, ps, base):
    ref = ps.trace(base)
    ok = ref["prim"] != mcrt.NO_PRIM
    return base[ok, :3] + base[ok, 3:] * ref["t"][ok, None]


def _assert_unflagged_equal(fast, flagged, ref):
    final = ~flagged
    for f in ("prim", "t", "u", "v", "interpolate"):
        assert np.array_equal(fast[f][final], ref[f][final]), (f, int((fast[f][final] != ref[f][final]).sum()))


def _assert_occlusion(ref, verdict, t, tgt):
    """verdict 'visible' <=> the reference-order closest hit is the target with the same t; 'occluded' never hides the target"""
    vis, occ = verdict == 0, verdict == 1
    assert np.array_equal(ref["prim"][vis], tgt[vis]) and np.array_equal(ref["t"][vis], t[vis])
    assert (ref["prim"][occ] != tgt[occ]).all()


@pytest.mark.parametrize("cid", sg.SCENES + ["pm_split"])
def test_generated_scenes_split_spheres_and_lights(cid, mcrt):
    """Each generated scene really splits what it is there for (the generators assert it too): every sphere and the only light have
    several references, and no scene is past the 4096 primitives below which the upload builds this tree."""
    scene = sg.split_scene(mcrt, cid)
    st = sg.split_stats(mcrt, scene)
    print(cid, st)
    assert st["prims"] < 4096 and st["refs"] > 1.3 * st["prims"] and st["split"] > 200
    assert st["split_lights"] == 1 and st["light_refs"] >= 5
    assert st["split_spheres"] == st["spheres"] == 16


@pytest.mark.parametrize("cid", CASES)
def test_tree_structure_and_coverage(cid, mcrt, scenes):
    """Children's boxes lie in their parents', every node is reached once, every primitive has a reference, and points sampled on each
    primitive (vertices, edges, interior; sphere surfaces) lie in the float box of at least one of its references' leaves."""
    scene, _, nodes, refs = scenes(cid)
    assert len(nodes) > 0
    a = scene.a
    n_prims = scene.n_prims
    assert refs.max() < n_prims and np.array_equal(np.unique(refs), np.arange(n_prims))
    assert len(refs) <= mcrt.BVH4_SPLIT_REF_BUDGET * n_prims
    reached = np.zeros(len(nodes), int)
    reached[0] = 1
    covered = np.zeros(len(refs), int)
    for i, n in enumerate(nodes):
        for c in range(4):
            ch = int(n["child"][c])
            if ch == 0:
                continue
            if ch & 0x80000000:
                f, k = (ch >> 8) & 0x7FFFFF, ch & 0xFF
                assert k >= 1 and f + k <= len(refs)
                covered[f:f + k] += 1
                continue
            reached[ch] += 1
            kid = nodes[ch]
            used = kid["child"] != 0
            assert (kid["lo"][:, used] >= n["lo"][:, c:c + 1]).all() and (kid["hi"][:, used] <= n["hi"][:, c:c + 1]).all()
    assert (reached == 1).all() and (covered == 1).all()

    # boxes of each primitive's references
    boxes = [[] for _ in range(n_prims)]
    for i, c, f, k in _leaves(nodes):
        lo, hi = nodes[i]["lo"][:, c].astype(np.float64), nodes[i]["hi"][:, c].astype(np.float64)
        for r in range(f, f + k):
            boxes[refs[r]].append((lo, hi))
    rng = np.random.default_rng(11)
    tv = [a[k].reshape(-1, 3) for k in ("tri_v0", "tri_v1", "tri_v2")]
    sph = a["sphere_origin_radius"].reshape(-1, 4)
    # the sampled points themselves are rounded (a wall's x = 0.3 x + 0.3 x + 0.4 x, off by an ulp): a few float64 ulps of the
    # scene's largest coordinate, which is 1.0e4 on the far scene
    tol = 1e-13 * _scale(scene)
    for p in range(n_prims):
        t, idx = int(a["prim_type"][p]), int(a["prim_index"][p])
        if t == 0:
            w = rng.dirichlet((1, 1, 1), 400)
            edge = rng.uniform(0, 1, (300, 1))
            w = np.concatenate([np.eye(3), w, np.concatenate([edge, 1 - edge, 0 * edge], 1), np.concatenate([0 * edge, edge, 1 - edge], 1),
                                np.concatenate([1 - edge, 0 * edge, edge], 1)])
            pts = w[:, :1] * tv[0][idx] + w[:, 1:2] * tv[1][idx] + w[:, 2:] * tv[2][idx]
        elif t == 1:
            d = rng.normal(size=(1000, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
            d = np.concatenate([d, np.eye(3), -np.eye(3)])
            pts = sph[idx, :3] + sph[idx, 3] * d
        else:
            continue    # quadrics are never split: their single reference's box is the quadric's box
        inside = np.zeros(len(pts), bool)
        for lo, hi in boxes[p]:
            inside |= ((pts >= lo - tol) & (pts <= hi + tol)).all(1)
        assert inside.all(), (cid, p, int((~inside).sum()))


@pytest.mark.parametrize("cid", CASES)
def test_unflagged_answers_equal_reference_order(cid, mcrt, scenes):
    scene, base, nodes, refs = scenes(cid)
    ps = port.PortScene(scene)
    try:
        rays = search_rays(mcrt, ps, base, np.random.default_rng(3))
        n_generic = len(rays) - 600                     # search_rays ends with 600 axis-parallel rays
        # far_small is 0.016 wide: degenerate_ray_families' rays from 1e6 away start 6e7 room sizes off, where the float64 sphere test
        # is decided by rounding (its discriminant cancels to noise) and can hit a sphere whose box the reference's slab test misses.
        # The tree without splits answers those rays the same way: a limit of the search on any tree, not of the split tree.
        if (scene.a["prim_type"] == 0).any() and cid != "far_small":
            rays = np.concatenate([rays, degenerate_ray_families(scene, n=4000)])
        ref = ps.trace(rays)
        fast, flagged, box, prim = ps.trace_fast(nodes, _scale(scene), rays, refs)
        _assert_unflagged_equal(fast, flagged, ref)
        print(f"{cid}: {int(flagged[:n_generic].sum())} of {n_generic} generic rays flagged")
        assert flagged[:n_generic].mean() < MAX_FLAGGED and flagged[n_generic:n_generic + 600].all()
        assert (~flagged[n_generic:]).sum() >= (500 if len(rays) > n_generic + 600 else 0) and box > 0 and prim > 0
        assert not flagged[:n_generic][ref["prim"][:n_generic] == mcrt.NO_PRIM].any()      # a generic miss is never ambiguous
    finally:
        ps.close()


@pytest.mark.parametrize("cid", sg.SCENES)
def test_rays_at_cut_lines_and_silhouettes(cid, mcrt, scenes):
    """Rays aimed where split primitives meet the faces of their references' boxes (split_scene_gen.adversarial_rays): from surfaces,
    along the cut planes at grazing angles, and tangent to split spheres at their cuts. Every unflagged answer is the reference-order
    answer bit for bit; occlusion queries towards the aimed-at primitive keep the invariant of the closest-hit comparison."""
    scene, base, nodes, refs = scenes(cid)
    ps = port.PortScene(scene)
    try:
        surface = _surface_points(mcrt, ps, base)
        rays, aim = sg.adversarial_rays(mcrt, scene, nodes, refs, surface, np.random.default_rng(9))
        ref = ps.trace(rays)
        fast, flagged, _, _ = ps.trace_fast(nodes, _scale(scene), rays, refs)
        _assert_unflagged_equal(fast, flagged, ref)
        hit_aim = ref["prim"] == aim
        print(f"{cid}: {len(rays)} rays, {int(hit_aim.sum())} hit the primitive aimed at, {flagged.mean():.4f} flagged")
        assert hit_aim.sum() > 2000 and (hit_aim & ~flagged).sum() > 1500
        assert flagged.mean() < MAX_FLAGGED_ADVERSARIAL
        sphere = scene.a["prim_type"][aim] == mcrt.PRIM_SPHERE
        assert (hit_aim & sphere & ~flagged).sum() > 200
        for fn in (ps.trace_visible, lambda *a: ps.trace_visible_peaks(*a)[:2]):
            verdict, t = fn(nodes, _scale(scene), rays, aim.astype(np.uint32), refs)
            _assert_occlusion(ref, verdict, t, aim)
            assert (verdict == 0).sum() > 1000 and (verdict == 1).sum() > 1000
    finally:
        ps.close()


@pytest.mark.parametrize("cid", ["c1_hexagon_diffuse_256", "c2_hexagon_room_96", "veach_mis_64", "smooth_mesh_64"] + sg.SCENES)
def test_occlusion_query_equals_closest_hit_comparison(cid, mcrt, scenes):
    """Shadow rays towards points on lights: verdict 'visible' <=> the reference-order closest hit is the light with the same t, in
    the restatement's order-free walk and in the device's visiting order. On the generated scenes the light has several references."""
    scene, base, nodes, refs = scenes(cid)
    ps = port.PortScene(scene)
    try:
        rng = np.random.default_rng(21)
        pts = _surface_points(mcrt, ps, base)
        a = scene.a
        lights = a["light_prim"]
        n = 20000
        tgt = lights[rng.integers(0, len(lights), n)].astype(np.uint32)
        lp = np.zeros((n, 3))
        for j in range(n):
            t, idx = int(a["prim_type"][tgt[j]]), int(a["prim_index"][tgt[j]])
            if t == 0:
                u, v = rng.uniform(0, 1, 2); su = np.sqrt(u)
                lp[j] = (1 - su) * a["tri_v0"].reshape(-1, 3)[idx] + (1 - v) * su * a["tri_v1"].reshape(-1, 3)[idx] + v * su * a["tri_v2"].reshape(-1, 3)[idx]
            else:
                sp = a["sphere_origin_radius"].reshape(-1, 4)[idx]
                d = rng.normal(size=3)
                lp[j] = sp[:3] + sp[3] * d / np.linalg.norm(d)
        o = pts[rng.integers(0, len(pts), n)]
        d = lp - o
        nrm = np.linalg.norm(d, axis=1, keepdims=True)
        keep = nrm[:, 0] > 1e-9
        rays = np.concatenate([o[keep], d[keep] / nrm[keep]], axis=1)
        tgt = tgt[keep]
        ref = ps.trace(rays)
        verdict, t = ps.trace_visible(nodes, _scale(scene), rays, tgt, refs)
        _assert_occlusion(ref, verdict, t, tgt)
        verdict2, t2, _ = ps.trace_visible_peaks(nodes, _scale(scene), rays, tgt, refs)
        _assert_occlusion(ref, verdict2, t2, tgt)
        print(f"{cid}: {int((verdict == 2).sum())} of {len(rays)} occlusion queries replayed")
        assert (verdict == 0).sum() > 100 and (verdict == 1).sum() > 100 and (verdict == 2).mean() < 0.05
    finally:
        ps.close()


@pytest.mark.parametrize("cid", ["clutter", "sphere_light"])
def test_render_cross_checked_over_split_tree(cid, mcrt, scenes):
    """A whole render by the restatement with every Scene::intersect call (camera, bounce and shadow rays; the shadow rays aim at the
    split light) also answered by the search over the split tree: no unflagged answer differs."""
    scene, _, nodes, refs = scenes(cid)
    cam = scene.cameras()[0].resized(48, 27, 2)
    ps = port.PortScene(scene)
    try:
        img, calls, flagged, mismatches = ps.render_rows_checked(nodes, _scale(scene), cam, 0, cam.height, cam.sqrtspp, 0x2468ACE, refs)
        ref, _ = ps.render_rows(cam, 0, cam.height, cam.sqrtspp, 0x2468ACE)
    finally:
        ps.close()
    print(f"{cid}: {calls} intersect calls, {flagged} flagged, {mismatches} mismatches")
    assert mismatches == 0 and calls > 10000 and flagged < 0.01 * calls
    assert np.array_equal(img, ref) and img.max() > 0


def test_fewer_primitive_tests_on_c2(mcrt, scenes):
    """The benchmark's scene (the hexagon room): the rebuilt tree tests fewer float64 primitives per ray than the reference's tree
    collapsed to 4-wide nodes, on camera rays and on rays between surfaces."""
    scene, base, nodes, refs = scenes("c2_hexagon_room_96")
    ps = port.PortScene(scene)
    try:
        rays = search_rays(mcrt, ps, base, np.random.default_rng(3))[:-600]
        _, _, _, prim0 = ps.trace_fast(mcrt.bvh4_host(scene), _scale(scene), rays)
        _, _, _, prim1 = ps.trace_fast(nodes, _scale(scene), rays, refs)
        assert prim1 < 0.85 * prim0, (prim0 / len(rays), prim1 / len(rays))
    finally:
        ps.close()
