"""CPU tests of the order-free search's BVH4 with spatial splits (buildBvh4Split in csrc/abi.cu, option bvh4_split; mcrt_bvh4_split_host
exposes it without a CUDA call). A leaf's (first, count) index a reference array that maps each reference to its ordered primitive; a
primitive cut by a spatial split has several references, each with a box clipped to its part of the primitive.

The search over such a tree is the search of tests/test_fast_search_cpu.py over a scene whose ordered primitives are the references
(Scene.reordered(refs)): the restatement there (oracle_trace_fast, oracle_trace_visible) then runs unchanged on the split tree, and a
hit on reference r is a hit on primitive refs[r]. That restatement treats a second reference of the best primitive as a competitor and
flags the ray, where the device (FastSearch::testLeaf) recognises the repeat by its ordered id: the restated flags are a superset of the
device's, and every unflagged answer must equal the reference-order answer."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases
from oracle import port
from test_fast_search_cpu import search_rays, degenerate_ray_families

CASES = [c for c in golden_cases() if c != "ior_test_nobvh_64" and not c.startswith("pm_")]


def _scale(scene):
    return float(np.float32(np.abs(scene.a["node_bounds"][:6]).max()))


def _leaves(nodes):
    """-> list of (node, slot, first, count) of every leaf reference"""
    out = []
    for i, n in enumerate(nodes):
        for c in range(4):
            ch = int(n["child"][c])
            if ch & 0x80000000:
                out.append((i, c, (ch >> 8) & 0x7FFFFF, ch & 0xFF))
    return out


def _split_trace(ps_refs, refs, nodes, scale, rays, NO_PRIM):
    hits, flagged, box, prim = ps_refs.trace_fast(nodes, scale, rays)
    hits = hits.copy()
    hit = hits["prim"] != NO_PRIM
    hits["prim"][hit] = refs[hits["prim"][hit]]
    return hits, flagged, box, prim


@pytest.mark.parametrize("cid", CASES)
def test_tree_structure_and_coverage(cid, mcrt):
    """Children's boxes lie in their parents', every node is reached once, every primitive has a reference, and points sampled on each
    primitive (vertices, edges, interior; sphere surfaces) lie in the float box of at least one of its references' leaves."""
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    nodes, refs = mcrt.bvh4_split_host(scene)
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
        tol = 1e-13 * _scale(scene)     # the sampled points themselves are rounded (a wall's x = 0.3 x + 0.3 x + 0.4 x, off by an ulp)
        for lo, hi in boxes[p]:
            inside |= ((pts >= lo - tol) & (pts <= hi + tol)).all(1)
        assert inside.all(), (cid, p, int((~inside).sum()))


@pytest.mark.parametrize("cid", CASES)
def test_unflagged_answers_equal_reference_order(cid, mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    nodes, refs = mcrt.bvh4_split_host(scene)
    ps, pr = port.PortScene(scene), port.PortScene(scene.reordered(refs))
    try:
        rays = search_rays(mcrt, ps, g["tr_rays"], np.random.default_rng(3))
        n_generic = len(rays) - 600                     # search_rays ends with 600 axis-parallel rays
        if (scene.a["prim_type"] == 0).any():
            rays = np.concatenate([rays, degenerate_ray_families(scene, n=4000)])
        ref = ps.trace(rays)
        fast, flagged, box, prim = _split_trace(pr, refs, nodes, _scale(scene), rays, mcrt.NO_PRIM)
        final = ~flagged
        for f in ("prim", "t", "u", "v", "interpolate"):
            assert np.array_equal(fast[f][final], ref[f][final]), (f, int((fast[f][final] != ref[f][final]).sum()))
        assert flagged[:n_generic].mean() < 0.02 and final[n_generic:].sum() >= (500 if len(rays) > n_generic + 600 else 0) and box > 0 and prim > 0
    finally:
        ps.close(); pr.close()


@pytest.mark.parametrize("cid", ["c1_hexagon_diffuse_256", "c2_hexagon_room_96", "veach_mis_64", "smooth_mesh_64"])
def test_occlusion_query_equals_closest_hit_comparison(cid, mcrt):
    """Shadow rays towards points on lights: verdict 'visible' <=> the reference-order closest hit is the light with the same t."""
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    g = np.load(os.path.join(GOLDEN, cid + ".npz"))
    nodes, refs = mcrt.bvh4_split_host(scene)
    ps, pr = port.PortScene(scene), port.PortScene(scene.reordered(refs))
    try:
        rng = np.random.default_rng(21)
        base = g["tr_rays"]
        ref0 = ps.trace(base)
        ok = ref0["prim"] != mcrt.NO_PRIM
        pts = base[ok, :3] + base[ok, 3:] * ref0["t"][ok, None]
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
                lp[j] = a["sphere_origin_radius"].reshape(-1, 4)[idx][:3]
        o = pts[rng.integers(0, len(pts), n)]
        d = lp - o
        nrm = np.linalg.norm(d, axis=1, keepdims=True)
        keep = nrm[:, 0] > 1e-9
        rays = np.concatenate([o[keep], d[keep] / nrm[keep]], axis=1)
        tgt = tgt[keep]
        first_ref = np.full(scene.n_prims, -1, np.int64)
        for r in range(len(refs) - 1, -1, -1):
            first_ref[refs[r]] = r
        ref = ps.trace(rays)
        verdict, t = pr.trace_visible(nodes, _scale(scene), rays, first_ref[tgt].astype(np.uint32))
        vis, occ = verdict == 0, verdict == 1
        assert np.array_equal(ref["prim"][vis], tgt[vis]) and np.array_equal(ref["t"][vis], t[vis])
        assert (ref["prim"][occ] != tgt[occ]).all()
        assert vis.sum() > 100 and occ.sum() > 100 and (verdict == 2).mean() < 0.05
    finally:
        ps.close(); pr.close()


def test_fewer_primitive_tests_on_c2(mcrt):
    """The benchmark's scene (the hexagon room): the rebuilt tree tests fewer float64 primitives per ray than the reference's tree
    collapsed to 4-wide nodes, on camera rays and on rays between surfaces."""
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "c2_hexagon_room_96.mcrtpack"))
    g = np.load(os.path.join(GOLDEN, "c2_hexagon_room_96.npz"))
    nodes, refs = mcrt.bvh4_split_host(scene)
    ps, pr = port.PortScene(scene), port.PortScene(scene.reordered(refs))
    try:
        rays = search_rays(mcrt, ps, g["tr_rays"], np.random.default_rng(3))[:-600]
        _, _, _, prim0 = ps.trace_fast(mcrt.bvh4_host(scene), _scale(scene), rays)
        _, _, _, prim1 = _split_trace(pr, refs, nodes, _scale(scene), rays, mcrt.NO_PRIM)
        assert prim1 < 0.85 * prim0, (prim0 / len(rays), prim1 / len(rays))
    finally:
        ps.close(); pr.close()
