"""Scenes on which the order-free search's BVH4 with spatial splits (buildBvh4Split, csrc/abi.cu) really cuts primitives: spheres and
lights included, so that the duplicate rule of FastSearch::testLeaf (a repeat of the best primitive is not its competitor, the occlusion
query skips every reference of its target) and the clipped boxes' coverage are both on the path of the tested rays. The golden scenes
barely split (no sphere and no light ever has a second reference). Seeded, below 4096 primitives (the upload's auto rule then builds
this tree), and assembled like tests/deep_scene_gen.py's scenes: the reference's tree is rebuilt by the CPU restatement of BVH::BVH.

  clutter       c2_hexagon_room_96 with CLUTTER small triangles (circumradius 1 % of the room), half scattered through the room and
                half around its 16 spheres, and one long thin emissive triangle running diagonally across the room as the only light
  sphere_light  the same clutter, the light one of the room's spheres made emissive: a split sphere is the occlusion target
  far           the clutter translated by FAR_OFFSET, where the float boxes' rounding is coarse against the primitives
  far_small     the far scene scaled by 1e-3 as a whole
  planes        triangles lying exactly on bin planes of the root box, triangles with an edge at a slope of about 1e-9 to a bin plane
                and slivers of aspect ratio about 1e6, each inside a cluster dense enough that the SAH cuts through it
  pm_split      pm_hexagon_room_64 with the clutter and a long thin light, for photon emission from a split light

Each generator asserts what it is there for (split spheres, a split light, more references than primitives): a builder change that
stops splitting them makes the scene fail instead of silently testing nothing."""
import os

import numpy as np

from conftest import GOLDEN
from deep_scene_gen import _small_triangles
from oracle import port

BASE = "c2_hexagon_room_96"
PM_BASE = "pm_hexagon_room_64"
CLUTTER = 1500
SEED = 5
FAR_OFFSET = np.array([1.0e4, -3.0e3, 7.0e3])
NB = 32                                  # buildBvh4Split's bins per axis
SCENES = ["clutter", "sphere_light", "far", "far_small", "planes"]


def _assemble(mcrt, base, tri, light_tri=None, light_sphere=None, scale=1.0, offset=(0.0, 0.0, 0.0)):
    """`base` (a Scene) with the triangles tri [n, 3, 3] appended in its first plain diffuse material, the whole scene then scaled by
    `scale` and moved by `offset`, and the reference's tree rebuilt. light_tri: index into tri of the triangle that becomes the only
    light; light_sphere: index of the base's sphere that becomes the only light (emissive, the other lamps stay as unlit surfaces)."""
    flat = base.unbuilt()
    a = dict(flat.a, **flat.extra)
    a["scene_ior"] = np.array([flat.ior])
    mats = a["materials"].copy()
    plain = (mats["dirac_delta"] == 0) & (mats["rough_specular"] == 0) & (mats["perfect_mirror"] == 0) & (mats["transparency"] == 0)
    diffuse = int(np.nonzero(plain & (mats["emissive"] == 0))[0][0])
    material = np.full(len(tri), diffuse)
    lamp = mats[diffuse].copy()
    lamp["emissive"] = 1; lamp["emittance"] = (200.0, 200.0, 200.0); lamp["reflectance"] = (0.0, 0.0, 0.0)
    mats["emissive"] = 0
    mats = np.concatenate([mats, [lamp]])
    a["materials"] = mats
    n_tri0, n_prim0, m = a["tri_vn_index"].size, a["prim_type"].size, len(tri)
    if light_tri is not None:
        material[light_tri] = len(mats) - 1
        light = n_prim0 + light_tri
    else:
        light = int(np.nonzero((a["prim_type"] == mcrt.PRIM_SPHERE) & (a["prim_index"] == light_sphere))[0][0])
        a["prim_material"] = a["prim_material"].copy()
        a["prim_material"][light] = len(mats) - 1
    scale = float(scale); offset = np.asarray(offset, np.float64)
    v0, v1, v2 = tri[:, 0], tri[:, 1], tri[:, 2]
    e1, e2 = v1 - v0, v2 - v0
    cross = np.cross(e1, e2)
    length = np.sqrt(np.sum(cross * cross, axis=1))
    assert (length > 0).all()
    for k, v in (("tri_v0", v0), ("tri_v1", v1), ("tri_v2", v2), ("tri_e1", e1), ("tri_e2", e2), ("tri_normal", cross / length[:, None])):
        a[k] = np.concatenate([a[k], v.reshape(-1)])
    a["tri_vn_index"] = np.concatenate([a["tri_vn_index"], np.full(m, -1, a["tri_vn_index"].dtype)])
    a["prim_type"] = np.concatenate([a["prim_type"], np.full(m, mcrt.PRIM_TRIANGLE, a["prim_type"].dtype)])
    a["prim_index"] = np.concatenate([a["prim_index"], (n_tri0 + np.arange(m)).astype(a["prim_index"].dtype)])
    a["prim_material"] = np.concatenate([a["prim_material"], material.astype(a["prim_material"].dtype)])
    a["prim_area"] = np.concatenate([a["prim_area"], 0.5 * length])
    a["prim_original"] = np.arange(n_prim0 + m, dtype=a["prim_original"].dtype)
    a["light_prim"] = np.array([light], dtype=a["light_prim"].dtype)
    a["light_cdf"] = np.array([1.0])
    bounds = np.asarray(base.extra["scene_bounds"], dtype=np.float64)
    bounds = np.concatenate([np.minimum(bounds[:3], tri.reshape(-1, 3).min(axis=0)), np.maximum(bounds[3:], tri.reshape(-1, 3).max(axis=0))])
    if scale != 1.0 or offset.any():
        # Triangle::Triangle and Sphere::Sphere of the moved scene: vertices, edges and areas in the new frame, normals unchanged
        for k in ("tri_v0", "tri_v1", "tri_v2"):
            a[k] = (a[k].reshape(-1, 3) * scale + offset).reshape(-1)
        for k in ("tri_e1", "tri_e2"):
            a[k] = a[k] * scale
        a["prim_area"] = a["prim_area"] * scale * scale
        sph = a["sphere_origin_radius"].reshape(-1, 4).copy()
        sph[:, :3] = sph[:, :3] * scale + offset; sph[:, 3] *= scale
        a["sphere_origin_radius"] = sph.reshape(-1)
        assert a["quadric_bounds"].size == 0
        bounds = np.concatenate([bounds[:3] * scale + offset, bounds[3:] * scale + offset])
        cam = a["camera_f64"].copy()
        cam[0:3] = cam[0:3] * scale + offset
        a["camera_f64"] = cam
    a["scene_bounds"] = bounds
    if "photon_emit_params" in a:
        p = a["photon_emit_params"].copy()
        p[3:9] = bounds
        a["photon_emit_params"] = p
    s = mcrt.Scene(a)
    bins = int(base.extra["bvh_params"][2])
    bvh_type = int(base.extra["bvh_params"][1])
    return s.with_bvh(port.bvh_build(s.prim_bounds(), a["scene_bounds"], bvh_type, bins, mcrt.BvhDesc))


def _base(mcrt, name=BASE):
    return mcrt.Scene.from_pack(os.path.join(GOLDEN, name + ".mcrtpack"))


def _clutter(base, rng, n=CLUTTER):
    """n small triangles: half at random points of the room, half just outside its spheres' surfaces, and a long thin triangle from
    one corner region of the room to the opposite one (the last)"""
    bounds = np.asarray(base.extra["scene_bounds"], dtype=np.float64)
    lo, hi = bounds[:3], bounds[3:]
    ext = hi - lo
    size = 0.01 * ext.max()
    n_room = n // 2
    room = lo + ext * (0.05 + 0.9 * rng.random((n_room, 3)))
    sph = base.a["sphere_origin_radius"].reshape(-1, 4)
    k = rng.integers(0, len(sph), n - n_room)
    d = rng.normal(size=(n - n_room, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    near = sph[k, :3] + d * sph[k, 3:4] * rng.uniform(1.02, 1.3, (n - n_room, 1))
    centre = np.concatenate([room, near])
    tri = _small_triangles(centre, np.full(len(centre), size), rng)
    a, b = lo + ext * (0.1, 0.3, 0.15), lo + ext * (0.9, 0.75, 0.85)
    side = np.cross(b - a, (0.0, 1.0, 0.0)); side *= 0.02 * ext.max() / np.linalg.norm(side)
    light = np.array([[a, b, a + side]])
    return np.concatenate([tri, light])


def split_stats(mcrt, scene, nodes=None, refs=None):
    """-> dict(prims, refs, split prims, split spheres, split lights (of all lights), most references of one primitive)"""
    if refs is None:
        nodes, refs = mcrt.bvh4_split_host(scene)
    per = np.bincount(refs, minlength=scene.n_prims)
    t = scene.a["prim_type"]
    lights = scene.a["light_prim"]
    return dict(prims=scene.n_prims, refs=len(refs), split=int((per > 1).sum()), split_spheres=int(((per > 1) & (t == mcrt.PRIM_SPHERE)).sum()),
                spheres=int((t == mcrt.PRIM_SPHERE).sum()), split_lights=int((per[lights] > 1).sum()), lights=len(lights),
                light_refs=int(per[lights].max()), most=int(per.max()))


def _check(mcrt, scene, spheres=True, light=True):
    assert scene.n_prims < 4096, scene.n_prims            # the upload's auto rule builds the split tree below 4096 primitives
    st = split_stats(mcrt, scene)
    assert st["refs"] > st["prims"], st
    if spheres:
        assert st["split_spheres"] > 0, st
    if light:
        assert st["split_lights"] == st["lights"] == 1, st
    return scene


def clutter(mcrt, seed=SEED):
    base = _base(mcrt)
    tri = _clutter(base, np.random.default_rng(seed))
    return _check(mcrt, _assemble(mcrt, base, tri, light_tri=len(tri) - 1))


def sphere_light(mcrt, seed=SEED):
    """the clutter without its long light; the room's largest sphere is the light"""
    base = _base(mcrt)
    tri = _clutter(base, np.random.default_rng(seed))[:-1]
    sph = base.a["sphere_origin_radius"].reshape(-1, 4)
    return _check(mcrt, _assemble(mcrt, base, tri, light_sphere=int(np.argmax(sph[:, 3]))))


def far(mcrt, scale=1.0, seed=SEED):
    base = _base(mcrt)
    tri = _clutter(base, np.random.default_rng(seed))
    return _check(mcrt, _assemble(mcrt, base, tri, light_tri=len(tri) - 1, scale=scale, offset=FAR_OFFSET * scale))


def planes(mcrt, seed=SEED):
    """The clutter plus, in dense clusters, triangles on bin planes x = lo + ext b / NB of the root box (the box of every primitive:
    the room's), triangles with an edge at a slope of about 1e-9 to such a plane, and slivers of aspect ratio about 1e6"""
    base = _base(mcrt)
    rng = np.random.default_rng(seed)
    clutter_tri = _clutter(base, rng)
    bounds = np.asarray(base.extra["scene_bounds"], dtype=np.float64)
    lo, hi = bounds[:3], bounds[3:]
    ext = hi - lo
    size = 0.01 * ext.max()
    special = []
    for j in range(24):
        k = j % 3
        b = 4 + (j * 5) % (NB - 8)
        plane = lo[k] + ext[k] * b / NB
        c = lo + ext * (0.15 + 0.7 * rng.random(3)); c[k] = plane
        ex, ey, ez = np.zeros(3), np.zeros(3), np.zeros(3); ex[(k + 1) % 3] = 1.0; ey[(k + 2) % 3] = 1.0; ez[k] = 1.0
        on = [c - size * ex, c + size * ex, c + size * ey]                                      # in the plane
        slope = [c - size * ex, c + size * ex + 2e-9 * size * ez, c + size * ey + 0.5 * size * ez]   # an edge at a slope of 1e-9
        sliver = [c - 2 * size * ex - 0.3 * size * ez, c + 2 * size * ex + 0.3 * size * ez,
                  c + 2 * size * ex + 0.3 * size * ez + 4e-6 * size * ey]                       # 4 size long, 4e-6 size wide, across it
        special += [on, slope, sliver]
        # a cluster around the plane's point, so that the SAH cuts there
        special += list(_small_triangles(c + rng.normal(0, 1.5 * size, (40, 3)), np.full(40, 0.3 * size), rng))
    tri = np.concatenate([clutter_tri[:-1], np.array(special), clutter_tri[-1:]])
    return _check(mcrt, _assemble(mcrt, base, tri, light_tri=len(tri) - 1))


def pm_split(mcrt, seed=SEED):
    """pm_hexagon_room_64 with the clutter; its long thin triangle is the only light"""
    base = _base(mcrt, PM_BASE)
    tri = _clutter(base, np.random.default_rng(seed))
    return _check(mcrt, _assemble(mcrt, base, tri, light_tri=len(tri) - 1), spheres=False)


def split_scene(mcrt, name):
    if name == "far_small":
        return far(mcrt, scale=1e-3)
    return dict(clutter=clutter, sphere_light=sphere_light, far=far, planes=planes, pm_split=pm_split)[name](mcrt)


def scene_scale(scene):
    """ctx->scene_scale as mcrt_scene_upload computes it (float)"""
    return float(np.float32(np.abs(scene.a["node_bounds"][:6]).max()))


def camera_rays(mcrt, scene, n=4000, seed=7):
    """n of the scene camera's rays at random pixels"""
    cam = scene.cameras()[0]
    rng = np.random.default_rng(seed)
    ps = port.PortScene(scene)
    try:
        pixel = rng.integers(0, cam.width * cam.height, n).astype(np.uint32)
        _, rays = ps.sample_pixels(cam, pixel, np.zeros(n, np.uint32), 7)
    finally:
        ps.close()
    return rays


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def cut_points(mcrt, scene, nodes, refs, rng, per_line=3):
    """Points where each split primitive meets a face of one of its references' leaf boxes: on triangles, points of the segment
    the face's plane cuts from the triangle; on spheres, points of the circle it cuts from the sphere; only those on the face
    itself (within the box). -> (points [n, 3], primitive [n], axis of the face [n], sphere centre and radius [n, 4] (NaN: triangle))"""
    a = scene.a
    per = np.bincount(refs, minlength=scene.n_prims)
    boxes = {}
    for i, n in enumerate(nodes):
        for c in range(4):
            ch = int(n["child"][c])
            if ch & 0x80000000:
                f, k = (ch >> 8) & 0x7FFFFF, ch & 0xFF
                for r in range(f, f + k):
                    if per[refs[r]] > 1:
                        boxes.setdefault(int(refs[r]), []).append((n["lo"][:, c].astype(np.float64), n["hi"][:, c].astype(np.float64)))
    tv = [a[k].reshape(-1, 3) for k in ("tri_v0", "tri_v1", "tri_v2")]
    sph = a["sphere_origin_radius"].reshape(-1, 4)
    pts, prim, axis, sphere = [], [], [], []
    for p, bl in boxes.items():
        t, idx = int(a["prim_type"][p]), int(a["prim_index"][p])
        for lo, hi in bl:
            slack = 1e-7 * (np.abs(lo) + np.abs(hi) + (hi - lo))
            for k in range(3):
                for c in (lo[k], hi[k]):
                    if t == mcrt.PRIM_TRIANGLE:
                        v = [tv[0][idx], tv[1][idx], tv[2][idx]]
                        ends = []
                        for e in range(3):
                            p0, p1 = v[e], v[(e + 1) % 3]
                            if (p0[k] - c) * (p1[k] - c) <= 0 and p0[k] != p1[k]:
                                ends.append(p0 + (c - p0[k]) / (p1[k] - p0[k]) * (p1 - p0))
                        if len(ends) < 2:
                            continue
                        s = np.concatenate([[0.0, 1.0], rng.random(per_line)])[:, None]
                        q = ends[0] + s * (ends[1] - ends[0])
                        q[:, k] = c
                        ctr = np.full((len(q), 4), np.nan)
                    else:
                        o, r = sph[idx, :3], sph[idx, 3]
                        h = c - o[k]
                        if abs(h) >= r:
                            continue
                        u, w = (k + 1) % 3, (k + 2) % 3
                        ang = rng.uniform(0, 2 * np.pi, 4 * per_line)
                        q = np.repeat(o[None], len(ang), 0)
                        q[:, k] = c
                        q[:, u] += np.sqrt(r * r - h * h) * np.cos(ang); q[:, w] += np.sqrt(r * r - h * h) * np.sin(ang)
                        ctr = np.repeat(sph[idx][None], len(q), 0)
                    keep = ((q >= lo - slack) & (q <= hi + slack)).all(1)
                    pts.append(q[keep]); prim.append(np.full(keep.sum(), p)); axis.append(np.full(keep.sum(), k)); sphere.append(ctr[keep])
    return np.concatenate(pts), np.concatenate(prim), np.concatenate(axis), np.concatenate(sphere)


def adversarial_rays(mcrt, scene, nodes, refs, surface, rng):
    """Rays at the cut points of every split primitive (cut_points): from random points of `surface` [m, 3]; along the face's plane at
    grazing angles of 1e-2 to 1e-8 through the point, from either side; and, for sphere points, tangent to the sphere at the point
    (the silhouette seen from the ray's origin) and just inside it. -> (rays [n, 6], primitive aimed at [n])"""
    pts, prim, axis, sphere = cut_points(mcrt, scene, nodes, refs, rng)
    n = len(pts)
    size = float(np.abs(scene.a["node_bounds"][3:6] - scene.a["node_bounds"][:3]).max())
    out, aim = [], []
    # from surfaces
    o = surface[rng.integers(0, len(surface), n)]
    d = pts - o
    ok = np.linalg.norm(d, axis=1) > 1e-6 * size
    out.append(np.concatenate([o[ok], _unit(d[ok])], 1)); aim.append(prim[ok])
    # along the cut plane, tilted out of it by 1e-2 ... 1e-8
    inplane = rng.normal(size=(n, 3)); inplane[np.arange(n), axis] = 0.0
    inplane = _unit(inplane)
    tilt = 10.0 ** -rng.uniform(2, 8, n) * rng.choice([-1.0, 1.0], n)
    d = inplane.copy(); d[np.arange(n), axis] = tilt
    d = _unit(d)
    length = size * rng.uniform(0.05, 0.5, (n, 1))
    out.append(np.concatenate([pts - d * length, d], 1)); aim.append(prim)
    # sphere silhouettes: tangent at the point, and 1e-9 of the radius inside it
    s = ~np.isnan(sphere[:, 0])
    if s.any():
        c, r, q = sphere[s, :3], sphere[s, 3:4], pts[s]
        nrm = _unit(q - c)
        tang = _unit(np.cross(nrm, rng.normal(size=nrm.shape)))
        for inset in (0.0, 1e-9, 1e-6):
            target = q - inset * r * nrm
            o = target - tang * r * rng.uniform(0.5, 3.0, (len(q), 1))
            out.append(np.concatenate([o, tang], 1)); aim.append(prim[s])
    return np.concatenate(out), np.concatenate(aim)
