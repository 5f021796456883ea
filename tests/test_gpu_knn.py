"""The photon-map k-NN search (knnSearchWarpT in csrc/photon.cuh, called through mcrt_knn_search) against a
brute-force float64 search, for every k where the kernel changes shape: both sides of each register-slot width
(knnSlotsFor: 1, 2, 4, 8 slots, then the shared-memory version above k = 256) and of the 48 KB dynamic
shared-memory limit (knnSharedBytes crosses it above k = 672).

Reference. Every query's distance to every photon in numpy float64, in the kernel's expression order: the
float32 position widened to double, dx = px - x, then (dx*dx + dy*dy) + dz*dz. kernels_f64.cu is built with
--fmad=false, so the returned distances must agree bit for bit. Coincident photons tie at the k-th distance;
any of them may be returned.

Frontier overflow. The search keeps at most KNN_FRONTIER = 256 pending octants per query; beyond that it drops
octants and mcrt_knn_search raises McrtError("k-NN frontier overflow"). Every result below is either exact or
that error - never a wrong answer. Queries in the hollow of a thin shell overflow for k up to 257 on the H100;
the plausible maps (clusters, planes, queries on or near photons) must not overflow at all."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_photon_octree_cpu import oracle_octree

pytestmark = pytest.mark.gpu

K_GRID = (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 672, 673, 768, 769, 1024)
K_MAX = 1024
DBL_MAX = np.finfo(np.float64).max
# scene bounds of the synthetic maps; every value is exact in float32, so clipped photons stay inside. The root
# splits at (0.5, 0.25, -0.25), its children at mid -/+ a quarter of the extent.
BOUNDS = np.array([-2.0, -1.0, -1.5, 3.0, 1.5, 1.0])
LO, HI = BOUNDS[:3], BOUNDS[3:]
MID = (LO + HI) / 2
SPLITS = [(MID[c], MID[c] - (HI[c] - LO[c]) / 4, MID[c] + (HI[c] - LO[c]) / 4) for c in range(3)]
CHUNK = 1 << 22   # distances per brute-force block (32 MB of float64)


@pytest.fixture(scope="module")
def pm(mcrt):
    """A photon-mapping context on the pm_hexagon_room_64 scene; the tests replace its photon maps."""
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "pm_hexagon_room_64.mcrtpack"))
    p = mcrt.PhotonMapper(scene, precision=mcrt.PRECISION_F64)
    yield p
    p.close()


@pytest.fixture(scope="module")
def empty_map(mcrt):
    return mcrt.build_photon_octree(np.zeros((0, 8), np.float32), 8, BOUNDS)[0]


# ------------------------------------------------------------------------------------------------- maps

def make_photons(pos, rng):
    """8-float photon records (flux xyz, position xyz, phi, theta) at `pos`, clipped into BOUNDS."""
    pos = np.clip(np.asarray(pos, np.float64).reshape(-1, 3), LO, HI)
    ph = np.empty((len(pos), 8), np.float32)
    ph[:, :3] = rng.uniform(0.0, 1.0, (len(pos), 3))
    ph[:, 3:6] = pos
    ph[:, 6] = rng.uniform(0.0, 2 * np.pi, len(pos))
    ph[:, 7] = rng.uniform(0.0, np.pi, len(pos))
    return ph


def build_map(mcrt, photons, leaf, check_builder=True):
    m, _ = mcrt.build_photon_octree(photons, leaf, BOUNDS)
    if check_builder:   # the k-NN results below are only as good as the octree they search
        host = oracle_octree(mcrt, photons, leaf, BOUNDS)
        for key in ("octant_bounds", "octant_start", "octant_count", "octant_next", "octant_leaf", "photons"):
            assert np.array_equal(host[key], m[key]), key
    return m


def positions(m):
    return m["photons"].reshape(-1, 8)[:, 3:6].astype(np.float64)


def uniform(rng, n):
    return rng.uniform(LO, HI, (n, 3))


def clusters(rng, n, n_clusters=12):
    centres = rng.uniform(LO + 0.3, HI - 0.3, (n_clusters, 3))
    sigma = np.exp(rng.uniform(np.log(0.01), np.log(0.2), (n_clusters, 1)))
    which = rng.integers(0, n_clusters, n)
    return centres[which] + rng.normal(0.0, 1.0, (n, 3)) * sigma[which]


SHELL_CENTRE = MID   # the root's split point: the centre query sits on all three root split planes


def shell(rng, n, radius=0.9, thickness=1e-3):
    d = rng.normal(0.0, 1.0, (n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return SHELL_CENTRE + d * radius * (1.0 + thickness * rng.normal(0.0, 1.0, (n, 1)))


def plane(rng, n):
    p = uniform(rng, n)
    p[:, 2] = MID[2]   # on the root's z split plane
    return p


def coincident(rng, n_blocks=8, block=1500, n_background=5000):
    """Blocks of identical positions, each larger than any k and than the leaf size (the builder's level-64 guard
    leaves), on a uniform background."""
    spots = rng.uniform(LO, HI, (n_blocks, 3)).astype(np.float32)
    return np.concatenate([np.repeat(spots, block, axis=0), uniform(rng, n_background)]), spots


# ---------------------------------------------------------------------------------------------- queries

def queries(m, rng, n_random=48, n_on=32, n_faces=32, n_far=8):
    """Random points in the box, points exactly on photons, on the root's and its children's split planes, on faces
    and corners of octant boxes, and points 10^3 box sizes away."""
    out = [uniform(rng, n_random)]
    pos = positions(m)
    if len(pos):
        out.append(pos[rng.integers(0, len(pos), n_on)])
    planes = uniform(rng, 3 * 3 * 4).reshape(3, 3, 4, 3)
    for c in range(3):
        for s in range(3):
            planes[c, s, :, c] = SPLITS[c][s]
    out.append(planes.reshape(-1, 3))
    out.append(np.array([[SPLITS[0][a], SPLITS[1][b], SPLITS[2][c]] for a in range(3) for b in range(3) for c in range(3)]))
    ob = m["octant_bounds"].reshape(-1, 6)
    if len(ob):
        box = ob[rng.integers(0, len(ob), n_faces)]
        p = rng.uniform(box[:, :3], box[:, 3:])
        snap = rng.random((n_faces, 3)) < 0.5
        side = rng.random((n_faces, 3)) < 0.5
        p[snap] = np.where(side, box[:, 3:], box[:, :3])[snap]
        out.append(p)
    d = rng.normal(0.0, 1.0, (n_far, 3))
    out.append(MID + d / np.linalg.norm(d, axis=1, keepdims=True) * 1e3 * np.linalg.norm(HI - LO))
    return np.concatenate(out)


# -------------------------------------------------------------------------------------------- reference

def dist2(q, pos):
    dx = q[:, None, 0] - pos[None, :, 0]
    dy = q[:, None, 1] - pos[None, :, 1]
    dz = q[:, None, 2] - pos[None, :, 2]
    return (dx * dx + dy * dy) + dz * dz


def brute_force(pos, q, k_max=K_MAX):
    """-> (index, d2), [len(q), min(k_max, n)]: every query's nearest photons by ascending d2."""
    n = len(pos)
    kk = min(k_max, n)
    idx = np.zeros((len(q), kk), np.int64)
    d2 = np.zeros((len(q), kk))
    if kk == 0:
        return idx, d2
    rows = max(1, CHUNK // n)
    for a in range(0, len(q), rows):
        d = dist2(q[a:a + rows], pos)
        part = np.argpartition(d, kk - 1, axis=1)[:, :kk]
        v = np.take_along_axis(d, part, 1)
        o = np.argsort(v, axis=1, kind="stable")
        idx[a:a + rows] = np.take_along_axis(part, o, 1)
        d2[a:a + rows] = np.take_along_axis(v, o, 1)
    return idx, d2


# ------------------------------------------------------------------------------------------------ device

def upload(pm, m, k, empty):
    """`m` as the global map and an empty caustic map (a scene without specular surfaces), at k."""
    pm._maps = (empty, m, k, 0)
    pm.upload_photons()


def search(pm, mcrt, q, which=1):
    """pm.knn on all of `q`; a batch that overflows the frontier is split until the overflowing queries are
    isolated. -> (index, d2, count, ok) with ok[i] False where query i overflowed."""
    try:
        idx, d2, cnt = pm.knn(which, q)
        return idx, d2, cnt, np.ones(len(q), bool)
    except mcrt.McrtError as e:
        if "frontier overflow" not in str(e):
            raise
        if len(q) == 1:
            k = pm.k_nearest
            return np.zeros((1, k), np.uint32), np.zeros((1, k)), np.zeros(1, np.uint32), np.zeros(1, bool)
    h = len(q) // 2
    a, b = search(pm, mcrt, q[:h], which), search(pm, mcrt, q[h:], which)
    return tuple(np.concatenate([x, y]) for x, y in zip(a, b))


def _rows(bad, what, k, tag):
    rows = np.flatnonzero(bad)
    return f"{tag} k={k}: {what} at {rows.size} queries, first {rows[:8].tolist()}"


def check_exact(pos, q, ref_idx, ref_d2, k, idx, d2, cnt, tag, no_prim):
    n = len(pos)
    kc = min(k, n)
    assert idx.shape == (len(q), k) and d2.shape == (len(q), k)
    assert np.all(cnt == kc), _rows(cnt != kc, f"count != {kc}", k, tag)
    pad = np.any(idx[:, kc:] != no_prim, axis=1) | np.any(d2[:, kc:] != DBL_MAX, axis=1)
    assert not pad.any(), _rows(pad, "padding not (NO_PRIM, DBL_MAX)", k, tag)
    if kc == 0:
        return
    gi, gd = idx[:, :kc].astype(np.int64), d2[:, :kc]
    assert np.all(gi < n), _rows(np.any(gi >= n, axis=1), "index out of range", k, tag)
    wrong = np.any(np.sort(gd, axis=1) != ref_d2[:, :kc], axis=1)
    assert not wrong.any(), _rows(wrong, "sorted d2 != the k smallest reference d2", k, tag)
    s = np.sort(gi, axis=1)
    dup = np.any(s[:, 1:] == s[:, :-1], axis=1)
    assert not dup.any(), _rows(dup, "repeated index", k, tag)
    p = pos[gi]
    dx, dy, dz = q[:, None, 0] - p[..., 0], q[:, None, 1] - p[..., 1], q[:, None, 2] - p[..., 2]
    mism = np.any((dx * dx + dy * dy) + dz * dz != gd, axis=1)
    assert not mism.any(), _rows(mism, "returned d2 != d2 of the returned index", k, tag)
    closer = ref_d2[:, :kc] < ref_d2[:, kc - 1:kc]
    rows = np.arange(len(q))[:, None]
    need = (rows * n + ref_idx[:, :kc])[closer]
    missing = ~np.isin(need, (rows * n + gi).ravel())
    assert not missing.any(), _rows(np.isin(np.arange(len(q)), need[missing] // n), "photon closer than the k-th missing", k, tag)


def run_grid(mcrt, pm, empty, m, q, tag, k_grid=K_GRID, may_overflow=None):
    """Every k of k_grid on map m: exact, or McrtError("frontier overflow") where may_overflow allows it."""
    pos = positions(m)
    ref_idx, ref_d2 = brute_force(pos, q, max(k_grid))
    allowed = np.zeros(len(q), bool) if may_overflow is None else np.broadcast_to(may_overflow, len(q))
    for k in k_grid:
        upload(pm, m, k, empty)
        idx, d2, cnt, ok = search(pm, mcrt, q)
        assert np.all(ok | allowed), _rows(~ok & ~allowed, "frontier overflow", k, tag)
        check_exact(pos, q[ok], ref_idx[ok], ref_d2[ok], k, idx[ok], d2[ok], cnt[ok], tag, mcrt.NO_PRIM)


# ------------------------------------------------------------------------------------------------- tests

LAYOUTS = {
    # name: (positions(rng), leaf size)
    "uniform_leaf1": (lambda rng: uniform(rng, 8000), 1),
    "uniform_leaf8": (lambda rng: uniform(rng, 40000), 8),
    "clusters_leaf200": (lambda rng: clusters(rng, 100000), 200),
    "plane_leaf8": (lambda rng: plane(rng, 40000), 8),
    "single_leaf": (lambda rng: clusters(rng, 256, 3), 1000),   # one leaf: the histogram bound runs at every k <= 256
}


@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_knn_matches_brute_force(name, mcrt, pm, empty_map):
    rng = np.random.default_rng(sorted(LAYOUTS).index(name) + 11)
    make, leaf = LAYOUTS[name]
    m = build_map(mcrt, make_photons(make(rng), rng), leaf)
    run_grid(mcrt, pm, empty_map, m, queries(m, rng), name)


def test_knn_thin_shell(mcrt, pm, empty_map):
    """A thin spherical shell at leaf size 8. From a point in its hollow every leaf is about equally far, so the
    best-first frontier keeps them all pending and outgrows KNN_FRONTIER: those queries may raise (the centre at
    k = 1 must), every other query is exact."""
    rng = np.random.default_rng(17)
    radius = 0.9
    m = build_map(mcrt, make_photons(shell(rng, 40000, radius), rng), 8)
    q = np.concatenate([queries(m, rng), SHELL_CENTRE[None], SHELL_CENTRE + uniform(rng, 8) * 0.1])
    hollow = np.linalg.norm(q - SHELL_CENTRE, axis=1) < 0.5 * radius
    run_grid(mcrt, pm, empty_map, m, q, "shell", may_overflow=hollow)
    upload(pm, m, 1, empty_map)
    with pytest.raises(mcrt.McrtError, match="frontier overflow"):
        pm.knn(1, SHELL_CENTRE[None])


def test_knn_coincident_blocks(mcrt, pm, empty_map):
    """Blocks of 1500 identical photons (more than any k, more than the leaf size of 200): queries on a block tie
    at d2 = 0 for every k; queries between blocks tie at the k-th distance."""
    rng = np.random.default_rng(3)
    pos, spots = coincident(rng)
    m = build_map(mcrt, make_photons(pos, rng), 200)
    s = spots.astype(np.float64)
    q = np.concatenate([queries(m, rng), s, (s[0] + s[1:]) / 2])
    run_grid(mcrt, pm, empty_map, m, q, "coincident")


@pytest.mark.parametrize("n", [0, 1, 672, 673, 674])
def test_knn_small_maps(n, mcrt, pm, empty_map):
    """Maps of 0, 1, k-1, k and k+1 photons for k = 673 (the first k past 48 KB), at every k of the grid: k is
    clamped to the map size, and the rest of each row is padding. The empty caustic map is queried too."""
    rng = np.random.default_rng(n)
    m = build_map(mcrt, make_photons(uniform(rng, n), rng), 64)
    q = queries(m, rng)
    run_grid(mcrt, pm, empty_map, m, q, f"n={n}")
    for k in (1, 673, 1024):
        upload(pm, m, k, empty_map)
        idx, d2, cnt = pm.knn(0, q)
        assert np.all(cnt == 0) and np.all(idx == mcrt.NO_PRIM) and np.all(d2 == DBL_MAX)


def test_knn_water_caustics_sized_map(mcrt, pm, empty_map):
    """One map of 2^20 photons at leaf size 200, the size of the water_caustics maps: half uniform, half clustered."""
    rng = np.random.default_rng(7)
    n = 1 << 20
    m = build_map(mcrt, make_photons(np.concatenate([uniform(rng, n // 2), clusters(rng, n - n // 2, 40)]), rng), 200,
                  check_builder=False)
    q = queries(m, rng, n_random=24, n_on=16, n_faces=16, n_far=4)
    run_grid(mcrt, pm, empty_map, m, q, "1M")


def test_knn_k_above_1024_is_refused(mcrt, pm, empty_map):
    rng = np.random.default_rng(1)
    m = build_map(mcrt, make_photons(uniform(rng, 2000), rng), 64)
    with pytest.raises(mcrt.McrtError, match="1024"):
        upload(pm, m, 1025, empty_map)


def comb_map(depth, rng, per_leaf=5):
    """A hand-made octree: a chain of inner octants 0..depth whose boxes contain the origin, each with 7 leaf
    children (the deepest: 8). A search from the origin pops the chain first and keeps every leaf pending, so
    the frontier holds 7 * depth + 8 octants after the last expansion. The last 4 children of the deepest
    octant - lanes 4..7 of that expansion - hold the photons nearest to the origin."""
    leaves = []   # (depth of the parent, child slot), in depth-first order
    leaves += [(depth, j) for j in range(8)]
    for i in range(depth - 1, -1, -1):
        leaves += [(i, j) for j in range(1, 8)]
    n_oct = depth + 1 + len(leaves)
    bounds = np.zeros((n_oct, 6))
    start = np.zeros(n_oct, np.uint64)
    count = np.zeros(n_oct, np.uint64)
    nxt = np.full(n_oct, 0xFFFFFFFF, np.uint32)
    leaf = np.zeros(n_oct, np.uint8)
    pos = []
    first_leaf = {}
    for li, (parent, j) in enumerate(leaves):
        o = depth + 1 + li
        first_leaf.setdefault(parent, o)
        near = parent == depth and j >= 4
        d = rng.normal(0.0, 1.0, 3)
        c = d / np.linalg.norm(d) * (rng.uniform(0.1, 0.12) if near else rng.uniform(0.3, 0.95))   # inside BOUNDS
        p = (c + rng.uniform(-0.01, 0.01, (per_leaf, 3))).astype(np.float32).astype(np.float64)
        bounds[o] = np.concatenate([p.min(axis=0), p.max(axis=0)])
        start[o], count[o], leaf[o] = li * per_leaf, per_leaf, 1
        last = li + 1 == len(leaves) or leaves[li + 1][0] != parent
        nxt[o] = 0xFFFFFFFF if last else o + 1
        pos.append(p)
    for i in range(depth + 1):
        bounds[i] = (-100, -100, -100, 100, 100, 100)
        count[i] = per_leaf * (8 + 7 * (depth - i))   # its subtree is a prefix of the photon array
        if i > 0:
            nxt[i] = first_leaf[i - 1]
    return {"octant_bounds": bounds.reshape(-1), "octant_start": start, "octant_count": count, "octant_next": nxt,
            "octant_leaf": leaf, "photons": make_photons(np.concatenate(pos), rng).reshape(-1)}


def test_knn_frontier_overflow_in_any_lane_raises(mcrt, pm, empty_map):
    """A frontier that overflows in lanes other than lane 0 of the expanding warp must still raise: the comb of
    depth 36 pushes the deepest octant's 8 children into slots 252..259, so only lanes 4..7 fall off - and their
    leaves hold the nearest photons. At depth 35 everything fits (slots 245..252) and the search is exact."""
    rng = np.random.default_rng(36)
    q = np.zeros((1, 3))
    fits = comb_map(35, rng)
    run_grid(mcrt, pm, empty_map, fits, q, "comb35", k_grid=(32,))
    over = comb_map(36, rng)
    upload(pm, over, 32, empty_map)
    with pytest.raises(mcrt.McrtError, match="frontier overflow"):
        pm.knn(1, q)
