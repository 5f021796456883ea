"""CPU property test of the radius estimate k_knn takes from a leaf's distance histogram before it fills its result set
(csrc/photon.cuh, knnSearchWarpT): 256 bins between the nearest and the farthest point of the octant's box, bound = upper edge of the
bin where the running count reaches k. It must be an UPPER bound of the k-th smallest distance of the leaf (so that tightening the
search radius with it cannot drop one of the k nearest photons) - restated here with the kernel's float64 expressions.

The kernel takes the estimate for leaves of k..256 photons, so k runs up to the leaf's photon count (leaves of exactly k photons
included); queries run from inside the box to 10^4 box sizes away, and boxes shrink until hi - lo is a few ulps of lo."""
import numpy as np
import pytest

BINS = 256


def bound_from_histogram(d2, lo, hi, k, max_d2=np.inf):
    scale = (BINS - 1) / (hi - lo)
    hist = np.zeros(BINS, dtype=np.int64)
    for v in d2:
        if v <= max_d2:
            q = (v - lo) * scale
            b = 0 if q <= 0.0 else (BINS - 1 if q >= BINS - 1 else int(q))
            hist[b] += 1
    run = np.cumsum(hist)
    if run[-1] < k:
        return None
    bsel = int(np.argmax(run >= k))
    return (lo + (bsel + 1) / scale) * (1.0 + 1e-9)


def leaf_distances(pts, bmin, bmax, p):
    """photon distances and BoundingBox::distance2 / max_distance2 of the octant box, as the kernel computes them"""
    d = p - pts
    d2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]
    near = np.maximum(np.maximum(bmin - p, p - bmax), 0.0)
    far = np.maximum(bmax - p, p - bmin)
    return d2, float(near[0] * near[0] + near[1] * near[1] + near[2] * near[2]), float(far[0] * far[0] + far[1] * far[1] + far[2] * far[2])


def assert_upper_bound(d2, lo, hi, k):
    n = len(d2)
    assert hi > lo   # the kernel skips the estimate otherwise
    s = np.sort(d2)
    kth = s[k - 1]
    bound = bound_from_histogram(d2, lo, hi, k)
    assert bound is not None and bound >= kth
    # with a tighter radius already in force only the photons inside it are counted
    cap = float(s[min(n - 1, k + 5)])
    b2 = bound_from_histogram(d2, lo, hi, k, cap)
    assert b2 is not None and b2 >= kth
    assert bound_from_histogram(d2, lo, hi, k, float(s[0]) * 0.5 if s[0] > 0 else -1.0) is None or k == 1


@pytest.mark.parametrize("seed", range(40))
def test_histogram_bound_is_an_upper_bound_of_the_kth_distance(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(50, 257))
    k = int(rng.integers(1, n + 1))
    bmin = rng.uniform(-5, 5, 3); bmax = bmin + rng.uniform(1e-3, 4, 3)
    style = seed % 4
    if style == 0: pts = rng.uniform(bmin, bmax, (n, 3))
    elif style == 1: pts = bmin + (bmax - bmin) * rng.beta(0.2, 0.2, (n, 3))          # piled up at the faces of the box
    elif style == 2: pts = np.tile(rng.uniform(bmin, bmax, 3), (n, 1))                # coincident photons
    else: pts = np.clip(rng.normal((bmin + bmax) / 2, (bmax - bmin) / 40, (n, 3)), bmin, bmax)
    pts = pts.astype(np.float32).astype(np.float64)                                    # photon positions are stored as float
    bmin, bmax = np.minimum(bmin, pts.min(axis=0)), np.maximum(bmax, pts.max(axis=0))  # octant boxes contain their photons
    p = rng.uniform(bmin - 2, bmax + 2) if seed % 3 else rng.uniform(bmin, bmax)       # query outside / inside the box
    assert_upper_bound(*leaf_distances(pts, bmin, bmax, p), k)


@pytest.mark.parametrize("seed", range(40))
def test_histogram_bound_far_queries(seed):
    """Queries 10^3..10^4 box sizes away: lo and hi are large and close, and the photons' distances crowd into few bins."""
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(1, 257))
    k = n if seed % 2 else int(rng.integers(1, n + 1))    # every other leaf holds exactly k photons
    size = 10.0 ** rng.uniform(-3, 1)
    pts = rng.uniform(-0.5, 0.5, (n, 3)) * size * rng.uniform(0.01, 1, 3) + rng.uniform(-5, 5, 3)
    if seed % 5 == 0: pts[: n // 2] = pts[0]                                            # a block of coincident photons
    pts = pts.astype(np.float32).astype(np.float64)
    bmin, bmax = pts.min(axis=0), pts.max(axis=0)                                        # tight boxes, as the octree builder stores them
    u = rng.normal(0, 1, 3); u /= np.linalg.norm(u)
    p = (bmin + bmax) / 2 + u * size * 10.0 ** rng.uniform(3, 4)
    d2, lo, hi = leaf_distances(pts, bmin, bmax, p)
    if n == 1 or np.all(bmin == bmax):
        assert hi == lo   # a point box: no estimate
        return
    assert_upper_bound(d2, lo, hi, k)


@pytest.mark.parametrize("seed", range(40))
def test_histogram_bound_thin_boxes(seed):
    """Boxes a few ulps of the query distance wide, seen along an axis: hi - lo is a few ulps of lo, the bin width is below
    the rounding of the distances, and photons land in bins that their rounded distances do not strictly order."""
    rng = np.random.default_rng(2000 + seed)
    n = int(rng.integers(2, 257))
    k = n if seed % 2 else int(rng.integers(1, n + 1))
    dist = rng.uniform(1.0, 8.0)
    width = int(rng.integers(1, 9)) * np.spacing(dist)
    pts = rng.uniform(0.0, width, (n, 3)).astype(np.float32).astype(np.float64)
    pts[0] = 0.0; pts[1] = np.float32(width)                                             # the box spans the full width
    bmin, bmax = pts.min(axis=0), pts.max(axis=0)
    axis, sign = int(rng.integers(0, 3)), float(rng.choice([-1.0, 1.0]))
    p = rng.uniform(bmin, bmax)
    p[axis] = bmax[axis] + dist if sign > 0 else bmin[axis] - dist
    d2, lo, hi = leaf_distances(pts, bmin, bmax, p)
    assert (hi - lo) <= 64 * np.spacing(lo)
    assert_upper_bound(d2, lo, hi, k)
