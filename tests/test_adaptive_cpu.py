"""Adaptive sampling bookkeeping without a GPU: the retirement rule of Progressive.render_adaptive (adaptive_retire)
and the per-tile pixel and sample counts, including edge tiles that the tile size does not divide."""
import numpy as np
import pytest


@pytest.mark.parametrize("rows,width,tile", [(54, 96, 16), (23, 37, 5), (7, 9, 16), (64, 64, 8), (1, 1, 1)])
def test_tile_pixel_counts_cover_the_grid(rows, width, tile, mcrt):
    ty, tx = mcrt.tile_grid(rows, width, tile)
    n = mcrt.tile_pixel_counts(rows, width, tile)
    assert n.shape == (ty, tx) and n.sum() == rows * width
    owner = np.zeros((rows, width), np.int64)      # each pixel's tile, from the definition
    for y in range(rows):
        for x in range(width):
            owner[y, x] = (y // tile) * tx + x // tile
    assert np.array_equal(np.bincount(owner.ravel(), minlength=ty * tx).reshape(ty, tx), n)
    assert n.max() <= tile * tile


def test_tile_samples_follow_the_active_mask(mcrt):
    rows, width, tile = 23, 37, 5                  # edge tiles of 3 rows and 2 columns
    n = mcrt.tile_pixel_counts(rows, width, tile)
    ty, tx = n.shape
    counts = np.zeros((ty, tx, 2), np.int64)
    active = np.ones((ty, tx), bool)
    rng = np.random.default_rng(3)
    paths = 0
    for k, samples in enumerate((3, 5, 2, 7, 1, 4)):
        if k in (2, 4):
            active &= rng.random((ty, tx)) < 0.6
        before = counts.copy()
        counts = mcrt.add_tile_samples(counts, active, k % 2, samples)
        assert np.array_equal(counts[~active], before[~active])          # retired tiles are frozen
        assert np.all(counts[active][:, k % 2] == before[active][:, k % 2] + samples)
        assert np.array_equal(counts[..., 1 - k % 2], before[..., 1 - k % 2])
        paths += int(n[active].sum()) * samples
    # the camera paths a run renders: every tile's pixels times its own count
    assert paths == int((n * counts.sum(-1)).sum())
    # active tiles all share one count: a pass is one sample range over a subset of the pixels
    assert len({tuple(c) for c in counts[active]}) <= 1


def random_case(rng, ty=6, tx=9):
    counts = rng.integers(0, 20, (ty, tx, 2))
    counts[0, 0] = (0, 30)                          # an empty half
    counts[0, 1] = (4, 0)
    counts[1, 1] = (3, 4)                           # below min_samples
    sums = np.stack([rng.exponential(1.0, (ty, tx)) * 1e-3, rng.exponential(1.0, (ty, tx))], -1)
    sums[2, 2, 0] = 0.0                             # a tile whose halves agree exactly
    active = rng.random((ty, tx)) < 0.8
    pixels = np.full((ty, tx), 16 * 16)
    pixels[-1, :] = 16 * 7
    pixels[:, -1] //= 2
    return active, counts, sums, pixels


@pytest.mark.parametrize("seed", range(20))
def test_retirement_rule(seed, mcrt):
    rng = np.random.default_rng(seed)
    active, counts, sums, pixels = random_case(rng)
    for target in (1e-3, 0.02, 0.05, 0.2, 10.0):
        for min_samples in (0, 8, 16):
            r = mcrt.adaptive_retire(active, counts, sums, pixels, target, min_samples)
            assert r.dtype == bool and r.shape == active.shape
            assert not np.any(r & ~active)                                   # only active tiles retire
            assert not np.any(r & ((counts[..., 0] == 0) | (counts[..., 1] == 0)))
            assert not np.any(r & (counts.sum(-1) < min_samples))
            bound = target ** 2 * sums[..., 1].sum() * pixels / pixels.sum()
            eligible = active & (counts > 0).all(-1) & (counts.sum(-1) >= min_samples)
            assert np.array_equal(r, eligible & (sums[..., 0] <= bound))


def test_retiring_every_tile_meets_the_target(mcrt):
    rng = np.random.default_rng(11)
    ty, tx = 5, 7
    counts = np.full((ty, tx, 2), 16)
    pixels = mcrt.tile_pixel_counts(70, 110, 16)
    assert pixels.shape == (ty, tx)
    hits = 0
    for _ in range(200):
        si2 = rng.exponential(1.0, (ty, tx))
        target = 0.05
        # noise within a random factor of each tile's share of the target
        share = target ** 2 * si2.sum() * pixels / pixels.sum()
        sv = share * rng.uniform(0.2, 1.05, (ty, tx))
        sums = np.stack([sv, si2], -1)
        r = mcrt.adaptive_retire(np.ones((ty, tx), bool), counts, sums, pixels, target, 16)
        if r.all():
            hits += 1
            assert sums[..., 0].sum() <= target ** 2 * sums[..., 1].sum() * (1 + 1e-12)
    assert hits > 0
