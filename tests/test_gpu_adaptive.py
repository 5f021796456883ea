"""Adaptive sampling (mcrt_render_accumulate_tiles_dev, mcrt_progressive_resolve_tiles_dev, Progressive.retire and
Progressive.render_adaptive). A pass over the active tiles renders the same samples of those pixels as a pass over
the whole frame, so every tile resolves to the uniform frame at its own sample count, up to the order of the float64
film additions (the bar of the progressive tests: rtol 1e-12, atol 1e-14)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-12, 1e-14
STATS = ("paths", "extension_rays", "shadow_rays")


@pytest.fixture(scope="module")
def tracers(mcrt):
    cache = {}

    def get(cid):
        if cid not in cache:
            scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
            g = np.load(os.path.join(GOLDEN, cid + ".npz"))
            cls = mcrt.PhotonMapper if scene.photon_maps() is not None else mcrt.PathTracer
            pt = cls(scene, precision=mcrt.PRECISION_F64, global_seed=int(g["seed"]))
            cache[cid] = (pt, scene, g)
        return cache[cid]
    yield get
    for pt, _, _ in cache.values():
        pt.close()


@pytest.fixture(scope="module")
def films():
    k = np.load(os.path.join(GOLDEN, "film_kat.npz"))
    return json.loads(str(k["films"])), int(k["seed"])


def zeros(*shape):
    import torch
    return torch.zeros(shape, dtype=torch.float64, device="cuda")


def pixels_of(mask, tile, rows, width):
    """Per-pixel bool [rows, width] of a tile mask."""
    return np.repeat(np.repeat(np.asarray(mask, bool), tile, 0), tile, 1)[:rows, :width]


def pattern(shape, k):
    """A fixed set of tiles: (ty + 2 tx) % 3 == k."""
    ty, tx = np.indices(shape)
    return (ty + 2 * tx) % 3 == k


# ---------------------------------------------------------------------------------------------- 1. every tile active
def accumulate_both_ways(mcrt, pt, cam, first, count, y_first=0, y_step=1, tile=16):
    import torch
    n_rows = len(range(y_first, cam.height, y_step))
    a, b = zeros(n_rows, cam.width, 3), zeros(n_rows, cam.width, 3)
    torch.cuda.synchronize()
    st_a = pt.render_accumulate_dev(cam, a.data_ptr(), None, first, count, y_first, y_step, n_rows)
    st_b = pt.render_accumulate_tiles_dev(cam, b.data_ptr(), None, first, count, tile,
                                          np.ones(mcrt.tile_grid(n_rows, cam.width, tile), bool), y_first, y_step, n_rows)
    A, B = a.cpu().numpy(), b.cpu().numpy()
    assert np.allclose(B, A, rtol=RTOL, atol=ATOL), np.abs(B - A).max()
    assert A.any()
    for k in STATS:
        assert st_a[k] == st_b[k], k
    assert st_b["paths"] == n_rows * cam.width * count


@pytest.mark.parametrize("cid", golden_cases())
def test_all_tiles_active_equals_accumulate(cid, mcrt, tracers):
    pt, scene, _ = tracers(cid)
    accumulate_both_ways(mcrt, pt, scene.cameras()[0], 2, 5)


def test_all_tiles_active_fast_mode_and_row_shard(mcrt, tracers):
    _, scene, g = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0]
    fast = mcrt.PathTracer(scene, precision=mcrt.PRECISION_F32, global_seed=int(g["seed"]))
    try:
        accumulate_both_ways(mcrt, fast, cam, 1, 6, tile=7)
    finally:
        fast.close()
    pt, _, _ = tracers("c2_hexagon_room_96")
    accumulate_both_ways(mcrt, pt, cam, 3, 4, y_first=1, y_step=3)
    pm, pscene, _ = tracers("pm_hexagon_room_64")
    accumulate_both_ways(mcrt, pm, pscene.cameras()[0], 0, 3, tile=5)


# ---------------------------------------------------------------------------------------------- 2. fixed schedule
PASSES = (2, 3, 1, 4, 2, 3)     # tiles retired after pass 2 have 5 samples, after pass 4 10, the rest 15


@pytest.mark.parametrize("cid,kw", [("c2_hexagon_room_96", {}), ("pm_hexagon_room_64", {}),
                                    ("c2_hexagon_room_96", {"y_first": 1, "y_step": 3}),
                                    ("c2_hexagon_room_96", {"tile": 7})])
def test_fixed_retirement_schedule(cid, kw, mcrt, tracers):
    pt, scene, _ = tracers(cid)
    cam = scene.cameras()[0]
    prog = mcrt.Progressive(pt, cam, **kw)
    tile, rows, width = prog.tile, prog.rows, cam.width
    assert prog.active.shape == mcrt.tile_grid(rows, width, tile)
    frozen = np.zeros((rows, width), bool)
    snapshot = None
    for k, s in enumerate(PASSES):
        prog.add(s)
        if snapshot is not None:   # the retired tiles' sums do not change, bit for bit
            for h in (0, 1):
                now = prog.rgb[h].cpu().numpy()
                assert np.array_equal(now[frozen], snapshot[h][frozen])
        if k in (1, 3):
            prog.retire(pattern(prog.active.shape, k // 2))
            frozen = pixels_of(~prog.active, tile, rows, width)
            snapshot = [prog.rgb[h].cpu().numpy() for h in (0, 1)]
    totals = prog.tile_counts.sum(-1)
    assert set(np.unique(totals)) == {5, 10, 15}
    assert np.array_equal(totals == 5, pattern(prog.active.shape, 0))
    assert prog.counts == [5, 10] and prog.samples == 15
    n_t = mcrt.tile_pixel_counts(rows, width, tile)
    assert prog.stats["paths"] == int((n_t * totals).sum())
    frame = prog.frame()
    assert frame.shape == (rows, width, 3)
    for c in (5, 10, 15):
        uniform = mcrt.Progressive(pt, cam, **kw)
        uniform.add(c)
        sel = pixels_of(totals == c, tile, rows, width)
        assert np.allclose(frame[sel], uniform.frame()[sel], rtol=RTOL, atol=ATOL), (c, np.abs(frame[sel] - uniform.frame()[sel]).max())
    err, tiles = prog.error()
    assert np.isfinite(err) and np.all(np.isfinite(tiles))


# ---------------------------------------------------------------------------------------------- 3. filters are additive
@pytest.mark.parametrize("name", ["mitchell", "lanczos_cached", "box_r1p5"])
def test_filtered_tile_passes_add_up(name, mcrt, films):
    import torch
    spec, seed = films
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "film_hexagon_room_64.mcrtpack"))
    cam = scene.cameras()[0]
    cam.film = spec[name]
    pt = mcrt.PathTracer(scene, precision=mcrt.PRECISION_F64, global_seed=seed)
    try:
        tile = 9
        grid = mcrt.tile_grid(cam.height, cam.width, tile)
        mask = np.random.default_rng(5).random(grid) < 0.4
        assert mask.any() and not mask.all()
        full = (zeros(cam.height, cam.width, 3), zeros(cam.height, cam.width))
        split = (zeros(cam.height, cam.width, 3), zeros(cam.height, cam.width))
        torch.cuda.synchronize()
        st = pt.render_accumulate_dev(cam, full[0].data_ptr(), full[1].data_ptr(), 1, 4)
        st_m = pt.render_accumulate_tiles_dev(cam, split[0].data_ptr(), split[1].data_ptr(), 1, 4, tile, mask)
        st_c = pt.render_accumulate_tiles_dev(cam, split[0].data_ptr(), split[1].data_ptr(), 1, 4, tile, ~mask)
        for f, s in zip(full, split):
            assert np.allclose(s.cpu().numpy(), f.cpu().numpy(), rtol=RTOL, atol=ATOL)
        for k in STATS:
            assert st_m[k] + st_c[k] == st[k]
    finally:
        pt.close()


# ---------------------------------------------------------------------------------------------- 4. the estimator
def resolve_reference_tiles(A, wA, B, wB, counts, tile):
    """float64 numpy restatement of mcrt_progressive_resolve_tiles_dev. wA/wB None: box film (weight = the tile's
    count). A or B None: that half has no samples in any tile. -> frame, frame error, tile errors, tile sums."""
    rows, width = (A if A is not None else B).shape[:2]
    ty, tx = -(-rows // tile), -(-width // tile)
    per_pixel = np.repeat(np.repeat(np.asarray(counts, np.float64), tile, 0), tile, 1)[:rows, :width]
    na, nb = per_pixel[..., 0], per_pixel[..., 1]
    both = (na > 0) & (nb > 0)
    zero = np.zeros((rows, width, 3))
    weighted = wA is not None or wB is not None
    wa = np.zeros((rows, width)) if A is None else (wA if weighted else na)
    wb = np.zeros((rows, width)) if B is None else (wB if weighted else nb)
    sa, sb = (zero if A is None else A), (zero if B is None else B)
    w = (wa + wb)[..., None]
    with np.errstate(divide="ignore", invalid="ignore"):
        frame = np.maximum(np.where(w == 0.0, 0.0, (sa + sb) / w), 0.0)
        scale = np.where(both, na * nb / (na + nb) ** 2, 0.0)[..., None]
        compare = (both & (wa != 0.0) & (wb != 0.0))[..., None]
        d = sa / wa[..., None] - sb / wb[..., None]
        v = np.where(compare, d * d * scale, 0.0)

    def rel(sv, si, has_both):
        if not has_both:
            return np.inf
        if sv == 0.0:
            return 0.0
        return np.sqrt(sv / si) if si > 0.0 else np.inf
    tiles, sums = np.zeros((ty, tx)), np.zeros((ty, tx, 2))
    for j in range(ty):
        for i in range(tx):
            sl = (slice(j * tile, (j + 1) * tile), slice(i * tile, (i + 1) * tile))
            sums[j, i] = v[sl].sum(), (frame[sl] ** 2).sum()
            tiles[j, i] = rel(*sums[j, i], counts[j, i, 0] > 0 and counts[j, i, 1] > 0)
    return frame, rel(v.sum(), (frame ** 2).sum(), bool(np.all(np.asarray(counts) > 0))), tiles, sums


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("tile", [1, 5, 16])
def test_estimator_with_tile_counts_matches_numpy(filtered, tile, mcrt, tracers):
    import torch
    pt, _, _ = tracers("c2_hexagon_room_96")
    rng = np.random.default_rng(17 + tile + filtered)
    rows, width = 23, 37                                   # tiles that divide neither
    ty, tx = mcrt.tile_grid(rows, width, tile)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda() if x is not None else None
    cases = []
    counts = rng.integers(1, 9, (ty, tx, 2))              # unequal nA, nB per tile
    counts[-1, 0] = (3, 0)                                 # a tile with an empty half: +inf
    cases.append(counts)
    cases.append(rng.integers(1, 9, (ty, tx, 2)))          # every tile has both halves: finite
    empty_b = rng.integers(1, 9, (ty, tx, 2))
    empty_b[..., 1] = 0                                    # B has no samples anywhere: passed as NULL
    cases.append(empty_b)
    for counts in cases:
        per_pixel = np.repeat(np.repeat(counts, tile, 0), tile, 1)[:rows, :width]
        A = rng.uniform(-0.05, 1.0, (rows, width, 3)) * per_pixel[..., :1]
        B = rng.uniform(-0.05, 1.0, (rows, width, 3)) * per_pixel[..., 1:]
        A[:3, :4] = B[:3, :4] = 0.0                        # a black corner: both halves agree
        wA = wB = None
        if filtered:
            wA = rng.uniform(0.2, 1.5, (rows, width)) * per_pixel[..., 0]
            wB = rng.uniform(0.2, 1.5, (rows, width)) * per_pixel[..., 1]
            wA[rng.random((rows, width)) < 0.05] = 0.0     # zero-weight pixels
        has_b = bool(counts[..., 1].any())
        tA, twA, tB, twB = dev(A), dev(wA), dev(B) if has_b else None, dev(wB) if has_b else None
        out = zeros(rows, width, 3)
        tiles, sums = zeros(ty, tx), zeros(ty, tx, 2)
        torch.cuda.synchronize()
        p = lambda t: t.data_ptr() if t is not None else None
        err = pt.progressive_resolve_tiles_dev(p(tA), p(twA), p(tB), p(twB), counts, width, rows, tile, out.data_ptr(),
                                               tiles.data_ptr(), sums.data_ptr())
        ref_frame, ref_err, ref_tiles, ref_sums = resolve_reference_tiles(A, wA, B if has_b else None, wB if has_b else None,
                                                                          counts, tile)
        assert np.allclose(out.cpu().numpy(), ref_frame, rtol=1e-12, atol=0)
        got_tiles = tiles.cpu().numpy()
        assert np.array_equal(np.isinf(got_tiles), np.isinf(ref_tiles))
        assert np.allclose(got_tiles, ref_tiles, rtol=1e-12, atol=0)
        assert np.allclose(sums.cpu().numpy(), ref_sums, rtol=1e-12, atol=1e-300)
        assert (err == np.inf) == (ref_err == np.inf) and np.isclose(err, ref_err, rtol=1e-12, atol=0)
        assert (err == np.inf) == bool(np.any(counts == 0))


def test_uniform_tile_counts_equal_the_scalar_resolve(mcrt, tracers):
    pt, scene, _ = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0]
    prog = mcrt.Progressive(pt, cam)
    for s in (2, 3):
        prog.add(s)
    frame, err, tiles, _ = prog._resolve()
    sums = prog.tile_sums()                                # through mcrt_progressive_resolve_tiles_dev
    frame_t, err_t, tiles_t, _ = prog._resolve()
    assert np.array_equal(frame_t, frame)
    assert np.isclose(err_t, err, rtol=1e-12) and np.allclose(tiles_t, tiles, rtol=1e-12)
    assert np.isclose(np.sqrt(sums[..., 0].sum() / sums[..., 1].sum()), err, rtol=1e-12)


# ---------------------------------------------------------------------------------------------- 5. render_adaptive
def check_history(mcrt, prog, target, min_samples):
    """Every recorded decision is the pure rule applied to the sums the run reported."""
    n_t = mcrt.tile_pixel_counts(prog.rows, prog.camera.width, prog.tile)
    active = np.ones(prog.active.shape, bool)
    first = 0
    for k, e in enumerate(prog.history):
        assert e["first"] == first and e["active"] == active.sum()
        assert np.all(e["tile_counts"][active].sum(-1) == first + e["count"])
        if np.isfinite(e["error"]):
            assert np.isclose(np.sqrt(e["tile_sums"][..., 0].sum() / e["tile_sums"][..., 1].sum()), e["error"], rtol=1e-9)
        if e["error"] <= target:
            assert k == len(prog.history) - 1 and prog.stop_reason == "target" and not e["retired"].any()
        else:
            want = mcrt.adaptive_retire(active, e["tile_counts"], e["tile_sums"], n_t, target, min_samples)
            assert np.array_equal(e["retired"], want), k
        active &= ~e["retired"]
        first += e["count"]
    assert np.array_equal(active, prog.active)
    return sum(int(e["retired"].sum()) for e in prog.history)


def test_render_adaptive_follows_its_rule(mcrt, tracers):
    pt, scene, _ = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0]
    probe = mcrt.Progressive(pt, cam)
    probe.render(4, 16)
    target = 0.6 * probe.error()[0]
    prog = mcrt.Progressive(pt, cam)
    frame = prog.render_adaptive(4, 128, target, min_samples=8)
    assert prog.stop_reason == "target" and prog.error()[0] <= target and prog.samples < 128
    assert check_history(mcrt, prog, target, 8) > 0           # some tiles retired before the frame met the target
    n_t = mcrt.tile_pixel_counts(prog.rows, cam.width, prog.tile)
    assert prog.stats["paths"] == int((n_t * prog.tile_counts.sum(-1)).sum())
    assert np.array_equal(frame, prog.frame())

    # no target that can be met: it runs until the active tiles reach max_samples
    capped = mcrt.Progressive(pt, cam)
    capped.render_adaptive(8, 32, 0.0, min_samples=8)
    assert capped.stop_reason == "max_samples" and capped.samples == 32
    check_history(mcrt, capped, 0.0, 8)
    assert all(e["error"] > 0.0 for e in capped.history)

    # nothing left to render
    done = mcrt.Progressive(pt, cam)
    done.add(4)
    done.retire(np.ones(done.active.shape, bool))
    done.render_adaptive(4, 64, 0.01)
    assert done.stop_reason == "no active tile" and done.history == [] and done.samples == 4


# ---------------------------------------------------------------------------------------------- 6. checkpoint / resume
def schedule(prog, steps):
    for s in steps:
        if isinstance(s, int):
            prog.add(s)
        else:
            prog.retire(pattern(prog.active.shape, s[1]))


STEPS = [2, 3, ("retire", 0), 1, 4, ("retire", 1), 2, 3]


@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "pm_hexagon_room_64"])
def test_resume_with_retired_tiles(cid, mcrt, tracers, tmp_path):
    pt, scene, g = tracers(cid)
    cam = scene.cameras()[0]
    whole = mcrt.Progressive(pt, cam)
    schedule(whole, STEPS)
    cls, seed = type(pt), int(g["seed"])
    path = str(tmp_path / "adaptive.npz")
    first = cls(scene, global_seed=seed)
    try:
        part = mcrt.Progressive(first, cam)
        schedule(part, STEPS[:4])
        part.save(path)
    finally:
        first.close()
    second = cls(scene, global_seed=seed)
    try:
        resumed = mcrt.Progressive.load(path, second, cam)
        assert np.array_equal(resumed.active, ~pattern(resumed.active.shape, 0))
        schedule(resumed, STEPS[4:])
        assert np.array_equal(resumed.active, whole.active)
        assert np.array_equal(resumed.tile_counts, whole.tile_counts) and resumed.counts == whole.counts
        assert np.allclose(resumed.frame(), whole.frame(), rtol=RTOL, atol=ATOL)
        with pytest.raises(mcrt.McrtError, match="tile differs"):
            mcrt.Progressive.load(path, second, cam, tile=8)
    finally:
        second.close()


def test_checkpoint_without_tile_state_loads_all_active(mcrt, tracers, tmp_path):
    pt, scene, _ = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0]
    path = str(tmp_path / "old.npz")
    prog = mcrt.Progressive(pt, cam)
    prog.add(1)
    prog.add(2)
    prog.save(path)
    with np.load(path) as z:                               # the format written before adaptive sampling
        data = {k: z[k] for k in z.files if k not in ("active", "tile_counts")}
    with open(path, "wb") as f:
        np.savez(f, **data)
    old = mcrt.Progressive.load(path, pt, cam)
    assert old.active.all() and np.all(old.tile_counts == [1, 2])
    schedule(old, [("retire", 0), 4, 3])
    ref = mcrt.Progressive(pt, cam)
    schedule(ref, [1, 2, ("retire", 0), 4, 3])
    assert np.array_equal(old.tile_counts, ref.tile_counts)
    assert np.allclose(old.frame(), ref.frame(), rtol=RTOL, atol=ATOL)


# ---------------------------------------------------------------------------------------------- 7. refused arguments
def test_refused_arguments(mcrt, tracers):
    import torch
    pt, scene, _ = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0]
    L = mcrt.lib()
    pt.set_film(cam)
    rgb = zeros(cam.height, cam.width, 3)
    wsum = zeros(cam.height, cam.width)
    torch.cuda.synchronize()
    st = mcrt.Stats()
    tile = 16
    grid = mcrt.tile_grid(cam.height, cam.width, tile)
    ones = np.ones(grid, np.uint8)
    none = np.zeros(grid, np.uint8)

    def accumulate(first, count, weight=None, tile=tile, mask=ones, y_first=0, y_step=1, n_rows=cam.height, camera=cam):
        m = mask.ctypes.data_as(C.c_void_p) if mask is not None else None
        return L.mcrt_render_accumulate_tiles_dev(pt.ctx, C.byref(camera.rec), y_first, y_step, n_rows, tile, m, first, count,
                                                  pt.global_seed, pt.kind, pt.precision, C.c_void_p(rgb.data_ptr()), weight,
                                                  C.byref(st))

    def refused(rc, words, code=-1):
        assert rc == code, rc
        msg = L.mcrt_last_error(pt.ctx).decode()
        assert words in msg, msg

    refused(accumulate(0, 1, tile=0), "tile is 0")
    refused(accumulate(0, 1, mask=None), "mask")
    refused(accumulate(0, 1, mask=none), "no active tile")
    refused(accumulate(0, 0), "sample_count")
    refused(accumulate(0xFFFFFFFF, 2), "2^32")
    refused(accumulate(0, 1, weight=C.c_void_p(wsum.data_ptr())), "weight")
    refused(accumulate(0, 1, y_first=cam.height), "row range")
    refused(accumulate(0, 1, y_step=0), "row range")
    cam_f = cam.resized(cam.width, cam.height)
    cam_f.film = {"filter": "mitchell-netravali"}
    pt.set_film(cam_f)
    try:
        half = np.ones(mcrt.tile_grid(len(range(0, cam.height, 2)), cam.width, tile), np.uint8)
        refused(accumulate(0, 1, weight=C.c_void_p(wsum.data_ptr()), mask=half, y_step=2, n_rows=len(range(0, cam.height, 2)),
                           camera=cam_f), "whole frame", code=-4)
        refused(accumulate(0, 1, camera=cam_f), "weight_sum_dev")
    finally:
        pt.set_film(cam)
    torch.cuda.synchronize()
    assert rgb.abs().sum().item() == 0.0 and wsum.abs().sum().item() == 0.0    # nothing was rendered

    out = zeros(cam.height, cam.width, 3)
    torch.cuda.synchronize()
    err = C.c_double()
    P = lambda t: C.c_void_p(t.data_ptr())
    counts = np.ones(grid + (2,), np.uint32)
    cp = lambda c: c.ctypes.data_as(C.c_void_p)

    def resolve(a, b, counts_ptr, tile=tile):
        return L.mcrt_progressive_resolve_tiles_dev(pt.ctx, a, None, b, None, counts_ptr, cam.width, cam.height, tile, P(out),
                                                    None, None, C.byref(err))
    refused(resolve(P(rgb), P(rgb), cp(counts), tile=0), "tile is 0")
    refused(resolve(P(rgb), P(rgb), None), "tile_samples")
    refused(resolve(P(rgb), P(rgb), cp(np.zeros_like(counts))), "no samples")
    refused(resolve(None, P(rgb), cp(counts)), "null sums")
    assert out.abs().sum().item() == 0.0


# ---------------------------------------------------------------------------------------------- 8. quality
def test_adaptive_error_against_an_independent_reference(mcrt, tracers, capsys):
    """The two-half estimate cannot see bias from retiring tiles too early; a 1024-spp frame of another seed can."""
    pt, scene, g = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54, 32)             # 1024 spp
    other = mcrt.PathTracer(scene, global_seed=int(g["seed"]) + 1)
    try:
        ref = other.render_rows(cam)
    finally:
        other.close()
    probe = mcrt.Progressive(pt, cam)
    probe.render(8, 64)
    target = probe.error()[0]                              # what uniform sampling reaches at about 64 spp
    prog = mcrt.Progressive(pt, cam)
    frame = prog.render_adaptive(8, 1024, target)
    assert prog.stop_reason == "target"
    measured = float(np.sqrt(np.sum((frame - ref) ** 2) / np.sum(ref ** 2)))
    n_t = mcrt.tile_pixel_counts(prog.rows, cam.width, prog.tile)
    adaptive_spp = float((n_t * prog.tile_counts.sum(-1)).sum()) / n_t.sum()
    uniform = mcrt.Progressive(pt, cam)
    # the probe's own error may differ from a rerun's in the last bits (order of the film additions)
    uniform.render(8, 1024, target_error=target * (1 + 1e-9))
    with capsys.disabled():
        print(f"\nc2_hexagon_room_96 96x54 target {target:.5f}: adaptive {adaptive_spp:.1f} spp on average "
              f"({len(prog.history)} passes, {int(prog.active.sum())}/{prog.active.size} tiles active at the end), "
              f"uniform {uniform.samples} spp; error against 1024 spp of another seed {measured:.5f} "
              f"({measured / target:.3f} x target)")
    assert measured <= 1.5 * target, (measured, target)
