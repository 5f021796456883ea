"""Progressive rendering (mcrt_render_accumulate_dev, mcrt_progressive_resolve_dev and the Progressive class): sample
passes of uneven sizes, resolved from the two halves A and B, must give the one-shot frame of the same samples up to the
order of the float64 film additions (the bar of test_render_is_repeatable_and_seed_dependent: rtol 1e-12, atol 1e-14),
and so meet the reference's golden images like mcrt_render_rows. The noise estimate is checked against a float64
numpy restatement and against the error measured between two independent seeds."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-12, 1e-14


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


def uneven(n):
    """Pass sizes 1, 2 and the rest of n samples (as many as fit)."""
    parts = []
    for s in (1, 2):
        if sum(parts) + s < n:
            parts.append(s)
    return parts + [n - sum(parts)]


def progressive(mcrt, pt, cam, passes, **kw):
    prog = mcrt.Progressive(pt, cam, **kw)
    for s in passes:
        prog.add(s)
    return prog


# ---------------------------------------------------------------------------------------------- 1. every golden case
@pytest.mark.parametrize("cid", golden_cases())
def test_passes_equal_one_shot_and_reference(cid, mcrt, tracers):
    pt, scene, g = tracers(cid)
    cam = scene.cameras()[0]
    n = cam.sqrtspp ** 2
    one = pt.render_rows(cam)
    st = pt.last_stats
    prog = progressive(mcrt, pt, cam, uneven(n))
    img = prog.frame()
    assert prog.samples == n and img.shape == one.shape
    assert np.allclose(img, one, rtol=RTOL, atol=ATOL), np.abs(img - one).max()
    ref = g["image"]
    rmse = float(np.sqrt(np.mean((img - ref) ** 2)))
    assert rmse / max(1.0, float(np.abs(ref).mean())) < (1e-6 if cid.startswith("pm_") else 1e-9), f"rmse {rmse:.3e}"
    assert prog.stats["paths"] == st["paths"] == cam.width * cam.height * n
    assert prog.stats["extension_rays"] == st["extension_rays"]


# ---------------------------------------------------------------------------------------------- 2. filters, fast mode
@pytest.mark.parametrize("name", ["mitchell", "lanczos_cached", "box_r1p5"])
def test_filtered_passes_equal_one_shot(name, mcrt, films):
    spec, seed = films
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "film_hexagon_room_64.mcrtpack"))
    cam = scene.cameras()[0]
    cam.film = spec[name]
    pt = mcrt.PathTracer(scene, precision=mcrt.PRECISION_F64, global_seed=seed)
    try:
        one = pt.render_rows(cam)
        prog = progressive(mcrt, pt, cam, uneven(cam.sqrtspp ** 2))
        assert prog.filtered
        assert np.allclose(prog.frame(), one, rtol=RTOL, atol=ATOL)
        k = np.load(os.path.join(GOLDEN, "film_kat.npz"))
        assert np.abs(prog.frame() - k["image_" + name]).max() <= 1e-9 * max(1.0, np.abs(k["image_" + name]).max())
    finally:
        pt.close()


def test_fast_mode_passes_equal_one_shot(mcrt, tracers):
    _, scene, g = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54, 4)
    pt = mcrt.PathTracer(scene, precision=mcrt.PRECISION_F32, global_seed=int(g["seed"]))
    try:
        one = pt.render_rows(cam)
        prog = progressive(mcrt, pt, cam, [1, 3, 12])
        assert np.allclose(prog.frame(), one, rtol=RTOL, atol=ATOL)
    finally:
        pt.close()


# ---------------------------------------------------------------------------------------------- 3. row shards
def test_strided_row_passes_equal_one_shot_rows(mcrt, tracers):
    pt, scene, _ = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54, 3)
    full = pt.render_rows(cam)
    world = 3
    for rank in range(world):
        prog = progressive(mcrt, pt, cam, [1, 3, 5], y_first=rank, y_step=world)
        assert np.allclose(prog.frame(), full[rank::world], rtol=RTOL, atol=ATOL)


def test_filtered_row_shards_add_up_to_the_frame(mcrt, films):
    """With a filter, each shard's unreduced sums cover any set of rows; their sum over the shards resolves to the frame."""
    import torch
    spec, seed = films
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "film_hexagon_room_64.mcrtpack"))
    cam = scene.cameras()[0]
    cam.film = spec["mitchell"]
    pt = mcrt.PathTracer(scene, precision=mcrt.PRECISION_F64, global_seed=seed)
    try:
        one = pt.render_rows(cam)
        n = cam.sqrtspp ** 2
        total = [torch.zeros((cam.height, cam.width, 3), dtype=torch.float64, device="cuda"),
                 torch.zeros((cam.height, cam.width), dtype=torch.float64, device="cuda")]
        for rank in range(3):
            prog = progressive(mcrt, pt, cam, uneven(n), y_first=rank, y_step=3)
            total[0] += prog.rgb[0] + prog.rgb[1]
            total[1] += prog.wsum[0] + prog.wsum[1]
        out = torch.empty_like(total[0])
        torch.cuda.synchronize()
        pt.progressive_resolve_dev(total[0].data_ptr(), total[1].data_ptr(), n, None, None, 0, cam.width, cam.height, 16, out.data_ptr())
        assert np.allclose(out.cpu().numpy(), one, rtol=RTOL, atol=ATOL)
    finally:
        pt.close()


# ---------------------------------------------------------------------------------------------- 4. checkpoint / resume
@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "pm_hexagon_room_64"])
def test_resume_from_checkpoint_equals_one_shot(cid, mcrt, tracers, tmp_path):
    pt, scene, g = tracers(cid)
    cam = scene.cameras()[0].resized(scene.cameras()[0].width, scene.cameras()[0].height, 3)
    one = pt.render_rows(cam)
    cls = type(pt)
    seed = int(g["seed"])
    first = cls(scene, global_seed=seed)
    prog = progressive(mcrt, first, cam, [1, 2, 3])
    path = str(tmp_path / "checkpoint.npz")
    prog.save(path)
    first.close()
    del prog

    second = cls(scene, global_seed=seed)
    try:
        resumed = mcrt.Progressive.load(path, second, cam)
        assert (resumed.samples, resumed.passes, resumed.counts) == (6, 3, [4, 2])
        resumed.add(3)
        assert resumed.counts == [4, 5]
        assert np.allclose(resumed.frame(), one, rtol=RTOL, atol=ATOL)
    finally:
        second.close()


def test_resume_is_refused_when_the_render_differs(mcrt, tracers, tmp_path):
    pt, scene, g = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0]
    seed = int(g["seed"])
    path = str(tmp_path / "c2.npz")
    progressive(mcrt, pt, cam, [1, 1]).save(path)
    assert mcrt.Progressive.load(path, pt, cam).samples == 2

    def refused(integrator, camera, what):
        with pytest.raises(mcrt.McrtError, match=what):
            mcrt.Progressive.load(path, integrator, camera)

    other = mcrt.PathTracer(scene, global_seed=seed + 1)
    refused(other, cam, "seed")
    other.close()
    fast = mcrt.PathTracer(scene, precision=mcrt.PRECISION_F32, global_seed=seed)
    refused(fast, cam, "precision")
    fast.close()
    moved = cam.resized(cam.width, cam.height)
    moved.rec.eye[0] += 1e-9
    refused(pt, moved, "camera")
    filtered = cam.resized(cam.width, cam.height)
    filtered.film = {"filter": "mitchell-netravali"}
    refused(pt, filtered, "film")
    c1, c1_scene, _ = tracers("oren_nayar_64")
    refused(c1, cam, "scene")
    edited = mcrt.Scene(dict(scene.a, **scene.extra))
    edited.a["materials"] = edited.a["materials"].copy()
    edited.a["materials"]["roughness"][0] += 0.25
    changed = mcrt.PathTracer(edited, global_seed=seed)
    refused(changed, cam, "scene")
    changed.close()

    # photon mapping: the integrator kind and the photons themselves are part of the identity
    pm, pscene, pg = tracers("pm_hexagon_room_64")
    pcam = pscene.cameras()[0]
    ppath = str(tmp_path / "pm.npz")
    progressive(mcrt, pm, pcam, [1, 1]).save(ppath)
    path_tracer = mcrt.PathTracer(pscene, global_seed=int(pg["seed"]))
    with pytest.raises(mcrt.McrtError, match="integrator"):
        mcrt.Progressive.load(ppath, path_tracer, pcam)
    path_tracer.close()
    caustic, glob, k, dv = pscene.photon_maps()
    glob = dict(glob, photons=glob["photons"].copy())
    glob["photons"][0] += 1e-3
    pm2 = mcrt.PhotonMapper(pscene, global_seed=int(pg["seed"]), photon_maps=(caustic, glob, k, dv))
    with pytest.raises(mcrt.McrtError, match="photon"):
        mcrt.Progressive.load(ppath, pm2, pcam)
    pm2.close()


# ---------------------------------------------------------------------------------------------- 5. the estimator
def resolve_reference(A, wA, nA, B, wB, nB, tile):
    """float64 numpy restatement of mcrt_progressive_resolve_dev. wA/wB None: box film (weight = sample count)."""
    rows, width = A.shape[:2]
    if wA is None:
        wA, wB = np.full((rows, width), float(nA)), np.full((rows, width), float(nB))
    w = (wA + wB)[..., None]
    with np.errstate(divide="ignore", invalid="ignore"):
        frame = np.where(w == 0.0, 0.0, (A + B) / w)
        frame = np.maximum(frame, 0.0)
        both = nA > 0 and nB > 0
        compare = (both & (wA != 0.0) & (wB != 0.0))[..., None]
        scale = nA * nB / float(nA + nB) ** 2 if both else 0.0
        d = A / wA[..., None] - B / wB[..., None]
        v = np.where(compare, d * d * scale, 0.0)

    def rel(sv, si):
        if not both:
            return np.inf
        if sv == 0.0:
            return 0.0
        return np.sqrt(sv / si) if si > 0.0 else np.inf
    ty, tx = -(-rows // tile), -(-width // tile)
    tiles = np.zeros((ty, tx))
    for j in range(ty):
        for i in range(tx):
            sl = (slice(j * tile, (j + 1) * tile), slice(i * tile, (i + 1) * tile))
            tiles[j, i] = rel(v[sl].sum(), (frame[sl] ** 2).sum())
    return frame, rel(v.sum(), (frame ** 2).sum()), tiles


def random_sums(rng, rows, width, n, filtered):
    rgb = rng.uniform(-0.05, 1.0, (rows, width, 3)) * n
    rgb[:3, :4] = 0.0                                      # a black corner: both halves agree
    if not filtered:
        return rgb, None
    w = rng.uniform(0.2, 1.5, (rows, width)) * n
    w[rng.random((rows, width)) < 0.05] = 0.0              # zero-weight pixels
    return rgb, w


@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("tile", [1, 5, 16, 64])
def test_estimator_matches_numpy(filtered, tile, mcrt, tracers):
    import torch
    pt, _, _ = tracers("c2_hexagon_room_96")
    rng = np.random.default_rng(7 + tile + filtered)
    rows, width = 23, 37                                   # tiles that divide neither
    for nA, nB in ((5, 3), (4, 4), (7, 0)):
        A, wA = random_sums(rng, rows, width, nA, filtered)
        B, wB = random_sums(rng, rows, width, max(nB, 1), filtered)
        if filtered:
            wA[5, 5] = wB[5, 5] = 0.0                      # a pixel no sample reached
        if nB == 0:                                        # an empty half is passed as NULL sums
            B[:] = 0.0
            if filtered:
                wB[:] = 0.0
        dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda() if x is not None else None
        tA, twA, tB, twB = dev(A), dev(wA), dev(B), dev(wB)
        out = torch.empty((rows, width, 3), dtype=torch.float64, device="cuda")
        tiles = torch.empty((-(-rows // tile), -(-width // tile)), dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        ptr = lambda t: t.data_ptr() if t is not None and nB else None
        err = pt.progressive_resolve_dev(tA.data_ptr(), twA.data_ptr() if filtered else None, nA, ptr(tB), ptr(twB), nB,
                                         width, rows, tile, out.data_ptr(), tiles.data_ptr())
        ref_frame, ref_err, ref_tiles = resolve_reference(A, wA, nA, B, wB, nB, tile)
        got_tiles = tiles.cpu().numpy()
        assert np.allclose(out.cpu().numpy(), ref_frame, rtol=1e-12, atol=0)
        assert np.allclose(got_tiles, ref_tiles, rtol=1e-12, atol=0)
        assert np.isclose(err, ref_err, rtol=1e-12, atol=0)
        if nB == 0:
            assert err == np.inf and np.all(got_tiles == np.inf)
        else:
            assert np.isfinite(err)
            if tile == 1:
                assert got_tiles[0, 0] == 0.0              # black in both halves
                if filtered:
                    assert got_tiles[5, 5] == 0.0          # no weight: a black pixel with no estimate



def test_estimator_against_independent_seeds(mcrt, tracers, capsys):
    """Owen-scrambled Sobol halves are not independent (each is better stratified than iid samples), so the estimate is
    expected to be conservative; it must never fall below 0.8x the error measured between two seeds."""
    pt, scene, g = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54, 8)             # 64 spp
    n = cam.sqrtspp ** 2
    seed = int(g["seed"])
    other = mcrt.PathTracer(scene, global_seed=seed + 1)
    try:
        i1, i2 = pt.render_rows(cam), other.render_rows(cam)
    finally:
        other.close()
    for pass_samples in (32, 8, 2):
        prog = progressive(mcrt, pt, cam, [pass_samples] * (n // pass_samples))
        est, _ = prog.error()
        frame = prog.frame()
        assert np.allclose(frame, i1, rtol=RTOL, atol=ATOL)
        measured = float(np.sqrt(np.sum((i1 - i2) ** 2) / 2 / np.sum(frame ** 2)))
        with capsys.disabled():
            print(f"\nc2_hexagon_room_96 96x54 {n} spp, passes of {pass_samples}: estimated {est:.5f}, "
                  f"measured between seeds {measured:.5f}, ratio {est / measured:.3f}")
        assert est >= 0.8 * measured, (pass_samples, est, measured)


# ---------------------------------------------------------------------------------------------- 6. stop at target
def test_render_stops_at_the_first_pass_within_target(mcrt, tracers):
    pt, scene, _ = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54, 8)
    probe = mcrt.Progressive(pt, cam)
    errs = []
    for _ in range(16):
        probe.add(4)
        errs.append(probe.error()[0])
    assert errs[0] == np.inf and all(np.isfinite(errs[1:]))
    # a rerun may differ in the last bits (order of the film additions): leave that much room
    target = errs[9] * (1 + 1e-9)
    expected = next(i for i, e in enumerate(errs) if e <= target) + 1
    prog = mcrt.Progressive(pt, cam)
    frame = prog.render(4, 64, target_error=target)
    assert prog.passes == expected and prog.samples == 4 * expected
    assert prog.error()[0] <= target
    single = progressive(mcrt, pt, cam, [prog.samples])
    assert single.error()[0] == np.inf
    assert np.allclose(frame, single.frame(), rtol=RTOL, atol=ATOL)
    # without a target it runs to max_samples
    full = mcrt.Progressive(pt, cam)
    full.render(24, 64)
    assert full.samples == 64 and full.passes == 3


# ---------------------------------------------------------------------------------------------- 7. refused arguments
def test_refused_arguments(mcrt, tracers):
    import torch
    pt, scene, g = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0]
    L = mcrt.lib()
    pt.set_film(cam)
    rgb = torch.zeros((cam.height, cam.width, 3), dtype=torch.float64, device="cuda")
    wsum = torch.zeros((cam.height, cam.width), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    st = mcrt.Stats()

    def accumulate(first, count, weight, y_first=0, y_step=1, n_rows=cam.height):
        return L.mcrt_render_accumulate_dev(pt.ctx, C.byref(cam.rec), y_first, y_step, n_rows, first, count, pt.global_seed,
                                            pt.kind, pt.precision, C.c_void_p(rgb.data_ptr()), weight, C.byref(st))

    def refused(rc, words):
        assert rc == -1, rc
        msg = L.mcrt_last_error(pt.ctx).decode()
        assert words in msg, msg

    refused(accumulate(0, 0, None), "sample_count")
    refused(accumulate(0xFFFFFFFF, 2, None), "2^32")
    refused(accumulate(2, 0xFFFFFFFF, None), "2^32")
    refused(accumulate(0, 1, C.c_void_p(wsum.data_ptr())), "weight")
    refused(accumulate(0, 1, None, y_first=cam.height), "row range")
    refused(accumulate(0, 1, None, y_step=0), "row range")
    assert rgb.abs().sum().item() == 0.0                     # nothing was rendered
    cam_f = cam.resized(cam.width, cam.height)
    cam_f.film = {"filter": "mitchell-netravali"}
    pt.set_film(cam_f)
    try:
        rc = L.mcrt_render_accumulate_dev(pt.ctx, C.byref(cam_f.rec), 0, 1, cam.height, 0, 1, pt.global_seed, pt.kind, pt.precision,
                                          C.c_void_p(rgb.data_ptr()), None, C.byref(st))
        refused(rc, "weight_sum_dev")
    finally:
        pt.set_film(cam)

    out = torch.empty_like(rgb)
    err = C.c_double()
    P = lambda t: C.c_void_p(t.data_ptr())
    refused(L.mcrt_progressive_resolve_dev(pt.ctx, P(rgb), None, 1, P(rgb), None, 1, cam.width, cam.height, 0, P(out), None,
                                           C.byref(err)), "tile")
    refused(L.mcrt_progressive_resolve_dev(pt.ctx, P(rgb), None, 0, None, None, 0, cam.width, cam.height, 16, P(out), None,
                                           C.byref(err)), "no samples")
    # the last sample of the 2^32 a pixel can have renders, and afterwards a real pass still matches one shot
    assert accumulate(0xFFFFFFFF, 1, None) == 0
    rgb.zero_()
    torch.cuda.synchronize()
    assert accumulate(0, cam.sqrtspp ** 2, None) == 0
    assert pt.progressive_resolve_dev(rgb.data_ptr(), None, cam.sqrtspp ** 2, None, None, 0, cam.width, cam.height, 16,
                                      out.data_ptr()) == np.inf
    assert np.allclose(out.cpu().numpy(), pt.render_rows(cam), rtol=RTOL, atol=ATOL)
