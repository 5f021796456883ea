"""Denoising film planes (mcrt_denoise_planes_dev, Progressive.denoise_planes / relight_denoised): the kernels against
their numpy restatement (tests/denoise_planes_ref.py), the guide's frame against mcrt_denoise_dev bit for bit,
every kind of plane render, quality against an independent high-sample reference, and the refusals."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import denoise_ref as dr
import denoise_planes_ref as dpr
from test_gpu_photon_light_groups import emit_params

pytestmark = pytest.mark.gpu

SIGMAS = ("sigma_color", "sigma_normal", "sigma_depth", "sigma_albedo")
DEFAULT_SIGMAS = dict(sigma_color=1.0, sigma_normal=64.0, sigma_depth=0.1, sigma_albedo=0.1)
INVALID = -1   # MCRT_ERR_INVALID


def load(mcrt, cid):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    return scene, int(np.load(os.path.join(GOLDEN, cid + ".npz"))["seed"])


@pytest.fixture(scope="module")
def c2(mcrt):
    scene, seed = load(mcrt, "c2_hexagon_room_96")
    pt = mcrt.PathTracer(scene, global_seed=seed)
    yield pt, scene, seed
    pt.close()


def zeros(*shape):
    import torch
    t = torch.zeros(shape, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    return t


def device(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a, np.float64)).cuda()
    torch.cuda.synchronize()
    return t


# ---------------------------------------------------------------------------------------------- 1. the kernels
def random_planes(rng, n_planes, h, w, tile, uneven):
    """Box-film planes whose sums are the guide's: -> (a, wa, b, wb, counts, features, planes a, planes b)."""
    ty, tx = -(-h // tile), -(-w // tile)
    counts = rng.integers(1, 9, (ty, tx, 2)) if uneven else np.full((ty, tx, 2), 4)
    wa, wb = dr.pixel_weights(counts, tile, h, w)
    base = rng.uniform(0.0, 2.0, (n_planes, h, w, 3)) / n_planes
    pa = np.maximum(0.0, base + rng.normal(0, 0.3 / n_planes, base.shape)) * wa[None, ..., None]
    pb = np.maximum(0.0, base + rng.normal(0, 0.3 / n_planes, base.shape)) * wb[None, ..., None]
    a, b = pa[0].copy(), pb[0].copy()
    for k in range(1, n_planes):   # the combine kernel's order
        a += pa[k]; b += pb[k]
    hits = rng.integers(0, 5, (h, w)).astype(np.float64)
    f = np.zeros((h, w, 8))
    f[..., 0:3] = rng.uniform(0, 1, (h, w, 3)).round(1) * hits[..., None]
    f[..., 3:6] = (rng.normal(size=(h, w, 3)) + [0, 0, 3]) * hits[..., None]
    f[..., 6] = rng.uniform(1, 3, (h, w)) * hits
    f[..., 7] = hits
    return a, wa, b, wb, counts, f, pa, pb


def run_planes(pt, a, b, pa, pb, counts, tile, f, params, with_frame=True):
    """-> (filtered plane sums A, B, guide frame or None, its error or None)"""
    n, h, w = pa.shape[:3]
    A, B, PA, PB, F = device(a), device(b), device(pa), device(pb), device(f)
    OA, OB, out = zeros(n, h, w, 3), zeros(n, h, w, 3), zeros(h, w, 3)
    err = pt.denoise_planes_dev(A.data_ptr(), B.data_ptr(), PA.data_ptr(), PB.data_ptr(), n, counts, tile, F.data_ptr(), w, h,
                                OA.data_ptr(), OB.data_ptr(), params, out.data_ptr() if with_frame else None)
    return OA.cpu().numpy(), OB.cpu().numpy(), out.cpu().numpy() if with_frame else None, err


def run_denoise(pt, a, b, counts, tile, f, params):
    h, w = a.shape[:2]
    A, B, F, out = device(a), device(b), device(f), zeros(h, w, 3)
    err = pt.denoise_dev(A.data_ptr(), None, B.data_ptr(), None, counts, tile, F.data_ptr(), w, h, out.data_ptr(), params)
    return out.cpu().numpy(), err


def params_of(mcrt, iterations, sig):
    return mcrt.DenoiseParams(iterations, 0, sig["sigma_color"], sig["sigma_normal"], sig["sigma_depth"], sig["sigma_albedo"])


@pytest.mark.parametrize("uneven", [False, True])
@pytest.mark.parametrize("tile", [1, 5, 16])
@pytest.mark.parametrize("iterations", [0, 1, 5])
@pytest.mark.parametrize("n_planes", [1, 4, 31])
@pytest.mark.parametrize("off", [None] + list(SIGMAS))
def test_kernels_match_the_restatement(uneven, tile, iterations, n_planes, off, mcrt, c2):
    if off is not None and (iterations != 5 or tile != 5 or n_planes != 4):
        pytest.skip("each sigma is switched off at 5 iterations, tile 5, 4 planes")
    pt = c2[0]
    rng = np.random.default_rng(zlib.crc32(repr((uneven, tile, iterations, n_planes, off)).encode()))
    a, wa, b, wb, counts, f, pa, pb = random_planes(rng, n_planes, 45, 67, tile, uneven)
    sig = dict(DEFAULT_SIGMAS)
    if off:
        sig[off] = 0.0
    params = params_of(mcrt, iterations, sig)
    oa, ob, frame, err = run_planes(pt, a, b, pa, pb, counts, tile, f, params)
    wa_, wb_, (want_frame, want_err, _), _ = dpr.denoise_planes(a, wa, b, wb, f, pa, pb, iterations, **sig)
    scale = max(pa.max(), pb.max())
    np.testing.assert_allclose(oa, wa_, rtol=1e-9, atol=1e-12 * scale)
    np.testing.assert_allclose(ob, wb_, rtol=1e-9, atol=1e-12 * scale)
    np.testing.assert_allclose(frame, want_frame, rtol=1e-9, atol=1e-12)
    # the guide's frame is mcrt_denoise_dev's, bit for bit; its error is summed with float64 atomics, whose order
    # differs from call to call, so it is compared to rounding here and bit for bit in the two-warp test below
    ref, ref_err = run_denoise(pt, a, b, counts, tile, f, params)
    assert np.array_equal(frame, ref)
    assert err == pytest.approx(ref_err, rel=1e-13)
    # the plane passes have no atomics: a second call gives the same bits, with or without the guide's frame
    oa2, ob2, _, none = run_planes(pt, a, b, pa, pb, counts, tile, f, params, with_frame=False)
    assert none is None and np.array_equal(oa2, oa) and np.array_equal(ob2, ob)


def test_a_plane_equal_to_the_guide_is_filtered_exactly_like_it(mcrt, c2):
    """Two warps: the guide's error has two float64 atomic additions per sum, which commute, so it is bit-exact too."""
    pt = c2[0]
    for h, w, tile in ((2, 32, 5), (45, 67, 16)):
        rng = np.random.default_rng(h * 1000 + w)
        a, wa, b, wb, counts, f, pa, pb = random_planes(rng, 3, h, w, tile, True)
        params = params_of(mcrt, 5, DEFAULT_SIGMAS)
        planes_a = np.concatenate([a[None], pa]); planes_b = np.concatenate([b[None], pb])
        oa, ob, frame, err = run_planes(pt, a, b, planes_a, planes_b, counts, tile, f, params)
        ref, ref_err = run_denoise(pt, a, b, counts, tile, f, params)
        assert np.array_equal(frame, ref)
        # plane 0 went through the same sums as the guide, so its resolve is the guide's denoised frame
        assert np.array_equal(dr.resolve(oa[0], wa, ob[0], wb), ref)
        if h == 2:
            assert err == ref_err


# ---------------------------------------------------------------------------------------------- 2. plane renders
KINDS = ["light_groups", "aovs", "lpes", "components", "ppm_components"]


@pytest.fixture(scope="module")
def pm_scene(mcrt):
    return load(mcrt, "pm_hexagon_room_64")


def make(mcrt, kind, c2, pm, y_step=1):
    """-> (render, a function that loads a checkpoint of it)"""
    if kind in ("light_groups", "aovs", "lpes"):
        pt, scene, _ = c2
        cam = scene.cameras()[0].resized(96, 54)
        kw = {"light_groups": dict(light_groups=mcrt.light_groups_by_emittance(scene)[0]), "aovs": dict(aovs=True),
              "lpes": dict(lpes=list(mcrt.AOV_LPES))}[kind]
        return mcrt.Progressive(pt, cam, y_step=y_step, **kw), lambda path: mcrt.Progressive.load(path, pt, cam, **kw)
    scene = pm.scene
    cam = scene.cameras()[0]
    if kind == "components":
        return mcrt.Progressive(pm, cam, components=True), lambda path: mcrt.Progressive.load(path, pm, cam, components=True)
    ep = emit_params(scene)
    args = (cam, 4000, ep["caustic_factor"], ep["max_photons_per_octree_leaf"])
    return (mcrt.ProgressivePhotonMapping(pm, *args, radius=0.2, components=True),
            lambda path: mcrt.ProgressivePhotonMapping.load(path, pm, *args, radius=0.2, components=True))


def restated(prog, weights):
    """relight_denoised(weights) and the denoised planes by the restatement, from the render's sums and guides."""
    h, w = prog.camera.height, prog.camera.width
    n = len(prog.lpes) if prog.lpes is not None else prog.n_planes
    wa, wb = dr.pixel_weights(prog.tile_counts, prog.tile, h, w)
    ga, gb = (x.cpu().numpy() for x in prog._halves())
    f = prog._feature_sums(8).cpu().numpy()
    oa, ob, _, _ = dpr.denoise_planes(ga, wa, gb, wb, f, prog.rgb[0].cpu().numpy()[:n], prog.rgb[1].cpu().numpy()[:n])
    wt = np.broadcast_to(np.asarray(weights, np.float64).reshape(n, -1), (n, 3))
    ca, cb = wt[0] * oa[0], wt[0] * ob[0]
    for k in range(1, n):   # the combine kernel's order
        ca = ca + wt[k] * oa[k]; cb = cb + wt[k] * ob[k]
    planes = np.stack([dr.resolve(oa[k], wa, ob[k], wb) for k in range(n)])
    return dr.resolve(ca, wa, cb, wb), planes


def check_render(prog, rng):
    """The denoised planes and relit frames against denoise() and the restatement."""
    planes, errors = prog.denoise_planes()
    n = planes.shape[0]
    assert errors.shape == (n,) and np.isfinite(errors).all() and (errors >= 0).all()
    dn, dn_err = prog.denoise()
    frame, err, tiles = prog.relight_denoised(np.ones(n))
    np.testing.assert_allclose(frame, dn, rtol=1e-12, atol=0)
    assert err == pytest.approx(dn_err, rel=1e-9) and tiles.shape == prog.active.shape
    w = rng.uniform(0.0, 2.0, (n, 3))
    got = prog.relight_denoised(w)[0]
    want, want_planes = restated(prog, w)
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-12 * want.max())
    np.testing.assert_allclose(planes, want_planes, rtol=1e-9, atol=1e-12 * want.max())
    return planes


@pytest.mark.parametrize("kind", KINDS)
def test_relight_denoised_on_every_plane_render(kind, mcrt, c2, pm_scene, tmp_path):
    scene, seed = pm_scene
    pm = mcrt.PhotonMapper(scene, global_seed=seed)
    try:
        prog, load_ck = make(mcrt, kind, c2, pm)
        rng = np.random.default_rng(zlib.crc32(kind.encode()))
        for _ in range(4):
            prog.add(4)
        with pytest.raises(mcrt.McrtError, match="denoise_planes"):
            prog.relight_denoised(np.ones(prog.n_planes))
        planes = check_render(prog, rng)
        # adaptive retirement: the top row of tiles keeps 16 samples while the others go on
        mask = np.zeros(prog.active.shape, bool); mask[0, :] = True
        prog.retire(mask)
        prog.add(4)
        with pytest.raises(mcrt.McrtError, match="denoise_planes"):
            prog.relight_denoised(np.ones(planes.shape[0]))
        prog.add(4)
        assert (prog.tile_counts[0] == 8).all() and (prog.tile_counts[1:] == 12).all()
        planes = check_render(prog, rng)
        # a resumed render denoises its planes like the original
        path = str(tmp_path / "ck.npz")
        prog.save(path)
        back = load_ck(path)
        with pytest.raises(mcrt.McrtError, match="denoise_planes"):
            back.relight_denoised(np.ones(planes.shape[0]))
        back_planes, _ = back.denoise_planes()
        assert np.array_equal(back_planes, planes)
        np.testing.assert_allclose(back.relight_denoised(np.ones(planes.shape[0]))[0], prog.relight_denoised(np.ones(planes.shape[0]))[0],
                                   rtol=1e-15, atol=0)
    finally:
        pm.close()


# ---------------------------------------------------------------------------------------------- 3. quality
QUALITY_BOUND = 0.7   # as test_gpu_denoise: denoised error / noisy error at 16 spp, against 1024 spp of another seed
RECOMPOSITE = [1, 1, 1, 1, 0, 0, 1, 1]   # the AOV planes without the reflections


@pytest.fixture(scope="module")
def quality(mcrt, c2):
    """Errors of a 16-spp AOV render at 320x180 against 1024 spp of another seed, printed as measured: per plane with
    some energy {name: (share of the beauty's energy, noisy, denoise_planes, denoise(weights=e_k))}, and the
    recomposite's (noisy, relight_denoised, denoise(weights=RECOMPOSITE))."""
    pt, scene, seed = c2
    cam = scene.cameras()[0].resized(320, 180)
    other = mcrt.PathTracer(scene, global_seed=seed + 1)
    try:
        ref_prog = mcrt.Progressive(other, cam, aovs=True)
        ref_prog.render(512, 1024)
        ref_planes, _ = ref_prog.aov_frames()
        ref_recomposite = ref_prog.relight(RECOMPOSITE)[0]
    finally:
        other.close()

    def rel(x, ref):
        return float(np.sqrt(np.sum((x - ref) ** 2) / np.sum(ref ** 2)))

    prog = mcrt.Progressive(pt, cam, aovs=True)
    prog.render(8, 16)
    noisy_planes, _ = prog.aov_frames()
    planes, _ = prog.denoise_planes()
    beauty = float(ref_planes.sum())
    per_plane = {}
    for k, name in enumerate(mcrt.AOV_NAMES):
        share = float(ref_planes[k].sum()) / beauty
        if share > 0.0:
            alone = prog.denoise(weights=np.eye(len(mcrt.AOV_NAMES))[k])[0]
            per_plane[name] = (share, rel(noisy_planes[k], ref_planes[k]), rel(planes[k], ref_planes[k]), rel(alone, ref_planes[k]))
    recomposite = (rel(prog.relight(RECOMPOSITE)[0], ref_recomposite), rel(prog.relight_denoised(RECOMPOSITE)[0], ref_recomposite),
                   rel(prog.denoise(weights=RECOMPOSITE)[0], ref_recomposite))
    lines = [f"  {n:22s} share {v[0]:.3f}: noisy {v[1]:.5f}, denoise_planes {v[2]:.5f}, denoise(weights=e_k) {v[3]:.5f}"
             for n, v in per_plane.items()]
    n, r, f = recomposite
    print(f"\nc2_hexagon_room_96 320x180, 16 spp against 1024 spp of another seed, per AOV plane:\n" + "\n".join(lines) +
          f"\n  recomposite {RECOMPOSITE}: noisy {n:.5f}, relight_denoised {r:.5f} ({r / n:.3f} x), "
          f"denoise(weights=...) {f:.5f} ({f / n:.3f} x)")
    return per_plane, recomposite


def test_relit_denoised_error_against_an_independent_reference(quality):
    noisy, relit, _ = quality[1]
    assert relit < QUALITY_BOUND * noisy


# Measured on the H100 (DESIGN.md §6): diffuse_direct, half of the frame's energy and its least noisy plane, goes from
# 0.0143 noisy to 0.0458 with the beauty's weights (0.0152 filtered alone), because the colour term lets the
# beauty's larger noise through and so blurs shadow edges only the direct light shows. Every other plane with energy
# is no worse than noisy. The bound stays as stated, and this test fails until the design meets it.
@pytest.mark.xfail(strict=True, reason="shared weights blur diffuse_direct: 0.0143 noisy, 0.0458 denoised (DESIGN.md §6)")
def test_every_major_plane_is_no_worse_denoised_than_noisy(quality):
    worse = {name: v for name, v in quality[0].items() if v[0] >= 0.1 and v[2] > v[1]}
    assert not worse, worse


# ---------------------------------------------------------------------------------------------- 4. refusals
def test_refused_arguments(mcrt, c2):
    L = mcrt.lib()
    pt, scene, _ = c2
    w, h, tile, n = 32, 16, 8, 3
    counts = np.full(mcrt.tile_grid(h, w, tile) + (2,), 2, np.uint32)
    A, B, F = zeros(h, w, 3), zeros(h, w, 3), zeros(h, w, 8)
    PA, PB = zeros(n, h, w, 3), zeros(n, h, w, 3)
    OA, OB, out = zeros(n, h, w, 3), zeros(n, h, w, 3), zeros(h, w, 3)
    for t in (OA, OB, out):
        t.fill_(float("nan"))
    import torch
    torch.cuda.synchronize()
    err = C.c_double(-1.0)
    P = lambda t, off=0: C.c_void_p(t.data_ptr() + off)   # noqa: E731

    def dn(a=P(A), b=P(B), pa=P(PA), pb=P(PB), k=n, c=counts, t=tile, f=P(F), width=w, height=h, params=None, oa=P(OA), ob=P(OB),
           o=P(out), e=C.byref(err)):
        cp = c.ctypes.data_as(C.c_void_p) if c is not None else None
        return L.mcrt_denoise_planes_dev(pt.ctx, a, b, pa, pb, k, cp, t, f, width, height, params, oa, ob, o, e)

    plane_bytes = h * w * 3 * 8
    cases = {
        "null a": dn(a=None), "null b": dn(b=None), "null planes a": dn(pa=None), "null planes b": dn(pb=None),
        "null counts": dn(c=None), "null features": dn(f=None), "null out a": dn(oa=None), "null out b": dn(ob=None),
        "tile 0": dn(t=0), "empty frame": dn(width=0), "no planes": dn(k=0),
        "empty half": dn(c=np.where(np.arange(counts.size).reshape(counts.shape) == 3, 0, counts).astype(np.uint32)),
        "iterations": dn(params=C.byref(mcrt.DenoiseParams(11, 0, 1.0, 64.0, 0.1, 0.1))),
        "negative sigma": dn(params=C.byref(mcrt.DenoiseParams(5, 0, -1.0, 64.0, 0.1, 0.1))),
        "nan sigma": dn(params=C.byref(mcrt.DenoiseParams(5, 0, 1.0, float("nan"), 0.1, 0.1))),
        "inf sigma": dn(params=C.byref(mcrt.DenoiseParams(5, 0, 1.0, 64.0, float("inf"), 0.1))),
        "out a is planes a": dn(oa=P(PA)), "out b inside planes a": dn(ob=P(PA, plane_bytes)),
        "out a overlaps planes b": dn(oa=P(PB, plane_bytes - 8)), "out b over the guide": dn(ob=P(A)),
        "outs overlap": dn(ob=P(OA, plane_bytes)), "frame over planes": dn(o=P(PB, 8)), "frame over out b": dn(o=P(OB)),
        "frame without error": dn(e=None), "error without frame": dn(o=None),
    }
    assert all(v == INVALID for v in cases.values()), cases
    for t in (OA, OB, out):   # nothing was written
        assert np.isnan(t.cpu().numpy()).all()
    assert err.value == -1.0


def test_refused_renders(mcrt, c2):
    pt, scene, _ = c2
    cam = scene.cameras()[0].resized(32, 16)
    plain = mcrt.Progressive(pt, cam)
    plain.render(2, 4)
    with pytest.raises(mcrt.McrtError, match="denoise_planes needs"):
        plain.denoise_planes()
    ids = mcrt.light_groups_by_emittance(scene)[0]
    shard = mcrt.Progressive(pt, cam, y_step=2, light_groups=ids)
    shard.render(2, 4)
    with pytest.raises(mcrt.McrtError, match="row set"):
        shard.denoise_planes()
    half = mcrt.Progressive(pt, cam, aovs=True)
    half.add(4)
    with pytest.raises(mcrt.McrtError, match="both halves"):
        half.denoise_planes()
    with pytest.raises(mcrt.McrtError, match="denoise_planes"):
        half.relight_denoised(np.ones(len(mcrt.AOV_NAMES)))
