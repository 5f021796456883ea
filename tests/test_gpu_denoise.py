"""Denoising progressive frames: the first-hit guides of mcrt_render_features_dev against the reference's camera rays
and hits, the kernels of mcrt_denoise_dev against their numpy restatement (oracle/denoise_ref.py), and the denoised
frame against an independent high-sample reference."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

from conftest import GOLDEN, golden_cases
from oracle import denoise_ref as dr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tracers(mcrt):
    cache = {}

    def get(cid, precision=None):
        key = (cid, precision)
        if key not in cache:
            scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
            g = np.load(os.path.join(GOLDEN, cid + ".npz"))
            cls = mcrt.PhotonMapper if scene.photon_maps() is not None else mcrt.PathTracer
            pt = cls(scene, precision=mcrt.PRECISION_F64 if precision is None else precision, global_seed=int(g["seed"]))
            cache[key] = (pt, scene, g)
        return cache[key]
    yield get
    for pt, _, _ in cache.values():
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


def features_of(pt, cam, first, count, precision=None):
    f = zeros(cam.height, cam.width, 8)
    pt.render_features_dev(cam, f.data_ptr(), first, count, precision)
    return f


def thin_lens(cam):
    from importlib import import_module
    mcrt = import_module("monte-carlo-ray-tracer_b200")
    r = cam.rec
    return mcrt.Camera(r.eye, r.forward, r.left, r.up, r.focal_length, r.sensor_width, cam.width, cam.height,
                       aperture_radius=0.05, focus_distance=3.0, thin_lens=True)


# ---------------------------------------------------------------------------------------------- 1. the guides
def box_cases():
    from importlib import import_module
    mcrt = import_module("monte-carlo-ray-tracer_b200")
    out = []
    for cid in golden_cases():
        scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
        if scene.cameras() and scene.cameras()[0].film_rec() is None:
            out.append(cid)
    return out + ["c2_hexagon_room_96:thin_lens"]


@pytest.mark.parametrize("case", box_cases())
def test_features_match_the_reference_hits(case, mcrt, tracers):
    from oracle import port
    cid, _, variant = case.partition(":")
    pt, scene, g = tracers(cid)
    cam = scene.cameras()[0].resized(40, 24)
    if variant == "thin_lens":
        cam = thin_lens(cam)
    n = cam.width * cam.height
    got = features_of(pt, cam, 0, 4).cpu().numpy().reshape(n, 8)
    pixel = np.repeat(np.arange(n, dtype=np.uint32), 4)
    sample = np.tile(np.arange(4, dtype=np.uint32), n)
    ps = port.PortScene(scene)
    try:
        _, rays = ps.sample_pixels(cam, pixel, sample, int(g["seed"]))
        hits = ps.trace(rays)
    finally:
        ps.close()
    per_sample = dr.hit_features(scene, rays, hits, mcrt.PRIM_TRIANGLE, mcrt.PRIM_SPHERE, mcrt.NO_PRIM).reshape(n, 4, 8)
    want = np.zeros((n, 8))
    for s in range(4):   # the kernel's order of additions
        want += per_sample[:, s]
    assert np.array_equal(got[:, 7], want[:, 7])
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
    assert want[:, 7].any()
    # consecutive ranges accumulate bit-identically to their union
    f = features_of(pt, cam, 0, 2)
    pt.render_features_dev(cam, f.data_ptr(), 2, 2)
    assert np.array_equal(f.cpu().numpy().reshape(n, 8), got)


@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "smooth_mesh_64", "quadric_64"])
def test_features_fast_mode_is_close(cid, mcrt, tracers):
    pt, scene, _ = tracers(cid)
    cam = scene.cameras()[0].resized(64, 36)
    a = features_of(pt, cam, 0, 4).cpu().numpy()
    b = features_of(pt, cam, 0, 4, mcrt.PRECISION_F32).cpu().numpy()
    differ = a[..., 7] != b[..., 7]
    assert differ.mean() <= 1e-3
    # float32 can also move a sample at an edge to the neighbouring surface with the same hit count: a few pixels
    same = ~differ & (a[..., 7] > 0)
    close = np.isclose(b[same], a[same], rtol=1e-3, atol=1e-3).all(-1)
    assert close.mean() >= 0.995
    np.testing.assert_allclose(b[same].mean(0), a[same].mean(0), rtol=1e-3, atol=1e-4)


# ---------------------------------------------------------------------------------------------- 2. the kernels
def random_inputs(rng, h, w, tile, box, uneven):
    ty, tx = -(-h // tile), -(-w // tile)
    counts = rng.integers(1, 9, (ty, tx, 2)) if uneven else np.full((ty, tx, 2), 4)
    if box:
        wa, wb = dr.pixel_weights(counts, tile, h, w)
    else:
        wa, wb = rng.uniform(0.5, 6.0, (h, w)), rng.uniform(0.5, 6.0, (h, w))
    base = rng.uniform(0.0, 2.0, (h, w, 3))
    a = (base + rng.normal(0, 0.3, (h, w, 3))) * wa[..., None]
    b = (base + rng.normal(0, 0.3, (h, w, 3))) * wb[..., None]
    hits = rng.integers(0, 5, (h, w)).astype(np.float64)
    f = np.zeros((h, w, 8))
    f[..., 0:3] = rng.uniform(0, 1, (h, w, 3)).round(1) * hits[..., None]
    f[..., 3:6] = (rng.normal(size=(h, w, 3)) + [0, 0, 3]) * hits[..., None]
    f[..., 6] = rng.uniform(1, 3, (h, w)) * hits
    f[..., 7] = hits
    return a, wa, b, wb, counts, f


def run_denoise(mcrt, pt, a, wa, b, wb, counts, tile, f, box, params):
    h, w = wa.shape
    A, B, F, out = device(a), device(b), device(f), zeros(h, w, 3)
    WA, WB = (None, None) if box else (device(wa), device(wb))
    err = pt.denoise_dev(A.data_ptr(), WA.data_ptr() if WA is not None else None, B.data_ptr(),
                         WB.data_ptr() if WB is not None else None, counts, tile, F.data_ptr(), w, h, out.data_ptr(), params)
    return out.cpu().numpy(), err


SIGMAS = ("sigma_color", "sigma_normal", "sigma_depth", "sigma_albedo")


@pytest.mark.parametrize("box", [True, False])
@pytest.mark.parametrize("uneven", [False, True])
@pytest.mark.parametrize("tile", [1, 5, 16])
@pytest.mark.parametrize("iterations", [0, 1, 5])
@pytest.mark.parametrize("off", [None] + list(SIGMAS))
def test_kernels_match_the_restatement(box, uneven, tile, iterations, off, mcrt, tracers):
    if off is not None and (iterations != 5 or tile != 5):
        pytest.skip("each sigma is switched off at 5 iterations, tile 5")
    pt, _, _ = tracers("c2_hexagon_room_96")
    rng = np.random.default_rng(zlib.crc32(repr((box, uneven, tile, iterations, off)).encode()))
    a, wa, b, wb, counts, f = random_inputs(rng, 45, 67, tile, box, uneven)
    sig = dict(sigma_color=1.0, sigma_normal=64.0, sigma_depth=0.1, sigma_albedo=0.1)
    if off:
        sig[off] = 0.0
    params = mcrt.DenoiseParams(iterations, 0, sig["sigma_color"], sig["sigma_normal"], sig["sigma_depth"], sig["sigma_albedo"])
    got, err = run_denoise(mcrt, pt, a, wa, b, wb, counts, tile, f, box, params)
    want, want_err, _ = dr.denoise(a, wa, b, wb, f, iterations, **sig)
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-12)
    assert err == pytest.approx(want_err, rel=1e-9)


# ---------------------------------------------------------------------------------------------- 3. identity
@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "smooth_mesh_64"])
def test_zero_iterations_is_the_resolve_and_equal_halves_are_unchanged(cid, mcrt, tracers):
    pt, scene, _ = tracers(cid)
    cam = scene.cameras()[0].resized(80, 45)
    prog = mcrt.Progressive(pt, cam, tile=7)
    prog.render(4, 12)
    frame, err = prog.frame(), prog.error()[0]
    out, derr = prog.denoise(iterations=0)
    np.testing.assert_allclose(out, frame, rtol=1e-14, atol=0)
    assert derr == pytest.approx(err, rel=1e-12)
    # halves equal: nothing to remove
    f = prog._feature_sums(8)
    same = zeros(cam.height, cam.width, 3)
    same.copy_(prog.rgb[0])
    o = zeros(cam.height, cam.width, 3)
    counts = np.full(prog.tile_counts.shape, 4)
    e = pt.denoise_dev(same.data_ptr(), None, same.data_ptr(), None, counts, prog.tile, f.data_ptr(), cam.width, cam.height,
                       o.data_ptr())
    np.testing.assert_allclose(o.cpu().numpy(), np.maximum(0.0, same.cpu().numpy() / 4), rtol=1e-14, atol=0)
    assert e == 0.0


# ---------------------------------------------------------------------------------------------- 4. quality
# Measured on the H100 (DESIGN.md §6): denoised / noisy 0.483 (C2) and 0.550 (smooth_mesh) at 16 spp; denoising a
# 1024-spp frame moved it 0.842x and 0.826x as far from the reference. The bounds keep a margin over both.
QUALITY_BOUND = 0.7          # denoised error / noisy error at 16 spp, against 1024 spp of another seed
CONVERGED_MARGIN = 1.0       # denoising a 1024-spp frame must not raise its error


@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "smooth_mesh_64"])
def test_denoised_error_against_an_independent_reference(cid, mcrt, tracers, capsys):
    pt, scene, g = tracers(cid)
    cam = scene.cameras()[0].resized(320, 180)
    other = mcrt.PathTracer(scene, global_seed=int(g["seed"]) + 1)
    try:
        ref_prog = mcrt.Progressive(other, cam)
        ref_prog.render(512, 1024)
        ref = ref_prog.frame()
        ref_dn, _ = ref_prog.denoise()
    finally:
        other.close()

    def rel(x):
        return float(np.sqrt(np.sum((x - ref) ** 2) / np.sum(ref ** 2)))

    prog = mcrt.Progressive(pt, cam)
    prog.render(8, 16)
    noisy = rel(prog.frame())
    dn, estimate = prog.denoise()
    denoised = rel(dn)
    # the reference's own noise: denoising a 1024-spp frame must not move it away from a second 1024-spp frame
    high = mcrt.Progressive(pt, cam)
    high.render(512, 1024)
    high_dn, _ = high.denoise()
    converged, converged_dn = rel(high.frame()), rel(high_dn)
    with capsys.disabled():
        print(f"\n{cid} 320x180: 16 spp error {noisy:.5f}, denoised {denoised:.5f} ({denoised / noisy:.3f} x), "
              f"residual estimate {estimate:.5f}; 1024 spp {converged:.5f}, denoised {converged_dn:.5f} "
              f"({converged_dn / converged:.3f} x); reference denoised vs itself {rel(ref_dn):.5f}")
    assert denoised < QUALITY_BOUND * noisy
    assert converged_dn <= CONVERGED_MARGIN * converged


# ---------------------------------------------------------------------------------------------- 5. everywhere
def test_after_adaptive_retirement(mcrt, tracers):
    pt, scene, _ = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(96, 54)
    prog = mcrt.Progressive(pt, cam)
    prog.render(8, 16)
    mask = np.zeros(prog.active.shape, bool); mask[0, :] = True
    prog.retire(mask)
    prog.add(8); prog.add(8)
    assert (prog.tile_counts[0, :] == 8).all() and (prog.tile_counts[1, :] == 16).all()
    out, err = prog.denoise()
    f = prog._feature_sums(8).cpu().numpy()
    wa, wb = dr.pixel_weights(prog.tile_counts, prog.tile, cam.height, cam.width)
    want, want_err, _ = dr.denoise(prog.rgb[0].cpu().numpy(), wa, prog.rgb[1].cpu().numpy(), wb, f)
    np.testing.assert_allclose(out, want, rtol=1e-9, atol=1e-12)
    assert err == pytest.approx(want_err, rel=1e-9)


@pytest.mark.parametrize("case", ["pm_hexagon_room_64", "mitchell", "fast"])
def test_denoise_works_where_progressive_does(case, mcrt, tracers, tmp_path):
    if case == "pm_hexagon_room_64":
        pt, scene, _ = tracers("pm_hexagon_room_64")
        cam = scene.cameras()[0].resized(64, 48)
    elif case == "mitchell":
        pt, scene, _ = tracers("c2_hexagon_room_96")
        c = scene.cameras()[0].resized(72, 40)
        r = c.rec
        cam = mcrt.Camera(r.eye, r.forward, r.left, r.up, r.focal_length, r.sensor_width, c.width, c.height,
                          film=dict(filter="mitchell-netravali"))
    else:
        pt, scene, _ = tracers("c2_hexagon_room_96", mcrt.PRECISION_F32)
        cam = scene.cameras()[0].resized(72, 40)
    prog = mcrt.Progressive(pt, cam)
    prog.render(4, 16)
    out, err = prog.denoise()
    assert np.isfinite(out).all() and (out >= 0).all() and 0 < err < prog.error()[0]
    f = prog._feature_sums(8).cpu().numpy()
    if prog.filtered:
        wa, wb = prog.wsum[0].cpu().numpy(), prog.wsum[1].cpu().numpy()
    else:
        wa, wb = dr.pixel_weights(prog.tile_counts, prog.tile, cam.height, cam.width)
    want, want_err, _ = dr.denoise(prog.rgb[0].cpu().numpy(), wa, prog.rgb[1].cpu().numpy(), wb, f)
    np.testing.assert_allclose(out, want, rtol=1e-9, atol=1e-12)
    # a resumed render denoises like the original
    path = str(tmp_path / "ck.npz")
    prog.save(path)
    resumed = mcrt.Progressive.load(path, pt, cam)
    out2, err2 = resumed.denoise()
    np.testing.assert_allclose(out2, out, rtol=1e-12, atol=1e-12)
    assert err2 == pytest.approx(err, rel=1e-12)


# ---------------------------------------------------------------------------------------------- 6. refusals
def test_refused_arguments(mcrt, tracers):
    L = mcrt.lib()
    pt, scene, _ = tracers("c2_hexagon_room_96")
    cam = scene.cameras()[0].resized(32, 16)
    w, h, tile = cam.width, cam.height, 8
    counts = np.full(mcrt.tile_grid(h, w, tile) + (2,), 2, np.uint32)
    A, B, F = zeros(h, w, 3), zeros(h, w, 3), zeros(h, w, 8)
    Wt = zeros(h, w)
    out = zeros(h, w, 3)
    out.fill_(float("nan"))
    err = C.c_double(-1.0)
    st = mcrt.Stats()
    P = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731

    def dn(a=P(A), aw=None, b=P(B), bw=None, c=counts, t=tile, f=P(F), width=w, height=h, params=None, o=P(out), e=C.byref(err)):
        cp = c.ctypes.data_as(C.c_void_p) if c is not None else None
        return L.mcrt_denoise_dev(pt.ctx, a, aw, b, bw, cp, t, f, width, height, params, o, e)

    INVALID, NO_SCENE = -1, -3   # MCRT_ERR_INVALID, MCRT_ERR_NO_SCENE
    cases = {
        "null a": dn(a=None), "null b": dn(b=None), "null counts": dn(c=None), "null features": dn(f=None),
        "null out": dn(o=None), "null error": dn(e=None), "tile 0": dn(t=0), "empty frame": dn(width=0),
        "one weight": dn(aw=P(Wt)),
        "empty half": dn(c=np.where(np.arange(counts.size).reshape(counts.shape) == 3, 0, counts).astype(np.uint32)),
        "iterations": dn(params=C.byref(mcrt.DenoiseParams(11, 0, 1.0, 64.0, 0.1, 0.1))),
        "negative sigma": dn(params=C.byref(mcrt.DenoiseParams(5, 0, -1.0, 64.0, 0.1, 0.1))),
        "nan sigma": dn(params=C.byref(mcrt.DenoiseParams(5, 0, 1.0, float("nan"), 0.1, 0.1))),
        "inf sigma": dn(params=C.byref(mcrt.DenoiseParams(5, 0, 1.0, 64.0, float("inf"), 0.1))),
        "features: count 0": L.mcrt_render_features_dev(pt.ctx, C.byref(cam.rec), 0, 0, 1, 0, P(F), C.byref(st)),
        "features: past 2^32": L.mcrt_render_features_dev(pt.ctx, C.byref(cam.rec), 0xFFFFFFFF, 2, 1, 0, P(F), C.byref(st)),
        "features: null camera": L.mcrt_render_features_dev(pt.ctx, None, 0, 1, 1, 0, P(F), C.byref(st)),
        "features: null buffer": L.mcrt_render_features_dev(pt.ctx, C.byref(cam.rec), 0, 1, 1, 0, None, C.byref(st)),
        "features: precision": L.mcrt_render_features_dev(pt.ctx, C.byref(cam.rec), 0, 1, 1, 7, P(F), C.byref(st)),
    }
    assert all(v == INVALID for v in cases.values()), cases
    assert np.isnan(out.cpu().numpy()).all()        # nothing was written
    assert not F.cpu().numpy().any()
    # no scene yet
    ctx = C.c_void_p()
    assert L.mcrt_init(0, C.byref(ctx)) == 0
    try:
        rc = L.mcrt_render_features_dev(ctx, C.byref(cam.rec), 0, 1, 1, 0, P(F), C.byref(st))
        assert rc == NO_SCENE
    finally:
        L.mcrt_destroy(ctx)
    # Progressive.denoise
    shard = mcrt.Progressive(pt, cam, y_first=0, y_step=2)
    shard.render(2, 4)
    with pytest.raises(mcrt.McrtError):
        shard.denoise()
    half = mcrt.Progressive(pt, cam)
    half.add(4)
    with pytest.raises(mcrt.McrtError):
        half.denoise()
    with pytest.raises(mcrt.McrtError):
        pt.denoise_dev(P(A).value, None, P(B).value, None, np.ones((1, 1, 2)), tile, P(F).value, w, h, P(out).value)
