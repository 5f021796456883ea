"""CPU checks of the denoiser: properties of its numpy restatement (oracle/denoise_ref.py), which the GPU tests hold the
CUDA kernels to, and the C ABI of mcrt_denoise_dev."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from oracle import denoise_ref as dr


def random_frame(rng, h=23, w=37, box=True, tile=8):
    a = rng.uniform(0.0, 2.0, (h, w, 3)); b = rng.uniform(0.0, 2.0, (h, w, 3))
    if box:
        counts = rng.integers(1, 9, (-(-h // tile), -(-w // tile), 2))
        wa, wb = dr.pixel_weights(counts, tile, h, w)
        a *= wa[..., None]; b *= wb[..., None]
    else:
        wa = rng.uniform(0.5, 4.0, (h, w)); wb = rng.uniform(0.5, 4.0, (h, w))
    f = np.zeros((h, w, 8))
    hits = rng.integers(0, 5, (h, w)).astype(np.float64)
    n = rng.normal(size=(h, w, 3))
    f[..., 0:3] = rng.uniform(0, 1, (h, w, 3)) * hits[..., None]
    f[..., 3:6] = n * hits[..., None]
    f[..., 6] = rng.uniform(1, 5, (h, w)) * hits
    f[..., 7] = hits
    return a, wa, b, wb, f


def test_zero_iterations_is_the_resolve():
    a, wa, b, wb, f = random_frame(np.random.default_rng(1))
    out, err, v = dr.denoise(a, wa, b, wb, f, iterations=0)
    ref = dr.resolve(a, wa, b, wb)
    np.testing.assert_allclose(out, ref, rtol=1e-14, atol=0)
    ia, ib = a / wa[..., None], b / wb[..., None]
    v_ref = ((ia - ib) ** 2).sum(-1) * wa * wb / (wa + wb) ** 2
    np.testing.assert_allclose(v, v_ref, rtol=1e-14)
    assert err == pytest.approx(np.sqrt(v_ref.sum() / (ref ** 2).sum()), rel=1e-12)


def test_constant_halves_come_out_unchanged():
    rng = np.random.default_rng(2)
    _, wa, _, wb, f = random_frame(rng)
    c = np.array([0.3, 1.5, 0.7])
    out, err, _ = dr.denoise(c * wa[..., None], wa, c * wb[..., None], wb, f, iterations=5)
    np.testing.assert_allclose(out, np.broadcast_to(c, out.shape), rtol=1e-13)
    assert err < 1e-14   # S / w rounds: the halves differ in the last bit


@pytest.mark.parametrize("box", [True, False])
def test_scaling_both_halves_scales_the_output(box):
    a, wa, b, wb, f = random_frame(np.random.default_rng(3), box=box)
    out, err, _ = dr.denoise(a, wa, b, wb, f, iterations=3)
    out4, err4, _ = dr.denoise(4.0 * a, wa, 4.0 * b, wb, f, iterations=3)
    np.testing.assert_allclose(out4, 4.0 * out, rtol=1e-12)
    assert err4 == pytest.approx(err, rel=1e-12)


def test_every_output_is_a_convex_combination_of_its_inputs():
    a, wa, b, wb, f = random_frame(np.random.default_rng(4))
    ia, ib = a / wa[..., None], b / wb[..., None]
    out, _, _ = dr.denoise(a, wa, b, wb, f, iterations=4)
    lo = np.minimum(ia.min(axis=(0, 1)), ib.min(axis=(0, 1)))
    hi = np.maximum(ia.max(axis=(0, 1)), ib.max(axis=(0, 1)))
    assert (out >= lo - 1e-12).all() and (out <= hi + 1e-12).all()
    # and every filtered half stays inside the range of that half
    ha, hb, va, vb, g, _ = dr.prep(a, wa, b, wb, f)
    na, nb, _, _ = dr.atrous(ha, hb, va, vb, g, 1, 1.0, 64.0, 0.1, 0.1)
    assert (na >= ia.min(axis=(0, 1)) - 1e-12).all() and (na <= ia.max(axis=(0, 1)) + 1e-12).all()


def test_a_normal_step_mixes_nothing_across_it():
    h, w = 16, 24
    rng = np.random.default_rng(5)
    wa = np.full((h, w), 4.0); wb = np.full((h, w), 4.0)
    left = np.arange(w) < w // 2
    colour = np.where(left[None, :, None], 1.0, 3.0) + rng.normal(0, 0.2, (h, w, 3))
    a = colour * wa[..., None]
    b = (colour + rng.normal(0, 0.2, (h, w, 3))) * wb[..., None]
    f = np.zeros((h, w, 8))
    f[..., 3:6] = np.where(left[None, :, None], [0.0, 0.0, 1.0], [1.0, 0.0, 0.0])
    f[..., 6] = 2.0; f[..., 7] = 1.0
    out, _, _ = dr.denoise(a, wa, b, wb, f, iterations=5, sigma_color=0.0, sigma_normal=1e6, sigma_depth=0.0, sigma_albedo=0.0)
    assert out[:, left].max() < 2.0 and out[:, ~left].min() > 2.0
    # switched off, the normal term lets the two planes mix
    mixed, _, _ = dr.denoise(a, wa, b, wb, f, iterations=5, sigma_color=0.0, sigma_normal=0.0, sigma_depth=0.0, sigma_albedo=0.0)
    assert mixed[:, left].max() > 2.0


def test_zero_variance_with_differing_colours_gives_weight_zero():
    w = dr.color_weight(np.array([0.5, 0.0, 0.5]), np.array([0.0, 0.0, 1.0]), 1.0)
    assert w[0] == 0.0 and w[1] == 1.0 and w[2] == 1.0
    # halves equal everywhere: zero variance, so no pixel mixes with a differently coloured neighbour
    rng = np.random.default_rng(6)
    h, wd = 9, 11
    c = rng.uniform(0, 1, (h, wd, 3))
    wa = np.full((h, wd), 2.0)
    f = np.zeros((h, wd, 8)); f[..., 5] = 1.0; f[..., 6] = 1.0; f[..., 7] = 1.0
    out, err, _ = dr.denoise(c * 2.0, wa, c * 2.0, wa, f, iterations=3)
    np.testing.assert_allclose(out, c, rtol=1e-14)
    assert err == 0.0


def test_invalid_pixels_keep_their_resolve_and_are_never_neighbours():
    a, wa, b, wb, f = random_frame(np.random.default_rng(7), box=False)
    wb[3:6, 4:9] = 0.0
    b[3:6, 4:9] = 0.0
    out, _, v = dr.denoise(a, wa, b, wb, f, iterations=3)
    np.testing.assert_array_equal(out[3:6, 4:9], dr.resolve(a, wa, b, wb)[3:6, 4:9])
    assert (v[3:6, 4:9] == 0).all()
    # changing an invalid pixel's sums changes no other pixel
    a2 = a.copy(); a2[4, 5] += 100.0
    out2, _, _ = dr.denoise(a2, wa, b, wb, f, iterations=3)
    mask = np.ones(wa.shape, bool); mask[4, 5] = False
    np.testing.assert_array_equal(out2[mask], out[mask])


def test_denoise_params_struct_matches_the_header(mcrt):
    assert C.sizeof(mcrt.DenoiseParams) == 8 + 4 * 8
    header = open(os.path.join(ROOT, "include", "mcrt_abi.h")).read()
    for key, macro in (("iterations", "ITERATIONS"), ("sigma_color", "SIGMA_COLOR"), ("sigma_normal", "SIGMA_NORMAL"),
                       ("sigma_depth", "SIGMA_DEPTH"), ("sigma_albedo", "SIGMA_ALBEDO")):
        m = re.search(r"#define MCRT_DENOISE_DEFAULT_%s ([0-9.]+)" % macro, header)
        assert m and float(m.group(1)) == mcrt.DENOISE_DEFAULTS[key], key


def test_denoise_entry_points_are_exported(mcrt):
    L = mcrt.lib()
    for sym in ("mcrt_render_features_dev", "mcrt_denoise_dev"):
        assert sym in mcrt.ABI_SYMBOLS and hasattr(L, sym)
