"""CPU checks of denoising film planes: properties of the numpy restatement (tests/denoise_planes_ref.py), which
the GPU tests hold mcrt_denoise_planes_dev to, and its C ABI as the package declares it."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from oracle import denoise_ref as dr
import denoise_planes_ref as dpr


def random_planes(rng, n_planes, h=23, w=37, tile=8):
    """Box-film planes that sum to the guide: -> (guide a, wa, guide b, wb, features, planes a, planes b)."""
    counts = rng.integers(1, 9, (-(-h // tile), -(-w // tile), 2))
    wa, wb = dr.pixel_weights(counts, tile, h, w)
    pa = rng.uniform(0.0, 1.0, (n_planes, h, w, 3)) * wa[None, ..., None]
    pb = rng.uniform(0.0, 1.0, (n_planes, h, w, 3)) * wb[None, ..., None]
    f = np.zeros((h, w, 8))
    hits = rng.integers(0, 5, (h, w)).astype(np.float64)
    f[..., 0:3] = rng.uniform(0, 1, (h, w, 3)).round(1) * hits[..., None]
    f[..., 3:6] = (rng.normal(size=(h, w, 3)) + [0, 0, 2]) * hits[..., None]
    f[..., 6] = rng.uniform(1, 5, (h, w)) * hits
    f[..., 7] = hits
    return pa.sum(0), wa, pb.sum(0), wb, f, pa, pb


def test_a_plane_equal_to_the_guide_resolves_to_the_denoised_frame():
    a, wa, b, wb, f, _, _ = random_planes(np.random.default_rng(1), 3)
    oa, ob, (frame, _, _), taps = dpr.denoise_planes(a, wa, b, wb, f, a[None], b[None], iterations=5)
    assert len(taps) == 5 and taps[0][0].shape == (25,) + wa.shape
    np.testing.assert_allclose(dr.resolve(oa[0], wa, ob[0], wb), frame, rtol=1e-12, atol=0)


def test_the_stored_weights_are_the_passes_weights():
    """Each pass's tap weights, applied to the guide's own means, give that pass's output bit for bit."""
    a, wa, b, wb, f, _, _ = random_planes(np.random.default_rng(2), 2)
    ha, hb, va, vb, g, valid = dr.prep(a, wa, b, wb, f)
    for step in (1, 2, 4):
        ta, tb = dpr.atrous_weights(ha, hb, va, vb, g, step, 1.0, 64.0, 0.1, 0.1)
        na, nb, nva, nvb = dr.atrous(ha, hb, va, vb, g, step, 1.0, 64.0, 0.1, 0.1)
        assert np.array_equal(dpr.filter_planes(ha[None], ta, step, valid)[0], na)
        assert np.array_equal(dpr.filter_planes(hb[None], tb, step, valid)[0], nb)
        assert (ta >= 0).all() and (ta[12] > 0).all()   # the centre tap always counts
        ha, hb, va, vb = na, nb, nva, nvb


def test_planes_that_sum_to_the_guide_have_filtered_sums_that_sum_to_its_filtered_sums():
    a, wa, b, wb, f, pa, pb = random_planes(np.random.default_rng(3), 8)
    oa, ob, _, _ = dpr.denoise_planes(a, wa, b, wb, f, pa, pb, iterations=5)
    ga, gb, _, _ = dpr.denoise_planes(a, wa, b, wb, f, a[None], b[None], iterations=5)
    np.testing.assert_allclose(oa.sum(0), ga[0], rtol=1e-12, atol=0)
    np.testing.assert_allclose(ob.sum(0), gb[0], rtol=1e-12, atol=0)


def test_permuting_scaling_and_zero_planes():
    a, wa, b, wb, f, pa, pb = random_planes(np.random.default_rng(4), 4)
    oa, ob, _, _ = dpr.denoise_planes(a, wa, b, wb, f, pa, pb, iterations=3)
    perm = [2, 0, 3, 1]
    qa, qb, _, _ = dpr.denoise_planes(a, wa, b, wb, f, pa[perm], pb[perm], iterations=3)
    assert np.array_equal(qa, oa[perm]) and np.array_equal(qb, ob[perm])
    sa, sb = pa.copy(), pb.copy()
    sa[1] *= 4.0; sb[1] *= 4.0       # a power of two scales exactly
    sa[3] = 0.0; sb[3] = 0.0
    ra, rb, _, _ = dpr.denoise_planes(a, wa, b, wb, f, sa, sb, iterations=3)
    np.testing.assert_allclose(ra[1], 4.0 * oa[1], rtol=1e-14); np.testing.assert_allclose(rb[1], 4.0 * ob[1], rtol=1e-14)
    assert not ra[3].any() and not rb[3].any()
    assert np.array_equal(ra[[0, 2]], oa[[0, 2]])   # the weights come from the guide alone


def test_zero_iterations_returns_the_input_sums():
    a, wa, b, wb, f, pa, pb = random_planes(np.random.default_rng(5), 3)
    oa, ob, (frame, _, _), taps = dpr.denoise_planes(a, wa, b, wb, f, pa, pb, iterations=0)
    assert taps == []
    np.testing.assert_allclose(oa, pa, rtol=1e-15, atol=0)
    np.testing.assert_allclose(ob, pb, rtol=1e-15, atol=0)
    np.testing.assert_allclose(frame, dr.resolve(a, wa, b, wb), rtol=1e-14, atol=0)


def test_invalid_pixels_keep_their_input_sums():
    a, wa, b, wb, f, pa, pb = random_planes(np.random.default_rng(6), 2)
    wb = wb.copy(); wb[3:6, 4:9] = 0.0
    pb = pb.copy(); pb[:, 3:6, 4:9] = 0.0
    oa, ob, _, _ = dpr.denoise_planes(a, wa, pb.sum(0), wb, f, pa, pb, iterations=3)
    assert np.array_equal(oa[:, 3:6, 4:9], pa[:, 3:6, 4:9]) and np.array_equal(ob[:, 3:6, 4:9], pb[:, 3:6, 4:9])


def test_denoise_planes_entry_point_is_exported_with_the_headers_arguments(mcrt):
    assert "mcrt_denoise_planes_dev" in mcrt.ABI_SYMBOLS
    L = mcrt.lib()
    assert hasattr(L, "mcrt_denoise_planes_dev")
    header = open(os.path.join(ROOT, "include", "mcrt_abi.h")).read()
    m = re.search(r"int mcrt_denoise_planes_dev\((.*?)\);", header, re.S)
    assert m
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    want = {"mcrt_ctx*": C.c_void_p, "const double*": C.c_void_p, "double*": C.c_void_p, "const uint32_t*": C.c_void_p,
            "uint32_t": C.c_uint32, "const mcrt_denoise_params*": C.POINTER(mcrt.DenoiseParams)}
    types = [want[p.rsplit(" ", 1)[0]] for p in params]
    types[-1] = C.POINTER(C.c_double)   # frame_error
    assert params[-1] == "double* frame_error"
    assert list(L.mcrt_denoise_planes_dev.argtypes) == types
