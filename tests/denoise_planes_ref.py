"""Numpy restatement of mcrt_denoise_planes_dev (csrc/denoise.cu), float64: every plane filtered with the tap weights
of the beauty frame's a-trous passes. Built on oracle/denoise_ref.py's restatement of mcrt_denoise_dev (prep, atrous,
denoise), whose weight arithmetic it repeats tap by tap. Test infrastructure only: the product runs the CUDA kernels.

Inputs as oracle/denoise_ref.py's, plus planes a_planes, b_planes [P, H, W, 3] of box-film sums."""
import numpy as np

from oracle.denoise_ref import H5, INVALID, atrous, color_weight, denoise, feature_weight, prep


def atrous_weights(a, b, var_a, var_b, g, step, sigma_color, sigma_normal, sigma_depth, sigma_albedo):
    """The tap weights of one atrous pass of step `step`, as k_denoise_atrous_weights stores them -> (wa, wb), each
    [25, H, W] in tap order 5 ky + kx; 0 for a tap the pass skips and for every tap of an invalid pixel."""
    h, w = var_a.shape
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    valid = g["flag"] != INVALID
    out_a = np.zeros((25, h, w)); out_b = np.zeros((25, h, w))
    for ky in range(5):
        for kx in range(5):
            dy, dx = (ky - 2) * step, (kx - 2) * step
            qy, qx = yy + dy, xx + dx
            inside = (qy >= 0) & (qy < h) & (qx >= 0) & (qx < w)
            qy = np.clip(qy, 0, h - 1); qx = np.clip(qx, 0, w - 1)
            p, q = (yy, xx), (qy, qx)
            hw = H5[ky] * H5[kx]
            if dx == 0 and dy == 0:
                wa = np.full((h, w), hw); wb = wa.copy()
            else:
                wf = feature_weight(g, p, q, sigma_normal, sigma_depth, sigma_albedo)
                d2a = ((a - a[q]) ** 2).sum(-1) / 3.0
                d2b = ((b - b[q]) ** 2).sum(-1) / 3.0
                wa = hw * wf * color_weight(d2b, var_b + var_b[q], sigma_color)
                wb = hw * wf * color_weight(d2a, var_a + var_a[q], sigma_color)
                use = inside & valid[q] & (wf != 0.0)
                wa = np.where(use, wa, 0.0); wb = np.where(use, wb, 0.0)
            out_a[5 * ky + kx] = np.where(valid, wa, 0.0)
            out_b[5 * ky + kx] = np.where(valid, wb, 0.0)
    return out_a, out_b


def filter_planes(x, taps, step, valid):
    """One k_denoise_atrous_planes pass: planes of means x [P, H, W, 3] filtered with one half's tap weights taps
    [25, H, W], summed in tap order; invalid pixels keep x."""
    h, w = taps.shape[1:]
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    acc = np.zeros_like(x); ws = np.zeros((h, w))
    for ky in range(5):
        for kx in range(5):
            qy = np.clip(yy + (ky - 2) * step, 0, h - 1); qx = np.clip(xx + (kx - 2) * step, 0, w - 1)
            t = taps[5 * ky + kx]
            acc += t[None, ..., None] * x[:, qy, qx]
            ws += t
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(valid[None, ..., None], acc / ws[None, ..., None], x)


def denoise_planes(a_rgb, wa, b_rgb, wb, features, a_planes, b_planes, iterations=5, sigma_color=1.0, sigma_normal=64.0,
                   sigma_depth=0.1, sigma_albedo=0.1):
    """mcrt_denoise_planes_dev: planes a_planes, b_planes [P, H, W, 3] (sums) filtered with the tap weights of the guide
    a_rgb, b_rgb -> (filtered plane sums A [P, H, W, 3], B, the guide's denoise() (frame, frame error, v'), the tap
    weights of each pass [(wa, wb)]). Invalid pixels keep their input sums."""
    a_rgb = np.asarray(a_rgb, np.float64); b_rgb = np.asarray(b_rgb, np.float64)
    wa = np.asarray(wa, np.float64); wb = np.asarray(wb, np.float64)
    a_planes = np.asarray(a_planes, np.float64); b_planes = np.asarray(b_planes, np.float64)
    a, b, var_a, var_b, g, valid = prep(a_rgb, wa, b_rgb, wb, features)
    v3 = valid[None, ..., None]
    with np.errstate(invalid="ignore", divide="ignore"):
        pa = np.where(v3, a_planes / wa[None, ..., None], 0.0)
        pb = np.where(v3, b_planes / wb[None, ..., None], 0.0)
    taps = []
    for k in range(iterations):
        t = atrous_weights(a, b, var_a, var_b, g, 1 << k, sigma_color, sigma_normal, sigma_depth, sigma_albedo)
        a, b, var_a, var_b = atrous(a, b, var_a, var_b, g, 1 << k, sigma_color, sigma_normal, sigma_depth, sigma_albedo)
        pa = filter_planes(pa, t[0], 1 << k, valid)
        pb = filter_planes(pb, t[1], 1 << k, valid)
        taps.append(t)
    out_a = np.where(v3, wa[None, ..., None] * pa, a_planes)
    out_b = np.where(v3, wb[None, ..., None] * pb, b_planes)
    guide = denoise(a_rgb, wa, b_rgb, wb, features, iterations, sigma_color, sigma_normal, sigma_depth, sigma_albedo)
    return out_a, out_b, guide, taps
