"""Numpy restatement of the cross-filtered a-trous denoiser of mcrt_denoise_dev (csrc/denoise.cu), float64, and of the
first-hit guides of mcrt_render_features_dev. Test infrastructure only: the product runs the CUDA kernels.

Inputs are whole frames: a_rgb, b_rgb [H, W, 3] sums; wa, wb [H, W] per-pixel weights of each half (the tile's count
with the box film, the weight sums with a filter); features [H, W, 8] {albedo.rgb, normal.xyz, t, hits} sums."""
import numpy as np

H5 = np.array([1.0, 4.0, 6.0, 4.0, 1.0]) / 16.0
SURFACE, BACKGROUND, INVALID = 0, 1, 2


def pixel_weights(tile_counts, tile, height, width):
    """Box-film weights [H, W] of each half from per-tile counts [tiles_y, tiles_x, 2]."""
    c = np.asarray(tile_counts, np.float64)
    ty = np.arange(height) // tile
    tx = np.arange(width) // tile
    return c[ty][:, tx, 0], c[ty][:, tx, 1]


def resolve(a_rgb, wa, b_rgb, wb):
    """k_progressive_resolve's frame: max(0, (A + B) / (wA + wB)), 0 where the weight is 0."""
    w = (wa + wb)[..., None]
    with np.errstate(invalid="ignore", divide="ignore"):
        v = np.where(w == 0.0, 0.0, (a_rgb + b_rgb) / w)
    return np.maximum(v, 0.0)


def relative_error(sum_v, sum_i2):
    if sum_v == 0.0:
        return 0.0
    return float(np.sqrt(sum_v / sum_i2)) if sum_i2 > 0.0 else float("inf")


def prep(a_rgb, wa, b_rgb, wb, features):
    """-> (A, B, var_A, var_B, guide dict, valid) as k_denoise_prep leaves them."""
    h, w = wa.shape
    valid = (wa != 0.0) & (wb != 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        ia = np.where(valid[..., None], a_rgb / wa[..., None], 0.0)
        ib = np.where(valid[..., None], b_rgb / wb[..., None], 0.0)
        d2 = ((a_rgb / wa[..., None] - b_rgb / wb[..., None]) ** 2).sum(-1) / 3.0
        va = np.where(valid, d2 * (wb / (wa + wb)), 0.0)
        vb = np.where(valid, d2 * (wa / (wa + wb)), 0.0)
    # 3x3 [1,2,1]x[1,2,1], normalised over the valid in-image pixels it covers
    sa = np.zeros((h, w)); sb = np.zeros((h, w)); sk = np.zeros((h, w))
    k1 = {-1: 1.0, 0: 2.0, 1: 1.0}
    pa, pb, pv = (np.pad(x, 1) for x in (va, vb, valid.astype(np.float64)))
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            k = k1[dx] * k1[dy]
            sl = (slice(1 + dy, 1 + dy + h), slice(1 + dx, 1 + dx + w))
            sa += k * pa[sl]; sb += k * pb[sl]; sk += k * pv[sl]
    with np.errstate(invalid="ignore", divide="ignore"):
        var_a = np.where(valid, sa / sk, 0.0)
        var_b = np.where(valid, sb / sk, 0.0)
    f = np.asarray(features, np.float64)
    hits = f[..., 7]
    surface = valid & (hits > 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        length = np.sqrt((f[..., 3:6] ** 2).sum(-1, keepdims=True))
        n = np.where(surface[..., None] & (length > 0), f[..., 3:6] * (1.0 / length), 0.0)
        z = np.where(surface, f[..., 6] / hits, 0.0)
        alb = np.where(surface[..., None], f[..., 0:3] / hits[..., None], 0.0)
    flag = np.where(~valid, INVALID, np.where(hits > 0, SURFACE, BACKGROUND))
    return ia, ib, var_a, var_b, {"n": n, "z": z, "albedo": alb, "flag": flag}, valid


def color_weight(d2, var_sum, sigma):
    if sigma == 0.0:
        return np.ones_like(d2)
    num = np.maximum(0.0, d2 - var_sum)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        w = np.exp(-num / (sigma * sigma * var_sum))
    return np.where(num == 0.0, 1.0, np.where(var_sum == 0.0, 0.0, w))


def feature_weight(g, p, q, sigma_normal, sigma_depth, sigma_albedo):
    """w_n w_z w_a between pixel sets p and q (index tuples of equal shape)."""
    fp, fq = g["flag"][p], g["flag"][q]
    w = np.ones(fp.shape)
    if sigma_normal != 0.0:
        w = w * np.maximum(0.0, (g["n"][p] * g["n"][q]).sum(-1)) ** sigma_normal
    if sigma_depth != 0.0:
        zp, zq = g["z"][p], g["z"][q]
        with np.errstate(invalid="ignore", divide="ignore"):
            w = w * np.exp(-np.abs(zp - zq) / (sigma_depth * np.maximum(zp, zq)))
    if sigma_albedo != 0.0:
        w = w * np.exp(-((g["albedo"][p] - g["albedo"][q]) ** 2).sum(-1) / (sigma_albedo * sigma_albedo))
    return np.where(fp != fq, 0.0, np.where(fp == BACKGROUND, 1.0, w))


def atrous(a, b, var_a, var_b, g, step, sigma_color, sigma_normal, sigma_depth, sigma_albedo):
    """One k_denoise_atrous pass of step `step` over both halves."""
    h, w = var_a.shape
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    valid = g["flag"] != INVALID
    acc_a = np.zeros_like(a); acc_b = np.zeros_like(b)
    ws_a = np.zeros((h, w)); ws_b = np.zeros((h, w)); vs_a = np.zeros((h, w)); vs_b = np.zeros((h, w))
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
            acc_a += wa[..., None] * a[q]; acc_b += wb[..., None] * b[q]
            ws_a += wa; ws_b += wb
            vs_a += wa * wa * var_a[q]; vs_b += wb * wb * var_b[q]
    with np.errstate(invalid="ignore", divide="ignore"):
        na = np.where(valid[..., None], acc_a / ws_a[..., None], a)
        nb = np.where(valid[..., None], acc_b / ws_b[..., None], b)
        nva = np.where(valid, vs_a / (ws_a * ws_a), var_a)
        nvb = np.where(valid, vs_b / (ws_b * ws_b), var_b)
    return na, nb, nva, nvb


def denoise(a_rgb, wa, b_rgb, wb, features, iterations=5, sigma_color=1.0, sigma_normal=64.0, sigma_depth=0.1,
            sigma_albedo=0.1):
    """-> (frame [H, W, 3], frame error, residual v' [H, W]) as mcrt_denoise_dev computes them."""
    a_rgb = np.asarray(a_rgb, np.float64); b_rgb = np.asarray(b_rgb, np.float64)
    wa = np.asarray(wa, np.float64); wb = np.asarray(wb, np.float64)
    a, b, var_a, var_b, g, valid = prep(a_rgb, wa, b_rgb, wb, features)
    for k in range(iterations):
        a, b, var_a, var_b = atrous(a, b, var_a, var_b, g, 1 << k, sigma_color, sigma_normal, sigma_depth, sigma_albedo)
    w = wa + wb
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.maximum(0.0, (wa[..., None] * a + wb[..., None] * b) / w[..., None])
        v = ((a - b) ** 2).sum(-1) * (wa * wb / (w * w))
    out = np.where(valid[..., None], out, resolve(a_rgb, wa, b_rgb, wb))
    v = np.where(valid, v, 0.0)
    return out, relative_error(v.sum(), (out ** 2).sum()), v


# ---------------------------------------------------------------------------------------------- first-hit guides
def _normalize(v):
    """vec.cuh normalize: v * (1 / sqrt(dot(v, v)))."""
    d = v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1] + v[..., 2] * v[..., 2]
    return v * (1.0 / np.sqrt(d))[..., None]


def _dot(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def hit_features(scene, rays, hits, prim_triangle=0, prim_sphere=1, no_prim=0xFFFFFFFF):
    """{albedo.rgb, shading normal.xyz, t, 1} [n, 8] of camera rays [n, 6] and their closest hits (HIT_DTYPE), in
    k_features' operation order; rows of misses are 0."""
    a = scene.a
    rays = np.asarray(rays, np.float64).reshape(-1, 6)
    n = len(rays)
    out = np.zeros((n, 8))
    hit = hits["prim"] != no_prim
    idx = np.nonzero(hit)[0]
    if not len(idx):
        return out
    prim = hits["prim"][idx].astype(np.int64)
    t = hits["t"][idx]; u = hits["u"][idx]; v = hits["v"][idx]
    o, d = rays[idx, :3], rays[idx, 3:]
    pos = o + d * t[:, None]
    ptype = a["prim_type"][prim]; pidx = a["prim_index"][prim].astype(np.int64)
    normal = np.zeros((len(idx), 3))
    tri = ptype == prim_triangle
    sph = ptype == prim_sphere
    quad = ~tri & ~sph
    normal[tri] = a["tri_normal"].reshape(-1, 3)[pidx[tri]]
    if sph.any():
        s = a["sphere_origin_radius"].reshape(-1, 4)[pidx[sph]]
        normal[sph] = (pos[sph] - s[:, :3]) / s[:, 3:4]
    if quad.any():
        G = a["quadric_G"].reshape(-1, 12)[pidx[quad]]
        p = pos[quad]
        g = np.stack([G[:, 0] * p[:, 0] + G[:, 3] * p[:, 1] + G[:, 6] * p[:, 2] + G[:, 9] * 1.0,
                      G[:, 1] * p[:, 0] + G[:, 4] * p[:, 1] + G[:, 7] * p[:, 2] + G[:, 10] * 1.0,
                      G[:, 2] * p[:, 0] + G[:, 5] * p[:, 1] + G[:, 8] * p[:, 2] + G[:, 11] * 1.0], -1)
        normal[quad] = _normalize(g)
    cos_theta = _dot(d, normal)
    shading = normal.copy()
    vn = np.full(len(idx), -1, np.int64)
    vn[tri] = a["tri_vn_index"][pidx[tri]]
    interp = vn >= 0
    if interp.any():
        vns = a["vertex_normals"].reshape(-1, 3, 3)[vn[interp]]
        uu, vv = u[interp][:, None], v[interp][:, None]
        sn = _normalize((1.0 - uu - vv) * vns[:, 0] + uu * vns[:, 1] + vv * vns[:, 2])
        flip = (cos_theta[interp] < 0) != (_dot(d[interp], sn) < 0)
        shading[interp] = np.where(flip[:, None], normal[interp], sn)
    shading = np.where((cos_theta > 0)[:, None], -shading, shading)
    m = a["materials"][a["prim_material"][prim]]
    specular = (m["perfect_mirror"] != 0) | (m["has_complex_ior"] != 0)
    albedo = np.where(specular[:, None], m["specular_reflectance"], m["reflectance"])
    out[idx, 0:3] = albedo
    out[idx, 3:6] = shading
    out[idx, 6] = t
    out[idx, 7] = 1.0
    return out
