"""ORACLE / TEST INFRASTRUCTURE - ctypes binding of the CPU restatement (oracle/mcrt_oracle.cpp).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module."""
import ctypes as C
import importlib
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "_build", "libmcrt_oracle.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            import importlib.util
            spec = importlib.util.spec_from_file_location("build_oracle", os.path.join(HERE, "build_oracle.py"))
            mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
            mod.build()
        L = C.CDLL(LIB_PATH)
        L.oracle_scene_create.restype = C.c_void_p
        L.oracle_scene_create.argtypes = [C.c_void_p]
        L.oracle_scene_destroy.argtypes = [C.c_void_p]
        L.oracle_sampler_stream.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p]
        L.oracle_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.oracle_sample_rays.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
        L.oracle_render_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64)]
        L.oracle_sample_pixels.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p]
        L.oracle_trace_fast.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_double, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                        C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.oracle_trace_visible.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.oracle_trace_peaks.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.oracle_trace_fast_peaks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                              C.c_void_p]
        L.oracle_trace_visible_peaks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                                 C.c_void_p, C.c_void_p]
        L.oracle_wide_stack_bound.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_double, C.c_void_p]
        L.oracle_render_rows_checked.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                                 C.c_uint32, C.c_void_p, C.c_void_p]
        L.oracle_bvh_build.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_void_p]
        L.oracle_bvh_free.argtypes = [C.c_void_p]
        L.oracle_octree_build.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p]
        L.oracle_octree_free.argtypes = [C.c_void_p]
        L.oracle_image_tonemap.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.oracle_render_film.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        L.oracle_photon_pass.restype = C.c_int
        L.oracle_photon_pass.argtypes = [C.c_void_p, C.c_uint64, C.c_double, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32,
                                         C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        L.oracle_photon_pass_free.argtypes = [C.c_void_p]
        L.oracle_pm_create.restype = C.c_void_p
        L.oracle_pm_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
        L.oracle_pm_destroy.argtypes = [C.c_void_p]
        L.oracle_pm_gather_radius.restype = C.c_int
        L.oracle_pm_gather_radius.argtypes = [C.c_void_p, C.c_double, C.c_double]
        L.oracle_pm_gather.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_pm_first_estimate.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_pm_sample_rays.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
        L.oracle_pm_sample_pixels.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p]
        L.oracle_pm_knn.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        L.oracle_pm_render_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _refs(refs):
    """-> (array to keep alive, pointer): the leaf references' ordered primitives of a tree with spatial splits
    (mcrt.bvh4_split_host), or a null pointer: leaves index ordered primitives"""
    if refs is None:
        return None, None
    refs = np.ascontiguousarray(refs, dtype=np.uint32)
    return refs, _p(refs)


def sampler_stream(pixel, sample, n_shuffles, seed):
    pixel = np.ascontiguousarray(pixel, dtype=np.uint32); sample = np.ascontiguousarray(sample, dtype=np.uint32)
    out = np.zeros((len(pixel), 7), dtype=np.uint32)
    lib().oracle_sampler_stream(_p(pixel), _p(sample), len(pixel), n_shuffles, seed, _p(out))
    return out


def bvh_build(prim_bounds, scene_bounds, bvh_type, bins_per_axis, desc_type):
    """BVH::BVH restated (scalar, host). bvh_type: 0 octree, 1 binary_sah, 2 quaternary_sah; desc_type: the
    product's BvhDesc ctypes struct (layout only). -> dict of node arrays + prim_order."""
    prim_bounds = np.ascontiguousarray(prim_bounds, dtype=np.float64).reshape(-1, 6)
    scene_bounds = np.ascontiguousarray(scene_bounds, dtype=np.float64).reshape(6)
    h, d = C.c_void_p(), desc_type()
    lib().oracle_bvh_build(_p(prim_bounds), len(prim_bounds), _p(scene_bounds), int(bvh_type), int(bins_per_axis), C.byref(h), C.addressof(d))

    def arr(ptr, count, dtype):
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(count * np.dtype(dtype).itemsize,)).view(dtype).copy() if count else np.zeros(0, dtype)
    out = dict(node_bounds=arr(d.node_bounds, d.n_nodes * 6, np.float64).reshape(-1, 6), node_first_prim=arr(d.node_first_prim, d.n_nodes, np.uint32),
               node_prim_count=arr(d.node_prim_count, d.n_nodes, np.uint32), node_next_sibling=arr(d.node_next_sibling, d.n_nodes, np.uint32),
               prim_order=arr(d.prim_order, d.n_prims, np.uint32))
    lib().oracle_bvh_free(h)
    return out


def build_photon_octree(photons, max_photons_per_octree_leaf, scene_bounds, desc_type, map_arrays):
    """Octree<Photon> + LinearOctree::compact restated (scalar, host). desc_type / map_arrays: the
    product's PhotonMapDesc struct and its numpy unpacker (layout only)."""
    photons = np.ascontiguousarray(photons, dtype=np.float32).reshape(-1, 8)
    bounds = np.ascontiguousarray(scene_bounds, dtype=np.float64)
    h, d = C.c_void_p(), desc_type()
    lib().oracle_octree_build(_p(photons), len(photons), int(max_photons_per_octree_leaf), _p(bounds), C.byref(h), C.addressof(d))
    out = map_arrays(d)
    lib().oracle_octree_free(h)
    return out


def image_tonemap(rgb, params):
    """Image::save restated; params = the product's ImageParams ctypes struct (layout only)."""
    rgb = np.ascontiguousarray(rgb, dtype=np.float64)
    h, w = rgb.shape[:2]
    out = np.zeros((h, w, 3), dtype=np.uint8)
    e, g = C.c_double(), C.c_double()
    lib().oracle_image_tonemap(_p(rgb), w, h, C.addressof(params), _p(out), C.byref(e), C.byref(g))
    return out, e.value, g.value


class PortScene:
    """The restatement's view of a flattened scene (takes the product package's Scene only as a
    container of the float64 arrays and the ctypes struct layout)."""

    def __init__(self, scene):
        self.scene = scene
        self._desc = scene.desc()
        self.h = lib().oracle_scene_create(C.addressof(self._desc))
        self.pkg = importlib.import_module("monte-carlo-ray-tracer_b200")

    def close(self):
        if self.h:
            lib().oracle_scene_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def trace(self, rays):
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        hits = np.zeros(len(rays), dtype=self.pkg.HIT_DTYPE)
        lib().oracle_trace(self.h, _p(rays), len(rays), _p(hits))
        return hits

    def sample_rays(self, rays, pixel, sample, seed):
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        pixel = np.ascontiguousarray(pixel, dtype=np.uint32); sample = np.ascontiguousarray(sample, dtype=np.uint32)
        out = np.zeros((len(rays), 3))
        lib().oracle_sample_rays(self.h, _p(rays), _p(pixel), _p(sample), len(rays), seed, _p(out))
        return out

    def render_film(self, camera, sqrtspp, seed):
        """Whole frame through Film::deposit with the camera's reconstruction filter."""
        rec = camera.film_rec()
        default_radius = [0.5, 2.0, 2.0, 1.39, 1.0, 1.71, 2.0]   # film.cpp:32-45
        if rec.radius <= 0.0:
            rec.radius = default_radius[rec.filter]
        out = np.zeros((camera.height, camera.width, 3))
        lib().oracle_render_film(self.h, C.addressof(camera.rec), C.addressof(rec), sqrtspp, seed, _p(out))
        return out

    def trace_fast(self, nodes, scene_scale, rays, refs=None):
        """The product's order-free search restated on the CPU over `nodes` (mcrt.bvh4_host, or mcrt.bvh4_split_host's nodes with its
        `refs`: a leaf's (first, count) then index refs, and a repeat of the best primitive is not its competitor). Hits name ordered
        primitives. -> (hits, ambiguous flags, box tests, primitive tests)"""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        nodes = np.ascontiguousarray(nodes)
        refs, rp = _refs(refs)
        hits = np.zeros(len(rays), dtype=self.pkg.HIT_DTYPE)
        flags = np.zeros(len(rays), dtype=np.uint8)
        bt, pt = C.c_uint64(), C.c_uint64()
        lib().oracle_trace_fast(self.h, _p(nodes), len(nodes), rp, float(scene_scale), _p(rays), len(rays), _p(hits), _p(flags), C.byref(bt),
                                C.byref(pt))
        return hits, flags.astype(bool), bt.value, pt.value

    def trace_visible(self, nodes, scene_scale, rays, target, refs=None):
        """The product's occlusion query restated on the CPU (refs as trace_fast's; every reference of the target, an ordered primitive, is
        skipped). -> (verdict 0 visible / 1 not / 2 tie-to-replay, t of the target)"""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        target = np.ascontiguousarray(target, dtype=np.uint32)
        nodes = np.ascontiguousarray(nodes)
        refs, rp = _refs(refs)
        verdict = np.zeros(len(rays), dtype=np.uint8); t = np.zeros(len(rays))
        lib().oracle_trace_visible(self.h, _p(nodes), rp, float(scene_scale), _p(rays), _p(target), len(rays), _p(verdict), _p(t))
        return verdict, t

    def trace_peaks(self, rays):
        """trace() and, per ray, the largest number of entries the reference-order heap held -> (hits, heap peaks)"""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        hits = np.zeros(len(rays), dtype=self.pkg.HIT_DTYPE)
        peak = np.zeros(len(rays), dtype=np.uint32)
        lib().oracle_trace_peaks(self.h, _p(rays), len(rays), _p(hits), _p(peak))
        return hits, peak

    def trace_fast_peaks(self, nodes, scene_scale, rays, refs=None):
        """trace_fast() and, per ray, the largest number of entries the order-free search's stack held -> (hits, flags, stack peaks);
        a ray whose peak exceeds the device's stack is flagged"""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        nodes = np.ascontiguousarray(nodes)
        refs, rp = _refs(refs)
        hits = np.zeros(len(rays), dtype=self.pkg.HIT_DTYPE)
        flags = np.zeros(len(rays), dtype=np.uint8)
        peak = np.zeros(len(rays), dtype=np.uint32)
        lib().oracle_trace_fast_peaks(self.h, _p(nodes), rp, float(scene_scale), _p(rays), len(rays), _p(hits), _p(flags), _p(peak))
        return hits, flags.astype(bool), peak

    def trace_visible_peaks(self, nodes, scene_scale, rays, target, refs=None):
        """The occlusion query in the device's visiting order -> (verdict as trace_visible, t of the target, stack peaks)"""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        target = np.ascontiguousarray(target, dtype=np.uint32)
        nodes = np.ascontiguousarray(nodes)
        refs, rp = _refs(refs)
        verdict = np.zeros(len(rays), dtype=np.uint8); t = np.zeros(len(rays)); peak = np.zeros(len(rays), dtype=np.uint32)
        lib().oracle_trace_visible_peaks(self.h, _p(nodes), rp, float(scene_scale), _p(rays), _p(target), len(rays), _p(verdict), _p(t), _p(peak))
        return verdict, t, peak

    def wide_stack_bound(self, rays, margin):
        """Per ray, an upper bound on the entries of fast mode's depth-first stack: the largest sum of (hit children - 1) along a path of
        boxes, grown by `margin`, that the ray hits"""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        out = np.zeros(len(rays), dtype=np.uint32)
        lib().oracle_wide_stack_bound(self.h, _p(rays), len(rays), float(margin), _p(out))
        return out

    def sample_pixels(self, camera, pixel, sample, seed):
        """-> (rgb [n,3], camera rays [n,6]) for (pixel, sample) pairs"""
        pixel = np.ascontiguousarray(pixel, dtype=np.uint32); sample = np.ascontiguousarray(sample, dtype=np.uint32)
        rgb = np.zeros((len(pixel), 3)); rays = np.zeros((len(pixel), 6))
        lib().oracle_sample_pixels(self.h, C.addressof(camera.rec), _p(pixel), _p(sample), len(pixel), seed, _p(rgb), _p(rays))
        return rgb, rays

    def render_rows_checked(self, nodes, scene_scale, camera, y0, y1, sqrtspp, seed, refs=None):
        """render_rows with every Scene::intersect call cross-checked against the order-free search over `nodes` (refs as trace_fast's)
        -> (image, calls, flagged, mismatches)"""
        nodes = np.ascontiguousarray(nodes)
        refs, rp = _refs(refs)
        out = np.zeros((y1 - y0, camera.width, 3))
        counts = np.zeros(3, dtype=np.uint64)
        lib().oracle_render_rows_checked(self.h, _p(nodes), rp, float(scene_scale), C.addressof(camera.rec), y0, y1, sqrtspp, seed, _p(out),
                                         _p(counts))
        return out, int(counts[0]), int(counts[1]), int(counts[2])

    def render_rows(self, camera, y0, y1, sqrtspp, seed):
        out = np.zeros((y1 - y0, camera.width, 3))
        rays = C.c_uint64()
        lib().oracle_render_rows(self.h, C.addressof(camera.rec), y0, y1, sqrtspp, seed, _p(out), C.byref(rays))
        return out, rays.value

    # ---------------------------------------------------------------------------------------- photon mapper
    def photon_pass(self, emissions, caustic_factor, max_photons_per_octree_leaf, scene_bounds, seed, pass_index=0):
        """PhotonMapper::PhotonMapper's photon pass restated -> (caustic map, global map, (caustic lights, global lights),
        total emissions, (caustic paths, global paths)). Maps are dicts as the product's _map_arrays returns; lights: the
        emitting light of each photon; paths: light << 32 | the light's emission index, the path that stored each photon.
        pass_index: pass i of progressive photon mapping (PhotonMapper.emit_pass), light l's emissions at the indices
        [i * n_l, (i + 1) * n_l); raises ValueError, as the product refuses it, when they do not fit 32 bits."""
        if not 0 <= int(pass_index) < 1 << 32:
            raise ValueError(f"pass index {pass_index} is outside [0, 2^32)")
        bounds = np.ascontiguousarray(scene_bounds, dtype=np.float64).reshape(6)
        h = C.c_void_p()
        d = [self.pkg.PhotonMapDesc(), self.pkg.PhotonMapDesc()]
        path_ptrs = (C.c_void_p * 2)()
        total = C.c_uint64()
        if lib().oracle_photon_pass(self.h, int(emissions), float(caustic_factor), int(max_photons_per_octree_leaf), _p(bounds),
                                    int(pass_index), int(seed), C.byref(h), C.addressof(d[0]), C.addressof(d[1]),
                                    C.cast(path_ptrs, C.POINTER(C.c_void_p)), C.byref(total)):
            raise ValueError(f"photon pass {pass_index}: the pass's emission indices do not fit 32 bits")
        try:
            maps = [self.pkg._map_arrays(m) for m in d]
            paths = tuple(np.ctypeslib.as_array(C.cast(path_ptrs[w], C.POINTER(C.c_uint64)), shape=(int(d[w].n_photons),)).copy()
                          if d[w].n_photons else np.zeros(0, np.uint64) for w in range(2))
        finally:
            lib().oracle_photon_pass_free(h)
        return maps[0], maps[1], tuple((p >> np.uint64(32)).astype(np.uint32) for p in paths), total.value, paths

    def photon_mapper(self, maps):
        """PhotonMapper::sampleRay restated over `maps` = (caustic, global, k, direct_visualization), the tuple
        PhotonMapper(photon_maps=...) takes."""
        return PortPhotonMapper(self, maps)


class PortPhotonMapper:
    """The restatement's PhotonMapper::sampleRay over given maps. Every call returns (rgb, components, counts): components
    [..., 4, 3] in the order of the product's PHOTON_COMPONENT_NAMES (emission, direct, caustic, global), counts a dict of
    rays (every Scene::intersect call), shadow_rays, knn_queries, knn_ties (queries whose k-th distance is shared by a
    photon left out: the reference's choice between them follows its octree walk, which the brute-force search does not
    restate), empty_queries (queries that took no photon) and photons (photons taken by all queries).
    gather_radius switches the estimates to progressive photon mapping's fixed-radius gather, as the product's."""

    def __init__(self, ps, maps):
        caustic, glob, k, dv = maps
        self.ps = ps
        self.k, self.direct_visualization = int(k), bool(dv)
        self._keep = [np.ascontiguousarray(m["photons"], dtype=np.float32) for m in (caustic, glob)]
        self._desc = []
        for ph in self._keep:
            d = ps.pkg.PhotonMapDesc()
            d.n_photons = ph.size // 8
            d.photons = ph.ctypes.data_as(C.c_void_p) if ph.size else None
            self._desc.append(d)
        self.h = lib().oracle_pm_create(ps.h, C.addressof(self._desc[0]), C.addressof(self._desc[1]), self.k, int(self.direct_visualization))

    def close(self):
        if self.h:
            lib().oracle_pm_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _counts(c):
        return dict(rays=int(c[0]), shadow_rays=int(c[1]), knn_queries=int(c[2]), knn_ties=int(c[3]), empty_queries=int(c[4]),
                    photons=int(c[5]))

    def gather_radius(self, r_caustic, r_global):
        """Following estimates take every photon within r_caustic / r_global of a query, normalised by r^2 (k_gather);
        (0, 0) returns to the k-NN estimate. Raises ValueError for the radii PhotonMapper.gather_radius refuses."""
        if lib().oracle_pm_gather_radius(self.h, float(r_caustic), float(r_global)):
            raise ValueError(f"gather radii ({r_caustic}, {r_global}): (0, 0) or two positive finite numbers")
        self.gather_radii = (float(r_caustic), float(r_global))

    def gather(self, which, points, radius):
        """brute-force fixed-radius search of map `which` -> (count uint32 [n], flux_sum [n, 3], cone_sum [n, 3]), as
        PhotonMapper.gather"""
        points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        n = len(points)
        cnt = np.zeros(n, np.uint32); flux = np.zeros((n, 3)); cone = np.zeros((n, 3))
        lib().oracle_pm_gather(self.h, int(which), _p(points), n, float(radius), _p(cnt), _p(flux), _p(cone))
        return cnt, flux, cone

    def first_estimate(self, which, rays, pixel, sample, seed, radius):
        """The estimate of map `which` that sampleRay makes at the first vertex of each camera sample, gathered within
        radius[i] (0: the k nearest photons) -> (estimate [n, 3], vertex position [n, 3] (NaN: no hit), bool [n]: the
        vertex is not a delta one, so the estimate ran)"""
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        pixel = np.ascontiguousarray(pixel, dtype=np.uint32); sample = np.ascontiguousarray(sample, dtype=np.uint32)
        radius = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, np.float64), (len(rays),)))
        n = len(rays)
        out = np.zeros((n, 3)); pos = np.zeros((n, 3)); ran = np.zeros(n, np.uint8)
        lib().oracle_pm_first_estimate(self.h, int(which), _p(rays), _p(pixel), _p(sample), n, int(seed), _p(radius), _p(out), _p(pos),
                                       _p(ran))
        return out, pos, ran.astype(bool)

    def knn(self, which, points):
        """brute-force k nearest photons of map `which` -> (index [n, k], distance2 [n, k] nearest first, count [n], ties)"""
        points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        n = len(points)
        d2 = np.zeros((n, self.k)); idx = np.zeros((n, self.k), np.uint32); cnt = np.zeros(n, np.uint32); ties = C.c_uint64()
        lib().oracle_pm_knn(self.h, int(which), _p(points), n, _p(d2), _p(idx), _p(cnt), C.byref(ties))
        return idx, d2, cnt, ties.value

    def sample_rays(self, rays, pixel, sample, seed):
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        pixel = np.ascontiguousarray(pixel, dtype=np.uint32); sample = np.ascontiguousarray(sample, dtype=np.uint32)
        rgb = np.zeros((len(rays), 3)); comp = np.zeros((len(rays), 4, 3)); c = np.zeros(6, np.uint64)
        lib().oracle_pm_sample_rays(self.h, _p(rays), _p(pixel), _p(sample), len(rays), seed, _p(rgb), _p(comp), _p(c))
        return rgb, comp, self._counts(c)

    def sample_pixels(self, camera, pixel, sample, seed):
        """-> (rgb [n, 3], components [n, 4, 3], camera rays [n, 6], counts)"""
        pixel = np.ascontiguousarray(pixel, dtype=np.uint32); sample = np.ascontiguousarray(sample, dtype=np.uint32)
        n = len(pixel)
        rgb = np.zeros((n, 3)); comp = np.zeros((n, 4, 3)); rays = np.zeros((n, 6)); c = np.zeros(6, np.uint64)
        lib().oracle_pm_sample_pixels(self.h, C.addressof(camera.rec), _p(pixel), _p(sample), n, seed, _p(rgb), _p(comp), _p(rays), _p(c))
        return rgb, comp, rays, self._counts(c)

    def render_rows(self, camera, y0, y1, sqrtspp, seed):
        """-> (frame [rows, width, 3], component frames [4, rows, width, 3] (per-pixel means), counts)"""
        out = np.zeros((y1 - y0, camera.width, 3)); comp = np.zeros((4, y1 - y0, camera.width, 3)); c = np.zeros(6, np.uint64)
        lib().oracle_pm_render_rows(self.h, C.addressof(camera.rec), y0, y1, sqrtspp, seed, _p(out), _p(comp), _p(c))
        return out, comp, self._counts(c)
