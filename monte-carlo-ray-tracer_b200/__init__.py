"""H100-native path-tracing integrator for the ray/BVH/BSDF hot path of
linusmossberg/monte-carlo-ray-tracer — Python host mirror over the C ABI (include/mcrt_abi.h).

The names follow the reference's classes for this path:
    Scene            flattened Scene + BVH          (source/scene/scene.hpp, source/bvh/bvh.hpp)
    Camera           camera state + sampleImage     (source/camera/camera.cpp:20-145)
    PathTracer       Integrator::sampleRay, batched (source/integrator/path-tracer/path-tracer.cpp)
    PhotonMapper     same with photon maps          (source/integrator/photon-mapper/photon-mapper.cpp)
Everything that computes runs in libmcrt_b200.so on the GPU; this module only marshals buffers.
There is no CPU fallback: importing works anywhere (so that symbols can be checked), but any compute
call without the built library or without a CUDA device raises."""
import ctypes as C
import math
import os
import struct

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MCRT_LIB", os.path.join(HERE, "libmcrt_b200.so"))  # MCRT_LIB: tuning variants

INTEGRATOR_PATH, INTEGRATOR_PHOTON = 0, 1
PRECISION_F64, PRECISION_F32 = 0, 1
PRIM_TRIANGLE, PRIM_SPHERE, PRIM_QUADRIC = 0, 1, 2
NO_PRIM = 0xFFFFFFFF

ABI_SYMBOLS = [
    "mcrt_abi_version", "mcrt_init", "mcrt_destroy", "mcrt_last_error", "mcrt_scene_upload",
    "mcrt_photon_upload", "mcrt_photon_emit", "mcrt_photon_download", "mcrt_octree_build",
    "mcrt_octree_free", "mcrt_render_rows", "mcrt_render_rows_dev", "mcrt_render_rows_strided_dev",
    "mcrt_trace_closest",
    "mcrt_sample_rays", "mcrt_sampler_stream", "mcrt_knn_search", "mcrt_set_option", "mcrt_set_film",
    "mcrt_obj_load", "mcrt_obj_free", "mcrt_obj_vertex_normals",
    "mcrt_bvh_build", "mcrt_bvh_free", "mcrt_image_tonemap", "mcrt_image_tonemap_dev",
    "mcrt_render_rows_strided_peers", "mcrt_frame_alloc", "mcrt_frame_open", "mcrt_frame_close", "mcrt_frame_free",
    "mcrt_render_film_sums_strided_dev", "mcrt_film_resolve_dev",
    "mcrt_bvh4_host", "mcrt_bvh4_host_free",
    "mcrt_fp64_peak", "mcrt_photon_emit_total", "mcrt_photon_emit_range", "mcrt_photon_build_dev",
    "mcrt_render_accumulate_dev", "mcrt_progressive_resolve_dev",
    "mcrt_render_accumulate_tiles_dev", "mcrt_progressive_resolve_tiles_dev",
    "mcrt_render_features_dev", "mcrt_denoise_dev", "mcrt_render_features_chain_dev",
    "mcrt_photon_emit_pass", "mcrt_photon_gather_radius", "mcrt_photon_gather_search",
    "mcrt_set_light_groups", "mcrt_render_accumulate_groups_dev", "mcrt_light_groups_combine_dev",
    "mcrt_render_accumulate_aovs_dev", "mcrt_photon_download_lights", "mcrt_render_accumulate_photon_components_dev",
    "mcrt_set_light_path_expressions", "mcrt_render_accumulate_lpe_dev", "mcrt_lpe_compile_host",
    "mcrt_lpe_compile_photon_host", "mcrt_photon_download_lpe_states",
]

# The light-path AOV planes of mcrt_render_accumulate_aovs_dev, in plane order (MCRT_AOV_* of include/mcrt_abi.h):
# the camera ray's own sky and emitter, then direct / indirect light by the lobe of the first scattering vertex
AOV_NAMES = ("background", "emission", "diffuse_direct", "diffuse_indirect", "reflection_direct", "reflection_indirect",
             "transmission_direct", "transmission_indirect")

# The photon mapper's component planes of mcrt_render_accumulate_photon_components_dev, in plane order (MCRT_PM_* of
# include/mcrt_abi.h): emitters seen from the camera, Monte Carlo direct light, the caustic-map and global-map estimates
PHOTON_COMPONENT_NAMES = ("emission", "direct", "caustic", "global")

# Light path expressions (mcrt_set_light_path_expressions): the event symbols of the compiled table (MCRT_LPE_SYM_* of
# include/mcrt_abi.h); label k of a table is symbol LPE_SYM_LABEL0 + k
LPE_SYM_RD, LPE_SYM_RS, LPE_SYM_RG, LPE_SYM_TS, LPE_SYM_TG, LPE_SYM_B, LPE_SYM_L, LPE_SYM_LABEL0 = range(8)
LPE_DEAD, LPE_MAX_STATES, LPE_MAX_SYMBOLS, LPE_MAX_EXPRESSIONS = 255, 255, 71, 32
# The light-path AOV planes of AOV_NAMES as light path expressions, in the same order
AOV_LPES = ("CB", "CL", "C<RD>[LB]", "C<RD>.+[LB]", "C[<RS><RG>][LB]", "C[<RS><RG>].+[LB]", "C<T.>[LB]", "C<T.>.+[LB]")


def PM_COMPONENT_LPES(direct_visualization):
    """The photon mapper's component planes of PHOTON_COMPONENT_NAMES as light path expressions, in the same order, for
    maps emitted with (True) or without (False) direct_visualization. N = [<RD><RG><TG>] is a non-delta event; the
    camera path reaches its first non-delta vertex x through smooth events <.S>*.

    Without direct visualization, light at x comes from next-event estimation (C S* x L, direct) and the caustic map
    (C S* x <.S> ..., caustic); the global map is gathered one non-delta bounce later (C S* x N ..., global).

    With it, both maps are gathered at x and no shadow ray is traced, so a direct photon stored at x reads C S* x L,
    the string next-event estimation would have: that string belongs to the global estimate, and the direct plane,
    which is then zero, takes "C.*B", which no photon-mapped path matches (the photon mapper has no sky)."""
    n = "[<RD><RG><TG>]"
    if direct_visualization:
        return ("C<.S>*L", "C.*B", f"C<.S>*{n}<.S>.*L", f"C<.S>*{n}({n}.*)?L")
    return ("C<.S>*L", f"C<.S>*{n}L", f"C<.S>*{n}{{1,2}}<.S>.*L", f"C<.S>*{n}{{2}}({n}.*)?L")


class McrtError(RuntimeError):
    pass


# ------------------------------------------------------------------------------------ ctypes structs
class DenoiseParams(C.Structure):
    _fields_ = [("iterations", C.c_uint32), ("_pad", C.c_uint32), ("sigma_color", C.c_double), ("sigma_normal", C.c_double),
                ("sigma_depth", C.c_double), ("sigma_albedo", C.c_double)]


# MCRT_DENOISE_DEFAULT_* of mcrt_abi.h
DENOISE_DEFAULTS = {"iterations": 5, "sigma_color": 1.0, "sigma_normal": 64.0, "sigma_depth": 0.1, "sigma_albedo": 0.1}
FEATURES_MAX_SPECULAR_DEPTH = 7   # MCRT_FEATURES_MAX_SPECULAR_DEPTH


class MaterialRec(C.Structure):
    _fields_ = [("reflectance", C.c_double * 3), ("specular_reflectance", C.c_double * 3),
                ("transmittance", C.c_double * 3), ("emittance", C.c_double * 3),
                ("roughness", C.c_double), ("specular_roughness", C.c_double), ("ior", C.c_double),
                ("transparency", C.c_double), ("complex_ior_real", C.c_double * 3),
                ("complex_ior_imag", C.c_double * 3), ("A", C.c_double), ("B", C.c_double),
                ("a", C.c_double * 2), ("has_complex_ior", C.c_uint32), ("perfect_mirror", C.c_uint32),
                ("rough", C.c_uint32), ("rough_specular", C.c_uint32), ("opaque", C.c_uint32),
                ("emissive", C.c_uint32), ("dirac_delta", C.c_uint32), ("_pad", C.c_uint32)]


MATERIAL_DTYPE = np.dtype([
    ("reflectance", "<f8", 3), ("specular_reflectance", "<f8", 3), ("transmittance", "<f8", 3),
    ("emittance", "<f8", 3), ("roughness", "<f8"), ("specular_roughness", "<f8"), ("ior", "<f8"),
    ("transparency", "<f8"), ("complex_ior_real", "<f8", 3), ("complex_ior_imag", "<f8", 3),
    ("A", "<f8"), ("B", "<f8"), ("a", "<f8", 2), ("has_complex_ior", "<u4"), ("perfect_mirror", "<u4"),
    ("rough", "<u4"), ("rough_specular", "<u4"), ("opaque", "<u4"), ("emissive", "<u4"),
    ("dirac_delta", "<u4"), ("_pad", "<u4")])
assert MATERIAL_DTYPE.itemsize == C.sizeof(MaterialRec)


class SceneDesc(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("n_nodes", C.c_uint32),
                ("node_bounds", C.c_void_p), ("node_first_prim", C.c_void_p),
                ("node_prim_count", C.c_void_p), ("node_next_sibling", C.c_void_p),
                ("n_prims", C.c_uint32),
                ("prim_type", C.c_void_p), ("prim_index", C.c_void_p), ("prim_material", C.c_void_p),
                ("prim_area", C.c_void_p),
                ("n_tris", C.c_uint32),
                ("tri_v0", C.c_void_p), ("tri_v1", C.c_void_p), ("tri_v2", C.c_void_p),
                ("tri_e1", C.c_void_p), ("tri_e2", C.c_void_p), ("tri_normal", C.c_void_p),
                ("tri_vn_index", C.c_void_p),
                ("n_vertex_normals", C.c_uint32), ("vertex_normals", C.c_void_p),
                ("n_spheres", C.c_uint32), ("sphere_origin_radius", C.c_void_p),
                ("n_quadrics", C.c_uint32),
                ("quadric_Q", C.c_void_p), ("quadric_G", C.c_void_p), ("quadric_bounds", C.c_void_p),
                ("n_materials", C.c_uint32), ("materials", C.c_void_p),
                ("n_lights", C.c_uint32), ("light_prim", C.c_void_p), ("light_cdf", C.c_void_p),
                ("scene_ior", C.c_double)]


class CameraRec(C.Structure):
    _fields_ = [("eye", C.c_double * 3), ("forward", C.c_double * 3), ("left", C.c_double * 3),
                ("up", C.c_double * 3), ("focal_length", C.c_double), ("sensor_width", C.c_double),
                ("aperture_radius", C.c_double), ("focus_distance", C.c_double),
                ("width", C.c_uint32), ("height", C.c_uint32), ("thin_lens", C.c_uint32), ("_pad", C.c_uint32)]


class FilmRec(C.Structure):
    _fields_ = [("filter", C.c_uint32), ("cache_size", C.c_uint32), ("radius", C.c_double)]


FILM_FILTERS = {"box": 0, "mitchell-netravali": 1, "catmull-rom": 2, "b-spline": 3, "hermite": 4, "gaussian": 5,
                "lanczos": 6}


class HitRec(C.Structure):
    _fields_ = [("t", C.c_double), ("u", C.c_double), ("v", C.c_double), ("prim", C.c_uint32),
                ("interpolate", C.c_uint32)]


HIT_DTYPE = np.dtype([("t", "<f8"), ("u", "<f8"), ("v", "<f8"), ("prim", "<u4"), ("interpolate", "<u4")])


class PhotonMapDesc(C.Structure):
    _fields_ = [("n_octants", C.c_uint32), ("octant_bounds", C.c_void_p), ("octant_start", C.c_void_p),
                ("octant_count", C.c_void_p), ("octant_next_sibling", C.c_void_p), ("octant_leaf", C.c_void_p),
                ("n_photons", C.c_uint64), ("photons", C.c_void_p)]


class ImageParams(C.Structure):
    """The camera's "image" object (image.cpp:10-35) without the size."""
    _fields_ = [("plain", C.c_uint32), ("tonemapper", C.c_uint32), ("exposure_scale", C.c_double),
                ("gain_scale", C.c_double)]

    @classmethod
    def from_json(cls, image):
        tm = str(image.get("tonemapper", "HABLE")).upper()
        return cls(int(bool(image.get("plain", False))), 1 if tm == "ACES" else 0,
                   math.pow(2, image.get("exposure_compensation", 0.0)), math.pow(2, image.get("gain_compensation", 0.0)))


class ObjMeshRec(C.Structure):
    _fields_ = [("n_vertices", C.c_uint64), ("n_normals", C.c_uint64), ("n_tri_v", C.c_uint64), ("n_tri_vt", C.c_uint64),
                ("n_tri_vn", C.c_uint64), ("vertices", C.c_void_p), ("normals", C.c_void_p), ("tri_v", C.c_void_p),
                ("tri_vt", C.c_void_p), ("tri_vn", C.c_void_p)]


class BvhDesc(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("n_prims", C.c_uint32), ("node_bounds", C.c_void_p),
                ("node_first_prim", C.c_void_p), ("node_prim_count", C.c_void_p), ("node_next_sibling", C.c_void_p),
                ("prim_order", C.c_void_p), ("build_rounds", C.c_uint32), ("kernel_launches", C.c_uint32)]


BVH_TYPES = {"octree": 0, "binary_sah": 1, "quaternary_sah": 2}


class PhotonEmitParams(C.Structure):
    _fields_ = [("emissions", C.c_uint64), ("caustic_factor", C.c_double), ("max_photons_per_octree_leaf", C.c_uint32),
                ("k_nearest_photons", C.c_uint32), ("direct_visualization", C.c_uint32), ("global_seed", C.c_uint32),
                ("scene_bounds", C.c_double * 6)]


class Stats(C.Structure):
    _fields_ = [("paths", C.c_uint64), ("extension_rays", C.c_uint64), ("shadow_rays", C.c_uint64),
                ("box_tests", C.c_uint64), ("prim_tests", C.c_uint64), ("knn_queries", C.c_uint64),
                ("wavefront_iterations", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("ior_stack_overflows", C.c_uint64), ("max_depth", C.c_uint32), ("_pad", C.c_uint32),
                ("gpu_ms_total", C.c_double), ("gpu_ms_generate", C.c_double), ("gpu_ms_extend", C.c_double),
                ("gpu_ms_shade", C.c_double), ("gpu_ms_shadow", C.c_double), ("gpu_ms_knn", C.c_double),
                ("extend_launches", C.c_uint64), ("shadow_launches", C.c_uint64),
                ("shadow_box_tests", C.c_uint64), ("shadow_prim_tests", C.c_uint64),
                ("extend_work_sum", C.c_uint64), ("extend_work_warpmax", C.c_uint64),
                ("replayed_rays", C.c_uint64)]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_ if not f.startswith("_")}


_lib = None


def lib():
    """The C-ABI library. Raises if it has not been built (no CPU fallback exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise McrtError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(LIB_PATH)
        L.mcrt_abi_version.restype = C.c_int
        L.mcrt_init.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.mcrt_destroy.argtypes = [C.c_void_p]
        L.mcrt_destroy.restype = None
        L.mcrt_last_error.argtypes = [C.c_void_p]
        L.mcrt_last_error.restype = C.c_char_p
        L.mcrt_scene_upload.argtypes = [C.c_void_p, C.POINTER(SceneDesc), C.POINTER(C.c_uint64)]
        L.mcrt_photon_upload.argtypes = [C.c_void_p, C.POINTER(PhotonMapDesc), C.POINTER(PhotonMapDesc),
                                         C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64)]
        L.mcrt_photon_emit.argtypes = [C.c_void_p, C.POINTER(PhotonEmitParams), C.c_int, C.POINTER(C.c_uint64),
                                       C.POINTER(C.c_uint64), C.POINTER(Stats)]
        L.mcrt_photon_emit_pass.argtypes = [C.c_void_p, C.POINTER(PhotonEmitParams), C.c_int, C.c_uint32, C.POINTER(C.c_uint64),
                                            C.POINTER(C.c_uint64), C.POINTER(Stats)]
        L.mcrt_photon_gather_radius.argtypes = [C.c_void_p, C.c_double, C.c_double]
        L.mcrt_photon_gather_search.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_double, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.POINTER(Stats)]
        L.mcrt_photon_download.argtypes = [C.c_void_p, C.c_int, C.POINTER(PhotonMapDesc)]
        L.mcrt_photon_download_lights.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64]
        L.mcrt_photon_download_lpe_states.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64]
        L.mcrt_octree_build.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.POINTER(C.c_void_p),
                                        C.POINTER(PhotonMapDesc), C.POINTER(C.c_double)]
        L.mcrt_octree_free.argtypes = [C.c_void_p]
        L.mcrt_octree_free.restype = None
        render_args = [C.c_void_p, C.POINTER(CameraRec), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                       C.c_int, C.c_int, C.c_void_p, C.POINTER(Stats)]
        L.mcrt_render_rows.argtypes = render_args
        L.mcrt_render_rows_dev.argtypes = render_args
        L.mcrt_render_rows_strided_dev.argtypes = [C.c_void_p, C.POINTER(CameraRec), C.c_uint32, C.c_uint32, C.c_uint32,
                                                   C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.POINTER(Stats)]
        L.mcrt_render_rows_strided_peers.argtypes = [C.c_void_p, C.POINTER(CameraRec), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                     C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_uint32, C.c_int, C.POINTER(Stats)]
        L.mcrt_frame_alloc.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p), C.c_void_p]
        L.mcrt_frame_open.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
        L.mcrt_frame_close.argtypes = [C.c_void_p, C.c_void_p]
        L.mcrt_frame_free.argtypes = [C.c_void_p, C.c_void_p]
        L.mcrt_fp64_peak.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        L.mcrt_bvh4_host.argtypes = [C.POINTER(SceneDesc), C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]
        L.mcrt_bvh4_host_free.argtypes = [C.c_void_p]
        L.mcrt_bvh4_host_free.restype = None
        L.mcrt_render_film_sums_strided_dev.argtypes = [C.c_void_p, C.POINTER(CameraRec), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                        C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(Stats)]
        L.mcrt_film_resolve_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        L.mcrt_render_accumulate_dev.argtypes = [C.c_void_p, C.POINTER(CameraRec), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                 C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(Stats)]
        L.mcrt_progressive_resolve_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
                                                   C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]
        L.mcrt_render_accumulate_tiles_dev.argtypes = [C.c_void_p, C.POINTER(CameraRec), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                       C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_void_p,
                                                       C.c_void_p, C.POINTER(Stats)]
        L.mcrt_progressive_resolve_tiles_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                         C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                         C.POINTER(C.c_double)]
        L.mcrt_set_light_groups.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
        L.mcrt_render_accumulate_groups_dev.argtypes = [C.c_void_p, C.POINTER(CameraRec), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                        C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_void_p,
                                                        C.c_uint32, C.POINTER(Stats)]
        L.mcrt_render_accumulate_aovs_dev.argtypes = L.mcrt_render_accumulate_groups_dev.argtypes
        L.mcrt_render_accumulate_photon_components_dev.argtypes = L.mcrt_render_accumulate_groups_dev.argtypes
        L.mcrt_set_light_path_expressions.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.mcrt_render_accumulate_lpe_dev.argtypes = L.mcrt_render_accumulate_groups_dev.argtypes
        L.mcrt_lpe_compile_host.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_char_p, C.c_uint32]
        L.mcrt_lpe_compile_photon_host.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32),
                                                   C.POINTER(C.c_uint32), C.c_void_p, C.c_char_p, C.c_uint32]
        L.mcrt_light_groups_combine_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_void_p]
        L.mcrt_render_features_dev.argtypes = [C.c_void_p, C.POINTER(CameraRec), C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                               C.c_void_p, C.POINTER(Stats)]
        L.mcrt_render_features_chain_dev.argtypes = [C.c_void_p, C.POINTER(CameraRec), C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                                     C.c_uint32, C.c_void_p, C.POINTER(Stats)]
        L.mcrt_denoise_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                       C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(DenoiseParams), C.c_void_p,
                                       C.POINTER(C.c_double)]
        L.mcrt_photon_emit_total.argtypes = [C.c_void_p, C.POINTER(PhotonEmitParams), C.POINTER(C.c_uint64)]
        L.mcrt_photon_emit_range.argtypes = [C.c_void_p, C.POINTER(PhotonEmitParams), C.c_int, C.c_uint64, C.c_uint64, C.POINTER(C.c_void_p),
                                             C.POINTER(C.c_uint64), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(Stats)]
        L.mcrt_photon_build_dev.argtypes = [C.c_void_p, C.POINTER(PhotonEmitParams), C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                            C.POINTER(C.c_double)]
        L.mcrt_trace_closest.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.POINTER(Stats)]
        L.mcrt_sample_rays.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32,
                                       C.c_int, C.c_int, C.c_void_p, C.POINTER(Stats)]
        L.mcrt_sampler_stream.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p]
        L.mcrt_knn_search.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.POINTER(Stats)]
        L.mcrt_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
        L.mcrt_set_film.argtypes = [C.c_void_p, C.POINTER(FilmRec)]
        L.mcrt_bvh_build.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_int,
                                     C.POINTER(C.c_void_p), C.POINTER(BvhDesc), C.POINTER(C.c_double)]
        L.mcrt_bvh_free.argtypes = [C.c_void_p]
        L.mcrt_bvh_free.restype = None
        L.mcrt_obj_load.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(ObjMeshRec), C.c_char_p, C.c_size_t]
        L.mcrt_obj_free.argtypes = [C.c_void_p]
        L.mcrt_obj_free.restype = None
        L.mcrt_obj_vertex_normals.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
        tm_args = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(ImageParams), C.c_void_p,
                   C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.mcrt_image_tonemap.argtypes = tm_args
        L.mcrt_image_tonemap_dev.argtypes = tm_args
        if L.mcrt_abi_version() != 1:
            raise McrtError("libmcrt_b200.so ABI version mismatch")
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None and a.size else None


# ------------------------------------------------------------------------------------ scene packs
_PACK_DTYPES = {0: np.uint8, 1: np.uint32, 2: np.int32, 3: np.uint64, 4: np.float32, 5: np.float64}


def read_pack(path):
    """Reads a scene pack written by host/exporter.cpp (PackWriter) → dict of numpy arrays."""
    if path.endswith(".xz"):   # large OBJ-scene packs are shipped xz-compressed (float64 arrays: ~5x)
        import lzma
        with lzma.open(path, "rb") as f:
            blob = f.read()
    else:
        with open(path, "rb") as f:
            blob = f.read()
    if blob[:8] != b"MCRTPK01":
        raise McrtError(f"{path}: not a scene pack")
    n, = struct.unpack_from("<I", blob, 8)
    out = {}
    for i in range(n):
        name, dtype, elem_size, count, offset = struct.unpack_from("<32sIIQQ", blob, 16 + 56 * i)
        name = name.split(b"\0")[0].decode()
        if dtype == 6:
            if name != "materials" or elem_size != MATERIAL_DTYPE.itemsize:
                raise McrtError(f"{path}: unexpected struct entry {name}")
            arr = np.frombuffer(blob, dtype=MATERIAL_DTYPE, count=count, offset=offset)
        else:
            arr = np.frombuffer(blob, dtype=_PACK_DTYPES[dtype], count=count, offset=offset)
        out[name] = arr.copy()
    return out


class Scene:
    """Flattened reference Scene (surfaces, materials, emissives, BVH) as float64 arrays."""

    _ARRAYS = ["node_bounds", "node_first_prim", "node_prim_count", "node_next_sibling", "prim_type",
               "prim_index", "prim_material", "prim_area", "tri_v0", "tri_v1", "tri_v2", "tri_e1", "tri_e2",
               "tri_normal", "tri_vn_index", "vertex_normals", "sphere_origin_radius", "quadric_Q",
               "quadric_G", "quadric_bounds", "materials", "light_prim", "light_cdf"]

    def __init__(self, arrays):
        self.a = {k: np.ascontiguousarray(arrays[k]) for k in self._ARRAYS}
        self.ior = float(np.asarray(arrays["scene_ior"]).reshape(-1)[0])
        self.extra = {k: v for k, v in arrays.items() if k not in self._ARRAYS}

    @classmethod
    def from_pack(cls, path):
        return cls(read_pack(path))

    @property
    def n_prims(self):
        return int(self.a["prim_type"].size)

    @property
    def n_nodes(self):
        return int(self.a["node_first_prim"].size)

    @property
    def n_lights(self):
        return int(self.a["light_prim"].size)

    def desc(self):
        a = self.a
        d = SceneDesc()
        d.abi_version = 1
        d.n_nodes = a["node_first_prim"].size
        d.n_prims = a["prim_type"].size
        d.n_tris = a["tri_vn_index"].size
        d.n_vertex_normals = a["vertex_normals"].size // 9
        d.n_spheres = a["sphere_origin_radius"].size // 4
        d.n_quadrics = a["quadric_bounds"].size // 6
        d.n_materials = a["materials"].size
        d.n_lights = a["light_prim"].size
        for k in self._ARRAYS:
            setattr(d, k, _ptr(a[k]))
        d.scene_ior = self.ior
        return d

    # -- inputs / outputs of BVH::BVH (mcrt_bvh_build)
    def prim_bounds(self):
        """Surface::Base::BB() of every primitive, [n_prims, 6] (triangle.cpp:115-122, sphere.cpp:56-62,
        quadric BB_)."""
        a = self.a
        out = np.zeros((self.n_prims, 6))
        t, i = a["prim_type"], a["prim_index"]
        tri = t == PRIM_TRIANGLE
        if tri.any():
            v = np.stack([a["tri_v0"].reshape(-1, 3), a["tri_v1"].reshape(-1, 3), a["tri_v2"].reshape(-1, 3)])[:, i[tri]]
            out[tri, :3] = v.min(axis=0); out[tri, 3:] = v.max(axis=0)
        sph = t == PRIM_SPHERE
        if sph.any():
            s = a["sphere_origin_radius"].reshape(-1, 4)[i[sph]]
            out[sph, :3] = s[:, :3] - s[:, 3:4]; out[sph, 3:] = s[:, :3] + s[:, 3:4]
        quad = t == PRIM_QUADRIC
        if quad.any():
            out[quad] = a["quadric_bounds"].reshape(-1, 6)[i[quad]]
        return out

    def reordered(self, order, bvh=None):
        """Scene whose primitive k is this scene's primitive order[k]; node arrays from `bvh` (a dict as
        returned by bvh_build) or none (Scene::intersect then scans all primitives, scene.cpp:159-171)."""
        order = np.asarray(order, dtype=np.int64)
        arrays = dict(self.a, **self.extra)
        arrays["scene_ior"] = np.array([self.ior])
        for k in ("prim_type", "prim_index", "prim_material", "prim_area"):
            arrays[k] = self.a[k][order]
        inverse = np.empty(len(order), dtype=np.int64)
        inverse[order] = np.arange(len(order))
        arrays["light_prim"] = inverse[self.a["light_prim"]].astype(np.uint32)
        if "prim_original" in arrays:
            arrays["prim_original"] = arrays["prim_original"][order]
        for k, dt in (("node_bounds", np.float64), ("node_first_prim", np.uint32), ("node_prim_count", np.uint32),
                      ("node_next_sibling", np.uint32)):
            arrays[k] = np.ascontiguousarray(bvh[k], dtype=dt).reshape(-1) if bvh is not None else np.zeros(0, dtype=dt)
        return Scene(arrays)

    def unbuilt(self):
        """The scene as BVH::BVH receives it: primitives in Scene::surfaces order, no hierarchy."""
        return self.reordered(np.argsort(self.extra["prim_original"], kind="stable"))

    def with_bvh(self, bvh):
        return self.reordered(bvh["prim_order"], bvh)

    def cameras(self):
        """Cameras stored in the pack (the exporter writes the one the scene was opened with)."""
        cams = []
        if "camera_f64" in self.extra:
            cams.append(Camera.from_pack_arrays(self.extra["camera_f64"], self.extra["camera_u32"],
                                                self.extra.get("camera_film_u32"), self.extra.get("camera_film_f64")))
        return cams

    def photon_maps(self):
        e = self.extra
        if "photon_params" not in e:
            return None
        maps = []
        for prefix in ("caustic", "global"):
            maps.append({k: e[f"{prefix}_{k}"] for k in
                         ("octant_bounds", "octant_start", "octant_count", "octant_next", "octant_leaf", "photons")})
        return maps[0], maps[1], int(e["photon_params"][0]), int(e["photon_params"][1])


class Camera:
    """Camera state after the reference's Camera::Camera (camera.cpp:20-64)."""

    def __init__(self, eye, forward, left, up, focal_length, sensor_width, width, height,
                 aperture_radius=-1.0, focus_distance=-1.0, thin_lens=False, sqrtspp=1, film=None):
        """film: None (default box film) or dict(filter=name|code, radius=None, cache_size=0), the camera's
        "film" object in the scene JSON (source/camera/film.cpp:19-59)."""
        self.film = dict(film) if film else None
        self.rec = CameraRec()
        for name, v in (("eye", eye), ("forward", forward), ("left", left), ("up", up)):
            for i in range(3):
                getattr(self.rec, name)[i] = float(v[i])
        self.rec.focal_length = focal_length
        self.rec.sensor_width = sensor_width
        self.rec.aperture_radius = aperture_radius
        self.rec.focus_distance = focus_distance
        self.rec.width, self.rec.height = int(width), int(height)
        self.rec.thin_lens = int(bool(thin_lens))
        self.sqrtspp = int(sqrtspp)

    @classmethod
    def from_pack_arrays(cls, f64, u32, film_u32=None, film_f64=None):
        film = None
        if film_u32 is not None and not (int(film_u32[0]) == 0 and float(film_f64[0]) == 0.5):
            film = dict(filter=int(film_u32[0]), cache_size=int(film_u32[1]), radius=float(film_f64[0]))
        return cls(f64[0:3], f64[3:6], f64[6:9], f64[9:12], f64[12], f64[13], u32[0], u32[1],
                   f64[14], f64[15], bool(u32[2]), int(u32[3]), film)

    def film_rec(self):
        """mcrt_film of this camera, or None for the default box film."""
        if not self.film:
            return None
        f = self.film.get("filter", "box")
        code = FILM_FILTERS[f.lower()] if isinstance(f, str) else int(f)
        radius = self.film.get("radius")
        return FilmRec(code, int(self.film.get("cache_size") or 0), float(radius) if radius else 0.0)

    @property
    def width(self):
        return self.rec.width

    @property
    def height(self):
        return self.rec.height

    def resized(self, width, height, sqrtspp=None):
        c = Camera(self.rec.eye, self.rec.forward, self.rec.left, self.rec.up, self.rec.focal_length,
                   self.rec.sensor_width, width, height, self.rec.aperture_radius, self.rec.focus_distance,
                   self.rec.thin_lens, self.sqrtspp if sqrtspp is None else sqrtspp, self.film)
        return c


class Integrator:
    """GPU context + uploaded scene. Mirrors class Integrator (source/integrator/integrator.hpp:7-30):
    owns the Scene, exposes sampleRay (batched) and is what Camera.sampleImage renders through."""

    kind = INTEGRATOR_PATH

    def __init__(self, scene, device=0, precision=PRECISION_F64, global_seed=0x12345678):
        self.scene = scene
        self.precision = precision
        self.global_seed = global_seed & 0xFFFFFFFF
        self.ctx = C.c_void_p()
        rc = lib().mcrt_init(device, C.byref(self.ctx))
        if rc:
            self.ctx = C.c_void_p()
            raise McrtError(f"mcrt_init(device={device}) failed with {rc}: no CUDA device? (there is no CPU fallback)")
        self.device = device
        self.h2d_bytes = 0
        self.upload_scene()
        self.last_stats = None

    def _check(self, rc):
        if rc:
            e = McrtError(f"mcrt error {rc}: {lib().mcrt_last_error(self.ctx).decode()}")
            e.code = rc       # the MCRT_ERR_* value
            raise e

    def set_option(self, key, value):
        self._check(lib().mcrt_set_option(self.ctx, key.encode(), float(value)))

    def upload_scene(self):
        d = self.scene.desc()
        n = C.c_uint64()
        # the library clears the group and LPE tables and forgets which table the maps were emitted under
        self._lpe_key = self._groups_key = self._photon_lpe_key = None
        self._check(lib().mcrt_scene_upload(self.ctx, C.byref(d), C.byref(n)))
        self.h2d_bytes = n.value
        return n.value

    def close(self):
        if getattr(self, "ctx", None):
            lib().mcrt_destroy(self.ctx)
            self.ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- Integrator::sampleRay, batched
    def sampleRay(self, rays, pixel, sample, precision=None):
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        pixel = np.ascontiguousarray(pixel, dtype=np.uint32)
        sample = np.ascontiguousarray(sample, dtype=np.uint32)
        out = np.zeros((len(rays), 3))
        st = Stats()
        self._check(lib().mcrt_sample_rays(self.ctx, _ptr(rays), _ptr(pixel), _ptr(sample), len(rays),
                                           self.global_seed, self.kind,
                                           self.precision if precision is None else precision, _ptr(out), C.byref(st)))
        self.last_stats = st.as_dict()
        return out

    # -- Scene::intersect, batched
    def intersect(self, rays, precision=None):
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        hits = np.zeros(len(rays), dtype=HIT_DTYPE)
        st = Stats()
        self._check(lib().mcrt_trace_closest(self.ctx, _ptr(rays), len(rays),
                                             self.precision if precision is None else precision, _ptr(hits), C.byref(st)))
        self.last_stats = st.as_dict()
        return hits

    # -- Camera::sampleImage for a block of rows (box film), host output
    def set_film(self, camera):
        """Film of the following renders = the camera's (Camera owns its Film, camera.cpp:34-37)."""
        rec = camera.film_rec()
        self._check(lib().mcrt_set_film(self.ctx, C.byref(rec) if rec is not None else None))

    def render_rows(self, camera, y0=0, y1=None, sqrtspp=None, precision=None, out=None):
        y1 = camera.height if y1 is None else y1
        self.set_film(camera)
        if out is None:
            out = np.zeros((y1 - y0, camera.width, 3))
        st = Stats()
        self._check(lib().mcrt_render_rows(self.ctx, C.byref(camera.rec), y0, y1,
                                           camera.sqrtspp if sqrtspp is None else sqrtspp, self.global_seed, self.kind,
                                           self.precision if precision is None else precision, _ptr(out), C.byref(st)))
        self.last_stats = st.as_dict()
        return out

    # -- same, framebuffer stays in HBM (raw device pointer, float64 [rows*W*3])
    def render_rows_dev(self, camera, out_dev_ptr, y0=0, y1=None, sqrtspp=None, precision=None):
        y1 = camera.height if y1 is None else y1
        self.set_film(camera)
        st = Stats()
        self._check(lib().mcrt_render_rows_dev(self.ctx, C.byref(camera.rec), y0, y1,
                                               camera.sqrtspp if sqrtspp is None else sqrtspp, self.global_seed,
                                               self.kind, self.precision if precision is None else precision,
                                               C.c_void_p(out_dev_ptr), C.byref(st)))
        self.last_stats = st.as_dict()
        return self.last_stats

    # -- interleaved rows y_first + k*y_step (multi-GPU sharding), framebuffer in HBM
    def render_rows_strided_peers(self, camera, frame_ptrs, y_first, y_step, n_rows, frame_is_float32=True, sqrtspp=None, precision=None):
        """Rows y_first + k*y_step rendered and resolved straight into the full-frame buffers `frame_ptrs` (this
        rank's and the peers', see distributed.PeerFrames): mcrt_render_rows_strided_peers."""
        self.set_film(camera)
        arr = (C.c_void_p * len(frame_ptrs))(*[C.c_void_p(int(q)) for q in frame_ptrs])
        st = Stats()
        self._check(lib().mcrt_render_rows_strided_peers(self.ctx, C.byref(camera.rec), y_first, y_step, n_rows,
                                                         camera.sqrtspp if sqrtspp is None else sqrtspp, self.global_seed, self.kind,
                                                         self.precision if precision is None else precision, arr, len(frame_ptrs),
                                                         1 if frame_is_float32 else 0, C.byref(st)))
        self.last_stats = st.as_dict()
        return self.last_stats

    def render_film_sums_strided_dev(self, camera, rgb_sum_ptr, weight_sum_ptr, y_first, y_step, n_rows, sqrtspp=None, precision=None):
        """Row shard of a render through the camera's reconstruction filter: unresolved whole-frame sums (device)."""
        self.set_film(camera)
        st = Stats()
        self._check(lib().mcrt_render_film_sums_strided_dev(self.ctx, C.byref(camera.rec), y_first, y_step, n_rows,
                                                            camera.sqrtspp if sqrtspp is None else sqrtspp, self.global_seed, self.kind,
                                                            self.precision if precision is None else precision,
                                                            C.c_void_p(rgb_sum_ptr), C.c_void_p(weight_sum_ptr), C.byref(st)))
        self.last_stats = st.as_dict()
        return self.last_stats

    def film_resolve_dev(self, rgb_sum_ptr, weight_sum_ptr, n_pixels, out_ptr):
        self._check(lib().mcrt_film_resolve_dev(self.ctx, C.c_void_p(rgb_sum_ptr), C.c_void_p(weight_sum_ptr), n_pixels, C.c_void_p(out_ptr)))

    # -- progressive rendering (see Progressive)
    def render_accumulate_dev(self, camera, rgb_sum_ptr, weight_sum_ptr, sample_first, sample_count, y_first=0, y_step=1,
                              n_rows=None, precision=None):
        """Adds samples [sample_first, sample_first + sample_count) of rows y_first + k*y_step into device sums
        (mcrt_render_accumulate_dev). weight_sum_ptr: None with the box film, whole-frame weight sums with a filter."""
        self.set_film(camera)
        n_rows = len(range(y_first, camera.height, y_step)) if n_rows is None else n_rows
        st = Stats()
        self._check(lib().mcrt_render_accumulate_dev(self.ctx, C.byref(camera.rec), y_first, y_step, n_rows, sample_first, sample_count,
                                                     self.global_seed, self.kind, self.precision if precision is None else precision,
                                                     C.c_void_p(rgb_sum_ptr), C.c_void_p(weight_sum_ptr) if weight_sum_ptr else None,
                                                     C.byref(st)))
        self.last_stats = st.as_dict()
        return self.last_stats

    def progressive_resolve_dev(self, a_rgb_ptr, a_weight_ptr, a_samples, b_rgb_ptr, b_weight_ptr, b_samples, width, rows, tile,
                                out_ptr, tile_error_ptr=None):
        """mcrt_progressive_resolve_dev: resolves A+B into out_ptr, per-tile errors into tile_error_ptr -> frame error."""
        def p(x):
            return C.c_void_p(x) if x else None
        err = C.c_double()
        self._check(lib().mcrt_progressive_resolve_dev(self.ctx, p(a_rgb_ptr), p(a_weight_ptr), a_samples, p(b_rgb_ptr), p(b_weight_ptr),
                                                       b_samples, width, rows, tile, p(out_ptr), p(tile_error_ptr), C.byref(err)))
        return err.value

    # -- adaptive sampling (see Progressive.render_adaptive)
    def render_accumulate_tiles_dev(self, camera, rgb_sum_ptr, weight_sum_ptr, sample_first, sample_count, tile, active,
                                    y_first=0, y_step=1, n_rows=None, precision=None):
        """mcrt_render_accumulate_tiles_dev: render_accumulate_dev restricted to the pixels of the active tiles.
        active: bool [ceil(n_rows / tile), ceil(width / tile)] over the row set's n_rows x width grid."""
        self.set_film(camera)
        n_rows = len(range(y_first, camera.height, y_step)) if n_rows is None else n_rows
        mask = np.ascontiguousarray(active, dtype=np.uint8)
        if mask.shape != tile_grid(n_rows, camera.width, tile):
            raise McrtError(f"tile mask has shape {mask.shape}, expected {tile_grid(n_rows, camera.width, tile)}")
        st = Stats()
        self._check(lib().mcrt_render_accumulate_tiles_dev(self.ctx, C.byref(camera.rec), y_first, y_step, n_rows, tile,
                                                           mask.ctypes.data_as(C.c_void_p), sample_first, sample_count,
                                                           self.global_seed, self.kind, self.precision if precision is None else precision,
                                                           C.c_void_p(rgb_sum_ptr), C.c_void_p(weight_sum_ptr) if weight_sum_ptr else None,
                                                           C.byref(st)))
        self.last_stats = st.as_dict()
        return self.last_stats

    def progressive_resolve_tiles_dev(self, a_rgb_ptr, a_weight_ptr, b_rgb_ptr, b_weight_ptr, tile_samples, width, rows, tile,
                                      out_ptr, tile_error_ptr=None, tile_sums_ptr=None):
        """mcrt_progressive_resolve_tiles_dev: progressive_resolve_dev with per-tile counts tile_samples
        [tiles_y, tiles_x, 2] = {nA, nB}; tile_sums_ptr (optional) receives {sum v, sum I^2} per tile -> frame error."""
        def p(x):
            return C.c_void_p(x) if x else None
        counts = np.ascontiguousarray(tile_samples, dtype=np.uint32)
        if counts.shape != tile_grid(rows, width, tile) + (2,):
            raise McrtError(f"tile_samples has shape {counts.shape}, expected {tile_grid(rows, width, tile) + (2,)}")
        err = C.c_double()
        self._check(lib().mcrt_progressive_resolve_tiles_dev(self.ctx, p(a_rgb_ptr), p(a_weight_ptr), p(b_rgb_ptr), p(b_weight_ptr),
                                                             counts.ctypes.data_as(C.c_void_p), width, rows, tile, p(out_ptr),
                                                             p(tile_error_ptr), p(tile_sums_ptr), C.byref(err)))
        return err.value

    # -- light groups (see Progressive's light_groups)
    def set_light_groups(self, ids, n_groups=None):
        """mcrt_set_light_groups: light l (the scene's l-th light_prim) goes to group ids[l]; the renders of
        render_accumulate_groups_dev then have n_groups + 1 planes, the last one the sky's. n_groups: max(ids) + 1 if None.
        ids None clears the table."""
        self._lpe_key = None   # the library clears the LPE table too
        if ids is None:
            self._check(lib().mcrt_set_light_groups(self.ctx, None, 0, 0))
            self._groups_key = None
            return
        ids = np.ascontiguousarray(ids, dtype=np.uint32).reshape(-1)
        n_groups = (int(ids.max()) + 1 if ids.size else 0) if n_groups is None else int(n_groups)
        table = ids if ids.size else np.zeros(1, np.uint32)   # a lightless scene's sky-only table: any non-null pointer
        self._groups_key = None
        self._check(lib().mcrt_set_light_groups(self.ctx, table.ctypes.data_as(C.c_void_p), ids.size, n_groups))
        self._groups_key = (tuple(int(g) for g in ids), n_groups)

    def render_accumulate_groups_dev(self, camera, planes_ptr, n_planes, sample_first, sample_count, tile=0, active=None,
                                     y_first=0, y_step=1, n_rows=None, precision=None):
        """mcrt_render_accumulate_groups_dev: render_accumulate_dev (active None) or render_accumulate_tiles_dev into the
        light-group planes planes_ptr [n_planes, n_rows, width, 3] (device)."""
        return self._render_accumulate_planes(lib().mcrt_render_accumulate_groups_dev, camera, planes_ptr, n_planes, sample_first,
                                              sample_count, tile, active, y_first, y_step, n_rows, precision)

    def render_accumulate_aovs_dev(self, camera, planes_ptr, sample_first, sample_count, tile=0, active=None,
                                   y_first=0, y_step=1, n_rows=None, precision=None):
        """mcrt_render_accumulate_aovs_dev: render_accumulate_dev (active None) or render_accumulate_tiles_dev into the
        light-path AOV planes planes_ptr [8, n_rows, width, 3] (device), in the order of AOV_NAMES."""
        return self._render_accumulate_planes(lib().mcrt_render_accumulate_aovs_dev, camera, planes_ptr, len(AOV_NAMES), sample_first,
                                              sample_count, tile, active, y_first, y_step, n_rows, precision)

    # -- light path expressions (see Progressive's lpes)
    def set_light_path_expressions(self, exprs):
        """mcrt_set_light_path_expressions: the renders of render_accumulate_lpe_dev then have one plane per expression,
        plane i the contributions whose event string exprs[i] matches. Labels L'g' name groups of the light-group table,
        so set_light_groups comes first (it clears this table). exprs None or empty clears the table."""
        exprs = list(exprs or ())
        arr = _lpe_strings(exprs)
        self._lpe_key = None
        self._check(lib().mcrt_set_light_path_expressions(self.ctx, C.cast(arr, C.c_void_p) if exprs else None, len(exprs)))
        # what the table is made of, for PhotonMapper.has_photon_lpe_states
        self._lpe_key = (tuple(str(e) for e in exprs), getattr(self, "_groups_key", None)) if exprs else None

    def render_accumulate_lpe_dev(self, camera, planes_ptr, n_planes, sample_first, sample_count, tile=0, active=None,
                                  y_first=0, y_step=1, n_rows=None, precision=None):
        """mcrt_render_accumulate_lpe_dev: render_accumulate_dev (active None) or render_accumulate_tiles_dev into the
        LPE planes planes_ptr [n_planes, n_rows, width, 3] (device), one per expression of set_light_path_expressions."""
        return self._render_accumulate_planes(lib().mcrt_render_accumulate_lpe_dev, camera, planes_ptr, n_planes, sample_first,
                                              sample_count, tile, active, y_first, y_step, n_rows, precision)

    def _render_accumulate_planes(self, fn, camera, planes_ptr, n_planes, sample_first, sample_count, tile, active, y_first,
                                  y_step, n_rows, precision):
        self.set_film(camera)
        n_rows = len(range(y_first, camera.height, y_step)) if n_rows is None else n_rows
        mask = None
        if active is not None:
            mask = np.ascontiguousarray(active, dtype=np.uint8)
            if mask.shape != tile_grid(n_rows, camera.width, tile):
                raise McrtError(f"tile mask has shape {mask.shape}, expected {tile_grid(n_rows, camera.width, tile)}")
        st = Stats()
        self._check(fn(self.ctx, C.byref(camera.rec), y_first, y_step, n_rows, tile,
                       mask.ctypes.data_as(C.c_void_p) if mask is not None else None, sample_first, sample_count,
                       self.global_seed, self.kind, self.precision if precision is None else precision,
                       C.c_void_p(planes_ptr), n_planes, C.byref(st)))
        self.last_stats = st.as_dict()
        return self.last_stats

    def light_groups_combine_dev(self, planes_ptr, n_planes, n_values, weights, out_ptr):
        """mcrt_light_groups_combine_dev: out = sum over g of weights[g] * plane g, added in order of g (device buffers of
        n_values float64 per plane). weights: [n_planes, 3] or [n_planes] (one weight for all three channels). The
        planes may be light-group or AOV planes: the kernel is a plain weighted sum."""
        w = light_group_weights(weights, n_planes)
        self._check(lib().mcrt_light_groups_combine_dev(self.ctx, C.c_void_p(planes_ptr), n_planes, n_values,
                                                        w.ctypes.data_as(C.c_void_p), C.c_void_p(out_ptr)))

    # -- denoising (see Progressive.denoise)
    def render_features_dev(self, camera, features_ptr, sample_first, sample_count, precision=None, specular_depth=0):
        """mcrt_render_features_dev: adds the first-hit guides {albedo.rgb, normal.xyz, t, hits} of samples
        [sample_first, sample_first + sample_count) of every pixel into device sums [height, width, 8].
        specular_depth > 0 (at most FEATURES_MAX_SPECULAR_DEPTH): mcrt_render_features_chain_dev, the guides of the
        first vertex after up to that many perfectly specular bounces of each sample's own path, with the albedo
        weighted by the chain's throughput and the depth measured along the chain."""
        st = Stats()
        precision = self.precision if precision is None else precision
        ptr = C.c_void_p(features_ptr) if features_ptr else None
        if specular_depth:
            rc = lib().mcrt_render_features_chain_dev(self.ctx, C.byref(camera.rec), sample_first, sample_count, self.global_seed,
                                                      precision, specular_depth, ptr, C.byref(st))
        else:
            rc = lib().mcrt_render_features_dev(self.ctx, C.byref(camera.rec), sample_first, sample_count, self.global_seed,
                                                precision, ptr, C.byref(st))
        self._check(rc)
        self.last_stats = st.as_dict()
        return self.last_stats

    def denoise_dev(self, a_rgb_ptr, a_weight_ptr, b_rgb_ptr, b_weight_ptr, tile_samples, tile, features_ptr, width, height,
                    out_ptr, params=None):
        """mcrt_denoise_dev: the denoised frame of halves A and B into out_ptr [height, width, 3] -> its residual error.
        tile_samples: {nA, nB} per tile [tiles_y, tiles_x, 2]; params: a DenoiseParams, or None for the defaults."""
        def p(x):
            return C.c_void_p(x) if x else None
        counts = np.ascontiguousarray(tile_samples, dtype=np.uint32)
        if counts.shape != tile_grid(height, width, tile) + (2,):
            raise McrtError(f"tile_samples has shape {counts.shape}, expected {tile_grid(height, width, tile) + (2,)}")
        err = C.c_double()
        self._check(lib().mcrt_denoise_dev(self.ctx, p(a_rgb_ptr), p(a_weight_ptr), p(b_rgb_ptr), p(b_weight_ptr),
                                           counts.ctypes.data_as(C.c_void_p), tile, p(features_ptr), width, height,
                                           C.byref(params) if params is not None else None, p(out_ptr), C.byref(err)))
        return err.value

    def frame_alloc(self, nbytes):
        """-> (device pointer, 64-byte CUDA IPC handle) of a zero-filled buffer other ranks can map"""
        ptr = C.c_void_p(); h = (C.c_ubyte * 64)()
        self._check(lib().mcrt_frame_alloc(self.ctx, nbytes, C.byref(ptr), h))
        return ptr.value, bytes(h)

    def frame_open(self, handle):
        ptr = C.c_void_p(); h = (C.c_ubyte * 64)(*handle)
        self._check(lib().mcrt_frame_open(self.ctx, h, C.byref(ptr)))
        return ptr.value

    def frame_close(self, ptr):
        self._check(lib().mcrt_frame_close(self.ctx, C.c_void_p(ptr)))

    def frame_free(self, ptr):
        self._check(lib().mcrt_frame_free(self.ctx, C.c_void_p(ptr)))

    def fp64_peak(self):
        """Measured DFMA thread-instructions per second of this GPU (mcrt_fp64_peak)."""
        v = C.c_double()
        self._check(lib().mcrt_fp64_peak(self.ctx, C.byref(v)))
        return v.value

    def render_rows_strided_dev(self, camera, out_dev_ptr, y_first, y_step, n_rows, sqrtspp=None, precision=None):
        self.set_film(camera)
        st = Stats()
        self._check(lib().mcrt_render_rows_strided_dev(self.ctx, C.byref(camera.rec), y_first, y_step, n_rows,
                                                       camera.sqrtspp if sqrtspp is None else sqrtspp,
                                                       self.global_seed, self.kind,
                                                       self.precision if precision is None else precision,
                                                       C.c_void_p(out_dev_ptr), C.byref(st)))
        self.last_stats = st.as_dict()
        return self.last_stats

    # -- Image::save without the file: float64 [H, W, 3] -> bytes [H, W, 3] in B,G,R order (the .tga payload)
    def tonemap(self, rgb, image=None):
        params = image if isinstance(image, ImageParams) else ImageParams.from_json(image or {})
        rgb = np.ascontiguousarray(rgb, dtype=np.float64)
        h, w = rgb.shape[:2]
        out = np.zeros((h, w, 3), dtype=np.uint8)
        e, g = C.c_double(), C.c_double()
        self._check(lib().mcrt_image_tonemap(self.ctx, _ptr(rgb), w, h, C.byref(params), _ptr(out), C.byref(e), C.byref(g)))
        return out, e.value, g.value

    def tonemap_dev(self, rgb_dev_ptr, out_dev_ptr, width, height, image=None):
        params = image if isinstance(image, ImageParams) else ImageParams.from_json(image or {})
        e, g = C.c_double(), C.c_double()
        self._check(lib().mcrt_image_tonemap_dev(self.ctx, C.c_void_p(rgb_dev_ptr), width, height, C.byref(params),
                                                 C.c_void_p(out_dev_ptr), C.byref(e), C.byref(g)))
        return e.value, g.value

    def sampler_stream(self, pixel, sample, n_shuffles):
        pixel = np.ascontiguousarray(pixel, dtype=np.uint32)
        sample = np.ascontiguousarray(sample, dtype=np.uint32)
        out = np.zeros((len(pixel), 7), dtype=np.uint32)
        self._check(lib().mcrt_sampler_stream(self.ctx, _ptr(pixel), _ptr(sample), len(pixel), n_shuffles,
                                              self.global_seed, _ptr(out)))
        return out


class PathTracer(Integrator):
    kind = INTEGRATOR_PATH


class PhotonMapper(Integrator):
    """Renders with the caustic/global photon maps the CPU photon pass produced (first pass stays on
    the CPU, SURVEY.md §8f); maps come from the scene pack or from explicit arrays.

    Light groups (set_light_groups, render_accumulate_groups_dev, Progressive(light_groups=...)) need maps that record
    which light emitted each photon: the maps of emit() / emit_pass() do (has_photon_lights, photon_lights); the maps of
    the scene pack, of photon_maps= and of emit_sharded do not.

    Components (render_accumulate_components_dev, Progressive(components=True)) split a frame by the estimator behind
    each contribution (PHOTON_COMPONENT_NAMES) and work with every kind of map.

    Light path expressions (render_accumulate_lpe_dev, Progressive(lpes=...)) need each photon's own events, which
    only maps of emit() / emit_pass() record, and only while the table is set: set_light_path_expressions, then emit
    (has_photon_lpe_states). Progressive does this itself, emitting again with the arguments of the last emit."""
    kind = INTEGRATOR_PHOTON

    def __init__(self, scene, device=0, precision=PRECISION_F64, global_seed=0x12345678, photon_maps=None, emit=None):
        """photon_maps: (caustic, global, k, direct_visualization) built by the reference's CPU pass (default: the
        ones in the scene pack); emit: dict(emissions, caustic_factor, max_photons_per_octree_leaf, k_nearest_photons,
        direct_visualization, scene_bounds) to run the photon pass on the GPU instead (mcrt_photon_emit)."""
        super().__init__(scene, device, precision, global_seed)
        if emit is not None:
            self.emit(**emit)
            return
        maps = photon_maps or scene.photon_maps()
        if maps is None:
            raise McrtError("PhotonMapper needs photon maps (scene pack exported with photon_map=True) or emit=...")
        self._maps = maps
        self.upload_photons()

    @property
    def has_photon_lights(self):
        """True when the current maps record the light that emitted each photon (maps of emit / emit_pass)."""
        return getattr(self, "_photon_lights", False)

    @property
    def has_photon_lpe_states(self):
        """True when the current maps were emitted (emit / emit_pass) while the current LPE table, with the same
        expressions and light groups, was set: each photon then carries the state of its own path."""
        key = getattr(self, "_photon_lpe_key", None)
        return key is not None and getattr(self, "_emitted", None) is not None and key == getattr(self, "_lpe_key", None)

    def photon_lpe_states(self, which):
        """The reverse-DFA state of each photon of map `which` before the event of its storage vertex, uint32 [n_photons],
        in the order of the photons of _maps[which] (mcrt_photon_download_lpe_states; lpe_compile_photon's rev_next)."""
        out = np.zeros(self.n_photons[which], np.uint32)
        self._check(lib().mcrt_photon_download_lpe_states(self.ctx, int(which), _ptr(out), out.size))
        return out

    def emit_again(self):
        """Repeats the last emit() / emit_pass() with the same arguments: the same photons (the passes are deterministic),
        now with the states of the LPE table set since. -> (n_caustic, n_global)"""
        if getattr(self, "_emit_args", None) is None:
            raise McrtError("the photon maps did not come from emit() / emit_pass()")
        return self.emit_pass(*self._emit_args)

    def photon_lights(self, which):
        """The index of the light that emitted each photon of map `which` (0 caustic, 1 global), uint32 [n_photons], in
        the order of the photons of _maps[which] (mcrt_photon_download_lights)."""
        if not self.has_photon_lights:
            raise McrtError("the photon maps carry no light index: only the maps of emit() / emit_pass() do")
        out = np.zeros(self.n_photons[which], np.uint32)
        self._check(lib().mcrt_photon_download_lights(self.ctx, int(which), _ptr(out), out.size))
        return out

    def set_light_groups(self, ids, n_groups=None):
        """Integrator.set_light_groups, for maps that carry light indices (has_photon_lights)."""
        if not self.has_photon_lights:
            raise McrtError("the photon mapper has no light groups with these maps: their photons carry no light index "
                            "(only the maps of emit() / emit_pass() do)")
        return super().set_light_groups(ids, n_groups)

    def render_accumulate_aovs_dev(self, *args, **kwargs):
        raise McrtError("the photon mapper has no light-path AOVs")

    def render_accumulate_components_dev(self, camera, planes_ptr, sample_first, sample_count, tile=0, active=None,
                                         y_first=0, y_step=1, n_rows=None, precision=None):
        """mcrt_render_accumulate_photon_components_dev: render_accumulate_dev (active None) or render_accumulate_tiles_dev
        into the component planes planes_ptr [4, n_rows, width, 3] (device), in the order of PHOTON_COMPONENT_NAMES.
        Works with every kind of map (scene pack, photon_maps=, emit, emit_pass, emit_sharded)."""
        return self._render_accumulate_planes(lib().mcrt_render_accumulate_photon_components_dev, camera, planes_ptr,
                                              len(PHOTON_COMPONENT_NAMES), sample_first, sample_count, tile, active, y_first,
                                              y_step, n_rows, precision)

    def _emit_params(self, emissions, caustic_factor, max_photons_per_octree_leaf, k_nearest_photons, direct_visualization, scene_bounds):
        p = PhotonEmitParams()
        p.emissions = int(emissions); p.caustic_factor = float(caustic_factor)
        p.max_photons_per_octree_leaf = int(max_photons_per_octree_leaf); p.k_nearest_photons = int(k_nearest_photons)
        p.direct_visualization = int(bool(direct_visualization)); p.global_seed = self.global_seed
        if scene_bounds is not None:
            b = scene_bounds
        elif self.scene.a["node_bounds"].size >= 6:
            b = self.scene.a["node_bounds"][:6]   # the BVH root's box
        elif "scene_bounds" in self.scene.extra:
            b = self.scene.extra["scene_bounds"]  # a scene without a BVH: the pack's scene box
        else:
            raise McrtError("the scene has no BVH and no scene bounds: pass scene_bounds")
        for i in range(6):
            p.scene_bounds[i] = float(b[i])
        return p

    def emit_sharded(self, rank, world, emissions, caustic_factor, max_photons_per_octree_leaf=200, k_nearest_photons=50,
                     direct_visualization=False, scene_bounds=None, precision=None):
        """The photon pass over `world` GPUs (SURVEY.md §8e): this rank emits its range of the emission index space
        (distributed.emission_range), the photon arrays are all-gathered (torch.distributed), and every rank builds the
        same two octrees from the concatenation. -> (n_caustic, n_global) of the whole maps."""
        import torch
        from . import distributed as mdist
        p = self._emit_params(emissions, caustic_factor, max_photons_per_octree_leaf, k_nearest_photons, direct_visualization, scene_bounds)
        prec = self.precision if precision is None else precision
        total = C.c_uint64()
        self._check(lib().mcrt_photon_emit_total(self.ctx, C.byref(p), C.byref(total)))
        first, count = mdist.emission_range(total.value, rank, world)
        ptr = [C.c_void_p(), C.c_void_p()]; n = [C.c_uint64(), C.c_uint64()]; st = Stats()
        self._check(lib().mcrt_photon_emit_range(self.ctx, C.byref(p), prec, first, count, C.byref(ptr[0]), C.byref(n[0]),
                                                 C.byref(ptr[1]), C.byref(n[1]), C.byref(st)))
        self.last_stats = st.as_dict()
        dev = torch.device("cuda", self.device)
        gathered = []
        for w in range(2):
            mine = mdist.device_view(ptr[w].value, n[w].value * 8, torch.float32, dev)
            gathered.append(mdist.all_gather_photons(mine, world, dev))
        ms = C.c_double()
        self._check(lib().mcrt_photon_build_dev(self.ctx, C.byref(p), C.c_void_p(gathered[0].data_ptr()), gathered[0].numel() // 8,
                                                C.c_void_p(gathered[1].data_ptr()), gathered[1].numel() // 8, C.byref(ms)))
        torch.cuda.synchronize(dev)
        self.last_stats["gpu_ms_knn"] = ms.value
        self.k_nearest = int(k_nearest_photons)
        self._host_maps = None
        self._emitted = (int(k_nearest_photons), int(bool(direct_visualization)))
        self._photon_lights = False   # the gathered arrays carry no light index
        self._emit_args = self._photon_lpe_key = None
        self.n_photons = (gathered[0].numel() // 8, gathered[1].numel() // 8)
        return self.n_photons

    def emit(self, emissions, caustic_factor, max_photons_per_octree_leaf=200, k_nearest_photons=50,
             direct_visualization=False, scene_bounds=None, precision=None):
        """PhotonMapper::PhotonMapper's first pass on the GPU; replaces the uploaded maps."""
        return self.emit_pass(0, emissions, caustic_factor, max_photons_per_octree_leaf, k_nearest_photons, scene_bounds,
                              direct_visualization, precision)

    def emit_pass(self, pass_index, emissions, caustic_factor, max_photons_per_octree_leaf=200, k_nearest_photons=50,
                  scene_bounds=None, direct_visualization=False, precision=None):
        """Photon pass `pass_index` of progressive photon mapping (mcrt_photon_emit_pass): light l's emissions take the
        reference's emission indices [pass_index * n_l, (pass_index + 1) * n_l) with the flux of a one-pass map, so every
        pass map is complete on its own and independent of the others. Pass 0 is emit(). Replaces the uploaded maps."""
        if not 0 <= int(pass_index) < 1 << 32:
            raise McrtError(f"pass index {pass_index} is outside [0, 2^32)")
        p = self._emit_params(emissions, caustic_factor, max_photons_per_octree_leaf, k_nearest_photons, direct_visualization, scene_bounds)
        nc, ng, st = C.c_uint64(), C.c_uint64(), Stats()
        self._check(lib().mcrt_photon_emit_pass(self.ctx, C.byref(p), self.precision if precision is None else precision,
                                                int(pass_index), C.byref(nc), C.byref(ng), C.byref(st)))
        self.last_stats = st.as_dict()
        self.k_nearest = int(k_nearest_photons)
        # the maps stay in HBM (octrees are built there too); host copies only when somebody asks
        self._host_maps = None
        self._emitted = (int(k_nearest_photons), int(bool(direct_visualization)))
        self._photon_lights = True
        self._emit_args = (pass_index, emissions, caustic_factor, max_photons_per_octree_leaf, k_nearest_photons, scene_bounds,
                           direct_visualization, precision)
        self._photon_lpe_key = getattr(self, "_lpe_key", None)
        self.n_photons = (nc.value, ng.value)
        return nc.value, ng.value

    @property
    def _maps(self):
        if self._host_maps is None and getattr(self, "_emitted", None) is not None:
            maps = []
            for which in (0, 1):
                d = PhotonMapDesc()
                self._check(lib().mcrt_photon_download(self.ctx, which, C.byref(d)))
                maps.append(_map_arrays(d))
            self._host_maps = (maps[0], maps[1]) + self._emitted
        return self._host_maps

    @_maps.setter
    def _maps(self, value):
        self._host_maps = value
        self._emitted = None
        self._photon_lights = False
        self._emit_args = self._photon_lpe_key = None

    @staticmethod
    def _map_desc(m):
        d = PhotonMapDesc()
        d.n_octants = m["octant_leaf"].size
        d.octant_bounds = _ptr(m["octant_bounds"]); d.octant_start = _ptr(m["octant_start"])
        d.octant_count = _ptr(m["octant_count"]); d.octant_next_sibling = _ptr(m["octant_next"])
        d.octant_leaf = _ptr(m["octant_leaf"])
        d.n_photons = m["photons"].size // 8
        d.photons = _ptr(m["photons"])
        return d

    def upload_photons(self):
        caustic, glob, k, dv = self._maps
        dc, dg = self._map_desc(caustic), self._map_desc(glob)
        n = C.c_uint64()
        self._check(lib().mcrt_photon_upload(self.ctx, C.byref(dc), C.byref(dg), k, dv, C.byref(n)))
        self.k_nearest = k
        return n.value

    def knn(self, which, points):
        points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        n, k = len(points), self.k_nearest
        idx = np.full((n, k), NO_PRIM, dtype=np.uint32); d2 = np.full((n, k), np.inf); cnt = np.zeros(n, dtype=np.uint32)
        st = Stats()
        self._check(lib().mcrt_knn_search(self.ctx, which, _ptr(points), n, _ptr(idx), _ptr(d2), _ptr(cnt), C.byref(st)))
        return idx, d2, cnt

    def gather_radius(self, r_caustic, r_global):
        """Following renders estimate radiance from every photon within r_caustic / r_global of a query (k_gather), with
        the k-NN formulas and r^2 in place of the k-th distance^2; (0, 0) returns to the reference's k-NN estimate, the
        default (mcrt_photon_gather_radius)."""
        self._check(lib().mcrt_photon_gather_radius(self.ctx, float(r_caustic), float(r_global)))
        self.gather_radii = (float(r_caustic), float(r_global))

    def gather(self, which, points, radius):
        """The fixed-radius search on caller points (mcrt_photon_gather_search) -> (count uint32 [n], flux_sum [n, 3],
        cone_sum [n, 3]): the photons of map `which` (0 caustic, 1 global) within `radius` (distance^2 <= radius^2), and
        the float64 sums of their flux, plain and weighted by max(0, 1 - d / radius)."""
        points = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        n = len(points)
        cnt = np.zeros(n, np.uint32); flux = np.zeros((n, 3)); cone = np.zeros((n, 3))
        st = Stats()
        self._check(lib().mcrt_photon_gather_search(self.ctx, which, _ptr(points), n, float(radius), _ptr(cnt), _ptr(flux),
                                                    _ptr(cone), C.byref(st)))
        return cnt, flux, cone


def _map_arrays(d):
    """PhotonMapDesc (host pointers) -> dict of numpy copies."""
    n, npn = d.n_octants, d.n_photons

    def arr(ptr, ctype, count, dtype):
        if not ptr or count == 0:
            return np.zeros(0, dtype=dtype)
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=(count,)).astype(dtype, copy=True)
    return {"octant_bounds": arr(d.octant_bounds, C.c_double, 6 * n, np.float64),
            "octant_start": arr(d.octant_start, C.c_uint64, n, np.uint64),
            "octant_count": arr(d.octant_count, C.c_uint64, n, np.uint64),
            "octant_next": arr(d.octant_next_sibling, C.c_uint32, n, np.uint32),
            "octant_leaf": arr(d.octant_leaf, C.c_uint8, n, np.uint8),
            "photons": arr(d.photons, C.c_float, 8 * npn, np.float32)}


def build_photon_octree(photons, max_photons_per_octree_leaf, scene_bounds, device=0):
    """mcrt_octree_build: the octree construction of mcrt_photon_emit on the GPU, on caller photons.
    -> (dict of octant_bounds, octant_start, octant_count, octant_next, octant_leaf, photons; gpu_ms)."""
    photons = np.ascontiguousarray(photons, dtype=np.float32).reshape(-1, 8)
    bounds = np.ascontiguousarray(scene_bounds, dtype=np.float64)
    ctx = C.c_void_p()
    rc = lib().mcrt_init(device, C.byref(ctx))
    if rc:
        raise McrtError(f"mcrt_init({device}) failed: {rc} (no CUDA device? there is no CPU fallback)")
    try:
        h, d, ms = C.c_void_p(), PhotonMapDesc(), C.c_double()
        rc = lib().mcrt_octree_build(ctx, _ptr(photons), len(photons), int(max_photons_per_octree_leaf), _ptr(bounds),
                                     C.byref(h), C.byref(d), C.byref(ms))
        if rc:
            raise McrtError(f"mcrt_octree_build failed ({rc}): {lib().mcrt_last_error(ctx).decode()}")
        out = _map_arrays(d)
        lib().mcrt_octree_free(h)
        return out, ms.value
    finally:
        lib().mcrt_destroy(ctx)


def load_obj(path, threads=0):
    """mcrt_obj_load: Scene::parseOBJ (scene.cpp:238-324), parallel. -> dict(vertices [n,3], normals [n,3],
    tri_v / tri_vt / tri_vn [m,3] uint64)."""
    h, d = C.c_void_p(), ObjMeshRec()
    err = C.create_string_buffer(512)
    rc = lib().mcrt_obj_load(os.fsencode(path), int(threads), C.byref(h), C.byref(d), err, 512)
    if rc:
        raise McrtError(err.value.decode() or f"mcrt_obj_load failed: {rc}")

    def arr(ptr, count, dtype):
        if not ptr or count == 0:
            return np.zeros((0, 3), dtype=dtype)
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(count * 3 * 8,)).view(dtype).reshape(-1, 3).copy()
    out = dict(vertices=arr(d.vertices, d.n_vertices, np.float64), normals=arr(d.normals, d.n_normals, np.float64),
               tri_v=arr(d.tri_v, d.n_tri_v, np.uint64), tri_vt=arr(d.tri_vt, d.n_tri_vt, np.uint64),
               tri_vn=arr(d.tri_vn, d.n_tri_vn, np.uint64))
    lib().mcrt_obj_free(h)
    return out


def vertex_normals(vertices, tri_v, threads=0):
    """mcrt_obj_vertex_normals: Scene::generateVertexNormals (scene.cpp:326-355). -> [n_vertices, 3]."""
    vertices = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
    tri_v = np.ascontiguousarray(tri_v, dtype=np.uint64).reshape(-1, 3)
    out = np.zeros_like(vertices)
    rc = lib().mcrt_obj_vertex_normals(_ptr(vertices), len(vertices), _ptr(tri_v), len(tri_v), int(threads), _ptr(out))
    if rc:
        raise McrtError("mcrt_obj_vertex_normals: triangle index out of range")
    return out


def bvh_build(prim_bounds, scene_bounds, bvh_type, bins_per_axis=0, device=0):
    """mcrt_bvh_build: the reference's BVH (bvh.cpp:13-78) over primitive boxes, built on the GPU.
    -> dict(node_bounds [n,6], node_first_prim, node_prim_count, node_next_sibling, prim_order, gpu_ms, rounds)."""
    prim_bounds = np.ascontiguousarray(prim_bounds, dtype=np.float64).reshape(-1, 6)
    scene_bounds = np.ascontiguousarray(scene_bounds, dtype=np.float64).reshape(6)
    code = BVH_TYPES[bvh_type.lower()] if isinstance(bvh_type, str) else int(bvh_type)
    ctx = C.c_void_p()
    rc = lib().mcrt_init(device, C.byref(ctx))
    if rc:
        raise McrtError(f"mcrt_init({device}) failed: {rc} (no CUDA device? there is no CPU fallback)")
    try:
        h, d, ms = C.c_void_p(), BvhDesc(), C.c_double()
        rc = lib().mcrt_bvh_build(ctx, _ptr(prim_bounds), len(prim_bounds), _ptr(scene_bounds), code, int(bins_per_axis),
                                  C.byref(h), C.byref(d), C.byref(ms))
        if rc:
            raise McrtError(f"mcrt_bvh_build failed ({rc}): {lib().mcrt_last_error(ctx).decode()}")

        def arr(ptr, count, dtype):
            return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(count * np.dtype(dtype).itemsize,)).view(dtype).copy()
        out = dict(node_bounds=arr(d.node_bounds, d.n_nodes * 6, np.float64).reshape(-1, 6),
                   node_first_prim=arr(d.node_first_prim, d.n_nodes, np.uint32),
                   node_prim_count=arr(d.node_prim_count, d.n_nodes, np.uint32),
                   node_next_sibling=arr(d.node_next_sibling, d.n_nodes, np.uint32),
                   prim_order=arr(d.prim_order, d.n_prims, np.uint32),
                   gpu_ms=ms.value, rounds=int(d.build_rounds), kernel_launches=int(d.kernel_launches))
        lib().mcrt_bvh_free(h)
        return out
    finally:
        lib().mcrt_destroy(ctx)


BVH4_NODE_DTYPE = np.dtype([("lo", "<f4", (3, 4)), ("hi", "<f4", (3, 4)), ("child", "<u4", (4,)), ("pad", "<u4", (4,))])


def bvh4_host(scene, max_leaf=0xFFFFFFFF):
    """The 4-wide float-box BVH of the order-free search as mcrt_scene_upload builds it (host only) -> structured array."""
    d = scene.desc()
    h, p, n = C.c_void_p(), C.c_void_p(), C.c_uint32()
    rc = lib().mcrt_bvh4_host(C.byref(d), max_leaf, C.byref(h), C.byref(p), C.byref(n))
    if rc:
        raise McrtError(f"mcrt_bvh4_host failed with {rc}")
    try:
        if n.value == 0:
            return np.zeros(0, BVH4_NODE_DTYPE)
        buf = (C.c_uint8 * (128 * n.value)).from_address(p.value)
        return np.frombuffer(buf, dtype=BVH4_NODE_DTYPE).copy()
    finally:
        lib().mcrt_bvh4_host_free(h)


def _lpe_strings(exprs):
    arr = (C.c_char_p * max(len(exprs), 1))()
    for i, e in enumerate(exprs):
        arr[i] = str(e).encode()
    return arr


def lpe_compile(exprs, n_groups=0):
    """The tables mcrt_set_light_path_expressions compiles from exprs (host only, mcrt_lpe_compile_host), with labels
    below n_groups -> {"next": uint8 [n_states, n_symbols] (LPE_DEAD: no expression can match any more), "accept": uint32
    [256] (bit i: expression i matches), "group_symbol": uint8 [n_groups] (the symbol of each group's lights)}. State 0
    follows the camera event C. Raises McrtError with the compiler's reason (and .code, the MCRT_ERR_* value)."""
    exprs = list(exprs)
    arr = _lpe_strings(exprs)
    nxt = np.zeros(LPE_MAX_STATES * LPE_MAX_SYMBOLS, np.uint8)
    acc = np.zeros(256, np.uint32)
    gs = np.zeros(max(int(n_groups), 1), np.uint8)
    ns, nsym = C.c_uint32(), C.c_uint32()
    err = C.create_string_buffer(1024)
    rc = lib().mcrt_lpe_compile_host(C.cast(arr, C.c_void_p) if exprs else None, len(exprs), int(n_groups),
                                     nxt.ctypes.data_as(C.c_void_p), acc.ctypes.data_as(C.c_void_p),
                                     gs.ctypes.data_as(C.c_void_p), C.byref(ns), C.byref(nsym), err, len(err))
    if rc:
        e = McrtError(f"mcrt_lpe_compile_host failed with {rc}: {err.value.decode()}")
        e.code = rc
        raise e
    return {"next": nxt[:ns.value * nsym.value].reshape(ns.value, nsym.value).copy(), "accept": acc,
            "group_symbol": gs[:int(n_groups)].copy()}


def lpe_compile_photon(exprs, n_groups=0):
    """lpe_compile plus the photon mapper's side of the table (mcrt_lpe_compile_photon_host): "rev_next": uint8
    [rev_n_states, n_symbols], the DFA of the reversed expressions, which reads a photon's events in emission order
    (its light's symbol first) from "rev_start" (LPE_DEAD when nothing can match); "join": uint32 [n_states,
    rev_n_states], the accept mask of a contribution whose camera prefix ends in forward state s and whose photon history
    ends in reverse state r. Raises McrtError (.code MCRT_ERR_UNSUPPORTED) when only the path tracer can take the table."""
    out = lpe_compile(exprs, n_groups)
    exprs = list(exprs)
    arr = _lpe_strings(exprs)
    rev = np.zeros(LPE_MAX_STATES * LPE_MAX_SYMBOLS, np.uint8)
    join = np.zeros(LPE_MAX_STATES * LPE_MAX_STATES, np.uint32)
    start, nr = C.c_uint32(), C.c_uint32()
    err = C.create_string_buffer(1024)
    rc = lib().mcrt_lpe_compile_photon_host(C.cast(arr, C.c_void_p) if exprs else None, len(exprs), int(n_groups),
                                            rev.ctypes.data_as(C.c_void_p), C.byref(start), C.byref(nr),
                                            join.ctypes.data_as(C.c_void_p), err, len(err))
    if rc:
        e = McrtError(f"mcrt_lpe_compile_photon_host failed with {rc}: {err.value.decode()}")
        e.code = rc
        raise e
    ns, nsym = out["next"].shape
    out.update(rev_next=rev[:nr.value * nsym].reshape(nr.value, nsym).copy(), rev_start=int(start.value),
               join=join[:ns * nr.value].reshape(ns, nr.value).copy())
    return out


def light_groups_by_emittance(scene, rtol=1e-12):
    """Groups the scene's lights by emittance: a light joins the first group whose first light's emittance equals its
    own in every channel to within rtol (relative; the default only absorbs the last-bit differences a mesh light's
    triangles get from their export), else it opens the next group. -> (ids uint32 [n_lights], the emittance of each
    group's first light float64 [n_groups, 3])."""
    a = scene.a
    lp = np.asarray(a["light_prim"], np.int64)
    em = np.ascontiguousarray(a["materials"]["emittance"][np.asarray(a["prim_material"], np.int64)[lp]], np.float64).reshape(-1, 3)
    ids = np.zeros(len(lp), np.uint32)
    groups = np.zeros((0, 3))
    for l, row in enumerate(em):
        same = np.nonzero((np.abs(groups - row) <= rtol * np.maximum(np.abs(groups), np.abs(row))).all(axis=1))[0]
        if same.size:
            ids[l] = same[0]
        else:
            ids[l] = len(groups)
            groups = np.concatenate([groups, row[None]])
    return ids, groups


def light_group_weights(weights, n_planes):
    """Weights of a light-group combination as float64 [n_planes, 3]: [n_planes, 3] as given, [n_planes] one weight for
    the three channels of a plane."""
    w = np.asarray(weights, np.float64)
    if w.shape == (n_planes,):
        w = np.repeat(w[:, None], 3, axis=1)
    if w.shape != (n_planes, 3):
        raise McrtError(f"light-group weights have shape {w.shape}, expected ({n_planes}, 3) or ({n_planes},)")
    return np.ascontiguousarray(w)


def light_groups_combine(planes, weights):
    """numpy restatement of mcrt_light_groups_combine_dev: sum over g of weights[g] * planes[g], in order of g, each
    product rounded before its addition. planes: [n_planes, ..., 3]."""
    planes = np.asarray(planes, np.float64)
    w = light_group_weights(weights, planes.shape[0])
    out = planes[0] * w[0]
    for g in range(1, planes.shape[0]):
        out = out + planes[g] * w[g]
    return out


def tile_grid(rows, width, tile):
    """(tiles_y, tiles_x) of the tile x tile blocks of a rows x width grid; the last row and column of blocks may be
    smaller than tile x tile."""
    return -(-int(rows) // int(tile)), -(-int(width) // int(tile))


def tile_pixel_counts(rows, width, tile):
    """Pixels of each tile of a rows x width grid, int64 [tiles_y, tiles_x]."""
    ty, tx = tile_grid(rows, width, tile)
    h = np.minimum(tile, rows - np.arange(ty, dtype=np.int64) * tile)
    w = np.minimum(tile, width - np.arange(tx, dtype=np.int64) * tile)
    return np.outer(h, w)


def add_tile_samples(tile_counts, active, half, samples):
    """Per-tile sample counts [tiles_y, tiles_x, 2] after a pass of `samples` samples into half `half` (0: A, 1: B)
    over the active tiles; retired tiles keep theirs."""
    out = np.array(tile_counts, dtype=np.int64, copy=True)
    out[np.asarray(active, bool), half] += int(samples)
    return out


def adaptive_retire(active, tile_counts, tile_sums, tile_pixels, target_error, min_samples):
    """The retirement rule of Progressive.render_adaptive -> bool [tiles_y, tiles_x], the active tiles to retire.

    A tile retires when both its halves have samples, it has at least min_samples samples, and its share of the
    noise is within its share of the target: sum v_t <= target^2 * sum I^2 (frame) * n_t / N, with n_t and N the
    pixels of the tile and of the frame and sum I^2 of the frame the total of the tiles'. If every tile meets it,
    sum over t of sum v_t <= target^2 * sum I^2: the frame meets the target."""
    counts = np.asarray(tile_counts, np.int64)
    sums = np.asarray(tile_sums, np.float64)
    n_t = np.asarray(tile_pixels, np.float64)
    bound = float(target_error) ** 2 * sums[..., 1].sum() * n_t / n_t.sum()
    return (np.asarray(active, bool) & (counts[..., 0] > 0) & (counts[..., 1] > 0) & (counts.sum(-1) >= min_samples)
            & (sums[..., 0] <= bound))


class Progressive:
    """A frame rendered in sample passes: it can be extended, stopped once it is good enough, checkpointed and resumed.

    Pass k adds the next range of samples of every pixel into sums A (even k) or B (odd k), torch CUDA tensors this
    object owns. Sample s of pixel p traces the same path whichever pass renders it, so the resolved frame equals the
    one-shot frame of the same samples up to the order of the float64 film additions. The difference between the two
    halves estimates the remaining noise (mcrt_progressive_resolve_dev). With the box film the sums cover the rows
    y_first + k*y_step, k < n_rows; with a reconstruction filter they, the frame and the tiles span the whole frame.

    Adaptive sampling (render_adaptive, retire): tiles of tile x tile pixels can be retired, and a retired tile never
    comes back. Passes then render only the active tiles (mcrt_render_accumulate_tiles_dev), so every active tile has
    `counts` samples and a retired tile keeps the counts it had (`tile_counts`); the frame is resolved with those
    per-tile counts (mcrt_progressive_resolve_tiles_dev). While every tile is active, add, frame and error run the
    uniform entry points. With a reconstruction filter, adaptive passes need the whole frame as the row set.

    Light groups (light_groups = a group id per light, e.g. light_groups_by_emittance(scene)[0]; box film; the path tracer,
    or the photon mapper with maps that record each photon's light, PhotonMapper.has_photon_lights): A and B then hold one plane per group and one for the sky, [G+1, rows, width, 3], filled by
    mcrt_render_accumulate_groups_dev. frame, error, render, render_adaptive and denoise work on the planes' sum, the
    beauty frame, so they behave as without groups; group_frames() resolves each plane, and relight(weights) and
    denoise(weights=...) work on any weighted sum (mcrt_light_groups_combine_dev), without rendering again.

    Light-path AOVs (aovs=True; box film, path tracer, not together with light groups): A and B hold the 8 planes of
    AOV_NAMES, [8, rows, width, 3], filled by mcrt_render_accumulate_aovs_dev. frame, error, render, render_adaptive
    and denoise work on the planes' sum, as with light groups; aov_frames() resolves each plane with its own noise
    estimate, and relight(weights) and denoise(weights=...) recomposite the frame from weighted planes.

    Photon-mapper components (components=True; box film, a PhotonMapper with any maps, not together with light groups
    or AOVs): A and B hold the 4 planes of PHOTON_COMPONENT_NAMES, [4, rows, width, 3], filled by
    mcrt_render_accumulate_photon_components_dev - emitters seen from the camera, direct light, the caustic-map and the
    global-map estimates. Everything works on the planes' sum as with AOVs; component_frames() resolves each plane with
    its own noise estimate, which shows which estimator still dominates the error, and relight(weights) /
    denoise(weights=...) recomposite the frame, e.g. relight([1, 1, 0, 1]) removes the caustics.

    Light path expressions (lpes = a list of expressions, see mcrt_set_light_path_expressions; box film, not together
    with AOVs or components; the path tracer, or the photon mapper with maps of emit() / emit_pass(), which this emits
    again with the same arguments once the table is set, so that every photon carries its path's state - the same
    photons, since the passes are deterministic): A and B hold one plane per expression and, last, the beauty plane "C.*",
    [len(lpes) + 1, rows, width, 3], filled by mcrt_render_accumulate_lpe_dev. Expressions may overlap or leave
    contributions out, so frame, error, render, render_adaptive and denoise work on the beauty plane alone and behave
    as without expressions. At most 31 expressions, since the beauty plane takes the table's 32nd. light_groups here only
    supplies the groups that labels L'g' name; without it labels are refused. lpe_frames() resolves each
    expression's plane with its own noise estimate; relight(weights) and denoise(weights=...) take one weight per
    expression (the beauty plane's weight is 0)."""

    _STATS = ("paths", "extension_rays", "shadow_rays")

    def __init__(self, integrator, camera, y_first=0, y_step=1, n_rows=None, tile=16, light_groups=None, aovs=False,
                 components=False, lpes=None):
        import torch
        if lpes is not None and integrator.kind == INTEGRATOR_PHOTON and getattr(integrator, "_emit_args", None) is None:
            raise McrtError("the photon mapper has light path expressions only with maps of emit() / emit_pass(): a photon's "
                            "events are recorded while it is emitted")
        if lpes is not None and (aovs or components):
            raise McrtError("light path expressions together with AOVs or components in one render are not supported")
        if components and integrator.kind != INTEGRATOR_PHOTON:
            raise McrtError("photon-mapper components need a PhotonMapper (the path tracer has light-path AOVs)")
        if components and (light_groups is not None or aovs):
            raise McrtError("photon-mapper components together with light groups or AOVs in one render are not supported")
        if light_groups is not None and integrator.kind == INTEGRATOR_PHOTON and not integrator.has_photon_lights:
            raise McrtError("the photon mapper has no light groups with these maps: their photons carry no light index "
                            "(only the maps of emit() / emit_pass() do)")
        if aovs and integrator.kind == INTEGRATOR_PHOTON:
            raise McrtError("the photon mapper has no light-path AOVs")
        if aovs and light_groups is not None:
            raise McrtError("light groups and light-path AOVs in one render are not supported")
        self.integrator, self.camera = integrator, camera
        self.y_first, self.y_step = int(y_first), int(y_step)
        self.n_rows = len(range(self.y_first, camera.height, self.y_step)) if n_rows is None else int(n_rows)
        self.tile = int(tile)
        rec = camera.film_rec()
        self.filtered = rec is not None and not (rec.filter == FILM_FILTERS["box"] and rec.radius in (0.0, 0.5))
        self.rows = camera.height if self.filtered else self.n_rows   # rows of the sums and of the resolved frame
        self.light_groups, self.n_planes = None, 1
        self.lpes, self.lpe_groups = None, None
        if lpes is not None:
            if self.filtered:
                raise McrtError("light path expressions take the box film only")
            self.lpes = [str(e) for e in lpes]
            if not self.lpes:
                raise McrtError("lpes: at least one expression")
            if len(self.lpes) > LPE_MAX_EXPRESSIONS - 1:
                raise McrtError(f"lpes: {len(self.lpes)} expressions, at most {LPE_MAX_EXPRESSIONS - 1}: the table holds "
                                f"{LPE_MAX_EXPRESSIONS}, and Progressive adds the beauty plane \"C.*\"")
            if light_groups is not None:
                self.lpe_groups = np.ascontiguousarray(light_groups, dtype=np.uint32).reshape(-1)
            self.n_planes = len(self.lpes) + 1
            self._set_lpe_tables()   # refuses a wrong expression or table before anything is allocated
            if integrator.kind == INTEGRATOR_PHOTON:
                integrator.emit_again()   # the same photons, now carrying their states under this table
            light_groups = None
        if light_groups is not None:
            if self.filtered:
                raise McrtError("light groups take the box film only")
            self.light_groups = np.ascontiguousarray(light_groups, dtype=np.uint32).reshape(-1)
            self.n_planes = (int(self.light_groups.max()) + 1 if self.light_groups.size else 0) + 1
            integrator.set_light_groups(self.light_groups, self.n_planes - 1)   # refuses a wrong table before anything is allocated
        self.aovs = bool(aovs)
        if self.aovs:
            if self.filtered:
                raise McrtError("light-path AOVs take the box film only")
            self.n_planes = len(AOV_NAMES)
        self.components = bool(components)
        if self.components:
            if self.filtered:
                raise McrtError("photon-mapper components take the box film only")
            self.n_planes = len(PHOTON_COMPONENT_NAMES)
        planes = (self.n_planes,) if self._planar or self.lpes is not None else ()
        dev = torch.device("cuda", integrator.device)
        self.rgb = [torch.zeros(planes + (self.rows, camera.width, 3), dtype=torch.float64, device=dev) for _ in range(2)]
        self.wsum = [torch.zeros((self.rows, camera.width), dtype=torch.float64, device=dev) for _ in range(2)] if self.filtered else None
        torch.cuda.synchronize(dev)   # the library renders on its own stream
        self.counts = [0, 0]          # samples per pixel in A and B (of the active tiles)
        self.passes = 0
        self.stats = dict.fromkeys(self._STATS, 0)
        self._resolved = None
        grid = tile_grid(self.rows, camera.width, self.tile)
        self.active = np.ones(grid, bool)                          # tiles that still receive samples
        self.tile_counts = np.zeros(grid + (2,), np.int64)          # samples per pixel of each tile in A and B
        self.history = []                                           # one record per render_adaptive pass
        self.stop_reason = None                                     # why the last render_adaptive stopped
        self._features = None                                       # ((samples, specular_depth), device sums [height, width, 8]) of features()

    @property
    def samples(self):
        return self.counts[0] + self.counts[1]

    @property
    def _planar(self):
        """A and B hold planes (light groups, AOVs or photon-mapper components) whose sum is the beauty frame's sums."""
        return self.light_groups is not None or self.aovs or self.components

    def _set_lpe_tables(self):
        # without light_groups the integrator's group table is cleared, so that labels L'g' are refused rather than
        # resolved against whatever table it holds, which the checkpoint's identity would not record
        if self.lpe_groups is not None:
            n_groups = int(self.lpe_groups.max()) + 1 if self.lpe_groups.size else 0
            self.integrator.set_light_groups(self.lpe_groups, n_groups)
        else:
            self.integrator.set_light_groups(None)
        self.integrator.set_light_path_expressions(self.lpes + ["C.*"])

    def add(self, samples):
        """Renders samples [self.samples, self.samples + samples) of the active tiles into A (even pass) or B (odd pass)."""
        half = self.passes % 2
        wsum = self.wsum[half].data_ptr() if self.filtered else None
        if self.light_groups is not None:
            self.integrator.set_light_groups(self.light_groups, self.n_planes - 1)   # the integrator may serve other renders
            st = self.integrator.render_accumulate_groups_dev(self.camera, self.rgb[half].data_ptr(), self.n_planes, self.samples,
                                                              int(samples), self.tile, None if self.active.all() else self.active,
                                                              self.y_first, self.y_step, self.n_rows)
        elif self.lpes is not None:
            self._set_lpe_tables()   # the integrator may serve other renders
            st = self.integrator.render_accumulate_lpe_dev(self.camera, self.rgb[half].data_ptr(), self.n_planes, self.samples,
                                                           int(samples), self.tile, None if self.active.all() else self.active,
                                                           self.y_first, self.y_step, self.n_rows)
        elif self.aovs:
            st = self.integrator.render_accumulate_aovs_dev(self.camera, self.rgb[half].data_ptr(), self.samples, int(samples), self.tile,
                                                            None if self.active.all() else self.active, self.y_first, self.y_step,
                                                            self.n_rows)
        elif self.components:
            st = self.integrator.render_accumulate_components_dev(self.camera, self.rgb[half].data_ptr(), self.samples, int(samples),
                                                                  self.tile, None if self.active.all() else self.active, self.y_first,
                                                                  self.y_step, self.n_rows)
        elif self.active.all():
            st = self.integrator.render_accumulate_dev(self.camera, self.rgb[half].data_ptr(), wsum, self.samples,
                                                       int(samples), self.y_first, self.y_step, self.n_rows)
        else:
            st = self.integrator.render_accumulate_tiles_dev(self.camera, self.rgb[half].data_ptr(), wsum, self.samples, int(samples),
                                                             self.tile, self.active, self.y_first, self.y_step, self.n_rows)
        self.counts[half] += int(samples)
        self.tile_counts = add_tile_samples(self.tile_counts, self.active, half, samples)
        self.passes += 1
        for k in self._STATS:
            self.stats[k] += st[k]
        self._resolved = None
        return st

    def _resolve(self, sums=False):
        """-> (frame, frame error, tile errors, tile sums {sum v, sum I^2} [tiles_y, tiles_x, 2] or None). sums: resolve
        through the per-tile entry point, which reports the tile sums, even while every tile is active."""
        if self._resolved is None or (sums and self._resolved[3] is None):
            self._resolved = self._resolve_halves(self._halves(), sums)
        return self._resolved

    def _halves(self, weights=None):
        """The sums of halves A and B, [rows, width, 3] each: with planes (light groups, AOVs, components) the combination
        of the planes with weights [n_planes, 3] or [n_planes] (None: every weight 1, the beauty frame's sums)."""
        import torch
        if self.lpes is not None:
            if weights is None:
                return [self.rgb[0][-1], self.rgb[1][-1]]   # the beauty plane
            w = light_group_weights(weights, len(self.lpes))
            weights = np.concatenate([w, np.zeros((1, 3))])   # the beauty plane's weight is 0
        elif not self._planar:
            if weights is not None:
                raise McrtError("weights need a render with light groups, AOVs, photon-mapper components or light path expressions")
            return self.rgb
        w = np.ones(self.n_planes) if weights is None else weights
        out = []
        for h in (0, 1):
            o = torch.empty(self.rgb[h].shape[1:], dtype=torch.float64, device=self.rgb[h].device)
            torch.cuda.synchronize(o.device)   # the library works on its own stream
            self.integrator.light_groups_combine_dev(self.rgb[h].data_ptr(), self.n_planes, o.numel(), w, o.data_ptr())
            out.append(o)
        return out

    def _resolve_halves(self, rgb, sums=False):
        """_resolve of the half sums rgb [A, B] (the weight sums are self.wsum's)."""
        import torch
        t = self.tile
        out = torch.empty_like(rgb[0])
        tiles = torch.empty(self.active.shape, dtype=torch.float64, device=out.device)
        if self.active.all() and not sums:
            ptrs = []
            for h in (0, 1):
                has = self.counts[h] > 0
                ptrs += [rgb[h].data_ptr() if has else None,
                         self.wsum[h].data_ptr() if has and self.filtered else None, self.counts[h]]
            err = self.integrator.progressive_resolve_dev(*ptrs, self.camera.width, self.rows, t, out.data_ptr(), tiles.data_ptr())
            return out.cpu().numpy(), err, tiles.cpu().numpy(), None
        tile_sums = torch.empty(self.active.shape + (2,), dtype=torch.float64, device=out.device)
        ptrs = []
        for h in (0, 1):
            has = bool(self.tile_counts[..., h].any())
            ptrs += [rgb[h].data_ptr() if has else None, self.wsum[h].data_ptr() if has and self.filtered else None]
        err = self.integrator.progressive_resolve_tiles_dev(*ptrs, self.tile_counts, self.camera.width, self.rows, t,
                                                            out.data_ptr(), tiles.data_ptr(), tile_sums.data_ptr())
        return out.cpu().numpy(), err, tiles.cpu().numpy(), tile_sums.cpu().numpy()

    # -- light groups
    def group_frames(self):
        """Each light-group plane resolved on its own, float64 [G+1, rows, width, 3]; the last plane is the sky's."""
        if self.light_groups is None:
            raise McrtError("group_frames needs a render with light groups")
        return np.stack([self._resolve_halves([self.rgb[0][g], self.rgb[1][g]])[0] for g in range(self.n_planes)])

    # -- light-path AOVs
    def aov_frames(self):
        """Each AOV plane resolved on its own (in the order of AOV_NAMES) -> (frames float64 [8, rows, width, 3], each
        plane's relative error float64 [8], estimated from the difference of its two halves like error()'s)."""
        if not self.aovs:
            raise McrtError("aov_frames needs a render with aovs=True")
        return self._plane_frames()

    # -- photon-mapper components
    def component_frames(self):
        """Each component plane resolved on its own (in the order of PHOTON_COMPONENT_NAMES) -> (frames float64
        [4, rows, width, 3], each plane's relative error float64 [4], estimated from the difference of its two halves
        like error()'s)."""
        if not self.components:
            raise McrtError("component_frames needs a render with components=True")
        return self._plane_frames()

    # -- light path expressions
    def lpe_frames(self):
        """Each expression's plane resolved on its own (in the order of lpes) -> (frames float64 [len(lpes), rows, width,
        3], each plane's relative error float64 [len(lpes)], estimated from the difference of its two halves like
        error()'s)."""
        if self.lpes is None:
            raise McrtError("lpe_frames needs a render with lpes")
        return self._plane_frames(len(self.lpes))

    def _plane_frames(self, n=None):
        """The first n (all) planes of A and B resolved on their own -> (frames [n, rows, width, 3], relative errors [n])."""
        res = [self._resolve_halves([self.rgb[0][k], self.rgb[1][k]]) for k in range(self.n_planes if n is None else n)]
        return np.stack([r[0] for r in res]), np.array([r[1] for r in res])

    def relight(self, weights):
        """The frame recomposited: the planes summed with weights [n_planes, 3] or [n_planes], resolved like frame()
        -> (frame, frame relative error, per-tile relative errors). Light groups: the last row weights the sky, and
        weight w_g on group g equals a render of the scene with group g's emittance scaled by w_g. AOVs: the rows weight
        the planes of AOV_NAMES, e.g. 0 on the reflection planes removes what the first vertex reflected. Components: the
        rows weight the planes of PHOTON_COMPONENT_NAMES, e.g. [1, 1, 0, 1] removes the caustics. Light path
        expressions: one row per expression; the beauty plane is left out."""
        frame, err, tiles, _ = self._resolve_halves(self._halves(weights))
        return frame, err, tiles

    def frame(self):
        """The resolved frame, float64 [rows, width, 3]."""
        return self._resolve()[0]

    def error(self):
        """-> (frame relative error, per-tile relative errors [tiles_y, tiles_x]); +inf until both halves have samples."""
        _, err, tiles, _ = self._resolve()
        return err, tiles

    def tile_sums(self):
        """-> {sum v, sum I^2} of each tile, float64 [tiles_y, tiles_x, 2] (mcrt_progressive_resolve_tiles_dev)."""
        return self._resolve(sums=True)[3]

    def render(self, pass_samples, max_samples, target_error=None):
        """Adds passes of pass_samples samples until max_samples, or until the first pass after which the frame error is
        at or below target_error. -> the frame."""
        while self.samples < max_samples:
            self.add(min(int(pass_samples), max_samples - self.samples))
            if target_error is not None and self.error()[0] <= target_error:
                break
        return self.frame()

    # -- adaptive sampling
    def retire(self, mask):
        """Retires the tiles where mask (bool [tiles_y, tiles_x]) is True: later passes skip them. A retired tile never
        comes back. The sums are unchanged, so the resolved frame is too."""
        mask = np.asarray(mask, bool)
        if mask.shape != self.active.shape:
            raise McrtError(f"tile mask has shape {mask.shape}, expected {self.active.shape}")
        self.active &= ~mask

    def render_adaptive(self, pass_samples, max_samples, target_error, min_samples=16):
        """Adds passes of pass_samples samples to the active tiles. After each pass it stops if the frame error is at
        or below target_error, as render does; otherwise it retires every active tile that adaptive_retire selects.
        It stops when no tile is active or the active tiles have max_samples samples. Each pass is recorded in
        self.history ({first, count, active, error, tile_counts, tile_sums, retired}); self.stop_reason says why it
        stopped ("target", "no active tile" or "max_samples"). -> the frame.

        Known limits: the criterion compares a tile's absolute noise with the frame's signal, so dark tiles retire
        early. A tile's estimate from few samples is itself noisy, which is what min_samples guards against. The two
        Owen-scrambled halves are not independent: with two large passes the estimate has read about 10 % low."""
        tile_pixels = tile_pixel_counts(self.rows, self.camera.width, self.tile)
        while True:
            if not self.active.any():
                self.stop_reason = "no active tile"
                break
            if self.samples >= max_samples:
                self.stop_reason = "max_samples"
                break
            first, count, n_active = self.samples, min(int(pass_samples), max_samples - self.samples), int(self.active.sum())
            self.add(count)
            _, err, _, sums = self._resolve(sums=True)
            entry = {"first": first, "count": count, "active": n_active, "error": err,
                     "tile_counts": self.tile_counts.copy(), "tile_sums": sums}
            if err <= target_error:
                entry["retired"] = np.zeros_like(self.active)
                self.history.append(entry)
                self.stop_reason = "target"
                break
            entry["retired"] = adaptive_retire(self.active, self.tile_counts, sums, tile_pixels, target_error, min_samples)
            self.retire(entry["retired"])
            self.history.append(entry)
        return self.frame()

    # -- denoising
    def _feature_sums(self, samples, specular_depth=0):
        """Device feature sums of samples [0, samples), computed once per (sample count, specular depth)."""
        import torch
        key = (int(samples), int(specular_depth))
        if self._features is None or self._features[0] != key:
            f = torch.zeros((self.camera.height, self.camera.width, 8), dtype=torch.float64, device=self.rgb[0].device)
            torch.cuda.synchronize(f.device)   # the library renders on its own stream
            self.integrator.render_features_dev(self.camera, f.data_ptr(), 0, key[0], specular_depth=key[1])
            self._features = (key, f)
        return self._features[1]

    def features(self, samples=8, specular_depth=0):
        """First-hit guides of the camera rays of samples [0, samples) of every pixel of the whole frame, as numpy:
        {albedo [H,W,3], normal [H,W,3] (normalised mean, 0 where nothing was hit), depth [H,W] (mean hit distance),
        coverage [H,W] (hits / samples)}. specular_depth > 0 takes them after up to that many perfectly specular
        bounces of each sample's path (Integrator.render_features_dev): the albedo is weighted by the chain's
        throughput and the depth is the distance along the chain. The device sums are kept and recomputed only when
        `samples` or `specular_depth` changes."""
        f = self._feature_sums(samples, specular_depth).cpu().numpy()
        hits = f[..., 7]
        with np.errstate(invalid="ignore", divide="ignore"):
            albedo = np.where(hits[..., None] > 0, f[..., 0:3] / hits[..., None], 0.0)
            depth = np.where(hits > 0, f[..., 6] / hits, 0.0)
            length = np.sqrt((f[..., 3:6] ** 2).sum(-1, keepdims=True))
            normal = np.where(length > 0, f[..., 3:6] / length, 0.0)
        return {"albedo": albedo, "normal": normal, "depth": depth, "coverage": hits / float(samples)}

    def denoise(self, iterations=None, sigma_color=None, sigma_normal=None, sigma_depth=None, sigma_albedo=None,
                feature_samples=8, specular_depth=0, weights=None):
        """The frame denoised by the cross-filtered a-trous filter of mcrt_denoise_dev, guided by features(feature_samples)
        -> (frame float64 [H, W, 3], residual error). The error is estimated like error()'s, from the difference of the
        two filtered halves: it measures the remaining noise, not the filter's bias. Arguments left None take the
        defaults of DENOISE_DEFAULTS. Uses the per-tile counts, so it works after adaptive retirement too.
        Raises McrtError unless the row set is the whole frame and every tile has samples in both halves.
        specular_depth > 0 guides the filter by features(feature_samples, specular_depth), taken after up to that
        many perfectly specular bounces, so glass and mirrors are guided by what they show; on the H100 measurements
        of DESIGN.md §6 that did not lower the denoised error at 8 feature samples, which is why 0 stays the default.

        Known limits: at specular_depth 0 the guides come from the first hit only, so glass and mirrors are guided by
        their own surface; rough and glossy lobes are never followed; the feature samples [0, F) also feed half A; the Owen-scrambled halves are not
        independent, so the residual estimate can read about 10 % low.

        weights (light groups, AOVs or components only): denoise the frame relit or recomposited with these weights (relight) instead of
        the beauty frame."""
        import torch
        if (self.y_first, self.y_step, self.n_rows) != (0, 1, self.camera.height):
            raise McrtError("denoise needs the whole frame as the row set (y_first 0, y_step 1, n_rows = height)")
        if not (self.tile_counts > 0).all():
            raise McrtError("denoise needs samples in both halves of every tile")
        given = {"iterations": iterations, "sigma_color": sigma_color, "sigma_normal": sigma_normal,
                 "sigma_depth": sigma_depth, "sigma_albedo": sigma_albedo}
        v = {k: DENOISE_DEFAULTS[k] if x is None else x for k, x in given.items()}
        params = DenoiseParams(int(v["iterations"]), 0, float(v["sigma_color"]), float(v["sigma_normal"]),
                               float(v["sigma_depth"]), float(v["sigma_albedo"]))
        rgb = self._halves(weights)
        feats = self._feature_sums(feature_samples, specular_depth)
        out = torch.empty_like(rgb[0])
        w = (self.wsum[0].data_ptr(), self.wsum[1].data_ptr()) if self.filtered else (None, None)
        err = self.integrator.denoise_dev(rgb[0].data_ptr(), w[0], rgb[1].data_ptr(), w[1], self.tile_counts, self.tile,
                                          feats.data_ptr(), self.camera.width, self.camera.height, out.data_ptr(), params)
        return out.cpu().numpy(), err

    # -- checkpoint / resume
    def _identity(self):
        """What a resumed render must match: every input that changes the samples' paths or where they land."""
        import hashlib
        ig, cam = self.integrator, self.camera
        h = hashlib.sha256()
        for k in Scene._ARRAYS:
            a = np.ascontiguousarray(ig.scene.a[k])
            h.update(k.encode() + str(a.dtype).encode() + str(a.shape).encode() + a.tobytes())
        h.update(np.float64(ig.scene.ior).tobytes())
        ident = {"seed": np.uint32(ig.global_seed), "precision": np.int32(ig.precision), "integrator": np.int32(ig.kind),
                 "camera": np.frombuffer(bytes(cam.rec), np.uint8),
                 "film": np.frombuffer(bytes(cam.film_rec()), np.uint8) if cam.film_rec() is not None else np.zeros(0, np.uint8),
                 "row_set": np.array([self.y_first, self.y_step, self.n_rows], np.int64),
                 "tile": np.int64(self.tile),   # the tile masks' shapes depend on it
                 "scene_digest": np.array(h.hexdigest())}
        if ig.kind == INTEGRATOR_PHOTON:
            ident.update(self._photon_identity())
        if self.light_groups is not None:
            ident["light_groups"] = self.light_groups.copy()
        if self.aovs:
            ident["aovs"] = np.int64(len(AOV_NAMES))
        if self.components:
            ident["photon_components"] = np.int64(len(PHOTON_COMPONENT_NAMES))
        if self.lpes is not None:
            ident["lpes"] = np.array(self.lpes)
            ident["lpe_groups"] = self.lpe_groups.copy() if self.lpe_groups is not None else np.zeros(0, np.int64)
        return ident

    def _photon_identity(self):
        """The photon maps' part of _identity: a digest of the uploaded maps, with light groups of each photon's light."""
        import hashlib
        ig = self.integrator
        caustic, glob, k, dv = ig._maps
        ph = hashlib.sha256(np.array([k, dv], np.int64).tobytes())
        for which, m in enumerate((caustic, glob)):
            rows = np.ascontiguousarray(np.asarray(m["photons"], np.float32).reshape(-1, 8))
            if self.light_groups is not None:
                # which light emitted a photon decides its plane: each row is the photon and its light index
                rows = np.concatenate([rows.view(np.uint32), ig.photon_lights(which)[:, None]], axis=1)
            rows = np.ascontiguousarray(rows).view(np.dtype((np.void, rows.shape[1] * 4))).ravel()
            ph.update(np.int64(len(rows)).tobytes() + np.sort(rows).tobytes())   # a set: order inside a leaf may differ
        return {"photon_digest": np.array(ph.hexdigest())}

    def save(self, path):
        """Writes an .npz checkpoint: the sums, the sample counts, the pass index, the active tiles and the per-tile
        counts, and the render's identity."""
        data = dict(self._identity(), counts=np.array(self.counts, np.int64), passes=np.int64(self.passes),
                    active=self.active.copy(), tile_counts=self.tile_counts.copy(),
                    rgb_a=self.rgb[0].cpu().numpy(), rgb_b=self.rgb[1].cpu().numpy())
        if self.filtered:
            data.update(wsum_a=self.wsum[0].cpu().numpy(), wsum_b=self.wsum[1].cpu().numpy())
        with open(path, "wb") as f:
            np.savez(f, **data)

    @classmethod
    def load(cls, path, integrator, camera, tile=None, light_groups=None, aovs=False, components=False, lpes=None):
        """Resumes a checkpoint written by save() with `integrator` and `camera` (and `tile`, the checkpoint's if None).
        Raises McrtError, and resumes nothing, when the seed, precision, integrator kind, camera, film, tile, scene,
        photon maps, light groups, AOVs, components or light path expressions (with their groups) differ from the
        checkpoint's. A checkpoint without tile state resumes with every tile active."""
        data = _read_checkpoint(path)
        y_first, y_step, n_rows = (int(v) for v in data["row_set"])
        p = cls(integrator, camera, y_first, y_step, n_rows, int(data["tile"]) if tile is None else int(tile), light_groups, aovs,
                components, **({"lpes": lpes} if lpes is not None else {}))
        p._restore(path, data)
        return p

    def _restore(self, path, data):
        """Takes over the sums, counts and tile state of checkpoint `data` after checking its identity."""
        import torch
        ident = self._identity()
        if ("light_groups" in data) != ("light_groups" in ident):
            raise McrtError(f"checkpoint {path}: light groups differ from this render's; not resuming")
        if ("aovs" in data) != ("aovs" in ident):
            raise McrtError(f"checkpoint {path}: light-path AOVs differ from this render's; not resuming")
        if ("photon_components" in data) != ("photon_components" in ident):
            raise McrtError(f"checkpoint {path}: photon-mapper components differ from this render's; not resuming")
        if ("lpes" in data) != ("lpes" in ident):
            raise McrtError(f"checkpoint {path}: light path expressions differ from this render's; not resuming")
        for k, want in ident.items():
            if k not in data or not np.array_equal(data[k], want):
                raise McrtError(f"checkpoint {path}: {k} differs from this render's; not resuming")
        for name, dst in (("rgb_a", self.rgb[0]), ("rgb_b", self.rgb[1])) + ((("wsum_a", self.wsum[0]), ("wsum_b", self.wsum[1])) if self.filtered else ()):
            if data[name].shape != tuple(dst.shape):
                raise McrtError(f"checkpoint {path}: {name} has shape {data[name].shape}, expected {tuple(dst.shape)}")
            dst.copy_(torch.from_numpy(data[name]))
        for name, want in (("active", self.active.shape), ("tile_counts", self.tile_counts.shape)):
            if name in data and data[name].shape != want:
                raise McrtError(f"checkpoint {path}: {name} has shape {data[name].shape}, expected {want}")
        torch.cuda.synchronize(self.rgb[0].device)
        self.counts = [int(c) for c in data["counts"]]
        self.passes = int(data["passes"])
        if "active" in data:
            self.active = data["active"].astype(bool)
            self.tile_counts = data["tile_counts"].astype(np.int64)
        else:
            self.tile_counts[...] = self.counts   # written before adaptive sampling: every tile has the uniform counts


def _read_checkpoint(path):
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def ppm_radii(r1, alpha, n):
    """The n gather radii of progressive photon mapping (Knaus & Zwicker 2011): r_1 = r1, then
    r_{i+1}^2 = r_i^2 (i + alpha) / (i + 1). With 0 < alpha < 1 the average of the passes' estimates converges:
    bias and variance both go to zero. -> float64 [n]."""
    r1, alpha, n = float(r1), float(alpha), int(n)
    if not (0.0 < alpha < 1.0):
        raise McrtError(f"alpha {alpha} is outside (0, 1)")
    if not (r1 > 0.0 and math.isfinite(r1)):
        raise McrtError(f"initial radius {r1} is not positive and finite")
    i = np.arange(1, max(n, 1), dtype=np.float64)
    r = np.empty(max(n, 0))
    if n > 0:
        r[0] = r1
        r[1:] = r1 * np.sqrt(np.cumprod((i + alpha) / (i + 1.0)))
    return r


class ProgressivePhotonMapping(Progressive):
    """Probabilistic progressive photon mapping (Knaus & Zwicker, "Progressive photon mapping: a probabilistic
    approach", TOG 2011) over the passes of Progressive: pass i emits its own photon map (PhotonMapper.emit_pass(i),
    the next emission indices of every light) and gathers with fixed radii r_i that shrink as ppm_radii, so the frame
    converges to the image, not to one map's answer. Even passes go to half A and odd ones to B, so the halves come
    from different maps and error(), render(target_error=...), render_adaptive and denoise() see the maps' noise too.

    radius: None picks the initial radii once from the pass-0 maps - for each map the median, over up to 4096 of its
    photons chosen with a fixed seed from the photons sorted by position, of the distance to the
    k_nearest_photons-th nearest photon (PhotonMapper.knn at the photons' positions; in a map of fewer photons, the
    farthest one); an empty caustic map takes the global radius. A number sets both, a pair (caustic, global) each.
    With few emissions per pass that radius is large, and its blur dominates the error for many passes: on the
    golden photon-mapping scene, a quarter of it reached the fixed k-NN map's error within 64 passes and the full
    radius did not (DESIGN.md section 6).

    light_groups: as Progressive's. Every pass emits its own map, and emitted maps record each photon's light, so the
    passes split their estimates by group; the pass-0 map is emitted before the table is set.

    lpes: as Progressive's. Every pass emits its map while the table is set, so every photon carries its path's state.

    components: as Progressive's. component_frames() then shows whether the caustic or the global estimate, whose radii
    shrink on their own schedules, still dominates the error.

    Each pass replaces the photon mapper's uploaded maps and leaves it in gather mode (gather_radius(0, 0) returns
    it to the k-NN estimate). The frame no longer equals a one-shot render; it equals the same sequence of passes.
    Every sample is weighted equally: with passes of equal size that is Knaus and Zwicker's plain average of the
    pass estimates, a shorter last pass deviates from it slightly. Checkpoints record the emissions, caustic factor,
    leaf size, alpha and the initial radii instead of the maps; load() resumes with the map of pass `passes`, which
    the next add() emits again (the passes are deterministic)."""

    def __init__(self, photon_mapper, camera, emissions, caustic_factor, max_photons_per_octree_leaf=200, alpha=2 / 3,
                 radius=None, k_nearest_photons=50, tile=16, light_groups=None, aovs=False, components=False, lpes=None):
        if not isinstance(photon_mapper, PhotonMapper):
            raise McrtError("ProgressivePhotonMapping needs a PhotonMapper")
        if aovs:
            raise McrtError("the photon mapper has no light-path AOVs")
        ppm_radii(1.0, alpha, 1)   # validates alpha
        self.emissions, self.caustic_factor = int(emissions), float(caustic_factor)
        self.max_photons_per_octree_leaf, self.k_nearest_photons = int(max_photons_per_octree_leaf), int(k_nearest_photons)
        self.alpha = float(alpha)
        if (light_groups is not None and not photon_mapper.has_photon_lights) or \
                (lpes is not None and getattr(photon_mapper, "_emit_args", None) is None):
            # Progressive sets the table on maps that carry light indices, and emits again the maps of emit_pass: the
            # pass-0 map
            photon_mapper.emit_pass(0, self.emissions, self.caustic_factor, self.max_photons_per_octree_leaf, self.k_nearest_photons)
        super().__init__(photon_mapper, camera, tile=tile, light_groups=light_groups, components=components,
                         **({"lpes": lpes} if lpes is not None else {}))
        if radius is None:
            radius = self._initial_radii()
        r = (float(radius), float(radius)) if np.ndim(radius) == 0 else tuple(float(x) for x in radius)
        if len(r) != 2:
            raise McrtError("radius: None, a number or a (caustic, global) pair")
        for x in r:
            ppm_radii(x, self.alpha, 1)   # validates the radius
        self.radius = r

    def _emit(self, pass_index):
        return self.integrator.emit_pass(pass_index, self.emissions, self.caustic_factor, self.max_photons_per_octree_leaf,
                                         self.k_nearest_photons)

    def _initial_radii(self):
        self._emit(0)
        ig, radii = self.integrator, [None, None]
        rng = np.random.default_rng(0x9E3779B9)
        for which, m in enumerate(ig._maps[:2]):
            pos = m["photons"].reshape(-1, 8)[:, 3:6].astype(np.float64)
            if len(pos) == 0:
                continue
            pos = pos[np.lexsort(pos.T[::-1])]   # the emission's atomics order the photons; the choice must not depend on it
            pick = np.sort(rng.choice(len(pos), min(4096, len(pos)), replace=False))
            _, d2, cnt = ig.knn(which, pos[pick])
            # the farthest of the cnt results (unsorted); a map with fewer than k photons returns them all, then padding
            kth = np.where(np.arange(d2.shape[1])[None, :] < cnt[:, None], d2, 0.0).max(axis=1)
            radii[which] = float(np.median(np.sqrt(kth)))
        if radii[1] is None:
            raise McrtError("the pass-0 global photon map is empty: no initial radius")
        return (radii[1] if radii[0] is None else radii[0], radii[1])

    def pass_radii(self, pass_index):
        """(caustic, global) gather radii of pass pass_index (0-based)."""
        return tuple(float(ppm_radii(r, self.alpha, int(pass_index) + 1)[-1]) for r in self.radius)

    def add(self, samples):
        """Emits the map of pass self.passes, gathers with that pass's radii and renders the next samples (Progressive.add)."""
        if self.lpes is not None:
            self._set_lpe_tables()   # the pass's photons carry their states under this render's table
        self._emit(self.passes)
        self.integrator.gather_radius(*self.pass_radii(self.passes))
        return super().add(samples)

    def _photon_identity(self):
        return {"ppm_emissions": np.int64(self.emissions), "ppm_caustic_factor": np.float64(self.caustic_factor),
                "ppm_leaf": np.int64(self.max_photons_per_octree_leaf), "ppm_alpha": np.float64(self.alpha),
                "ppm_radius": np.array(self.radius, np.float64)}

    @classmethod
    def load(cls, path, photon_mapper, camera, emissions, caustic_factor, max_photons_per_octree_leaf=200, alpha=2 / 3,
             radius=None, k_nearest_photons=50, tile=None, light_groups=None, components=False, lpes=None):
        """Resumes a checkpoint written by save(). Raises McrtError, and resumes nothing, when the seed, precision,
        camera, film, tile, scene, emissions, caustic factor, leaf size, alpha, initial radii, light groups, components
        or light path expressions differ from the checkpoint's (radius None derives them from the pass-0 maps again)."""
        data = _read_checkpoint(path)
        p = cls(photon_mapper, camera, emissions, caustic_factor, max_photons_per_octree_leaf, alpha, radius, k_nearest_photons,
                int(data["tile"]) if tile is None else int(tile), light_groups, components=components, lpes=lpes)
        p._restore(path, data)
        return p


def shard_rows(height, rank, world_size):
    """Row block of `rank` (SURVEY.md §8e): contiguous blocks, remainder spread over the first ranks."""
    base, rem = divmod(height, world_size)
    y0 = rank * base + min(rank, rem)
    return y0, y0 + base + (1 if rank < rem else 0)
