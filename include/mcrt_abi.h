/*
 * mcrt_abi.h — C ABI of the H100-native path-tracing integrator.
 *
 * Drop-in boundary for the ray/BVH/BSDF hot path of linusmossberg/monte-carlo-ray-tracer.
 * The reference has no FFI; the interface this replaces is the C++ virtual
 *     glm::dvec3 Integrator::sampleRay(Ray)            (source/integrator/integrator.hpp:20)
 * and its only caller, the per-pixel loop in
 *     Camera::samplePixel / Camera::sampleImage        (source/camera/camera.cpp:66-145).
 * Because one scalar ray per virtual call cannot feed a GPU, the batch boundary sits at
 * the body of Camera::sampleImage ("render these rows of this camera"), plus batched
 * sampleRay / Scene::intersect entry points with the reference's per-call semantics.
 *
 * Conventions
 *   - plain C, no torch / C++ types; every pointer is a HOST pointer unless the name ends
 *     in _dev; the caller owns host buffers, the context owns device memory.
 *   - return 0 on success, a negative mcrt_status on failure; mcrt_last_error() gives text.
 *   - one context per GPU, driven from one host thread at a time.
 *   - all scene arrays are the *built* state of the reference's Scene/BVH/Material objects
 *     in float64 (the reference computes in double), flattened by the exporter
 *     (monte-carlo-ray-tracer_b200/host/exporter.cpp). Layouts for the device (FP64 parity
 *     arrays, FP32 wide-node arrays) are derived inside mcrt_scene_upload.
 */
#ifndef MCRT_ABI_H
#define MCRT_ABI_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MCRT_ABI_VERSION 1

typedef enum mcrt_status {
    MCRT_OK = 0,
    MCRT_ERR_INVALID = -1,   /* bad argument / inconsistent scene description        */
    MCRT_ERR_CUDA = -2,      /* CUDA runtime error (text in mcrt_last_error)          */
    MCRT_ERR_NO_SCENE = -3,  /* render/trace called before mcrt_scene_upload          */
    MCRT_ERR_UNSUPPORTED = -4, /* feature outside the hot path (e.g. non-box film)     */
    MCRT_ERR_NO_PHOTONS = -5 /* photon-mapped render without mcrt_photon_upload       */
} mcrt_status;

/* Primitive type tags: Surface::{Triangle,Sphere,Quadric} (source/surface/surface.hpp:54-116). */
enum { MCRT_PRIM_TRIANGLE = 0, MCRT_PRIM_SPHERE = 1, MCRT_PRIM_QUADRIC = 2 };

/* Integrator kinds: PathTracer / PhotonMapper (source/camera/camera.cpp:22-29). */
enum { MCRT_INTEGRATOR_PATH = 0, MCRT_INTEGRATOR_PHOTON = 1 };

/* Arithmetic of the device path.
 *   MCRT_PRECISION_F64: parity mode — double, operation order of the reference, no FMA
 *                       contraction, reference's best-first traversal order.
 *   MCRT_PRECISION_F32: fast mode — float, wide-node stack traversal, scale-aware offsets. */
enum { MCRT_PRECISION_F64 = 0, MCRT_PRECISION_F32 = 1 };

/* Material record: the built state of class Material (source/material/material.hpp:37-54)
 * including the derived flags/constants of Material::computeProperties (material.cpp:97-111). */
typedef struct mcrt_material {
    double reflectance[3];
    double specular_reflectance[3];
    double transmittance[3];
    double emittance[3];          /* radiosity after Scene::generateEmissives (scene.cpp:202) */
    double roughness, specular_roughness, ior, transparency;
    double complex_ior_real[3], complex_ior_imag[3];
    double A, B;                  /* Oren–Nayar constants (material.cpp:106-108)              */
    double a[2];                  /* GGX alpha (material.cpp:110)                             */
    uint32_t has_complex_ior, perfect_mirror;
    uint32_t rough, rough_specular, opaque, emissive, dirac_delta;
    uint32_t _pad;
} mcrt_material;

/* Flattened Scene + BVH (source/scene/scene.hpp, source/bvh/bvh.hpp:68-108). */
typedef struct mcrt_scene_desc {
    uint32_t abi_version;             /* MCRT_ABI_VERSION */
    /* BVH::linear_tree in depth-first order; n_nodes == 0 means "no bvh object" and the
     * linear-scan branch of Scene::intersect (scene.cpp:159-173) is taken. */
    uint32_t n_nodes;
    const double* node_bounds;        /* [n_nodes][6]  min.xyz, max.xyz                       */
    const uint32_t* node_first_prim;  /* [n_nodes]     LinearNode::start_surface              */
    const uint32_t* node_prim_count;  /* [n_nodes]     LinearNode::num_surfaces (0 = inner)   */
    const uint32_t* node_next_sibling;/* [n_nodes]     0 = none                               */
    /* BVH::ordered_surfaces (or Scene::surfaces without a BVH). */
    uint32_t n_prims;
    const uint8_t* prim_type;         /* [n_prims] MCRT_PRIM_*                                */
    const uint32_t* prim_index;       /* [n_prims] index into the per-type arrays             */
    const uint32_t* prim_material;    /* [n_prims] index into materials                       */
    const double* prim_area;          /* [n_prims] Surface::Base::area_                       */
    /* triangles (source/surface/surface.hpp:92-96) */
    uint32_t n_tris;
    const double* tri_v0;             /* [n_tris][3] */
    const double* tri_v1;
    const double* tri_v2;
    const double* tri_e1;             /* stored, not recomputed: keeps the reference's rounding */
    const double* tri_e2;
    const double* tri_normal;         /* face normal_ */
    const int32_t* tri_vn_index;      /* [n_tris] index into vertex_normals or -1             */
    uint32_t n_vertex_normals;
    const double* vertex_normals;     /* [n_vertex_normals][9]  n0,n1,n2                      */
    /* spheres (surface.hpp:68-69) */
    uint32_t n_spheres;
    const double* sphere_origin_radius; /* [n_spheres][4] */
    /* quadrics (surface.hpp:114-115, clip box = Base::BB_) */
    uint32_t n_quadrics;
    const double* quadric_Q;          /* [n_quadrics][16] column-major dmat4                  */
    const double* quadric_G;          /* [n_quadrics][12] column-major dmat4x3                */
    const double* quadric_bounds;     /* [n_quadrics][6]                                      */
    /* materials: one entry per distinct Material object */
    uint32_t n_materials;
    const mcrt_material* materials;
    /* Scene::emissives / cumulative_emissives_importance (scene.cpp:178-209) */
    uint32_t n_lights;
    const uint32_t* light_prim;       /* [n_lights] ordered-primitive index of each emissive  */
    const double* light_cdf;          /* [n_lights]                                           */
    double scene_ior;                 /* Scene::ior */
} mcrt_scene_desc;

/* Camera state after Camera::Camera (source/camera/camera.cpp:20-64). */
typedef struct mcrt_camera {
    double eye[3], forward[3], left[3], up[3];
    double focal_length, sensor_width, aperture_radius, focus_distance;
    uint32_t width, height;
    uint32_t thin_lens;
    uint32_t _pad;
} mcrt_camera;

/* Ray as the reference's Ray(start, direction, medium_ior) (source/ray/ray.cpp:13-14). */
typedef struct mcrt_ray {
    double origin[3];
    double direction[3];
} mcrt_ray;

/* Result of Scene::intersect (source/ray/intersection.hpp:9-23). prim == 0xFFFFFFFF: miss. */
typedef struct mcrt_hit {
    double t, u, v;
    uint32_t prim;
    uint32_t interpolate;
} mcrt_hit;

/* LinearOctree<Photon> (source/octree/linear-octree.hpp:19-29, photon.hpp:35-37). */
typedef struct mcrt_photon_map_desc {
    uint32_t n_octants;
    const double* octant_bounds;        /* [n_octants][6]                                     */
    const uint64_t* octant_start;       /* start_data                                         */
    const uint64_t* octant_count;       /* contained_data                                     */
    const uint32_t* octant_next_sibling;/* 0xFFFFFFFF = none                                  */
    const uint8_t* octant_leaf;
    uint64_t n_photons;
    const float* photons;               /* [n_photons][8] flux.xyz, pos.xyz, phi, theta       */
} mcrt_photon_map_desc;

typedef struct mcrt_stats {
    uint64_t paths;            /* camera paths started                                        */
    uint64_t extension_rays;   /* closest-hit queries for path extension (incl. primary)      */
    uint64_t shadow_rays;      /* closest-hit queries for next-event estimation               */
    uint64_t box_tests;        /* AABB slab tests executed by the traversal kernels           */
    uint64_t prim_tests;       /* primitive intersection tests executed                       */
    uint64_t knn_queries;      /* photon-map k-NN queries                                     */
    uint64_t wavefront_iterations;
    uint64_t kernel_launches;
    uint64_t ior_stack_overflows;
    uint32_t max_depth;
    uint32_t _pad;
    double gpu_ms_total;       /* CUDA-event time of the render, first launch → last          */
    /* per-stage sums of CUDA-event times; filled only with option "stage_timing" = 1 */
    double gpu_ms_generate, gpu_ms_extend, gpu_ms_shade, gpu_ms_shadow, gpu_ms_knn;
    uint64_t extend_launches, shadow_launches;
    uint64_t shadow_box_tests, shadow_prim_tests; /* k_shadow's share of box_tests / prim_tests */
    /* k_extend warp-tail diagnostic: sum over rays of (box+prim tests) / sum over warps of
     * 32*max over the warp's rays = the lane utilisation lost to uneven ray lengths alone */
    uint64_t extend_work_sum, extend_work_warpmax; /* builds with -DMCRT_TAIL_DIAGNOSTIC only, else 0 */
    /* parity mode: closest-hit queries whose two nearest candidates lay within rounding distance of each
     * other and were therefore re-traced in the reference's own visiting order (csrc/bvh4.cuh) */
    uint64_t replayed_rays;
} mcrt_stats;

typedef struct mcrt_ctx mcrt_ctx;

int mcrt_abi_version(void);

/* Create a context on CUDA device `device`. */
int mcrt_init(int device, mcrt_ctx** out_ctx);
void mcrt_destroy(mcrt_ctx* ctx);
const char* mcrt_last_error(const mcrt_ctx* ctx);

/* Replaces the Scene held by Integrator (integrator.hpp:25): copies the description to the
 * device and derives both device layouts. Returns bytes copied host→device in *h2d_bytes. */
int mcrt_scene_upload(mcrt_ctx* ctx, const mcrt_scene_desc* scene, uint64_t* h2d_bytes);

/* Replaces PhotonMapper's caustic_map/global_map members (photon-mapper.hpp:27-28). */
int mcrt_photon_upload(mcrt_ctx* ctx, const mcrt_photon_map_desc* caustic_map,
                       const mcrt_photon_map_desc* global_map, uint32_t k_nearest,
                       uint32_t direct_visualization, uint64_t* h2d_bytes);

/* Film reconstruction filter, the "film" object of a camera in the scene JSON
 * (source/camera/film.cpp:19-59). Default (never set): box, radius 0.5, no cache. */
enum { MCRT_FILM_BOX = 0, MCRT_FILM_MITCHELL_NETRAVALI = 1, MCRT_FILM_CATMULL_ROM = 2, MCRT_FILM_B_SPLINE = 3,
       MCRT_FILM_HERMITE = 4, MCRT_FILM_GAUSSIAN = 5, MCRT_FILM_LANCZOS = 6 };
typedef struct mcrt_film {
    uint32_t filter;        /* MCRT_FILM_* */
    uint32_t cache_size;    /* 0: evaluate the filter function, else nearest-neighbour lookup table */
    double radius;          /* <= 0: the filter's default radius (film.cpp:32-43) */
} mcrt_film;

/* SURVEY.md §8f-4 ("next"): Film::deposit with the reference's reconstruction filters for the
 * following renders of this context (source/camera/film.cpp:61-113, filter.hpp). With a filter other
 * than the default box, samples splat into neighbouring pixels, so mcrt_render_rows* must then
 * cover the whole frame (rows cannot be sharded without halo exchange). NULL restores the default. */
int mcrt_set_film(mcrt_ctx* ctx, const mcrt_film* film);

/* Parameters of the photon pass, the "photon_map" object of the scene JSON
 * (source/integrator/photon-mapper/photon-mapper.cpp:28-38). */
typedef struct mcrt_photon_emit_params {
    uint64_t emissions;                    /* "emissions" (before the caustic_factor scaling)  */
    double caustic_factor;
    uint32_t max_photons_per_octree_leaf;
    uint32_t k_nearest_photons;
    uint32_t direct_visualization;
    uint32_t global_seed;
    double scene_bounds[6];                /* Scene::BB() = root box of both octrees            */
} mcrt_photon_emit_params;

/* SURVEY.md §8f-1 ("next"): replaces the first pass of PhotonMapper::PhotonMapper
 * (photon-mapper.cpp:24-223) — photon emission + tracing (emitPhoton, :225-277) on the GPU, then
 * Octree<Photon> construction + LinearOctree::compact (octree.cpp:34-81, linear-octree.cpp:201-244)
 * — and installs the two maps in the context exactly as mcrt_photon_upload would. The photon
 * multiset and the octree structure equal the reference's (photons inside one leaf may be stored
 * in a different order: the reference's order depends on its thread schedule). The octrees are
 * built on the device from the emission buffers (the photons never visit the host); in `stats`,
 * gpu_ms_total is the emission wavefront and gpu_ms_knn the octree construction. */
int mcrt_photon_emit(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, int precision,
                     uint64_t* n_caustic, uint64_t* n_global, mcrt_stats* stats);

/* The photon pass in pieces, for sharding it over GPUs (SURVEY.md §8e: emission sharded by ranges of the
 * reference's EmissionWork index space, photon-mapper.cpp:61-78, photons all-gathered, every rank builds the
 * same octrees):
 *   mcrt_photon_emit_total   size of the emission index space (sum over lights of their emission counts)
 *   mcrt_photon_emit_range   emits work items [work_first, work_first + work_count); the photons stay in device
 *                            buffers of the context - 8 floats per photon {flux.xyz, pos.xyz, phi, theta} - whose
 *                            addresses are returned (valid until the next emission / mcrt_destroy)
 *   mcrt_photon_build_dev    builds both octrees from device photon arrays (this rank's, or the concatenation
 *                            of all ranks') and installs them like mcrt_photon_upload
 * mcrt_photon_emit == total, range(0, total), build. */
int mcrt_photon_emit_total(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, uint64_t* total_emissions);
int mcrt_photon_emit_range(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, int precision,
                           uint64_t work_first, uint64_t work_count, const float** caustic_dev, uint64_t* n_caustic,
                           const float** global_dev, uint64_t* n_global, mcrt_stats* stats);
int mcrt_photon_build_dev(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, const float* caustic_dev,
                          uint64_t n_caustic, const float* global_dev, uint64_t n_global, double* build_ms);

/* One pass of progressive photon mapping (Knaus & Zwicker, "Progressive photon mapping: a probabilistic
 * approach", TOG 2011): mcrt_photon_emit, except that light l's emissions are the reference's emission
 * indices [pass * n_l, (pass + 1) * n_l), n_l being its count in the emission plan. The photon flux stays
 * light_flux / n_l, so every pass map is a complete map on its own; the index offset continues each light's
 * Owen-scrambled Sobol sequence, so passes stay stratified against each other, and passes 0..P-1 hold the
 * photons of one mcrt_photon_emit whose per-light counts are P * n_l (with 1/P of their flux). Pass 0 is
 * mcrt_photon_emit. MCRT_ERR_INVALID when (pass + 1) * n_l exceeds 2^32 for a light (the sample index is
 * 32 bits). */
int mcrt_photon_emit_pass(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, int precision, uint32_t pass,
                          uint64_t* n_caustic, uint64_t* n_global, mcrt_stats* stats);

/* Fixed-radius photon gather for the following photon-mapped renders of this context, in place of the
 * reference's k-NN estimate: every photon within r of a query enters it, with the k-NN formulas and r^2 in
 * place of the k-th distance^2 - caustic 3/(pi r^2) sum flux f/pdf (1 - d/r), global 1/(pi r^2) sum flux f/pdf.
 * The kernel (k_gather) replaces k_knn; its time is reported in gpu_ms_knn, the same stage slot.
 * (0, 0) returns to the k-NN estimate, the default; otherwise both radii must be positive and finite
 * (MCRT_ERR_INVALID). The radii stay set when maps are replaced. */
int mcrt_photon_gather_radius(mcrt_ctx* ctx, double r_caustic, double r_global);

/* The traversal of the fixed-radius gather on caller points (which: 0 caustic, 1 global map): for each point
 * out_count[i] photons lie within `radius` (float64 distance2 <= radius^2, inclusive), out_flux_sum[i][3] is the
 * float64 sum of their float32 flux and out_cone_sum[i][3] the same weighted by max(0, 1 - d / radius).
 * Host buffers. MCRT_ERR_UNSUPPORTED if a traversal stack overflowed. */
int mcrt_photon_gather_search(mcrt_ctx* ctx, int which, const double* points_xyz, size_t n, double radius,
                              uint32_t* out_count, double* out_flux_sum, double* out_cone_sum, mcrt_stats* stats);

/* Host view of the maps built by mcrt_photon_emit (which: 0 caustic, 1 global). The pointers stay
 * valid until the next mcrt_photon_emit / mcrt_destroy. */
int mcrt_photon_download(mcrt_ctx* ctx, int which, mcrt_photon_map_desc* out);

/* The index of the light that emitted each photon of a built map (which: 0 caustic, 1 global), out[n] HOST, in the
 * order mcrt_photon_download returns the photons; n must be the map's photon count. Maps emitted by mcrt_photon_emit /
 * mcrt_photon_emit_pass carry these indices; maps of mcrt_photon_upload and mcrt_photon_build_dev do not
 * (MCRT_ERR_UNSUPPORTED), and neither do maps emitted before the last mcrt_scene_upload. */
int mcrt_photon_download_lights(mcrt_ctx* ctx, int which, uint32_t* out, uint64_t n);
/* The reverse-DFA state (mcrt_lpe_compile_photon_host) of each photon of a built map before the event of the vertex
 * where it was stored, out[n] HOST, in mcrt_photon_download's order; n must be the map's photon count. Only maps emitted
 * by mcrt_photon_emit / _emit_pass while an LPE table the photon mapper takes was set carry them (else
 * MCRT_ERR_UNSUPPORTED). A photon whose state is MCRT_LPE_DEAD is still stored: it counts for every estimate's radius. */
int mcrt_photon_download_lpe_states(mcrt_ctx* ctx, int which, uint32_t* out, uint64_t n);

/* The octree construction step of mcrt_photon_emit alone, on caller photons: Octree<Photon>
 * insertion + LinearOctree::compact (octree.cpp:34-81, linear-octree.cpp:201-244) on the GPU.
 * photons: HOST, [n][8] floats {flux.xyz, pos.xyz, phi, theta} (copied to the device); the result
 * (same octants as the reference's LinearOctree; photons of a leaf in input order) is copied back:
 * *out points into host memory owned by *handle, release it with mcrt_octree_free. */
int mcrt_octree_build(mcrt_ctx* ctx, const float* photons, uint64_t n, uint32_t max_photons_per_octree_leaf,
                      const double* scene_bounds6, void** handle, mcrt_photon_map_desc* out, double* gpu_ms);
void mcrt_octree_free(void* handle);

/* SURVEY.md §8f-3 ("next"): scene ingest. Scene::parseOBJ (source/scene/scene.cpp:238-324) as a
 * parallel mmap-based reader with identical results: "v" / "vn" lines and the first three corners
 * of every "f" line, zero-based (idx - 1 in size_t arithmetic). tri_vt / tri_vn hold only the faces
 * whose three corners all carry that index, exactly as the reference's separate lists do. Host
 * code, no GPU involved. *out points into memory owned by *handle (mcrt_obj_free). A missing file
 * or a negative index (the reference prints / throws) returns MCRT_ERR_INVALID with the message. */
typedef struct mcrt_obj_mesh {
    uint64_t n_vertices, n_normals, n_tri_v, n_tri_vt, n_tri_vn;
    const double* vertices;     /* [n_vertices][3] */
    const double* normals;      /* [n_normals][3] */
    const uint64_t* tri_v;      /* [n_tri_v][3] */
    const uint64_t* tri_vt;     /* [n_tri_vt][3] */
    const uint64_t* tri_vn;     /* [n_tri_vn][3] */
} mcrt_obj_mesh;
int mcrt_obj_load(const char* path, int threads, void** handle, mcrt_obj_mesh* out, char* err, size_t errlen);
void mcrt_obj_free(void* handle);
/* Scene::generateVertexNormals (scene.cpp:326-355): normalised sum of face normal x area x corner
 * angle over the incident triangles, added in triangle order (bit-identical sums), parallel over
 * vertices. out_normals: [n_vertices][3]. */
int mcrt_obj_vertex_normals(const double* vertices, uint64_t n_vertices, const uint64_t* tri_v, uint64_t n_triangles,
                            int threads, double* out_normals);

/* SURVEY.md §8f-4 ("next", image half): Image::save (source/camera/image.cpp:37-51) without the file:
 * auto exposure (getExposure, image.cpp:63-73: histogram median -> 0.5), tone-mapping operator
 * (pixel-operators.cpp:7-51), auto gain (getGain, image.cpp:78-88: 99th percentile -> 0.99), sRGB
 * gamma (srgb.hpp:54-62) and truncation to bytes in B,G,R order. `params` = the camera's "image"
 * object (image.cpp:10-35). rgb: [height][width][3] float64 as mcrt_render_rows returns it;
 * out_bgr: [height][width][3] bytes = the reference's .tga after its 18-byte header.
 * mcrt_image_tonemap takes HOST buffers, mcrt_image_tonemap_dev DEVICE pointers (e.g. the
 * framebuffer of mcrt_render_rows_dev, so that 6 MB of bytes leave the GPU instead of 50 MB). */
enum { MCRT_TONEMAP_HABLE = 0, MCRT_TONEMAP_ACES = 1, MCRT_TONEMAP_LINEAR = 2 };
typedef struct mcrt_image_params {
    uint32_t plain;                 /* "plain": no tone mapping, no auto exposure / gain */
    uint32_t tonemapper;            /* MCRT_TONEMAP_HABLE (default) | MCRT_TONEMAP_ACES */
    double exposure_scale;          /* 2^exposure_compensation, Image::exposure_scale (image.cpp:21) */
    double gain_scale;              /* 2^gain_compensation, Image::gain_scale (image.cpp:22) */
} mcrt_image_params;
int mcrt_image_tonemap(mcrt_ctx* ctx, const double* rgb, uint32_t width, uint32_t height, const mcrt_image_params* params,
                       uint8_t* out_bgr, double* exposure_factor, double* gain_factor);
int mcrt_image_tonemap_dev(mcrt_ctx* ctx, const double* rgb_dev, uint32_t width, uint32_t height,
                           const mcrt_image_params* params, uint8_t* out_bgr_dev, double* exposure_factor, double* gain_factor);

/* SURVEY.md §8f-2 ("next"): BVH construction on the GPU. Replaces BVH::BVH (source/bvh/bvh.cpp:13-78):
 * the binned-SAH builders recursiveBuildBinarySAH / recursiveBuildQuaternarySAH (bvh.cpp:165-432),
 * the octree-derived hierarchy (bvh.cpp:130-163, octree.cpp:34-81), arbitrarySplit and compact
 * (bvh.cpp:434-474). The result is the reference's tree node for node (same boxes, same
 * depth-first order, same ordered_surfaces), because every decision of those builders depends
 * only on counts and min/max unions.
 *   prim_bounds   [n_prims][6] = Surface::Base::BB() {min.xyz, max.xyz} in Scene::surfaces order
 *   scene_bounds  Scene::BB() (the root box, bvh.cpp:20)
 *   type          the "bvh" object's "type" (bvh.cpp:24-56), bins_per_axis its "bins_per_axis"
 *                 (<= 0: the reference's default, 16 binary / 8 quaternary)
 * *out points into memory owned by *handle (release with mcrt_bvh_free): node arrays in the layout
 * mcrt_scene_desc takes, and prim_order[i] = index into the caller's primitives of ordered
 * primitive i. gpu_ms (optional): device time of the build. */
enum { MCRT_BVH_OCTREE = 0, MCRT_BVH_BINARY_SAH = 1, MCRT_BVH_QUATERNARY_SAH = 2 };
typedef struct mcrt_bvh_desc {
    uint32_t n_nodes, n_prims;
    const double* node_bounds;            /* [n_nodes][6] */
    const uint32_t* node_first_prim;      /* LinearNode::start_surface */
    const uint32_t* node_prim_count;      /* LinearNode::num_surfaces (0 = inner node) */
    const uint32_t* node_next_sibling;    /* LinearNode::next_sibling */
    const uint32_t* prim_order;           /* [n_prims] */
    uint32_t build_rounds, kernel_launches;
} mcrt_bvh_desc;
int mcrt_bvh_build(mcrt_ctx* ctx, const double* prim_bounds, uint32_t n_prims, const double* scene_bounds6, int type,
                   int bins_per_axis, void** handle, mcrt_bvh_desc* out, double* gpu_ms);
void mcrt_bvh_free(void* handle);

/* Replaces Camera::sampleImage (camera.cpp:101-145) for rows [y0, y1) with the default box
 * film (film.cpp:13-17): out_rgb[(y-y0)*W+x][3] = mean over sqrtspp² samples of
 * Integrator::sampleRay, clamped at 0 (film.cpp:112). Sample s of pixel p uses
 * Sampler::initiate(p) / setIndex(s) with `global_seed` (sampler.hpp:30-44,58).
 * out_rgb is a HOST buffer of (y1-y0)*W*3 doubles. */
int mcrt_render_rows(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y0, uint32_t y1,
                     uint32_t sqrtspp, uint32_t global_seed, int integrator_kind,
                     int precision, double* out_rgb, mcrt_stats* stats);

/* Same, but the framebuffer stays resident in HBM (device pointer, doubles); used by the
 * multi-GPU all-gather and by the HBM-resident throughput measurement. */
int mcrt_render_rows_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y0, uint32_t y1,
                         uint32_t sqrtspp, uint32_t global_seed, int integrator_kind,
                         int precision, double* out_rgb_dev, mcrt_stats* stats);

/* Interleaved row sharding for multi-GPU renders (SURVEY.md §8e): renders image rows
 * y_first + k*y_step for k in [0, n_rows) into out_rgb_dev[k*W + x][3] (device pointer). Every
 * rank gets statistically identical rows, so per-rank cost is balanced. */
int mcrt_render_rows_strided_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first,
                                 uint32_t y_step, uint32_t n_rows, uint32_t sqrtspp,
                                 uint32_t global_seed, int integrator_kind, int precision,
                                 double* out_rgb_dev, mcrt_stats* stats);

/* Row-sharded render with the frame exchange fused into the film resolve (SURVEY.md §8e, replaces the NCCL
 * all-gather of the framebuffer): the rows y_first + k*y_step this rank renders are written straight into
 * frames[0..n_frames) - the FULL-frame buffers [height][width][3] of every rank, float32 ("float3
 * framebuffer") or float64 - at their final position. frames[] are device pointers valid on this device:
 * the rank's own buffer from mcrt_frame_alloc and the peers' buffers mapped with mcrt_frame_open (CUDA IPC;
 * the stores cross NVLink). The caller synchronises the ranks (barrier) before reading a frame and before
 * the next render overwrites it. */
int mcrt_render_rows_strided_peers(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first,
                                   uint32_t y_step, uint32_t n_rows, uint32_t sqrtspp,
                                   uint32_t global_seed, int integrator_kind, int precision,
                                   void* const* frames, uint32_t n_frames, int frame_is_float32,
                                   mcrt_stats* stats);
/* Reconstruction filters across row shards (film.cpp:61-79): with a filter set by mcrt_set_film a sample splats
 * into neighbouring rows, so a rank that renders rows y_first + k*y_step accumulates into whole-frame buffers and
 * returns them UNRESOLVED: rgb_sum_dev[height*width][3] and weight_sum_dev[height*width] (device, float64; zeroed
 * first, then accumulated as mcrt_render_accumulate_dev does). The
 * host adds them over the ranks (an all-reduce) and calls mcrt_film_resolve_dev, Film::Splat::get (film.cpp:106-113). */
int mcrt_render_film_sums_strided_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step,
                                      uint32_t n_rows, uint32_t sqrtspp, uint32_t global_seed, int integrator_kind,
                                      int precision, double* rgb_sum_dev, double* weight_sum_dev, mcrt_stats* stats);
int mcrt_film_resolve_dev(mcrt_ctx* ctx, const double* rgb_sum_dev, const double* weight_sum_dev, uint64_t n_pixels,
                          double* out_rgb_dev);

/* Progressive rendering. Sample s of pixel p traces the same path whichever call renders it, so sums over disjoint
 * sample ranges add up to the one-shot frame's sums (up to the order of the float64 film additions).
 * mcrt_render_accumulate_dev adds samples [sample_first, sample_first + sample_count) of every pixel of rows
 * y_first + k*y_step, k < n_rows, into caller-owned device sums (not zeroed, not resolved). Box film:
 * rgb_sum_dev[n_rows*W][3], weight_sum_dev NULL (the weight is the sample count). Reconstruction filter
 * (mcrt_set_film): whole-frame rgb_sum_dev[H*W][3] and weight_sum_dev[H*W]; any set of rows may be accumulated.
 * MCRT_ERR_INVALID: sample_count 0, sample_first + sample_count > 2^32, a weight pointer with the box film or
 * none with a filter, and every argument mcrt_render_rows_strided_dev refuses. */
int mcrt_render_accumulate_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                               uint32_t sample_first, uint32_t sample_count, uint32_t global_seed, int integrator_kind,
                               int precision, double* rgb_sum_dev, double* weight_sum_dev, mcrt_stats* stats);
/* Resolves two sets of sums A and B (a_samples / b_samples samples per pixel) into out_rgb_dev[rows*width][3] =
 * max((A+B)/(wA+wB), 0), with w the sample count (box film, weight pointers NULL) or the weight sums (filter; the
 * pixel is 0 where the weight is 0), and estimates the remaining noise. Per pixel and channel
 * v = (A/wA - B/wB)^2 * nA*nB/(nA+nB)^2, unbiased for the variance of the combined mean if the halves are independent
 * (pixels where a half has zero weight contribute no v). tile_error_dev[ceil(rows/tile)][ceil(width/tile)]
 * (optional) and *frame_error (optional) = sqrt(sum v / sum I^2) over the tile / the frame, I the resolved value;
 * 0 where sum v is 0, +inf where sum I^2 is 0 < sum v. A half may be empty (samples 0, sums NULL): the frame is
 * resolved and every error is +inf. MCRT_ERR_INVALID: tile 0, no samples in either half. */
int mcrt_progressive_resolve_dev(mcrt_ctx* ctx, const double* a_rgb_dev, const double* a_weight_dev, uint64_t a_samples,
                                 const double* b_rgb_dev, const double* b_weight_dev, uint64_t b_samples,
                                 uint32_t width, uint32_t rows, uint32_t tile, double* out_rgb_dev,
                                 double* tile_error_dev, double* frame_error);

/* Adaptive sampling. The n_rows x width grid of a row set is cut into tile x tile blocks (the last row and column of
 * blocks may be smaller); active_tiles (HOST) holds one byte per block, [ceil(n_rows/tile)][ceil(width/tile)],
 * nonzero = active. mcrt_render_accumulate_tiles_dev adds samples [sample_first, sample_first + sample_count) of
 * every pixel of the active blocks into caller-owned sums, exactly as mcrt_render_accumulate_dev does for all pixels
 * (same sums layout; the other pixels' sums are not touched). MCRT_ERR_INVALID: tile 0, a null mask, a mask with no
 * active block, and every argument mcrt_render_accumulate_dev refuses. MCRT_ERR_UNSUPPORTED: a reconstruction filter
 * with a row set other than the whole frame (its splats cross blocks, whose resolve spans the whole frame). */
int mcrt_render_accumulate_tiles_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                                     uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                                     uint32_t global_seed, int integrator_kind, int precision, double* rgb_sum_dev,
                                     double* weight_sum_dev, mcrt_stats* stats);
/* mcrt_progressive_resolve_dev with per-tile sample counts: tile_samples (HOST) [ceil(rows/tile)][ceil(width/tile)][2]
 * = {nA, nB} of each tile's pixels; they set a box-film pixel's weights and every pixel's scale nA*nB/(nA+nB)^2.
 * With a filter, a pixel near a tile border also holds splats of samples of neighbouring tiles, which may have other
 * counts: its own tile's counts in the scale are then an approximation. A tile with an empty half has error +inf,
 * and so does the frame if any tile has one. tile_sums_dev (optional, device) receives {sum v, sum I^2} of each tile,
 * [n_tiles][2]. MCRT_ERR_INVALID: a null tile_samples and every argument mcrt_progressive_resolve_dev refuses (a half
 * "has samples" when any tile has samples in it). */
int mcrt_progressive_resolve_tiles_dev(mcrt_ctx* ctx, const double* a_rgb_dev, const double* a_weight_dev,
                                       const double* b_rgb_dev, const double* b_weight_dev, const uint32_t* tile_samples,
                                       uint32_t width, uint32_t rows, uint32_t tile, double* out_rgb_dev,
                                       double* tile_error_dev, double* tile_sums_dev, double* frame_error);

/* Light groups. Radiance is linear in emittance, so the path tracer can deposit each contribution into the plane of the
 * emitter it comes from, and one render yields every group's share of the frame. mcrt_set_light_groups assigns light l
 * (the scene's l-th light_prim) to group group_of_light[l] < n_groups; plane n_groups holds the sky, so a render has
 * n_groups + 1 planes. group_of_light NULL with n_lights = n_groups = 0 clears the table; a scene without lights sets
 * its sky-only table with any non-NULL pointer and n_lights = n_groups = 0. mcrt_scene_upload clears the table too.
 * MCRT_ERR_NO_SCENE before an upload. MCRT_ERR_INVALID: n_lights other than the scene's light count, an id >= n_groups,
 * n_groups = 2^32 - 1. MCRT_ERR_UNSUPPORTED: an emissive primitive the scene does not list as a light (its
 * contributions would have no group). The other entry points ignore the table. */
int mcrt_set_light_groups(mcrt_ctx* ctx, const uint32_t* group_of_light, uint32_t n_lights, uint32_t n_groups);
/* mcrt_render_accumulate_dev (active_tiles NULL) or mcrt_render_accumulate_tiles_dev (active_tiles HOST, same mask
 * layout) into light-group planes: planes_dev[n_planes][n_rows*W][3], plane g the sums of group g's lights and plane
 * n_groups the sky's. Every contribution lands in exactly one plane, so the planes add up to the sums of the one-plane
 * entry points over the same samples; the box film's weight is the sample count. The photon mapper splits its photon
 * estimates by the light each photon came from, so it needs maps that carry light indices (mcrt_photon_download_lights);
 * the photon mapper adds no sky, so its sky plane stays zero. MCRT_ERR_INVALID: no group table, n_planes !=
 * n_groups + 1, a null planes_dev, and every argument the one-plane entry points refuse. MCRT_ERR_UNSUPPORTED: a
 * reconstruction filter, the photon mapper with maps that carry no light index (or with no maps). Nothing is written
 * when a call is refused. */
int mcrt_render_accumulate_groups_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                                      uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                                      uint32_t global_seed, int integrator_kind, int precision, double* planes_dev,
                                      uint32_t n_planes, mcrt_stats* stats);
/* Relighting: out_dev[i] = sum over g = 0, 1, ... n_planes - 1 of weights[g][i % 3] * planes_dev[g * n_values + i]
 * (weights HOST [n_planes][3]; each product rounded, then added, in order of g, in float64). On unresolved sums the
 * result is the sums of the scene with group g's emittance scaled by weights[g] (plane n_planes - 1: the sky), and
 * feeds mcrt_progressive_resolve[_tiles]_dev and mcrt_denoise_dev as they are. out_dev must not overlap planes_dev.
 * MCRT_ERR_INVALID: null pointers, n_planes 0, n_values not a multiple of 3. The function is a plain weighted sum of
 * planes, so it recombines the light-path AOV planes of mcrt_render_accumulate_aovs_dev the same way. */
int mcrt_light_groups_combine_dev(mcrt_ctx* ctx, const double* planes_dev, uint32_t n_planes, uint64_t n_values,
                                  const double* weights, double* out_dev);

/* Light-path AOVs: the path tracer's contributions split by the kind of scattering they come through. The reference's
 * material model picks exactly one interaction type (reflection, refraction or diffuse) per vertex, and next-event
 * estimation and BSDF sampling at that vertex both use it, so "the lobe of the first scattering vertex" (the camera ray's
 * hit) is one value per path. A contribution is direct when its light path has exactly one scattering vertex: light
 * sampled from the first vertex, or the sky or an emitter reached by the ray leaving it; every later contribution is
 * indirect.
 *   plane 0 MCRT_AOV_BACKGROUND                the sky seen by the camera ray (it hits nothing)
 *   plane 1 MCRT_AOV_EMISSION                  an emitter seen by the camera ray
 *   plane 2 / 3 MCRT_AOV_DIFFUSE_DIRECT / _INDIRECT            the first vertex scattered diffusely
 *   plane 4 / 5 MCRT_AOV_REFLECTION_DIRECT / _INDIRECT         ... reflected: mirrors, conductors, GGX, the Fresnel
 *                                                              reflection of dielectric and coated materials
 *   plane 6 / 7 MCRT_AOV_TRANSMISSION_DIRECT / _INDIRECT       ... refracted
 * Every contribution lands in exactly one plane, so the planes add up to the beauty sums. */
enum {
    MCRT_AOV_BACKGROUND = 0, MCRT_AOV_EMISSION = 1, MCRT_AOV_DIFFUSE_DIRECT = 2, MCRT_AOV_DIFFUSE_INDIRECT = 3,
    MCRT_AOV_REFLECTION_DIRECT = 4, MCRT_AOV_REFLECTION_INDIRECT = 5, MCRT_AOV_TRANSMISSION_DIRECT = 6,
    MCRT_AOV_TRANSMISSION_INDIRECT = 7, MCRT_AOV_COUNT = 8
};
/* mcrt_render_accumulate_dev (active_tiles NULL) or mcrt_render_accumulate_tiles_dev (active_tiles HOST, same mask
 * layout) into the AOV planes planes_dev[MCRT_AOV_COUNT][n_rows*W][3] (path tracer, box film; the box film's weight is
 * the sample count). The planes add up to the sums of the one-plane entry points over the same samples, and
 * mcrt_light_groups_combine_dev, mcrt_progressive_resolve[_tiles]_dev and mcrt_denoise_dev take them or their weighted
 * sums. MCRT_ERR_INVALID: n_planes != MCRT_AOV_COUNT, a null planes_dev, and every argument the one-plane entry points
 * refuse. MCRT_ERR_UNSUPPORTED: a reconstruction filter, the photon mapper. Nothing is written when a call is refused.
 * The light-group table plays no part here, and the other entry points write no AOVs. */
int mcrt_render_accumulate_aovs_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                                    uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                                    uint32_t global_seed, int integrator_kind, int precision, double* planes_dev,
                                    uint32_t n_planes, mcrt_stats* stats);

/* Photon-mapper components: the photon mapper's contributions split by the estimator that made them. Its sampleRay
 * (photon-mapper.cpp:299-332) deposits at exactly one of four kinds of site, so every deposit lands in one plane:
 *   plane 0 MCRT_PM_EMISSION   an emitter seen from the camera, directly or through an unbroken chain of delta bounces
 *   plane 1 MCRT_PM_DIRECT     Monte Carlo direct light: next-event estimation and the BSDF-sampled emitter hit it is
 *                              combined with by MIS (an emitter hit after the first non-delta vertex)
 *   plane 2 MCRT_PM_CAUSTIC    every caustic-map density estimate
 *   plane 3 MCRT_PM_GLOBAL     every global-map density estimate
 * No estimate is split inside itself: each query deposits its whole estimate into one plane, so the planes add up to
 * the one-plane sums up to the order of the float64 film additions. The photon mapper adds no sky, so there is no
 * background plane. With direct_visualization the first non-delta vertex queries both maps and the path ends there: the
 * direct plane stays zero and no shadow ray is traced. */
enum {
    MCRT_PM_EMISSION = 0, MCRT_PM_DIRECT = 1, MCRT_PM_CAUSTIC = 2, MCRT_PM_GLOBAL = 3, MCRT_PM_COMPONENT_COUNT = 4
};
/* mcrt_render_accumulate_dev (active_tiles NULL) or mcrt_render_accumulate_tiles_dev (active_tiles HOST, same mask
 * layout) into the component planes planes_dev[MCRT_PM_COMPONENT_COUNT][n_rows*W][3] (photon mapper, box film; the box
 * film's weight is the sample count). Any photon maps serve: those of mcrt_photon_upload, mcrt_photon_emit[_pass] and
 * mcrt_photon_build_dev. mcrt_light_groups_combine_dev, mcrt_progressive_resolve[_tiles]_dev and mcrt_denoise_dev take
 * the planes or their weighted sums. MCRT_ERR_UNSUPPORTED: the path tracer (it has light-path AOVs instead), a
 * reconstruction filter. MCRT_ERR_INVALID: an integrator kind outside MCRT_INTEGRATOR_*, n_planes !=
 * MCRT_PM_COMPONENT_COUNT, a null planes_dev, and every argument the one-plane entry points refuse. MCRT_ERR_NO_PHOTONS: no photon maps, as the one-plane photon render. Nothing is
 * written when a call is refused. The light-group table plays no part here. */
int mcrt_render_accumulate_photon_components_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step,
                                                 uint32_t n_rows, uint32_t tile, const uint8_t* active_tiles,
                                                 uint32_t sample_first, uint32_t sample_count, uint32_t global_seed,
                                                 int integrator_kind, int precision, double* planes_dev, uint32_t n_planes,
                                                 mcrt_stats* stats);

/* Light path expressions (LPEs): film planes chosen by regular expressions over each path-tracer contribution's event
 * string. The string is C (the camera), then the event of each scattering vertex before the contribution, then its
 * source: L for an emitter (hit, or sampled by next-event estimation at the last vertex), L'g' for an emitter whose
 * light is in group g of the mcrt_set_light_groups table, B for the sky. Vertex events are <RD> (diffuse), <RS> / <RG>
 * (reflection, smooth / rough: GGX and rough dielectrics), <TS> / <TG> (refraction, smooth / rough).
 * Syntax (a subset of OSL's, anchored to the whole string, whitespace ignored): the events above, <XY> with X in {R,T,.}
 * and Y in {D,G,S,.}, the shorthands D = <.D>, G = <.G>, S = <.S>, R = <R.>, T = <T.>, '.' for any one event, sets
 * [...] and [^...] of events, ( ), |, and the repetitions * + ? {n} {n,} {n,m} (n, m <= 1000). '.' matches L and B
 * too: the indirect diffuse light is C<RD>.+[LB], while C<RD>.+ also takes the direct C<RD>L and C<RD>B.
 * The compiled union is a DFA: state 0 follows C, a state from which no expression can match any more is
 * MCRT_LPE_DEAD, and every state carries a 32-bit accept mask, bit i for expression i. Symbols are the MCRT_LPE_SYM_*
 * events, then one per distinct label (ascending group index); the lights of every unlabelled group read
 * MCRT_LPE_SYM_L, which L matches together with every label. */
enum {
    MCRT_LPE_SYM_RD = 0, MCRT_LPE_SYM_RS = 1, MCRT_LPE_SYM_RG = 2, MCRT_LPE_SYM_TS = 3, MCRT_LPE_SYM_TG = 4,
    MCRT_LPE_SYM_B = 5, MCRT_LPE_SYM_L = 6, MCRT_LPE_SYM_LABEL0 = 7,
    MCRT_LPE_MAX_EXPRESSIONS = 32, MCRT_LPE_MAX_LABELS = 64, MCRT_LPE_MAX_STATES = 255, MCRT_LPE_DEAD = 255,
    MCRT_LPE_MAX_SYMBOLS = MCRT_LPE_SYM_LABEL0 + MCRT_LPE_MAX_LABELS
};
/* Compiles exprs[n] and uploads the tables; exprs NULL with n = 0 clears them. Labels need the light-group table
 * (mcrt_set_light_groups) and a group index below its n_groups; mcrt_set_light_groups and mcrt_scene_upload clear the
 * LPE table. MCRT_ERR_NO_SCENE before an upload. MCRT_ERR_INVALID: a syntax error (the message names the expression and
 * the character offset), n > MCRT_LPE_MAX_EXPRESSIONS, more than MCRT_LPE_MAX_LABELS distinct labels, an unknown label.
 * MCRT_ERR_UNSUPPORTED: more than MCRT_LPE_MAX_STATES live states. A refused call leaves no table. */
int mcrt_set_light_path_expressions(mcrt_ctx* ctx, const char* const* exprs, uint32_t n);
/* mcrt_render_accumulate_dev (active_tiles NULL) or mcrt_render_accumulate_tiles_dev (active_tiles HOST, same mask
 * layout) into planes_dev[n][n_rows*W][3], plane i the sums of the contributions whose event string expression i
 * matches (path tracer, box film; the box film's weight is the sample count). Planes may overlap, or leave a
 * contribution out; a path ends at the vertex where its state becomes MCRT_LPE_DEAD, and next-event estimation that no
 * expression accepts traces no shadow ray, so every plane keeps its value while fewer rays are traced.
 * MCRT_ERR_INVALID: no LPE table, n_planes other than its expression count, a null planes_dev, and every argument the
 * one-plane entry points refuse. MCRT_ERR_UNSUPPORTED: a reconstruction filter. Nothing is written when a call is
 * refused. The other entry points ignore the table.
 * The photon mapper (integrator_kind MCRT_INTEGRATOR_PHOTON) gives every photon term of its k-NN or gather estimates a
 * string of its own: C, the camera's events up to the gather vertex x, x's event, then the photon's events from the one
 * before x back to its first bounce (e_m .. e_1), then its light, C c1..ck x e_m..e_1 L'g'. Emitter hits and next-event
 * estimation read as the path tracer's. Expressions select which terms land in a plane; they change neither the photons
 * an estimate finds nor the radius it is normalised by. A camera path whose every possible photon term no expression
 * accepts issues no k-NN query. The photon mapper needs maps emitted by mcrt_photon_emit / _emit_pass while this same
 * table (same expressions, groups and light symbols) was set; the first refusal, MCRT_ERR_UNSUPPORTED, is of any other
 * maps (none, mcrt_photon_upload, mcrt_photon_build_dev, no or another table, before the last mcrt_scene_upload), the
 * second, MCRT_ERR_UNSUPPORTED, of a table whose reversed expressions need more than MCRT_LPE_MAX_STATES states. */
int mcrt_render_accumulate_lpe_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                                   uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                                   uint32_t global_seed, int integrator_kind, int precision, double* planes_dev,
                                   uint32_t n_planes, mcrt_stats* stats);
/* Test hook (host only, no CUDA call): the tables mcrt_set_light_path_expressions would upload, with labels below
 * n_groups. next[MCRT_LPE_MAX_STATES * MCRT_LPE_MAX_SYMBOLS] receives [*n_states][*n_symbols], accept[256] the accept
 * masks (accept[MCRT_LPE_DEAD] = 0), group_symbol[n_groups] (NULL when n_groups is 0) the symbol of each group's
 * lights. error[error_capacity] receives the reason of a refusal (or ""). Returns what mcrt_set_light_path_expressions
 * would. */
int mcrt_lpe_compile_host(const char* const* exprs, uint32_t n, uint32_t n_groups, uint8_t* next, uint32_t* accept,
                          uint8_t* group_symbol, uint32_t* n_states, uint32_t* n_symbols, char* error, uint32_t error_capacity);
/* Test hook (host only, no CUDA call): the photon mapper's side of the same tables. rev_next[MCRT_LPE_MAX_STATES *
 * MCRT_LPE_MAX_SYMBOLS] receives [*rev_n_states][n_symbols], the DFA of the reversed expressions, which reads a
 * photon's events in emission order (its light's symbol first) from *rev_start (MCRT_LPE_DEAD when nothing can match);
 * join[MCRT_LPE_MAX_STATES * MCRT_LPE_MAX_STATES] receives [n_states][*rev_n_states], the accept mask of a contribution
 * whose camera prefix ends in forward state s and whose photon history ends in reverse state r. Returns what
 * mcrt_lpe_compile_host would, or MCRT_ERR_UNSUPPORTED, with the reason in error, when the path tracer would take the
 * table and the photon mapper would refuse it. */
int mcrt_lpe_compile_photon_host(const char* const* exprs, uint32_t n, uint32_t n_groups, uint8_t* rev_next, uint32_t* rev_start,
                                 uint32_t* rev_n_states, uint32_t* join, char* error, uint32_t error_capacity);

/* Denoising a progressive frame (mcrt_denoise_dev) needs per-pixel guides: the first hits of the camera rays of samples
 * [sample_first, sample_first + sample_count) of every pixel of the whole width x height frame add
 * {albedo.rgb, shading normal.xyz, t, 1} per hit into features_dev [height*width][8] (device, float64); a miss adds
 * nothing. Albedo is the specular reflectance of perfect mirrors and complex-IOR materials, the reflectance of every
 * other material; the shading normal faces the ray. The sums are added to, never zeroed; each pixel adds its samples
 * in increasing order, so consecutive ranges accumulate bit-identically to their union. The guides are per pixel
 * (a box footprint) whatever film is set, and depend on the scene, camera, seed and sample range only.
 * MCRT_ERR_INVALID: a null camera or buffer, sample_count 0, sample_first + sample_count > 2^32, an empty frame or
 * more than 2^32 pixels, an unknown precision. MCRT_ERR_NO_SCENE before mcrt_scene_upload. */
int mcrt_render_features_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t sample_first, uint32_t sample_count,
                             uint32_t global_seed, int precision, double* features_dev, mcrt_stats* stats);

#define MCRT_FEATURES_MAX_SPECULAR_DEPTH 7

/* mcrt_render_features_dev with the guides taken after perfectly specular bounces, so glass and mirrors are guided by
 * what they show. Each sample follows its own path, exactly as the path tracer traces it (same sampler dimensions,
 * IOR history, ray offsets), with throughput T = prod f/pdf and distance L = sum t. A hit on a material without
 * dirac_delta, the hit at depth specular_depth, or a hit whose sampled bounce is rejected or leaves T at 0 is the end
 * vertex; it adds {T * albedo, shading normal, L + t, 1} with mcrt_render_features_dev's albedo and normal. A miss
 * anywhere on the chain adds nothing. No Russian roulette: a pure delta chain this short would not roulette. At
 * specular_depth 0 the sums are mcrt_render_features_dev's bit for bit; accumulation, order and determinism are the
 * same. Refuses everything mcrt_render_features_dev refuses, and specular_depth > MCRT_FEATURES_MAX_SPECULAR_DEPTH
 * (MCRT_ERR_INVALID); a refused call launches nothing. */
int mcrt_render_features_chain_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t sample_first, uint32_t sample_count,
                                   uint32_t global_seed, int precision, uint32_t specular_depth, double* features_dev,
                                   mcrt_stats* stats);

/* Parameters of mcrt_denoise_dev; a NULL pointer selects the MCRT_DENOISE_DEFAULT_* values. */
typedef struct mcrt_denoise_params {
    uint32_t iterations;   /* 0..10 a-trous passes of steps 1, 2, 4, ...; 0 = the two halves' plain resolve */
    uint32_t _pad;
    double sigma_color, sigma_normal, sigma_depth, sigma_albedo;   /* >= 0, finite; 0 switches the term off */
} mcrt_denoise_params;

#define MCRT_DENOISE_MAX_ITERATIONS 10
#define MCRT_DENOISE_DEFAULT_ITERATIONS 5
#define MCRT_DENOISE_DEFAULT_SIGMA_COLOR 1.0
#define MCRT_DENOISE_DEFAULT_SIGMA_NORMAL 64.0
#define MCRT_DENOISE_DEFAULT_SIGMA_DEPTH 0.1
#define MCRT_DENOISE_DEFAULT_SIGMA_ALBEDO 0.1

/* Cross-filtered a-trous denoiser over the two halves of a progressive frame (whole frame, float64). The sums and
 * weights are those mcrt_progressive_resolve_tiles_dev takes, with tile_samples (HOST) {nA, nB}[n_tiles] (uniform
 * renders pass equal counts); features_dev are mcrt_render_features_dev's sums. Each half is filtered with edge-stopping
 * weights from the guides (normal, relative depth, albedo) and a colour term measured on the other half, so the
 * difference of the filtered halves still estimates the residual noise: out_rgb_dev [height*width][3] receives
 * max(0, (wA A' + wB B') / (wA + wB)) and *frame_error sqrt(sum v' / sum out^2) with v' = sum_c (A' - B')^2 wA wB /
 * (wA + wB)^2 (0 if sum v' = 0, +inf if sum out^2 = 0 < sum v'). A pixel with zero weight in a half is output as its
 * plain resolve. Device buffers except tile_samples, params and frame_error. MCRT_ERR_INVALID: a null buffer, an
 * empty frame or more than 2^32 pixels, tile 0, a tile with an empty half, weight sums given for one half only,
 * iterations > MCRT_DENOISE_MAX_ITERATIONS, a negative or non-finite sigma. */
int mcrt_denoise_dev(mcrt_ctx* ctx, const double* a_rgb_dev, const double* a_weight_dev,
                     const double* b_rgb_dev, const double* b_weight_dev, const uint32_t* tile_samples,
                     uint32_t tile, const double* features_dev, uint32_t width, uint32_t height,
                     const mcrt_denoise_params* params, double* out_rgb_dev, double* frame_error);

/* Denoising film planes (light groups, AOVs, components, LPE planes; box film, whole frame): every plane is filtered with
 * the edge weights mcrt_denoise_dev computes for the guide frame, the box-film half sums a_rgb_dev / b_rgb_dev. The
 * filter is linear once its weights are fixed, so planes that sum to the guide give filtered sums that sum to the
 * guide's, up to rounding. a_planes_dev / b_planes_dev [n_planes][height*width][3] are each half's plane sums;
 * a_out_planes_dev / b_out_planes_dev (same layout) receive the filtered sums, unresolved, which
 * mcrt_progressive_resolve[_tiles]_dev resolves (with its residual-noise estimate) and mcrt_light_groups_combine_dev
 * recomposites; a pixel with an empty half keeps its input sums. out_rgb_dev and frame_error (optional, given together
 * or not at all) receive exactly what mcrt_denoise_dev writes for the guide. Scratch: 400 B per pixel plus 48 B per
 * pixel per plane, kept by the context. MCRT_ERR_INVALID, writing nothing: every argument mcrt_denoise_dev refuses,
 * n_planes 0, an output buffer that overlaps an input or another output, out_rgb_dev without frame_error or the
 * reverse. */
int mcrt_denoise_planes_dev(mcrt_ctx* ctx, const double* a_rgb_dev, const double* b_rgb_dev,
                            const double* a_planes_dev, const double* b_planes_dev, uint32_t n_planes,
                            const uint32_t* tile_samples, uint32_t tile, const double* features_dev,
                            uint32_t width, uint32_t height, const mcrt_denoise_params* params,
                            double* a_out_planes_dev, double* b_out_planes_dev,
                            double* out_rgb_dev, double* frame_error);

/* A device buffer that other processes on the node can map: *dev_ptr (zero-filled) and its 64-byte CUDA IPC
 * handle, to be sent to the peers by whatever channel the host uses (torch.distributed in this repository). */
int mcrt_frame_alloc(mcrt_ctx* ctx, uint64_t bytes, void** dev_ptr, unsigned char ipc_handle[64]);
int mcrt_frame_open(mcrt_ctx* ctx, const unsigned char ipc_handle[64], void** dev_ptr);
int mcrt_frame_close(mcrt_ctx* ctx, void* peer_ptr);
int mcrt_frame_free(mcrt_ctx* ctx, void* dev_ptr);

/* Test hook (host only, no CUDA call): the 4-wide float-box BVH mcrt_scene_upload derives from the scene's tree for the
 * order-free closest-hit search (csrc/bvh4.cuh). nodes128: n_nodes records of 128 bytes {float lo[3][4], hi[3][4];
 * uint32 child[4], pad[4]}; child = 0 empty | inner node index | 0x80000000 | first_prim << 8 | count. max_leaf: 0 keeps the
 * reference's leaves, n cuts larger leaves into runs of n, 0xFFFFFFFF = the upload's own rule. */
int mcrt_bvh4_host(const mcrt_scene_desc* scene, uint32_t max_leaf, void** handle, const void** nodes128, uint32_t* n_nodes);
void mcrt_bvh4_host_free(void* handle);

/* Test hook (host only, no CUDA call): the 4-wide BVH with spatial splits that mcrt_scene_upload builds for small scenes
 * (option bvh4_split). Nodes as mcrt_bvh4_host's, but a leaf's first / count index refs[], the ordered primitive of each
 * reference; a primitive cut by a spatial split has several references. node_cost: cost of a node visit in primitive
 * tests; ref_budget: references per primitive at most (>= 1). */
int mcrt_bvh4_split_host(const mcrt_scene_desc* scene, double node_cost, double ref_budget, void** handle, const void** nodes128,
                         uint32_t* n_nodes, const uint32_t** refs, uint32_t* n_refs);
void mcrt_bvh4_split_host_free(void* handle);

/* Measured FP64 issue rate of this GPU (independent DFMA chains on every SM), thread-instructions per second:
 * the denominator of bench.py's FP64 roofline for the float64 kernels. */
int mcrt_fp64_peak(mcrt_ctx* ctx, double* dfma_per_second);

/* Batched Scene::intersect (scene.cpp:151-176): closest hit per ray. `medium_ior` is not
 * needed by the query. Host buffers. */
int mcrt_trace_closest(mcrt_ctx* ctx, const mcrt_ray* rays, size_t n, int precision,
                       mcrt_hit* hits, mcrt_stats* stats);

/* Batched Integrator::sampleRay (integrator.hpp:20): ray i is traced as sample `sample[i]`
 * of pixel `pixel[i]` (the sampler state the reference keeps thread_local), medium = scene
 * ior; out_rgb[i][3] receives the radiance estimate. Host buffers. */
int mcrt_sample_rays(mcrt_ctx* ctx, const mcrt_ray* rays, const uint32_t* pixel,
                     const uint32_t* sample, size_t n, uint32_t global_seed,
                     int integrator_kind, int precision, double* out_rgb, mcrt_stats* stats);

/* Test hook for the Owen-scrambled Sobol sampler (sampler.hpp:13-91): for each i, after
 * initiate(pixel[i]), setIndex(sample[i]) and `n_shuffles` calls of shuffle(), writes the
 * seven dimensions get<0,7>() as raw uint32 (before the 2^-32 scaling). Host buffers. */
int mcrt_sampler_stream(mcrt_ctx* ctx, const uint32_t* pixel, const uint32_t* sample, size_t n,
                        uint32_t n_shuffles, uint32_t global_seed, uint32_t* out_u32x7);

/* Batched LinearOctree<Photon>::knnSearch (linear-octree.cpp:24-117) on the uploaded map
 * (which: 0 caustic, 1 global). out_index[i][k] photon indices (ordered_data order, unsorted,
 * 0xFFFFFFFF padded), out_dist2[i][k]; out_count[i] results found. Host buffers. */
int mcrt_knn_search(mcrt_ctx* ctx, int which, const double* points_xyz, size_t n,
                    uint32_t* out_index, double* out_dist2, uint32_t* out_count,
                    mcrt_stats* stats);

/* Tunables (pool size etc.); unknown keys return MCRT_ERR_INVALID. */
int mcrt_set_option(mcrt_ctx* ctx, const char* key, double value);

#ifdef __cplusplus
}
#endif
#endif /* MCRT_ABI_H */
