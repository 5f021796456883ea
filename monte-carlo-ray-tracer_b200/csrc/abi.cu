// C ABI of the H100 path-tracing integrator (include/mcrt_abi.h): context, scene upload (derives
// the float64 parity layout and the float32 wide-node layout from the flattened reference scene),
// the wavefront render loop and the batched sampleRay / Scene::intersect / sampler entry points.
// There is deliberately no CPU fallback: without a CUDA device every entry point fails.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "mcrt_abi.h"
#include "launch.h"
#include "bvh_build.h"
#include "image.h"
#include "denoise.h"
#include "lpe.h"

using namespace mcrt;

// internal "integrator" of runWavefront: the photon emission pass (not an ABI value)
static const int MCRT_INTERNAL_EMIT = 100;

#define CK(call)                                                                              \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess)                                                                \
        {                                                                                     \
            ctx->error = std::string(#call) + ": " + cudaGetErrorString(e_);                  \
            return MCRT_ERR_CUDA;                                                             \
        }                                                                                     \
    } while (0)

namespace
{
    template <class R> struct SceneArrays
    {
        std::vector<WideChild<R>> wide;
        std::vector<V4<R>> geom;
        std::vector<PrimShade<R>> shade;
        std::vector<V4<R>> vnormals;
        std::vector<Quadric<R>> quadrics;
        std::vector<Material<R>> materials;
        std::vector<Light<R>> lights;
        DeviceScene<R> dev;
    };

    template <class R> struct WaveBuffers
    {
        PathBuffer<R> buf[2];
        ShadowRecord<R>* shadow = nullptr;
        V4<R>* hits = nullptr;
        uint32_t capacity = 0;
    };
}

struct mcrt_ctx
{
    int device = 0;
    int sm_count = 132;   // H100 SXM; mcrt_init reads the device's own count
    cudaStream_t stream = nullptr;
    std::string error;

    bool has_scene = false;
    std::vector<void*> scene_allocs;
    DeviceScene<double> scene64;
    DeviceScene<float> scene32;
    float scene_scale = 1.0f;
    uint32_t n_bvh4_nodes = 0;
    uint32_t bvh4_max_leaf = 0xFFFFFFFFu;   // auto; 0: keep the reference's leaves; n: cut larger leaves into runs of n (option / MCRT_BVH4_MAX_LEAF)
    int dynamic_fetch = -1;       // -1 auto (scenes with >= 2048 BVH4 nodes without spatial splits), 0 off, 1 on
    int bvh4_split = -1;          // BVH4 with spatial splits (buildBvh4Split): -1 auto (below 4096 primitives, leaves cut by the auto rule), 0 off, 1 on
    double bvh4_split_cost = 0.5; // buildBvh4Split's node cost in primitive tests (MCRT_BVH4_SPLIT_COST)
    PeerFrames peer_out{};   // n_frames != 0: the next resolve writes into these frames (mcrt_render_rows_strided_peers)
    int exact_traversal = 0;   // 1: every ray takes the reference-order replay (traverseReferenceOrder)

    WaveBuffers<double> wave64;
    WaveBuffers<float> wave32;
    std::vector<void*> wave_allocs64, wave_allocs32;

    uint32_t* d_sobol_bytes = nullptr;
    Counters* d_counters = nullptr;
    Counters* h_counters = nullptr; // pinned, 2 slots
    double* d_film = nullptr;
    size_t film_values = 0;
    // reconstruction filter (mcrt_set_film); the default box film needs none of this
    bool film_default = true;
    mcrt_film film = {MCRT_FILM_BOX, 0u, 0.5};
    double* d_film_wsum = nullptr;
    size_t film_wsum_values = 0;
    double* d_film_cache = nullptr;
    double* d_host_out = nullptr;      // staging of mcrt_render_rows (host-buffer entry point)
    size_t host_out_values = 0;
    double* d_resolve_scratch = nullptr;   // per-tile noise sums of mcrt_progressive_resolve_dev (grow-only)
    size_t resolve_scratch_values = 0;
    double* d_denoise_scratch = nullptr;   // state, guides, tile counts and sums of mcrt_denoise_dev (grow-only)
    size_t denoise_scratch_values = 0;
    double* d_denoise_planes_scratch = nullptr;   // tap weights and plane states of mcrt_denoise_planes_dev (grow-only)
    size_t denoise_planes_scratch_values = 0;
    uint32_t* d_pixel_list = nullptr;      // pixels of the active tiles of mcrt_render_accumulate_tiles_dev (grow-only)
    size_t pixel_list_values = 0;
    std::vector<uint32_t> h_pixel_list;
    // light groups (mcrt_set_light_groups); mcrt_scene_upload clears them
    bool has_light_groups = false;
    bool emissive_unlit = false;            // the scene has an emissive primitive that is not one of its lights
    uint32_t n_light_groups = 0;
    uint32_t* d_group_of_light = nullptr;   // [n_lights] (grow-only)
    size_t group_of_light_values = 0;
    double* d_group_weights = nullptr;      // [n_planes][3] of mcrt_light_groups_combine_dev (grow-only)
    size_t group_weight_values = 0;
    std::vector<uint32_t> h_group_of_light; // host copy of the table, for the LPE light symbols
    // light path expressions (mcrt_set_light_path_expressions); mcrt_scene_upload and mcrt_set_light_groups clear them
    uint32_t lpe_n = 0;                     // expressions = planes of an LPE render; 0: no table
    uint32_t lpe_symbols = 0;
    uint8_t* d_lpe_next = nullptr;          // [MCRT_LPE_MAX_STATES][MCRT_LPE_MAX_SYMBOLS] at most, [states][lpe_symbols] used
    uint32_t* d_lpe_accept = nullptr;       // [256]
    uint8_t* d_lpe_light_symbol = nullptr;  // [n_lights] (grow-only)
    size_t lpe_light_values = 0;
    // the photon mapper's side of the table (lpe.h): reversed expressions' DFA, join with the forward states
    uint8_t* d_lpe_rev_next = nullptr;      // [MCRT_LPE_MAX_STATES][MCRT_LPE_MAX_SYMBOLS] at most, [states][lpe_symbols] used
    uint32_t* d_lpe_join = nullptr;         // [MCRT_LPE_MAX_STATES][MCRT_LPE_MAX_STATES] at most, [states][lpe_rev_states] used
    uint8_t* d_lpe_join_any = nullptr;      // [256]
    uint32_t lpe_rev_states = 0, lpe_rev_start = MCRT_LPE_DEAD;
    std::string lpe_photon_error;           // non-empty: the photon mapper refuses the table, for this reason
    // the table's content (every compiled array and the lights' symbols): maps emitted under a table carry its identity,
    // so that setting the same expressions and groups again keeps them valid
    std::string lpe_identity;
    cudaEvent_t ev_start = nullptr, ev_stop = nullptr, ev_poll[2] = { nullptr, nullptr };

    // photon maps (PhotonMapper::caustic_map / global_map) + k-NN query queues
    bool has_photons = false;
    std::vector<void*> photon_allocs;
    DevicePhotonMap photon_map[2];
    uint32_t k_nearest = 0, direct_visualization = 0;
    // maps built by mcrt_photon_emit (host copies, also what mcrt_photon_download returns)
    struct HostPhotonMap
    {
        std::vector<double> octant_bounds;
        std::vector<uint64_t> octant_start, octant_count;
        std::vector<uint32_t> octant_next;
        std::vector<uint8_t> octant_leaf;
        std::vector<float> photons;
    } built_map[2];
    bool built_valid = false;
    // the uploaded maps carry the emitting light of each photon (maps of mcrt_photon_emit / _emit_pass), even when a map
    // holds no photon; maps of mcrt_photon_upload and mcrt_photon_build_dev do not
    bool photon_lights = false;
    // the identity (lpe_identity) of the LPE table the maps were emitted under, empty without one; photon_lpe_states: the
    // maps carry each photon's reverse-DFA state (the table was one the photon mapper takes)
    std::string photon_lpe_identity;
    bool photon_lpe_states = false;
    // maps built on the device by mcrt_photon_emit / mcrt_octree_build; host copies are made on demand
    PhotonOctreeDevice built_dev[2];
    bool built_host_current[2] = { false, false };
    double photon_build_ms = 0.0;
    // emission pass inputs (device), set by mcrt_photon_emit around runWavefront
    const unsigned long long* d_emit_offsets = nullptr;
    const void* d_emit_flux = nullptr;
    float4* d_emit_photons[2] = { nullptr, nullptr };
    uint32_t* d_emit_lights[2] = { nullptr, nullptr };   // the emitting light of each photon of d_emit_photons
    uint32_t* d_emit_lpe_states[2] = { nullptr, nullptr };   // ... and its reverse-DFA state (emission under an LPE table)
    unsigned long long emit_capacity[2] = { 0, 0 };
    std::vector<void*> emit_allocs;          // emission buffers (kept until the next emission / mcrt_destroy)
    unsigned long long emit_stored[2] = { 0, 0 };
    unsigned long long emit_work_first = 0;   // first emission index of the range being emitted (mcrt_photon_emit_range)
    uint32_t emit_pass = 0;                   // photon pass being emitted (mcrt_photon_emit_pass)
    double gather_r2[2] = { 0.0, 0.0 };       // fixed gather radius^2 of the caustic / global map; 0: k-NN (mcrt_photon_gather_radius)
    double emit_non_caustic_reject = 1.0;
    void* knn_queue64 = nullptr; void* knn_queue32 = nullptr;
    uint32_t knn_capacity64 = 0, knn_capacity32 = 0;

    std::vector<cudaEvent_t> stage_events; // 6 per wavefront iteration when stage_timing is on (the 6th: before k_knn)
    std::vector<uint8_t> prim_interpolates; // host copy: ordered prim has vertex normals

    // ray-coherence sort buffers (shared by both precisions)
    std::vector<void*> sort_allocs;
    RaySort sort{};
    uint32_t sort_capacity = 0;
    double scene_bmin[3] = { 0, 0, 0 }, scene_bmax[3] = { 1, 1, 1 };

    // options
    int sort_rays = 1;
    int sort_shade = 0;
    // 1: k_shade walks paths grouped by the material class of their hit. Off by default: on the H100 the class key, its
    // scan and scatter (three launches per bounce) and the gathers through shade_order cost more than the coherent
    // material branches save - C2 parity 1653 against 1713 ms per frame, fast mode 1213 against 1287 (DESIGN.md §3)
    int sort_shade_class = 0;
    int sort_prim_key = -1;   // -1 auto (>= 4096 primitives), 0 origin-cell keys, 1 source-primitive keys
    uint32_t pool_paths = 1u << 23;   // measured on C2: 2 Mi 2269, 4 Mi 2378, 8 Mi 2463, 16 Mi 2503 Mray/s (coarser bins fill better)
    int blocks_per_sm = 16;   // grid = SMs x this for the grid-stride stage kernels (more CTAs than fit at once keep every SM busy to the end of a stage)
    double ray_eps_scale = 1e-5;
    int poll_interval = 4;
    int stage_timing = 0;
};

namespace
{
    template <class T>
    int devAlloc(mcrt_ctx* ctx, std::vector<void*>& track, T** out, size_t count)
    {
        *out = nullptr;
        if (count == 0) count = 1;
        void* p = nullptr;
        CK(cudaMalloc(&p, count * sizeof(T)));
        track.push_back(p);
        *out = static_cast<T*>(p);
        return MCRT_OK;
    }

    template <class T>
    int devUpload(mcrt_ctx* ctx, std::vector<void*>& track, const T** out, const std::vector<T>& v, uint64_t& bytes)
    {
        T* p = nullptr;
        int rc = devAlloc(ctx, track, &p, v.size());
        if (rc) return rc;
        if (!v.empty())
        {
            CK(cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
            bytes += v.size() * sizeof(T);
        }
        *out = p;
        return MCRT_OK;
    }

    void freeAll(std::vector<void*>& track)
    {
        for (void* p : track) cudaFree(p);
        track.clear();
    }

    template <class R> V3<R> v3(const double* p) { return V3<R>((R)p[0], (R)p[1], (R)p[2]); }

    // Build the per-precision host arrays from the float64 description.
    template <class R>
    int buildArrays(mcrt_ctx* ctx, const mcrt_scene_desc& s, SceneArrays<R>& a)
    {
        // ---- geometry slots + shading records
        a.geom.resize(3 * (size_t)s.n_prims);
        a.shade.resize(s.n_prims);
        for (uint32_t i = 0; i < s.n_prims; i++)
        {
            const uint32_t type = s.prim_type[i], idx = s.prim_index[i];
            PrimShade<R>& ps = a.shade[i];
            ps.nx = ps.ny = ps.nz = R(0);
            ps.area = (R)s.prim_area[i];
            ps.material = s.prim_material[i];
            ps.vn_index = -1;
            ps.type = type;
            ps.light = NO_PRIM;
            if (ps.material >= s.n_materials) { ctx->error = "prim_material out of range"; return MCRT_ERR_INVALID; }
            if (type == MCRT_PRIM_TRIANGLE)
            {
                if (idx >= s.n_tris) { ctx->error = "triangle index out of range"; return MCRT_ERR_INVALID; }
                a.geom[3 * i + 0] = V4<R>(v3<R>(s.tri_v0 + 3 * idx), R(PRIM_TRIANGLE));
                a.geom[3 * i + 1] = V4<R>(v3<R>(s.tri_e1 + 3 * idx), R(0));
                a.geom[3 * i + 2] = V4<R>(v3<R>(s.tri_e2 + 3 * idx), R(0));
                ps.nx = (R)s.tri_normal[3 * idx]; ps.ny = (R)s.tri_normal[3 * idx + 1]; ps.nz = (R)s.tri_normal[3 * idx + 2];
                ps.vn_index = s.tri_vn_index[idx];
                if (ps.vn_index >= (int32_t)s.n_vertex_normals) { ctx->error = "vertex normal index out of range"; return MCRT_ERR_INVALID; }
            }
            else if (type == MCRT_PRIM_SPHERE)
            {
                if (idx >= s.n_spheres) { ctx->error = "sphere index out of range"; return MCRT_ERR_INVALID; }
                const double* sp = s.sphere_origin_radius + 4 * idx;
                a.geom[3 * i + 0] = V4<R>(v3<R>(sp), R(PRIM_SPHERE));
                a.geom[3 * i + 1] = V4<R>((R)sp[3], R(0), R(0), R(0));
                a.geom[3 * i + 2] = V4<R>(R(0), R(0), R(0), R(0));
            }
            else if (type == MCRT_PRIM_QUADRIC)
            {
                if (idx >= s.n_quadrics) { ctx->error = "quadric index out of range"; return MCRT_ERR_INVALID; }
                a.geom[3 * i + 0] = V4<R>(R(idx), R(0), R(0), R(PRIM_QUADRIC));
                a.geom[3 * i + 1] = V4<R>(R(0), R(0), R(0), R(0));
                a.geom[3 * i + 2] = V4<R>(R(0), R(0), R(0), R(0));
            }
            else
            {
                ctx->error = "unknown primitive type";
                return MCRT_ERR_INVALID;
            }
        }

        a.vnormals.resize(3 * (size_t)s.n_vertex_normals);
        for (uint32_t i = 0; i < s.n_vertex_normals; i++)
            for (int k = 0; k < 3; k++)
                a.vnormals[3 * i + k] = V4<R>(v3<R>(s.vertex_normals + 9 * i + 3 * k), R(0));

        a.quadrics.resize(s.n_quadrics);
        for (uint32_t i = 0; i < s.n_quadrics; i++)
        {
            for (int k = 0; k < 16; k++) a.quadrics[i].Q[k] = (R)s.quadric_Q[16 * i + k];
            for (int k = 0; k < 12; k++) a.quadrics[i].G[k] = (R)s.quadric_G[12 * i + k];
            for (int k = 0; k < 3; k++) { a.quadrics[i].bmin[k] = (R)s.quadric_bounds[6 * i + k]; a.quadrics[i].bmax[k] = (R)s.quadric_bounds[6 * i + 3 + k]; }
        }

        a.materials.resize(s.n_materials);
        for (uint32_t i = 0; i < s.n_materials; i++)
        {
            const mcrt_material& m = s.materials[i];
            Material<R>& o = a.materials[i];
            o.reflectance = v3<R>(m.reflectance);
            o.specular_reflectance = v3<R>(m.specular_reflectance);
            o.transmittance = v3<R>(m.transmittance);
            o.emittance = v3<R>(m.emittance);
            o.ior_real = v3<R>(m.complex_ior_real);
            o.ior_imag = v3<R>(m.complex_ior_imag);
            o.roughness = (R)m.roughness; o.specular_roughness = (R)m.specular_roughness;
            o.ior = (R)m.ior; o.transparency = (R)m.transparency;
            o.A = (R)m.A; o.B = (R)m.B; o.ax = (R)m.a[0]; o.ay = (R)m.a[1];
            o.flags = (m.has_complex_ior ? MAT_COMPLEX_IOR : 0u) | (m.perfect_mirror ? MAT_PERFECT_MIRROR : 0u) |
                      (m.rough ? MAT_ROUGH : 0u) | (m.rough_specular ? MAT_ROUGH_SPECULAR : 0u) |
                      (m.opaque ? MAT_OPAQUE : 0u) | (m.emissive ? MAT_EMISSIVE : 0u) |
                      (m.dirac_delta ? MAT_DIRAC_DELTA : 0u);
        }

        a.lights.resize(s.n_lights);
        for (uint32_t i = 0; i < s.n_lights; i++)
        {
            const uint32_t prim = s.light_prim[i];
            if (prim >= s.n_prims) { ctx->error = "light_prim out of range"; return MCRT_ERR_INVALID; }
            const uint32_t type = s.prim_type[prim], idx = s.prim_index[prim];
            Light<R>& l = a.lights[i];
            l.prim = prim; l.type = type;
            l.cdf = (R)s.light_cdf[i];
            l.area = (R)s.prim_area[prim];
            l.emittance = v3<R>(s.materials[s.prim_material[prim]].emittance);
            l.p0 = l.p1 = l.p2 = l.normal = V3<R>(R(0));
            if (type == MCRT_PRIM_TRIANGLE)
            {
                l.p0 = v3<R>(s.tri_v0 + 3 * idx); l.p1 = v3<R>(s.tri_v1 + 3 * idx); l.p2 = v3<R>(s.tri_v2 + 3 * idx);
                l.normal = v3<R>(s.tri_normal + 3 * idx);
            }
            else if (type == MCRT_PRIM_SPHERE)
            {
                l.p0 = v3<R>(s.sphere_origin_radius + 4 * idx);
                l.p1 = V3<R>((R)s.sphere_origin_radius[4 * idx + 3], R(0), R(0));
            }
            else
            {
                ctx->error = "quadric lights are not supported by the reference (scene.cpp:125-132)";
                return MCRT_ERR_INVALID;
            }
            a.shade[prim].light = i;
        }
        return MCRT_OK;
    }

    // Children-contiguous layout of the BVH (see scene.cuh). Child order inside a block = the
    // reference's next_sibling chain, which the parity traversal depends on.
    template <class R>
    int buildWide(mcrt_ctx* ctx, const mcrt_scene_desc& s, SceneArrays<R>& a)
    {
        DeviceScene<R>& d = a.dev;
        d.root_is_leaf = 0; d.root_first_prim = 0; d.root_prim_count = 0; d.n_wide_root = 0;
        for (int k = 0; k < 3; k++) { d.root_bmin[k] = R(0); d.root_bmax[k] = R(0); }
        if (s.n_nodes == 0) return MCRT_OK;
        auto lower = [&](double v) { R r = (R)v; if ((double)r > v) r = std::nextafter(r, (R)-INFINITY); return r; };
        auto upper = [&](double v) { R r = (R)v; if ((double)r < v) r = std::nextafter(r, (R)INFINITY); return r; };
        // float bounds are rounded outwards so that no double-precision hit is lost; exact in double
        for (int k = 0; k < 3; k++) { d.root_bmin[k] = lower(s.node_bounds[k]); d.root_bmax[k] = upper(s.node_bounds[3 + k]); }
        if (s.node_prim_count[0])
        {
            d.root_is_leaf = 1; d.root_first_prim = s.node_first_prim[0]; d.root_prim_count = s.node_prim_count[0];
            return MCRT_OK;
        }
        auto childrenOf = [&](uint32_t node, std::vector<uint32_t>& out)
        {
            out.clear();
            uint32_t c = node + 1;
            while (c != 0 && c < s.n_nodes) { out.push_back(c); c = s.node_next_sibling[c]; }
        };
        // breadth-first so that siblings' blocks are close together
        struct Pending { uint32_t node; uint32_t record; }; // record = index of the child record to patch
        std::vector<uint32_t> kids;
        std::vector<Pending> queue;
        childrenOf(0, kids);
        d.n_wide_root = (uint32_t)kids.size();
        auto emitBlock = [&](const std::vector<uint32_t>& ks) -> int
        {
            if (ks.size() > 8) { ctx->error = "BVH arity > 8 unsupported"; return MCRT_ERR_UNSUPPORTED; }
            for (uint32_t c : ks)
            {
                WideChild<R> w;
                std::memset(&w, 0, sizeof(w));
                for (int k = 0; k < 3; k++) { w.bmin[k] = lower(s.node_bounds[6 * c + k]); w.bmax[k] = upper(s.node_bounds[6 * c + 3 + k]); }
                if (s.node_prim_count[c]) { w.a = s.node_first_prim[c]; w.b = s.node_prim_count[c] | WIDE_LEAF; }
                else { w.a = 0; w.b = 0; queue.push_back({ c, (uint32_t)a.wide.size() }); }
                a.wide.push_back(w);
            }
            return MCRT_OK;
        };
        int rc = emitBlock(kids);
        if (rc) return rc;
        for (size_t q = 0; q < queue.size(); q++)
        {
            const Pending pnd = queue[q];
            childrenOf(pnd.node, kids);
            a.wide[pnd.record].a = (uint32_t)a.wide.size();
            a.wide[pnd.record].b = (uint32_t)kids.size();
            rc = emitBlock(kids);
            if (rc) return rc;
        }
        return MCRT_OK;
    }


    // The reference's tree collapsed to <= 4 children per node for traverseFast (bvh4.cuh). Any tree over
    // the same ordered primitives with exactly containing boxes serves: the boxes only decide which
    // primitives get tested. Inner children are pulled up greedily by box area (largest first) while
    // the node has room; nodes with more than 4 children (the reference's octree type has up to 8) get
    // intermediate nodes over consecutive runs of children. Float boxes are rounded outwards.
    int buildBvh4(uint32_t max_leaf_option, const mcrt_scene_desc& s, std::vector<Bvh4Node>& out)
    {
        out.clear();
        if (s.n_nodes == 0) return MCRT_OK;
        if (s.n_prims >= BVH4_MAX_PRIMS) return MCRT_OK;   // leaf references hold 23 bits: such scenes use the replay traversal
        auto lower = [](double v) { float r = (float)v; if ((double)r > v) r = std::nextafter(r, -INFINITY); return r; };
        auto upper = [](double v) { float r = (float)v; if ((double)r < v) r = std::nextafter(r, INFINITY); return r; };
        struct Item { int64_t node; std::vector<Item> group; double box[6]; uint32_t first, count; };   // node >= 0: reference node; -1: run of items; -2: part of a reference leaf
        // leaves larger than max_leaf are cut into runs of consecutive primitives with their own boxes (lanes of a
        // warp then spend similar time per leaf, and the tighter boxes cull more)
        // auto: cut leaves to 2 primitives on tiny scenes (the reference's leaves hold up to 8 in the 44-primitive hexagon
        // room), keep the reference's leaves on big ones, where the extra nodes cost more than the tighter boxes save
        const uint32_t max_leaf = max_leaf_option == 0xFFFFFFFFu ? (s.n_prims < 4096u ? 2u : 0u) : max_leaf_option;
        auto primBox = [&](uint32_t prim, double* b)
        {
            const uint32_t type = s.prim_type[prim], idx = s.prim_index[prim];
            if (type == MCRT_PRIM_TRIANGLE)
            {
                for (int k = 0; k < 3; k++)
                {
                    const double a0 = s.tri_v0[3 * (size_t)idx + k], a1 = s.tri_v1[3 * (size_t)idx + k], a2 = s.tri_v2[3 * (size_t)idx + k];
                    b[k] = std::min(a0, std::min(a1, a2)); b[3 + k] = std::max(a0, std::max(a1, a2));
                }
            }
            else if (type == MCRT_PRIM_SPHERE)
            {
                const double* sp = s.sphere_origin_radius + 4 * (size_t)idx;
                for (int k = 0; k < 3; k++) { b[k] = sp[k] - sp[3]; b[3 + k] = sp[k] + sp[3]; }
            }
            else for (int k = 0; k < 6; k++) b[k] = s.quadric_bounds[6 * (size_t)idx + k];
        };
        auto itemOfNode = [&](uint32_t n)
        {
            Item it; it.node = n; it.first = s.node_first_prim[n]; it.count = s.node_prim_count[n];
            for (int k = 0; k < 6; k++) it.box[k] = s.node_bounds[6 * (size_t)n + k];
            if (max_leaf && it.count > max_leaf)
            {
                // a reference leaf with more primitives than max_leaf: a run of part-leaves (shape() groups them by four)
                it.node = -1;
                for (uint32_t f = it.first; f < it.first + it.count; f += max_leaf)
                {
                    Item part; part.node = -2; part.first = f; part.count = std::min(max_leaf, it.first + it.count - f);
                    for (int k = 0; k < 3; k++) { part.box[k] = 1e300; part.box[3 + k] = -1e300; }
                    for (uint32_t q = f; q < f + part.count; q++)
                    {
                        double b[6]; primBox(q, b);
                        // never outside the reference's leaf box (sphere / quadric boxes are what the reference stores anyway)
                        for (int k = 0; k < 3; k++) { part.box[k] = std::min(part.box[k], b[k]); part.box[3 + k] = std::max(part.box[3 + k], b[3 + k]); }
                    }
                    it.group.push_back(part);
                }
            }
            return it;
        };
        auto area = [](const double* b) { const double x = b[3] - b[0], y = b[4] - b[1], z = b[5] - b[2]; return x * y + y * z + z * x; };
        auto childrenOf = [&](uint32_t node, std::vector<Item>& kids)
        {
            uint32_t c = node + 1;
            while (c != 0 && c < s.n_nodes) { kids.push_back(itemOfNode(c)); c = s.node_next_sibling[c]; }
        };
        auto isInner = [&](const Item& it) { return it.node == -1 || (it.node >= 0 && s.node_prim_count[it.node] == 0); };
        auto expand = [&](const Item& it, std::vector<Item>& kids) { if (it.node < 0) kids = it.group; else { kids.clear(); childrenOf((uint32_t)it.node, kids); } };
        auto shape = [&](std::vector<Item>& kids)
        {
            // pull grandchildren up while there is room
            while (kids.size() < 4)
            {
                int pick = -1; double pick_area = -1.0; std::vector<Item> sub, best_sub;
                for (size_t i = 0; i < kids.size(); i++)
                {
                    if (!isInner(kids[i])) continue;
                    expand(kids[i], sub);
                    if (sub.empty() || kids.size() - 1 + sub.size() > 4) continue;
                    const double a = area(kids[i].box);
                    if (a > pick_area) { pick_area = a; pick = (int)i; best_sub = sub; }
                }
                if (pick < 0) break;
                kids.erase(kids.begin() + pick);
                kids.insert(kids.begin() + pick, best_sub.begin(), best_sub.end());
            }
            // too many: intermediate nodes over consecutive runs
            while (kids.size() > 4)
            {
                std::vector<Item> packed;
                for (size_t i = 0; i < kids.size(); i += 4)
                {
                    const size_t e = std::min(kids.size(), i + 4);
                    if (e - i == 1) { packed.push_back(kids[i]); continue; }
                    Item g; g.node = -1; g.group.assign(kids.begin() + i, kids.begin() + e);
                    for (int k = 0; k < 3; k++) { g.box[k] = 1e300; g.box[3 + k] = -1e300; }
                    for (const Item& c : g.group) for (int k = 0; k < 3; k++) { g.box[k] = std::min(g.box[k], c.box[k]); g.box[3 + k] = std::max(g.box[3 + k], c.box[3 + k]); }
                    packed.push_back(std::move(g));
                }
                kids.swap(packed);
            }
        };
        auto leafRef = [&](const Item& it, uint32_t& ref) -> bool
        {
            const uint32_t first = it.first, count = it.count;
            if (count > 255u) return false;
            ref = BVH4_LEAF | (first << 8) | count;
            return true;
        };
        struct Pending { Item item; uint32_t parent, slot; };
        std::vector<Pending> queue;   // breadth-first: the top of the tree is contiguous
        auto emit = [&](std::vector<Item>& kids, uint32_t self) -> int
        {
            shape(kids);
            Bvh4Node n;
            std::memset(&n, 0, sizeof(n));
            for (int c = 0; c < 4; c++) for (int k = 0; k < 3; k++) { n.lo[k][c] = 3.0e38f; n.hi[k][c] = -3.0e38f; }
            for (size_t c = 0; c < kids.size(); c++)
            {
                for (int k = 0; k < 3; k++) { n.lo[k][c] = lower(kids[c].box[k]); n.hi[k][c] = upper(kids[c].box[3 + k]); }
                if (!isInner(kids[c]))
                {
                    if (!leafRef(kids[c], n.child[c])) return 1;
                }
                else queue.push_back({ kids[c], self, (uint32_t)c });
            }
            out[self] = n;
            return 0;
        };
        std::vector<Item> kids;
        out.emplace_back();
        if (s.node_prim_count[0]) kids.push_back(itemOfNode(0));   // the root is a leaf: one child
        else childrenOf(0, kids);
        bool too_big = emit(kids, 0) != 0;
        for (size_t q = 0; q < queue.size() && !too_big; q++)
        {
            const Pending pn = queue[q];   // copy: emit() grows the queue
            const uint32_t self = (uint32_t)out.size();
            out.emplace_back();
            out[pn.parent].child[pn.slot] = self;
            expand(pn.item, kids);
            too_big = emit(kids, self) != 0;
        }
        if (too_big) out.clear();   // a leaf with more than 255 primitives: the replay traversal handles the scene
        return MCRT_OK;
    }

    // A BVH4 for traverseFast built anew with spatial splits (Stich, Friedrich and Dietrich, "Spatial Splits in Bounding Volume
    // Hierarchies", HPG 2009): binned SAH over object and spatial splits, the binary tree collapsed to <= 4 children per node like
    // buildBvh4's. A spatial split cuts a primitive into references with a box each, clipped to its part of the primitive: a large
    // triangle lying diagonally to the axes (the hexagon room's walls) is then tested only by rays that come near it. Leaf
    // references (first, count) index `refs`, which maps each reference to its ordered primitive. The search stays exact because
    // the float boxes conservatively contain what they hold: every point of a primitive lies in the box of at least one of its
    // references. Triangles are clipped in float64 and each clipped coordinate is widened by a bound on its rounding error
    // (2^-40 of the magnitudes involved, and more where an edge crosses the plane at a grazing angle); spheres keep their box
    // intersected with the cuts (interval operations, exact); quadrics are never split. `node_cost` is the cost of visiting a
    // node (four box tests) in float64 primitive tests; references are capped at `ref_budget` times the primitive count.
    int buildBvh4Split(const mcrt_scene_desc& s, double node_cost, double ref_budget, std::vector<Bvh4Node>& out, std::vector<uint32_t>& refs)
    {
        out.clear(); refs.clear();
        if (s.n_nodes == 0 || s.n_prims == 0 || s.n_prims >= BVH4_MAX_PRIMS) return MCRT_OK;
        auto lower = [](double v) { float r = (float)v; if ((double)r > v) r = std::nextafter(r, -INFINITY); return r; };
        auto upper = [](double v) { float r = (float)v; if ((double)r < v) r = std::nextafter(r, INFINITY); return r; };
        struct Ref { uint32_t prim; double b[6]; };
        struct SNode { double b[6]; int32_t kid[2]; uint32_t first, count; };   // kid[0] < 0: leaf over refs[first, first + count)
        constexpr int NB = 32;
        constexpr uint32_t MAX_LEAF = 2;
        const double eps = std::ldexp(1.0, -40);
        auto empty = [](double* b) { for (int k = 0; k < 3; k++) { b[k] = 1e300; b[3 + k] = -1e300; } };
        auto grow = [](double* b, const double* c) { for (int k = 0; k < 3; k++) { b[k] = std::min(b[k], c[k]); b[3 + k] = std::max(b[3 + k], c[3 + k]); } };
        auto area = [](const double* b) { const double x = b[3] - b[0], y = b[4] - b[1], z = b[5] - b[2]; return (x < 0 || y < 0 || z < 0) ? 0.0 : x * y + y * z + z * x; };
        auto isEmpty = [](const double* b) { return b[0] > b[3] || b[1] > b[4] || b[2] > b[5]; };
        auto vert = [&](const double* base, uint32_t idx, double* p) { for (int k = 0; k < 3; k++) p[k] = base[3 * (size_t)idx + k]; };

        // The part of primitive `prim` inside the box c (the reference's box with one face moved to a cut), boxed conservatively.
        auto clip = [&](uint32_t prim, const double* c, double* out_b)
        {
            empty(out_b);
            const uint32_t type = s.prim_type[prim], idx = s.prim_index[prim];
            if (type == MCRT_PRIM_TRIANGLE)
            {
                // Sutherland-Hodgman against the six planes of c; every vertex carries its error bound
                struct P { double x[3]; double e; };
                P poly[16], next[16];
                int n = 3;
                vert(s.tri_v0, idx, poly[0].x); vert(s.tri_v1, idx, poly[1].x); vert(s.tri_v2, idx, poly[2].x);
                for (int i = 0; i < 3; i++) poly[i].e = 0.0;
                for (int plane = 0; plane < 6 && n > 0; plane++)
                {
                    const int k = plane % 3;
                    const bool is_lo = plane < 3;
                    const double pos = c[plane];
                    auto inside = [&](const P& p) { return is_lo ? p.x[k] >= pos : p.x[k] <= pos; };
                    int m = 0;
                    for (int i = 0; i < n; i++)
                    {
                        const P& a = poly[i];
                        const P& b = poly[(i + 1) % n];
                        const bool ia = inside(a), ib = inside(b);
                        if (ia) next[m++] = a;
                        if (ia != ib)
                        {
                            const double den = b.x[k] - a.x[k];
                            const double t = std::min(1.0, std::max(0.0, (pos - a.x[k]) / den));
                            P q;
                            double span = 0.0;
                            for (int j = 0; j < 3; j++) { q.x[j] = a.x[j] + t * (b.x[j] - a.x[j]); span = std::max(span, std::fabs(b.x[j] - a.x[j])); }
                            q.x[k] = pos;
                            const double mag = std::fabs(pos) + std::fabs(a.x[k]) + std::fabs(b.x[k]);
                            q.e = std::max(a.e, b.e) + span * std::min(1.0, eps * mag / std::fabs(den)) +
                                  eps * (std::fabs(q.x[0]) + std::fabs(q.x[1]) + std::fabs(q.x[2]) + span);
                            next[m++] = q;
                        }
                    }
                    n = m;
                    for (int i = 0; i < n; i++) poly[i] = next[i];
                }
                for (int i = 0; i < n; i++)
                    for (int k = 0; k < 3; k++)
                    {
                        out_b[k] = std::min(out_b[k], poly[i].x[k] - poly[i].e - eps * std::fabs(poly[i].x[k]));
                        out_b[3 + k] = std::max(out_b[3 + k], poly[i].x[k] + poly[i].e + eps * std::fabs(poly[i].x[k]));
                    }
            }
            else
            {
                const double* sp = s.sphere_origin_radius + 4 * (size_t)idx;
                for (int k = 0; k < 3; k++) { out_b[k] = sp[k] - sp[3]; out_b[3 + k] = sp[k] + sp[3]; }
            }
            // never outside c: every point of the primitive inside c is inside this
            for (int k = 0; k < 3; k++) { out_b[k] = std::max(out_b[k], c[k]); out_b[3 + k] = std::min(out_b[3 + k], c[3 + k]); }
        };
        // ref cut at `pos` on axis k -> left / right parts (an empty box: nothing of the primitive on that side)
        auto cut = [&](const Ref& r, int k, double pos, Ref& l, Ref& rr)
        {
            double c[6];
            l.prim = rr.prim = r.prim;
            std::memcpy(c, r.b, sizeof(c)); c[3 + k] = std::min(c[3 + k], pos); clip(r.prim, c, l.b);
            std::memcpy(c, r.b, sizeof(c)); c[k] = std::max(c[k], pos); clip(r.prim, c, rr.b);
        };

        std::vector<Ref> all(s.n_prims);
        bool quadrics = false;
        for (uint32_t i = 0; i < s.n_prims; i++)
        {
            Ref& r = all[i];
            r.prim = i;
            const uint32_t type = s.prim_type[i], idx = s.prim_index[i];
            if (type == MCRT_PRIM_TRIANGLE)
            {
                double v[3][3];
                vert(s.tri_v0, idx, v[0]); vert(s.tri_v1, idx, v[1]); vert(s.tri_v2, idx, v[2]);
                for (int k = 0; k < 3; k++) { r.b[k] = std::min(v[0][k], std::min(v[1][k], v[2][k])); r.b[3 + k] = std::max(v[0][k], std::max(v[1][k], v[2][k])); }
            }
            else if (type == MCRT_PRIM_SPHERE)
            {
                const double* sp = s.sphere_origin_radius + 4 * (size_t)idx;
                for (int k = 0; k < 3; k++) { r.b[k] = sp[k] - sp[3]; r.b[3 + k] = sp[k] + sp[3]; }
            }
            else { quadrics = true; for (int k = 0; k < 6; k++) r.b[k] = s.quadric_bounds[6 * (size_t)idx + k]; }
        }
        const size_t budget = (size_t)(ref_budget * s.n_prims);
        size_t n_refs = all.size();
        std::vector<SNode> nodes;

        // binary SBVH, depth first; returns the node index
        std::function<int32_t(std::vector<Ref>&)> build = [&](std::vector<Ref>& rs) -> int32_t
        {
            SNode nd;
            empty(nd.b);
            for (const Ref& r : rs) grow(nd.b, r.b);
            nd.kid[0] = nd.kid[1] = -1; nd.first = 0; nd.count = (uint32_t)rs.size();
            const int32_t self = (int32_t)nodes.size();
            nodes.push_back(nd);
            const size_t n = rs.size();
            auto makeLeaf = [&]() { nodes[self].first = (uint32_t)refs.size(); for (const Ref& r : rs) refs.push_back(r.prim); return self; };
            if (n <= 1) return makeLeaf();
            const double pa = std::max(area(nd.b), 1e-300);
            double best = INFINITY; int best_axis = -1, best_bin = -1; bool best_spatial = false;
            double cbox[6]; empty(cbox);
            for (const Ref& r : rs) for (int k = 0; k < 3; k++) { const double cc = 0.5 * (r.b[k] + r.b[3 + k]); cbox[k] = std::min(cbox[k], cc); cbox[3 + k] = std::max(cbox[3 + k], cc); }
            auto centroidBin = [&](const Ref& r, int k) { const double ext = cbox[3 + k] - cbox[k]; int b = (int)(NB * ((0.5 * (r.b[k] + r.b[3 + k]) - cbox[k]) / ext)); return std::min(NB - 1, std::max(0, b)); };
            // object splits: centroid bins
            for (int k = 0; k < 3; k++)
            {
                if (!(cbox[3 + k] > cbox[k])) continue;
                double bb[NB][6]; uint32_t cnt[NB] = {};
                for (int b = 0; b < NB; b++) empty(bb[b]);
                for (const Ref& r : rs) { const int b = centroidBin(r, k); grow(bb[b], r.b); cnt[b]++; }
                double right[NB][6]; uint32_t rc[NB];
                double acc[6]; empty(acc); uint32_t ac = 0;
                for (int b = NB - 1; b >= 1; b--) { grow(acc, bb[b]); ac += cnt[b]; std::memcpy(right[b], acc, sizeof(acc)); rc[b] = ac; }
                empty(acc); ac = 0;
                for (int b = 0; b < NB - 1; b++)
                {
                    grow(acc, bb[b]); ac += cnt[b];
                    if (ac == 0 || rc[b + 1] == 0) continue;
                    const double cost = node_cost + (area(acc) * ac + area(right[b + 1]) * rc[b + 1]) / pa;
                    if (cost < best) { best = cost; best_axis = k; best_bin = b; best_spatial = false; }
                }
            }
            // spatial splits: bins over the node's box, references chopped at every bin boundary they cross
            bool has_quadric = false;
            if (quadrics) for (const Ref& r : rs) has_quadric |= s.prim_type[r.prim] == MCRT_PRIM_QUADRIC;
            if (!has_quadric && n_refs + n <= budget)
            {
                for (int k = 0; k < 3; k++)
                {
                    const double lo = nd.b[k], ext = nd.b[3 + k] - nd.b[k];
                    if (!(ext > 0.0)) continue;
                    auto plane = [&](int b) { return lo + ext * b / NB; };
                    auto binOf = [&](double x) { return std::min(NB - 1, std::max(0, (int)(NB * ((x - lo) / ext)))); };
                    double bb[NB][6]; uint32_t enter[NB] = {}, leave[NB] = {};
                    for (int b = 0; b < NB; b++) empty(bb[b]);
                    for (const Ref& r : rs)
                    {
                        const int b0 = binOf(r.b[k]), b1 = binOf(r.b[3 + k]);
                        enter[b0]++; leave[b1]++;
                        Ref cur = r, l, rr;
                        for (int b = b0; b < b1; b++)
                        {
                            cut(cur, k, plane(b + 1), l, rr);
                            if (!isEmpty(l.b)) grow(bb[b], l.b);
                            cur = rr;
                            if (isEmpty(cur.b)) break;
                        }
                        if (!isEmpty(cur.b)) grow(bb[b1], cur.b);
                    }
                    double right[NB][6]; uint32_t rc[NB];
                    double acc[6]; empty(acc); uint32_t ac = 0;
                    for (int b = NB - 1; b >= 1; b--) { grow(acc, bb[b]); ac += leave[b]; std::memcpy(right[b], acc, sizeof(acc)); rc[b] = ac; }
                    empty(acc); ac = 0;
                    for (int b = 0; b < NB - 1; b++)
                    {
                        grow(acc, bb[b]); ac += enter[b];
                        if (ac == 0 || rc[b + 1] == 0 || (ac == n && rc[b + 1] == n)) continue;
                        const double cost = node_cost + (area(acc) * ac + area(right[b + 1]) * rc[b + 1]) / pa;
                        if (cost < best) { best = cost; best_axis = k; best_bin = b; best_spatial = true; }
                    }
                }
            }
            if (n <= MAX_LEAF && (double)n <= best) return makeLeaf();
            std::vector<Ref> ls, rrs;
            if (best_spatial)
            {
                const int k = best_axis;
                const double lo = nd.b[k], ext = nd.b[3 + k] - nd.b[k];
                const double pos = lo + ext * (best_bin + 1) / NB;
                for (const Ref& r : rs)
                {
                    if (r.b[3 + k] <= pos) ls.push_back(r);
                    else if (r.b[k] >= pos) rrs.push_back(r);
                    else
                    {
                        Ref l, rr;
                        cut(r, k, pos, l, rr);
                        if (!isEmpty(l.b)) ls.push_back(l);
                        if (!isEmpty(rr.b)) rrs.push_back(rr);
                    }
                }
                if (ls.empty() || rrs.empty() || (ls.size() == n && rrs.size() == n)) { ls.clear(); rrs.clear(); }
                else n_refs += ls.size() + rrs.size() - n;
            }
            else if (best_axis >= 0)
            {
                for (const Ref& r : rs) (centroidBin(r, best_axis) <= best_bin ? ls : rrs).push_back(r);
            }
            if (ls.empty() || rrs.empty())
            {
                // no usable split (coincident centroids): halves in centroid order along the widest axis
                ls.clear(); rrs.clear();
                int k = 0;
                for (int j = 1; j < 3; j++) if (nd.b[3 + j] - nd.b[j] > nd.b[3 + k] - nd.b[k]) k = j;
                std::vector<Ref> sorted = rs;
                std::stable_sort(sorted.begin(), sorted.end(), [&](const Ref& a, const Ref& b) { return a.b[k] + a.b[3 + k] < b.b[k] + b.b[3 + k]; });
                ls.assign(sorted.begin(), sorted.begin() + n / 2);
                rrs.assign(sorted.begin() + n / 2, sorted.end());
            }
            rs.clear(); rs.shrink_to_fit();
            const int32_t l = build(ls);
            const int32_t r = build(rrs);
            nodes[self].kid[0] = l; nodes[self].kid[1] = r;
            return self;
        };
        build(all);
        if (refs.size() >= BVH4_MAX_PRIMS) { out.clear(); refs.clear(); return MCRT_OK; }

        // collapse to 4-wide nodes: pull up the grandchildren of the largest inner child while there is room, breadth first
        auto isInner = [&](int32_t i) { return nodes[i].kid[0] >= 0; };
        struct Pending { int32_t node; uint32_t parent, slot; };
        std::vector<Pending> queue;
        auto emit = [&](int32_t bnode, uint32_t self)
        {
            std::vector<int32_t> kids;
            if (isInner(bnode)) kids = { nodes[bnode].kid[0], nodes[bnode].kid[1] };
            else kids = { bnode };   // the root is a leaf
            while (kids.size() < 4)
            {
                int pick = -1; double pick_area = -1.0;
                for (size_t i = 0; i < kids.size(); i++)
                    if (isInner(kids[i]) && area(nodes[kids[i]].b) > pick_area) { pick_area = area(nodes[kids[i]].b); pick = (int)i; }
                if (pick < 0) break;
                const int32_t c = kids[pick];
                kids[pick] = nodes[c].kid[0];
                kids.insert(kids.begin() + pick + 1, nodes[c].kid[1]);
            }
            Bvh4Node n;
            std::memset(&n, 0, sizeof(n));
            for (int c = 0; c < 4; c++) for (int k = 0; k < 3; k++) { n.lo[k][c] = 3.0e38f; n.hi[k][c] = -3.0e38f; }
            for (size_t c = 0; c < kids.size(); c++)
            {
                const SNode& sn = nodes[kids[c]];
                for (int k = 0; k < 3; k++) { n.lo[k][c] = lower(sn.b[k]); n.hi[k][c] = upper(sn.b[3 + k]); }
                if (!isInner(kids[c])) n.child[c] = BVH4_LEAF | (sn.first << 8) | sn.count;
                else queue.push_back({ kids[c], self, (uint32_t)c });
            }
            out[self] = n;
        };
        out.emplace_back();
        emit(0, 0);
        for (size_t q = 0; q < queue.size(); q++)
        {
            const Pending pn = queue[q];
            const uint32_t self = (uint32_t)out.size();
            out.emplace_back();
            out[pn.parent].child[pn.slot] = self;
            emit(pn.node, self);
        }
        return MCRT_OK;
    }

    template <class R>
    int uploadArrays(mcrt_ctx* ctx, const mcrt_scene_desc& s, SceneArrays<R>& a, uint64_t& bytes)
    {
        DeviceScene<R>& d = a.dev;
        int rc;
        if ((rc = devUpload(ctx, ctx->scene_allocs, &d.wide, a.wide, bytes))) return rc;
        if ((rc = devUpload(ctx, ctx->scene_allocs, &d.geom, a.geom, bytes))) return rc;
        if ((rc = devUpload(ctx, ctx->scene_allocs, &d.shade, a.shade, bytes))) return rc;
        if ((rc = devUpload(ctx, ctx->scene_allocs, &d.vnormals, a.vnormals, bytes))) return rc;
        if ((rc = devUpload(ctx, ctx->scene_allocs, &d.quadrics, a.quadrics, bytes))) return rc;
        if ((rc = devUpload(ctx, ctx->scene_allocs, &d.materials, a.materials, bytes))) return rc;
        if ((rc = devUpload(ctx, ctx->scene_allocs, &d.lights, a.lights, bytes))) return rc;
        {
            // shade classes: distinct (material flags, has vertex normals) combinations present in the scene
            std::vector<uint32_t> combos;
            std::vector<uint8_t> cls(s.n_prims ? s.n_prims : 1, 1);
            for (uint32_t i = 0; i < s.n_prims; i++)
            {
                const uint32_t combo = (a.materials[a.shade[i].material].flags << 1) | (a.shade[i].vn_index >= 0 ? 1u : 0u);
                size_t k = 0;
                while (k < combos.size() && combos[k] != combo) k++;
                if (k == combos.size()) combos.push_back(combo);
                cls[i] = (uint8_t)(1u + (k < SHADE_CLASS_BINS - 1u ? k : SHADE_CLASS_BINS - 2u));
            }
            if ((rc = devUpload(ctx, ctx->scene_allocs, &d.shade_class, cls, bytes))) return rc;
        }
        d.n_nodes = s.n_nodes; d.n_prims = s.n_prims; d.n_lights = s.n_lights;
        d.prims_class = PRIMS_TRI;
        for (uint32_t i = 0; i < s.n_prims; i++)
        {
            if (s.prim_type[i] == MCRT_PRIM_SPHERE && d.prims_class == PRIMS_TRI) d.prims_class = PRIMS_TRI_SPHERE;
            else if (s.prim_type[i] != MCRT_PRIM_TRIANGLE && s.prim_type[i] != MCRT_PRIM_SPHERE) { d.prims_class = PRIMS_ALL; break; }
        }
        d.material_flags_any = 0;   // selects the k_shade feature set (kernels_impl.cuh)
        for (const auto& m : a.materials) d.material_flags_any |= m.flags;
        d.scene_ior = (R)s.scene_ior;
        d.scene_scale = (R)ctx->scene_scale;
        return MCRT_OK;
    }

    template <class R>
    int ensureWave(mcrt_ctx* ctx, WaveBuffers<R>& w, std::vector<void*>& track)
    {
        if (w.capacity == ctx->pool_paths) return MCRT_OK;
        freeAll(track);
        w.capacity = 0;
        const size_t n = ctx->pool_paths;
        int rc;
        for (int b = 0; b < 2; b++)
        {
            if ((rc = devAlloc(ctx, track, &w.buf[b].ray_o, n))) return rc;
            if ((rc = devAlloc(ctx, track, &w.buf[b].ray_d, n))) return rc;
            if ((rc = devAlloc(ctx, track, &w.buf[b].thr, n))) return rc;
            if ((rc = devAlloc(ctx, track, &w.buf[b].iors_a, n))) return rc;
            if ((rc = devAlloc(ctx, track, &w.buf[b].iors_b, n))) return rc;
            if ((rc = devAlloc(ctx, track, &w.buf[b].meta, n))) return rc;
            if ((rc = devAlloc(ctx, track, &w.buf[b].meta2, n))) return rc;
        }
        if ((rc = devAlloc(ctx, track, &w.shadow, n))) return rc;
        if ((rc = devAlloc(ctx, track, &w.hits, n))) return rc;
        w.capacity = ctx->pool_paths;
        return MCRT_OK;
    }

    int ensureSort(mcrt_ctx* ctx)
    {
        if (ctx->sort_capacity == ctx->pool_paths) return MCRT_OK;
        freeAll(ctx->sort_allocs);
        ctx->sort_capacity = 0;
        const size_t n = ctx->pool_paths;
        int rc;
        RaySort& r = ctx->sort;
        for (int b = 0; b < 2; b++)
        {
            if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.path_key[b], n))) return rc;
            if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.path_rank[b], n))) return rc;
        }
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.path_order, n))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.shadow_key, n))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.shadow_rank, n))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.shadow_order, n))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.shade_key, n))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.shade_rank, n))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.shade_order, n))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.hist_shade, (size_t)SORT_BINS))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.hist_path, (size_t)SORT_BINS))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.hist_shadow, (size_t)SORT_BINS))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.bin_start, (size_t)SORT_BINS))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.block_offset, (size_t)2 * SORT_SCAN_BLOCKS))) return rc;
        if ((rc = devAlloc(ctx, ctx->sort_allocs, &r.done_counter, (size_t)1))) return rc;
        CK(cudaMemset(r.done_counter, 0, sizeof(uint32_t)));
        ctx->sort_capacity = ctx->pool_paths;
        return MCRT_OK;
    }

    int ensureFilm(mcrt_ctx* ctx, size_t values)
    {
        if (ctx->film_values >= values && ctx->d_film) return MCRT_OK;
        if (ctx->d_film) cudaFree(ctx->d_film);
        ctx->d_film = nullptr; ctx->film_values = 0;
        CK(cudaMalloc((void**)&ctx->d_film, values * sizeof(double)));
        ctx->film_values = values;
        return MCRT_OK;
    }

    template <class R> DeviceScene<R>& sceneOf(mcrt_ctx* ctx);
    template <> DeviceScene<double>& sceneOf<double>(mcrt_ctx* ctx) { return ctx->scene64; }
    template <> DeviceScene<float>& sceneOf<float>(mcrt_ctx* ctx) { return ctx->scene32; }
    template <class R> WaveBuffers<R>& waveOf(mcrt_ctx* ctx);
    template <> WaveBuffers<double>& waveOf<double>(mcrt_ctx* ctx) { return ctx->wave64; }
    template <> WaveBuffers<float>& waveOf<float>(mcrt_ctx* ctx) { return ctx->wave32; }
    template <class R> std::vector<void*>& waveAllocsOf(mcrt_ctx* ctx);
    template <> std::vector<void*>& waveAllocsOf<double>(mcrt_ctx* ctx) { return ctx->wave_allocs64; }
    template <> std::vector<void*>& waveAllocsOf<float>(mcrt_ctx* ctx) { return ctx->wave_allocs32; }

    void fillStats(mcrt_stats* st, const Counters& c, uint64_t iterations, uint64_t launches, double ms)
    {
        if (!st) return;
        std::memset(st, 0, sizeof(*st));
        st->paths = c.paths;
        st->extension_rays = c.extension_rays;
        st->shadow_rays = c.shadow_rays;
        st->box_tests = c.box_tests;
        st->prim_tests = c.prim_tests;
        st->knn_queries = c.knn_queries;
        st->wavefront_iterations = iterations;
        st->kernel_launches = launches;
        st->ior_stack_overflows = c.ior_stack_overflows;
        st->max_depth = c.max_depth;
        st->gpu_ms_total = ms;
        st->shadow_box_tests = c.shadow_box_tests;
        st->shadow_prim_tests = c.shadow_prim_tests;
        st->extend_work_sum = c.work_sum;
        st->extend_work_warpmax = c.work_warpmax;
        st->replayed_rays = c.replayed_rays;
    }

    template <class R> DeviceCamera<R> deviceCamera(const mcrt_camera& cam)
    {
        DeviceCamera<R> c;
        std::memset(&c, 0, sizeof(c));
        c.eye = v3<R>(cam.eye); c.forward = v3<R>(cam.forward);
        c.left = v3<R>(cam.left); c.up = v3<R>(cam.up);
        c.focal_length = (R)cam.focal_length; c.sensor_width = (R)cam.sensor_width;
        c.aperture_radius = (R)cam.aperture_radius; c.focus_distance = (R)cam.focus_distance;
        c.width = cam.width; c.height = cam.height; c.thin_lens = cam.thin_lens;
        return c;
    }

    // offset of spawned rays along the normal: C::EPSILON in parity mode, scale-aware in fast mode
    template <class R> R rayEps(const mcrt_ctx* ctx)
    {
        return Mode<R>::parity ? (R)1e-9 : (R)(ctx->ray_eps_scale * ctx->scene_scale);
    }

    // Accumulate mode of runWavefront: the samples are added into the caller's device sums, which are neither
    // zeroed before the render nor resolved after it (mcrt_render_accumulate_dev, mcrt_render_film_sums_strided_dev).
    struct FilmSums
    {
        double* rgb;    // box film [n_pixels][3] in film_index order; filtered film [height*width][3]
        double* wsum;   // filtered film [height*width]; null with the box film
        uint32_t n_planes = 0;   // box film only: rgb holds this many planes of the mode below; 0: one plane
        // FILM_MODE_GROUPS: light-group planes (mcrt_render_accumulate_groups_dev); FILM_MODE_AOV: planes each deposit site
        // names, the MCRT_AOV_COUNT light-path planes of the path tracer (mcrt_render_accumulate_aovs_dev) or the
        // MCRT_PM_COMPONENT_COUNT estimator planes of the photon mapper (mcrt_render_accumulate_photon_components_dev);
        // FILM_MODE_LPE: one plane per light path expression (mcrt_render_accumulate_lpe_dev). Without planes
        // runWavefront picks FILM_MODE_BOX or FILM_MODE_SPLAT.
        FilmMode mode = FILM_MODE_BOX;
    };

    // The wavefront loop shared by mcrt_render_rows(_dev) and mcrt_sample_rays. Camera work item w is sample
    // sample_first + w / n_pixels of pixel w % n_pixels, or of pixel d_pixel_list[w % n_pixels] when a list is given
    // (n_pixels is then its length). accum == null: the film lives in the context, is zeroed first and resolved into
    // out_dev at the end.
    template <class R>
    int runWavefront(mcrt_ctx* ctx, const mcrt_camera* cam, uint32_t row_first, uint32_t row_step, uint32_t n_pixels, uint32_t spp,
                     uint64_t total_work, uint32_t global_seed, int integrator, const double* d_user_rays,
                     const uint32_t* d_user_pixel, const uint32_t* d_user_sample, size_t film_pixels,
                     double film_weight, double* out_dev, mcrt_stats* stats, uint32_t sample_first = 0,
                     const FilmSums* accum = nullptr, const uint32_t* d_pixel_list = nullptr)
    {
        if (!ctx->has_scene) { ctx->error = "no scene uploaded"; return MCRT_ERR_NO_SCENE; }
        if (integrator == MCRT_INTEGRATOR_PHOTON && !ctx->has_photons)
        {
            ctx->error = "photon-mapped render requested without mcrt_photon_upload";
            return MCRT_ERR_NO_PHOTONS;
        }
        WaveBuffers<R>& wb = waveOf<R>(ctx);
        int rc;
        if ((rc = ensureWave(ctx, wb, waveAllocsOf<R>(ctx)))) return rc;
        if (!accum && (rc = ensureFilm(ctx, film_pixels * 3))) return rc;
        const bool filtered = cam && !d_user_rays && !ctx->film_default && integrator != MCRT_INTERNAL_EMIT;
        if (filtered && !accum && ctx->film_wsum_values < film_pixels)
        {
            if (ctx->d_film_wsum) cudaFree(ctx->d_film_wsum);
            ctx->d_film_wsum = nullptr; ctx->film_wsum_values = 0;
            CK(cudaMalloc((void**)&ctx->d_film_wsum, film_pixels * sizeof(double)));
            ctx->film_wsum_values = film_pixels;
        }
        KnnQuery<R>* knn_queue = nullptr;
        const uint32_t knn_capacity = 2u * ctx->pool_paths; // a path emits at most caustic + global per bounce
        if (integrator == MCRT_INTEGRATOR_PHOTON)
        {
            void*& q = Mode<R>::parity ? ctx->knn_queue64 : ctx->knn_queue32;
            uint32_t& cap = Mode<R>::parity ? ctx->knn_capacity64 : ctx->knn_capacity32;
            if (cap != knn_capacity)
            {
                if (q) cudaFree(q);
                q = nullptr; cap = 0;
                CK(cudaMalloc(&q, (size_t)knn_capacity * sizeof(KnnQuery<R>)));
                cap = knn_capacity;
            }
            knn_queue = static_cast<KnnQuery<R>*>(q);
        }

        cudaStream_t s = ctx->stream;
        const int grid = ctx->sm_count * ctx->blocks_per_sm;
        WaveParams<R> p;
        std::memset(&p, 0, sizeof(p));
        p.scene = sceneOf<R>(ctx);
        if (ctx->exact_traversal) p.scene.bvh4 = nullptr;
        p.scene.dynamic_fetch = (ctx->dynamic_fetch < 0 ? ctx->n_bvh4_nodes >= 2048u : ctx->dynamic_fetch != 0) ? 1u : 0u;
        if (cam) p.camera = deviceCamera<R>(*cam);
        p.buf[0] = wb.buf[0]; p.buf[1] = wb.buf[1];
        p.shadow = wb.shadow;
        p.hits = wb.hits;
        p.counters = ctx->d_counters;
        p.sobol_bytes = ctx->d_sobol_bytes;
        double* const film_rgb = accum ? accum->rgb : ctx->d_film;
        double* const film_wsum = accum ? accum->wsum : ctx->d_film_wsum;
        p.film = film_rgb;
        p.film_mode = filtered ? FILM_MODE_SPLAT : FILM_MODE_BOX;
        if (accum && accum->n_planes)
        {
            p.film_mode = accum->mode;
            p.group_of_light = ctx->d_group_of_light;
            p.plane_values = film_pixels * 3;
            p.n_planes = accum->n_planes;
            if (accum->mode == FILM_MODE_LPE)
            {
                p.lpe_next = ctx->d_lpe_next;
                p.lpe_accept = ctx->d_lpe_accept;
                p.lpe_light_symbol = ctx->d_lpe_light_symbol;
                p.lpe_symbols = ctx->lpe_symbols;
            }
        }
        if (filtered)
        {
            p.filmp.rgb = film_rgb; p.filmp.wsum = film_wsum;
            p.filmp.cache = ctx->film.cache_size ? ctx->d_film_cache : nullptr;
            p.filmp.radius = ctx->film.radius;
            p.filmp.two_inv_radius = 2.0 / ctx->film.radius;
            p.filmp.inv_dx = ctx->film.cache_size ? (double)(ctx->film.cache_size - 1) / ctx->film.radius : 0.0;
            p.filmp.filter = ctx->film.filter; p.filmp.cache_size = ctx->film.cache_size;
            p.filmp.width = cam->width; p.filmp.height = cam->height;
        }
        p.user_rays = d_user_rays; p.user_pixel = d_user_pixel; p.user_sample = d_user_sample;
        p.pixel_list = d_pixel_list;
        p.capacity = wb.capacity;
        p.global_seed = global_seed;
        p.spp = spp;
        p.row_first = row_first;
        p.row_step = row_step;
        p.n_pixels = n_pixels;
        p.integrator = (uint32_t)integrator;
        p.ray_eps = rayEps<R>(ctx);
        std::memset(&p.sort, 0, sizeof(p.sort));
        if (ctx->sort_rays)
        {
            if ((rc = ensureSort(ctx))) return rc;
            p.sort = ctx->sort;
            p.sort.shade_sorted = ctx->sort_shade ? 1u : 0u;
            if (!ctx->sort_shade_class || integrator == MCRT_INTERNAL_EMIT) p.sort.shade_order = nullptr;
            {
                // source-primitive keys for scenes with enough primitives to index space finely
                const uint32_t n_prims = sceneOf<R>(ctx).n_prims;
                const double cells = (double)(1u << (3 * SORT_ORIGIN_BITS));
                // fewer primitives than cells: the scale would not fit 32 bits, and origin cells are finer anyway
                const bool use_prim = (ctx->sort_prim_key < 0 ? n_prims >= 4096u : ctx->sort_prim_key != 0) && (double)n_prims >= cells;
                p.sort.prim_scale = use_prim ? (uint32_t)(cells * 4294967296.0 / (double)n_prims * 0.999999) : 0u;
            }
            for (int k = 0; k < 3; k++)
            {
                const double ext = ctx->scene_bmax[k] - ctx->scene_bmin[k];
                p.sort.key_min[k] = (float)ctx->scene_bmin[k];
                p.sort.key_scale[k] = ext > 0.0 ? (float)((double)(1u << SORT_ORIGIN_BITS) / ext) : 0.0f;
            }
        }

        const bool emitting = integrator == MCRT_INTERNAL_EMIT;
        if (emitting)
        {
            p.emit.emit_offsets = ctx->d_emit_offsets;
            p.emit.photon_flux = static_cast<const V4<R>*>(ctx->d_emit_flux);
            p.emit.photons[0] = ctx->d_emit_photons[0]; p.emit.photons[1] = ctx->d_emit_photons[1];
            p.emit.lights[0] = ctx->d_emit_lights[0]; p.emit.lights[1] = ctx->d_emit_lights[1];
            p.emit.capacity[0] = ctx->emit_capacity[0]; p.emit.capacity[1] = ctx->emit_capacity[1];
            p.emit.non_caustic_reject = (R)ctx->emit_non_caustic_reject;
            p.emit.pass = ctx->emit_pass;
            if (ctx->d_emit_lpe_states[0])
            {
                p.emit.lpe_states[0] = ctx->d_emit_lpe_states[0]; p.emit.lpe_states[1] = ctx->d_emit_lpe_states[1];
                p.emit.lpe_rev_next = ctx->d_lpe_rev_next;
                p.emit.lpe_rev_start = ctx->lpe_rev_start;
                p.lpe_light_symbol = ctx->d_lpe_light_symbol;
                p.lpe_symbols = ctx->lpe_symbols;
            }
        }
        if (integrator == MCRT_INTEGRATOR_PHOTON)
        {
            p.pm.map[0] = ctx->photon_map[0]; p.pm.map[1] = ctx->photon_map[1];
            p.pm.queries = knn_queue;
            p.pm.k_nearest = ctx->k_nearest;
            p.pm.direct_visualization = ctx->direct_visualization;
            p.pm.query_capacity = knn_capacity;
            p.pm.gather_r2[0] = ctx->gather_r2[0]; p.pm.gather_r2[1] = ctx->gather_r2[1];
            if (ctx->photon_lights) { p.pm.lights[0] = ctx->built_dev[0].lights; p.pm.lights[1] = ctx->built_dev[1].lights; }
            if (p.film_mode == FILM_MODE_LPE)
            {
                p.pm.lpe_states[0] = ctx->built_dev[0].lpe_states; p.pm.lpe_states[1] = ctx->built_dev[1].lpe_states;
                p.pm.lpe_join = ctx->d_lpe_join;
                p.pm.lpe_join_any = ctx->d_lpe_join_any;
                p.pm.lpe_rev_states = ctx->lpe_rev_states;
            }
        }

        Counters init;
        std::memset(&init, 0, sizeof(init));
        init.total_work = total_work;
        if (sample_first)
        {
            // work item w is sample w / n_pixels of pixel w % n_pixels: starting the work index at sample_first * n_pixels
            // renders samples sample_first.. without a kernel change (< 2^64: both factors are below 2^32)
            init.next_work = (uint64_t)sample_first * n_pixels;
            init.total_work = init.next_work + total_work;
        }
        if (integrator == MCRT_INTERNAL_EMIT) { init.next_work = ctx->emit_work_first; init.total_work = ctx->emit_work_first + total_work; }
        ctx->h_counters[0] = init;
        CK(cudaEventRecord(ctx->ev_start, s));   // the timed region includes the counter upload and the film / histogram memsets
        CK(cudaMemcpyAsync(ctx->d_counters, &ctx->h_counters[0], sizeof(Counters), cudaMemcpyHostToDevice, s));
        if (!accum)
        {
            CK(cudaMemsetAsync(ctx->d_film, 0, film_pixels * 3 * sizeof(double), s));
            if (filtered) CK(cudaMemsetAsync(ctx->d_film_wsum, 0, film_pixels * sizeof(double), s));
        }
        const bool sorting = ctx->sort_rays != 0;
        if (sorting)
        {
            CK(cudaMemsetAsync(p.sort.hist_path, 0, SORT_BINS * sizeof(uint32_t), s));
            CK(cudaMemsetAsync(p.sort.hist_shadow, 0, SORT_BINS * sizeof(uint32_t), s));
            CK(cudaMemsetAsync(ctx->sort.hist_shade, 0, SORT_BINS * sizeof(uint32_t), s));
        }
        auto sortPaths = [&](int buffer)
        {
            launchSortScan(p.sort.hist_path, p.sort, s);
            launchSortScatter(p.sort.path_key[buffer], p.sort.path_rank[buffer], p.sort, p.sort.path_order,
                              &ctx->d_counters->n_cur, grid, s);
        };

        uint64_t launches = 0, iterations = 0;

        if (emitting) Launch<R>::emitGenerate(p, 0, grid, s);
        else Launch<R>::generate(p, 0, grid, s);
        launchAdvance(ctx->d_counters, s);
        launches += 2;
        if (sorting) { sortPaths(0); launches += 2; }

        // Enqueue iterations ahead of the GPU; poll the queue counters through pinned memory every
        // poll_interval iterations with one poll of look-ahead, so the device never waits on the host.
        int pending[2] = { 0, 0 };
        int slot = 0;
        bool done = false;
        while (!done)
        {
            for (int k = 0; k < ctx->poll_interval; k++)
            {
                const int cur = (int)(iterations & 1u);
                cudaEvent_t* ev = nullptr;
                if (ctx->stage_timing)
                {
                    while (ctx->stage_events.size() < 6 * (iterations + 1))
                    {
                        cudaEvent_t e;
                        CK(cudaEventCreate(&e));
                        ctx->stage_events.push_back(e);
                    }
                    ev = &ctx->stage_events[6 * iterations];
                    cudaEventRecord(ev[0], s);
                }
                Launch<R>::extend(p, cur, grid, s);
                if (ev) cudaEventRecord(ev[1], s);
                if (p.sort.shade_order)
                {
                    // group the paths by the material class of what they hit (counted with the shade stage)
                    Launch<R>::shadeKey(p, grid, s);
                    launchSortScan(p.sort.hist_shade, p.sort, s);
                    launchSortScatter(p.sort.shade_key, p.sort.shade_rank, p.sort, p.sort.shade_order, &ctx->d_counters->n_cur, grid, s);
                    launches += 3;
                }
                if (emitting)
                {
                    Launch<R>::emitShade(p, cur, grid, s);
                }
                else if (integrator == MCRT_INTEGRATOR_PHOTON)
                {
                    Launch<R>::shadePhoton(p, cur, grid, s);
                    if (ev) cudaEventRecord(ev[5], s);
                    Launch<R>::knn(p, grid, s);
                    launches += 1;
                }
                else
                {
                    Launch<R>::shade(p, cur, grid, s);
                }
                if (ev) cudaEventRecord(ev[2], s);
                if (!emitting)
                {
                    if (sorting)
                    {
                        launchSortScan(p.sort.hist_shadow, p.sort, s);
                        launchSortScatter(p.sort.shadow_key, p.sort.shadow_rank, p.sort, p.sort.shadow_order,
                                          &ctx->d_counters->n_shadow, grid, s);
                        launches += 2;
                    }
                    Launch<R>::shadow(p, grid, s);
                }
                if (ev) cudaEventRecord(ev[3], s);
                if (emitting) Launch<R>::emitGenerate(p, cur ^ 1, grid, s);
                else Launch<R>::generate(p, cur ^ 1, grid, s);
                launchAdvance(ctx->d_counters, s);
                if (sorting) { sortPaths(cur ^ 1); launches += 2; }
                if (ev) cudaEventRecord(ev[4], s);
                launches += 5;
                iterations++;
            }
            CK(cudaMemcpyAsync(&ctx->h_counters[slot], ctx->d_counters, sizeof(Counters), cudaMemcpyDeviceToHost, s));
            CK(cudaEventRecord(ctx->ev_poll[slot], s));
            pending[slot] = 1;
            const int other = slot ^ 1;
            if (pending[other])
            {
                CK(cudaEventSynchronize(ctx->ev_poll[other]));
                const Counters& c = ctx->h_counters[other];
                if (c.n_cur == 0 && c.next_work >= c.total_work) done = true;
                pending[other] = 0;
            }
            slot = other;
        }

        if (!emitting && !accum)
        {
            if (filtered) launchResolveFilmWeighted(ctx->d_film, ctx->d_film_wsum, out_dev, film_pixels, grid, s);
            else if (ctx->peer_out.n_frames) launchResolveFilmPeers(ctx->d_film, ctx->peer_out, film_pixels * 3, film_weight, grid, s);
            else launchResolveFilm(ctx->d_film, out_dev, film_pixels * 3, film_weight, grid, s);
            launches += 1;
        }
        CK(cudaEventRecord(ctx->ev_stop, s));
        CK(cudaMemcpyAsync(&ctx->h_counters[0], ctx->d_counters, sizeof(Counters), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        CK(cudaGetLastError());
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop));
        const Counters& c = ctx->h_counters[0];
        fillStats(stats, c, iterations, launches, ms);
        if (stats)
        {
            stats->extend_launches = iterations;
            stats->shadow_launches = iterations;
            if (ctx->stage_timing)
            {
                for (uint64_t it = 0; it < iterations; it++)
                {
                    cudaEvent_t* ev = &ctx->stage_events[6 * it];
                    if (integrator == MCRT_INTEGRATOR_PHOTON) { float tk = 0; cudaEventElapsedTime(&tk, ev[5], ev[2]); stats->gpu_ms_knn += tk; }
                    float t01 = 0, t12 = 0, t23 = 0, t34 = 0;
                    cudaEventElapsedTime(&t01, ev[0], ev[1]); cudaEventElapsedTime(&t12, ev[1], ev[2]);
                    cudaEventElapsedTime(&t23, ev[2], ev[3]); cudaEventElapsedTime(&t34, ev[3], ev[4]);
                    stats->gpu_ms_extend += t01; stats->gpu_ms_shade += t12;
                    stats->gpu_ms_shadow += t23; stats->gpu_ms_generate += t34;
                }
            }
        }
        if (c.traversal_overflow)
        {
            ctx->error = "traversal stack/heap overflow: result would differ from the reference";
            return MCRT_ERR_UNSUPPORTED;
        }
        if (c.ior_stack_overflows)
        {
            // RefractionHistory::iors is an unbounded vector in the reference (ray.cpp:74-98); the device
            // stack holds IOR_STACK_CAPACITY nested media. Beyond that externalIOR would be wrong: refuse.
            ctx->error = "more than 8 nested dielectric media on a path (refraction-history stack overflow): result would differ from the reference";
            return MCRT_ERR_UNSUPPORTED;
        }
        if (emitting && c.photon_overflow)
        {
            ctx->error = "photon arrays overflowed";
            return MCRT_ERR_UNSUPPORTED;
        }
        return MCRT_OK;
    }

    // ---------------------------------------------------------------------------------------
    // Octree<Photon> + LinearOctree::compact on the host (octree.cpp:34-81, linear-octree.cpp:201-244).
    // Samples [sample_first, sample_first + spp) of every pixel of rows y_first + k*y_step, k < n_rows: resolved into
    // out_dev, or added into the caller's sums when accum is given. d_pixel_list (accumulate mode only): only the n_list
    // pixels it lists (positions in the n_rows x width grid) are rendered.
    int renderDispatch(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                       uint32_t sample_first, uint64_t spp, uint32_t global_seed, int integrator_kind, int precision,
                       double* out_dev, mcrt_stats* stats, const FilmSums* accum = nullptr,
                       const uint32_t* d_pixel_list = nullptr, uint32_t n_list = 0)
    {
        if (!camera || n_rows == 0 || y_step == 0 || spp == 0 || camera->width == 0 ||
            (uint64_t)y_first + (uint64_t)(n_rows - 1) * y_step >= camera->height)
        {
            ctx->error = "mcrt_render_rows: invalid camera / row range / sample count";
            return MCRT_ERR_INVALID;
        }
        if ((uint64_t)sample_first + spp > 0x100000000ull)
        {
            ctx->error = "sample range beyond 2^32 samples per pixel";
            return MCRT_ERR_INVALID;
        }
        if (!ctx->film_default && !accum && (y_first != 0 || y_step != 1 || n_rows != camera->height))
        {
            ctx->error = "a reconstruction filter other than the default box splats across rows: render the whole frame in one call";
            return MCRT_ERR_UNSUPPORTED;
        }
        const uint64_t n_pixels64 = (uint64_t)camera->width * n_rows;
        if (n_pixels64 > 0xFFFFFFFFull) { ctx->error = "row block too large"; return MCRT_ERR_INVALID; }
        const uint32_t n_pixels = (uint32_t)n_pixels64;
        const uint32_t n_work = d_pixel_list ? n_list : n_pixels;   // pixels the camera work covers
        const uint64_t total = (uint64_t)n_work * spp;
        // a filtered film accumulates at image positions (samples splat across rows): its buffers span the whole frame
        const size_t film_pixels = ctx->film_default ? (size_t)n_pixels : (size_t)camera->width * camera->height;
        if (precision == MCRT_PRECISION_F64)
            return runWavefront<double>(ctx, camera, y_first, y_step, n_work, (uint32_t)spp, total, global_seed, integrator_kind,
                                        nullptr, nullptr, nullptr, film_pixels, (double)spp, out_dev, stats, sample_first, accum,
                                        d_pixel_list);
        if (precision == MCRT_PRECISION_F32)
            return runWavefront<float>(ctx, camera, y_first, y_step, n_work, (uint32_t)spp, total, global_seed, integrator_kind,
                                       nullptr, nullptr, nullptr, film_pixels, (double)spp, out_dev, stats, sample_first, accum,
                                       d_pixel_list);
        ctx->error = "unknown precision";
        return MCRT_ERR_INVALID;
    }

    // One-shot frame: sqrtspp² samples per pixel (Camera::sampleImage)
    int renderFrame(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                    uint32_t sqrtspp, uint32_t global_seed, int integrator_kind, int precision, double* out_dev,
                    mcrt_stats* stats, const FilmSums* accum = nullptr)
    {
        if (sqrtspp == 0 || sqrtspp > 65535u)
        {
            ctx->error = "mcrt_render_rows: invalid camera / row range / sqrtspp";
            return MCRT_ERR_INVALID;
        }
        return renderDispatch(ctx, camera, y_first, y_step, n_rows, 0u, (uint64_t)sqrtspp * sqrtspp, global_seed,
                              integrator_kind, precision, out_dev, stats, accum);
    }

    // Arguments of the accumulate entry points: a sample count and sums that match the film
    int checkAccumulateSums(mcrt_ctx* ctx, const char* fn, uint32_t sample_count, const double* rgb_sum_dev,
                            const double* weight_sum_dev)
    {
        const std::string name(fn);
        if (!rgb_sum_dev) { ctx->error = name + ": null rgb sums"; return MCRT_ERR_INVALID; }
        if (sample_count == 0) { ctx->error = name + ": sample_count is 0"; return MCRT_ERR_INVALID; }
        if (ctx->film_default && weight_sum_dev)
        {
            ctx->error = name + ": the box film is weighted by the sample count; weight_sum_dev must be NULL";
            return MCRT_ERR_INVALID;
        }
        if (!ctx->film_default && !weight_sum_dev)
        {
            ctx->error = name + ": a reconstruction filter needs weight_sum_dev";
            return MCRT_ERR_INVALID;
        }
        return MCRT_OK;
    }
}

extern "C" int mcrt_photon_upload(mcrt_ctx* ctx, const mcrt_photon_map_desc* caustic_map, const mcrt_photon_map_desc* global_map,
                                  uint32_t k_nearest, uint32_t direct_visualization, uint64_t* h2d_bytes);

extern "C"
{

int mcrt_abi_version(void) { return MCRT_ABI_VERSION; }

int mcrt_init(int device, mcrt_ctx** out_ctx)
{
    if (!out_ctx) return MCRT_ERR_INVALID;
    *out_ctx = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return MCRT_ERR_CUDA;
    mcrt_ctx* ctx = new mcrt_ctx();
    if (const char* e = std::getenv("MCRT_BVH4_MAX_LEAF")) ctx->bvh4_max_leaf = (uint32_t)std::atoi(e);   // tuning experiments
    if (const char* e = std::getenv("MCRT_BVH4_SPLIT")) ctx->bvh4_split = std::atoi(e);
    if (const char* e = std::getenv("MCRT_BVH4_SPLIT_COST")) ctx->bvh4_split_cost = std::atof(e);
    ctx->device = device;
    auto fail = [&](int rc) { mcrt_destroy(ctx); return rc; };
    if (cudaSetDevice(device) != cudaSuccess) return fail(MCRT_ERR_CUDA);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(MCRT_ERR_CUDA);
    ctx->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) return fail(MCRT_ERR_CUDA);
    if (cudaMalloc((void**)&ctx->d_counters, sizeof(Counters)) != cudaSuccess) return fail(MCRT_ERR_CUDA);
    if (cudaMallocHost((void**)&ctx->h_counters, 2 * sizeof(Counters)) != cudaSuccess) return fail(MCRT_ERR_CUDA);
    {
        std::vector<uint32_t> tab(6 * 4 * 256);
        makeSobolByteTable(tab.data());
        if (cudaMalloc((void**)&ctx->d_sobol_bytes, tab.size() * 4) != cudaSuccess) return fail(MCRT_ERR_CUDA);
        if (cudaMemcpy(ctx->d_sobol_bytes, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) return fail(MCRT_ERR_CUDA);
    }
    if (cudaEventCreate(&ctx->ev_start) != cudaSuccess || cudaEventCreate(&ctx->ev_stop) != cudaSuccess) return fail(MCRT_ERR_CUDA);
    for (int i = 0; i < 2; i++)
        if (cudaEventCreateWithFlags(&ctx->ev_poll[i], cudaEventDisableTiming) != cudaSuccess) return fail(MCRT_ERR_CUDA);
    *out_ctx = ctx;
    return MCRT_OK;
}

void mcrt_destroy(mcrt_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    freeAll(ctx->scene_allocs);
    freeAll(ctx->wave_allocs64);
    freeAll(ctx->wave_allocs32);
    freeAll(ctx->sort_allocs);
    freeAll(ctx->photon_allocs);
    if (ctx->knn_queue64) cudaFree(ctx->knn_queue64);
    if (ctx->knn_queue32) cudaFree(ctx->knn_queue32);
    if (ctx->d_film) cudaFree(ctx->d_film);
    if (ctx->d_film_wsum) cudaFree(ctx->d_film_wsum);
    if (ctx->d_film_cache) cudaFree(ctx->d_film_cache);
    if (ctx->d_host_out) cudaFree(ctx->d_host_out);
    if (ctx->d_resolve_scratch) cudaFree(ctx->d_resolve_scratch);
    if (ctx->d_denoise_scratch) cudaFree(ctx->d_denoise_scratch);
    if (ctx->d_denoise_planes_scratch) cudaFree(ctx->d_denoise_planes_scratch);
    if (ctx->d_pixel_list) cudaFree(ctx->d_pixel_list);
    if (ctx->d_group_of_light) cudaFree(ctx->d_group_of_light);
    if (ctx->d_group_weights) cudaFree(ctx->d_group_weights);
    if (ctx->d_lpe_next) cudaFree(ctx->d_lpe_next);
    if (ctx->d_lpe_accept) cudaFree(ctx->d_lpe_accept);
    if (ctx->d_lpe_light_symbol) cudaFree(ctx->d_lpe_light_symbol);
    if (ctx->d_lpe_rev_next) cudaFree(ctx->d_lpe_rev_next);
    if (ctx->d_lpe_join) cudaFree(ctx->d_lpe_join);
    if (ctx->d_lpe_join_any) cudaFree(ctx->d_lpe_join_any);
    if (ctx->d_counters) cudaFree(ctx->d_counters);
    if (ctx->d_sobol_bytes) cudaFree(ctx->d_sobol_bytes);
    if (ctx->h_counters) cudaFreeHost(ctx->h_counters);
    if (ctx->ev_start) cudaEventDestroy(ctx->ev_start);
    if (ctx->ev_stop) cudaEventDestroy(ctx->ev_stop);
    for (int i = 0; i < 2; i++) if (ctx->ev_poll[i]) cudaEventDestroy(ctx->ev_poll[i]);
    for (cudaEvent_t e : ctx->stage_events) cudaEventDestroy(e);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* mcrt_last_error(const mcrt_ctx* ctx)
{
    return ctx ? ctx->error.c_str() : "null context";
}

int mcrt_set_option(mcrt_ctx* ctx, const char* key, double value)
{
    if (!ctx || !key) return MCRT_ERR_INVALID;
    std::string k(key);
    if (k == "pool_paths") { if (value < 1024 || value > 268435456.0) return MCRT_ERR_INVALID; ctx->pool_paths = (uint32_t)value; }
    else if (k == "blocks_per_sm") { if (value < 1 || value > 32) return MCRT_ERR_INVALID; ctx->blocks_per_sm = (int)value; }
    else if (k == "ray_eps_scale") { if (value <= 0) return MCRT_ERR_INVALID; ctx->ray_eps_scale = value; }
    else if (k == "poll_interval") { if (value < 1 || value > 1024) return MCRT_ERR_INVALID; ctx->poll_interval = (int)value; }
    else if (k == "stage_timing") { ctx->stage_timing = value != 0.0; }
    else if (k == "sort_rays") { ctx->sort_rays = value != 0.0; }
    else if (k == "sort_shade") { ctx->sort_shade = value != 0.0; }
    else if (k == "sort_shade_class") { ctx->sort_shade_class = value != 0.0; }
    else if (k == "sort_prim_key") { ctx->sort_prim_key = (int)value; }
    else if (k == "exact_traversal") { ctx->exact_traversal = value != 0.0; }
    else if (k == "dynamic_fetch") { ctx->dynamic_fetch = (int)value; }
    else if (k == "bvh4_split") { if (value < -1 || value > 1) return MCRT_ERR_INVALID; ctx->bvh4_split = (int)value; }   // takes effect at the next mcrt_scene_upload
    else if (k == "bvh4_max_leaf") { if (value < 0 || value > 255) return MCRT_ERR_INVALID; ctx->bvh4_max_leaf = (uint32_t)value; }   // takes effect at the next mcrt_scene_upload
    else { ctx->error = "unknown option " + k; return MCRT_ERR_INVALID; }
    return MCRT_OK;
}

int mcrt_scene_upload(mcrt_ctx* ctx, const mcrt_scene_desc* scene, uint64_t* h2d_bytes)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!scene || scene->abi_version != MCRT_ABI_VERSION) { ctx->error = "scene description missing or ABI version mismatch"; return MCRT_ERR_INVALID; }
    if (scene->n_prims == 0 || scene->n_materials == 0) { ctx->error = "empty scene"; return MCRT_ERR_INVALID; }
    if (scene->n_prims >= (1u << 24)) { ctx->error = "more than 2^24 primitives"; return MCRT_ERR_UNSUPPORTED; }
    CK(cudaSetDevice(ctx->device));
    const mcrt_scene_desc& s = *scene;

    // structural validation of the BVH links (a malformed tree must not hang the device)
    for (uint32_t i = 0; i < s.n_nodes; i++)
    {
        if (s.node_next_sibling[i] != 0 && (s.node_next_sibling[i] <= i || s.node_next_sibling[i] >= s.n_nodes))
        { ctx->error = "node_next_sibling must point forward"; return MCRT_ERR_INVALID; }
        if ((uint64_t)s.node_first_prim[i] + s.node_prim_count[i] > s.n_prims)
        { ctx->error = "node primitive range out of bounds"; return MCRT_ERR_INVALID; }
        if (s.node_prim_count[i] == 0 && i + 1 >= s.n_nodes)
        { ctx->error = "inner node without children"; return MCRT_ERR_INVALID; }
    }
    for (uint32_t i = 1; i < s.n_lights; i++)
    {
        if (s.light_cdf[i] < s.light_cdf[i - 1]) { ctx->error = "light_cdf must be non-decreasing"; return MCRT_ERR_INVALID; }
    }

    freeAll(ctx->scene_allocs);
    ctx->has_scene = false;
    ctx->has_light_groups = false;
    ctx->n_light_groups = 0;
    ctx->lpe_n = 0;
    ctx->photon_lights = false;   // the maps' light indices name the lights of the previous scene
    ctx->photon_lpe_identity.clear();
    ctx->photon_lpe_states = false;

    // scene scale for the fast mode's ray offsets
    double scale = 0.0;
    auto grow = [&](const double* p, int n) { for (int i = 0; i < n; i++) { double v = p[i] < 0 ? -p[i] : p[i]; if (v < 1e300 && v > scale) scale = v; } };
    if (s.n_nodes) grow(s.node_bounds, 6);
    else
    {
        grow(s.tri_v0, 3 * s.n_tris); grow(s.tri_v1, 3 * s.n_tris); grow(s.tri_v2, 3 * s.n_tris);
        for (uint32_t i = 0; i < s.n_spheres; i++) { double m = 0; for (int k = 0; k < 3; k++) { double v = s.sphere_origin_radius[4 * i + k]; v = v < 0 ? -v : v; if (v > m) m = v; } m += s.sphere_origin_radius[4 * i + 3]; if (m > scale) scale = m; }
        grow(s.quadric_bounds, 6 * s.n_quadrics);
    }
    ctx->scene_scale = scale > 0.0 ? (float)scale : 1.0f;
    {
        // bounds for the sort key grid: root node box, or the union of primitive extents without a BVH
        double lo[3] = { 1e300, 1e300, 1e300 }, hi[3] = { -1e300, -1e300, -1e300 };
        auto add = [&](const double* q) { for (int k = 0; k < 3; k++) { if (q[k] < lo[k]) lo[k] = q[k]; if (q[k] > hi[k]) hi[k] = q[k]; } };
        if (s.n_nodes) { add(s.node_bounds); add(s.node_bounds + 3); }
        else
        {
            for (uint32_t i = 0; i < s.n_tris; i++) { add(s.tri_v0 + 3 * i); add(s.tri_v1 + 3 * i); add(s.tri_v2 + 3 * i); }
            for (uint32_t i = 0; i < s.n_spheres; i++)
            {
                const double* sp = s.sphere_origin_radius + 4 * i;
                double a[3] = { sp[0] - sp[3], sp[1] - sp[3], sp[2] - sp[3] }, b[3] = { sp[0] + sp[3], sp[1] + sp[3], sp[2] + sp[3] };
                add(a); add(b);
            }
            for (uint32_t i = 0; i < s.n_quadrics; i++) { add(s.quadric_bounds + 6 * i); add(s.quadric_bounds + 6 * i + 3); }
        }
        for (int k = 0; k < 3; k++)
        {
            const bool ok = lo[k] <= hi[k] && lo[k] > -1e290 && hi[k] < 1e290;
            ctx->scene_bmin[k] = ok ? lo[k] : -1.0;
            ctx->scene_bmax[k] = ok ? hi[k] : 1.0;
        }
    }

    uint64_t bytes = 0;
    int rc;
    {
        SceneArrays<double> a;
        if ((rc = buildArrays(ctx, s, a))) return rc;
        std::memset(&a.dev, 0, sizeof(a.dev));
        if ((rc = buildWide(ctx, s, a))) return rc;
        if ((rc = uploadArrays(ctx, s, a, bytes))) return rc;
        std::vector<Bvh4Node> bvh4;
        if ((rc = buildBvh4(ctx->bvh4_max_leaf, s, bvh4))) return rc;
        ctx->n_bvh4_nodes = (uint32_t)bvh4.size();   // dynamic fetch's auto rule counts the tree without spatial splits
        a.dev.bvh4 = nullptr; a.dev.bvh4_geom = nullptr; a.dev.bvh4_prim = nullptr;
        std::vector<uint32_t> refs;
        std::vector<V4<double>> ref_geom;
        if (!bvh4.empty())
        {
            // spatial splits where buildBvh4 cuts the reference's leaves (small scenes); big scenes keep the reference's leaves
            const bool split = ctx->bvh4_split < 0 ? ctx->bvh4_max_leaf == 0xFFFFFFFFu && s.n_prims < 4096u : ctx->bvh4_split != 0;
            if (split)
            {
                std::vector<Bvh4Node> split_nodes;
                if ((rc = buildBvh4Split(s, ctx->bvh4_split_cost, 2.0, split_nodes, refs))) return rc;
                if (!split_nodes.empty()) bvh4.swap(split_nodes);
                else refs.clear();
            }
            if (refs.empty())
            {
                refs.resize(s.n_prims);
                for (uint32_t i = 0; i < s.n_prims; i++) refs[i] = i;
                a.dev.bvh4_geom = a.dev.geom;
            }
            else
            {
                ref_geom.resize(3 * refs.size());
                for (size_t r = 0; r < refs.size(); r++) for (int j = 0; j < 3; j++) ref_geom[3 * r + j] = a.geom[3 * (size_t)refs[r] + j];
                if ((rc = devUpload(ctx, ctx->scene_allocs, &a.dev.bvh4_geom, ref_geom, bytes))) return rc;
            }
            if ((rc = devUpload(ctx, ctx->scene_allocs, &a.dev.bvh4_prim, refs, bytes))) return rc;
            if ((rc = devUpload(ctx, ctx->scene_allocs, &a.dev.bvh4, bvh4, bytes))) return rc;
        }
        CK(cudaStreamSynchronize(ctx->stream)); // host vectors die at scope exit
        ctx->scene64 = a.dev;
    }
    {
        SceneArrays<float> a;
        if ((rc = buildArrays(ctx, s, a))) return rc;
        std::memset(&a.dev, 0, sizeof(a.dev));
        if ((rc = buildWide(ctx, s, a))) return rc;
        if ((rc = uploadArrays(ctx, s, a, bytes))) return rc;
        CK(cudaStreamSynchronize(ctx->stream));
        ctx->scene32 = a.dev;
    }
    ctx->prim_interpolates.assign(s.n_prims, 0);
    for (uint32_t i = 0; i < s.n_prims; i++)
        if (s.prim_type[i] == MCRT_PRIM_TRIANGLE && s.tri_vn_index[s.prim_index[i]] >= 0) ctx->prim_interpolates[i] = 1;
    {
        // light groups need every emitter the paths can hit to be a light (buildArrays has checked the indices)
        std::vector<uint8_t> lit(s.n_prims, 0);
        for (uint32_t i = 0; i < s.n_lights; i++) lit[s.light_prim[i]] = 1;
        ctx->emissive_unlit = false;
        for (uint32_t i = 0; i < s.n_prims && !ctx->emissive_unlit; i++)
            ctx->emissive_unlit = s.materials[s.prim_material[i]].emissive && !lit[i];
    }
    ctx->has_scene = true;
    if (h2d_bytes) *h2d_bytes = bytes;
    return MCRT_OK;
}

int mcrt_photon_upload(mcrt_ctx* ctx, const mcrt_photon_map_desc* caustic_map, const mcrt_photon_map_desc* global_map,
                       uint32_t k_nearest, uint32_t direct_visualization, uint64_t* h2d_bytes)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!caustic_map || !global_map || k_nearest == 0) { ctx->error = "mcrt_photon_upload: invalid arguments"; return MCRT_ERR_INVALID; }
    if (k_nearest > 1024) { ctx->error = "k_nearest_photons > 1024 unsupported"; return MCRT_ERR_UNSUPPORTED; }
    CK(cudaSetDevice(ctx->device));
    // the maps mcrt_photon_emit built live in photon_allocs too: forget them before they are freed
    ctx->built_valid = false;
    for (int w = 0; w < 2; w++) { ctx->built_dev[w] = PhotonOctreeDevice(); ctx->built_host_current[w] = false; ctx->photon_map[w] = DevicePhotonMap(); }
    freeAll(ctx->photon_allocs);
    ctx->has_photons = false;
    ctx->photon_lights = false;
    ctx->photon_lpe_identity.clear();
    ctx->photon_lpe_states = false;
    uint64_t bytes = 0;
    const mcrt_photon_map_desc* maps[2] = { caustic_map, global_map };
    for (int w = 0; w < 2; w++)
    {
        const mcrt_photon_map_desc& m = *maps[w];
        if (m.n_photons >= 0xFFFFFFFFull) { ctx->error = "photon map with >= 2^32 photons unsupported"; return MCRT_ERR_UNSUPPORTED; }
        std::vector<DeviceOctant> oct(m.n_octants);
        for (uint32_t i = 0; i < m.n_octants; i++)
        {
            DeviceOctant& o = oct[i];
            for (int k = 0; k < 3; k++) { o.bmin[k] = m.octant_bounds[6 * i + k]; o.bmax[k] = m.octant_bounds[6 * i + 3 + k]; }
            o.start = m.octant_start[i]; o.count = m.octant_count[i];
            o.leaf = m.octant_leaf[i];
            o.n_children = 0;
            for (int k = 0; k < 8; k++) o.children[k] = OCTANT_NULL;
            if (o.start + o.count > m.n_photons) { ctx->error = "octant photon range out of bounds"; return MCRT_ERR_INVALID; }
            if (!o.leaf)
            {
                // children = node+1 followed along next_sibling (linear-octree.cpp:88-103)
                uint32_t c = i + 1;
                while (c != OCTANT_NULL)
                {
                    if (c <= i || c >= m.n_octants || o.n_children >= 8) { ctx->error = "malformed octree links"; return MCRT_ERR_INVALID; }
                    o.children[o.n_children++] = c;
                    c = m.octant_next_sibling[c];
                }
            }
        }
        const DeviceOctant* d_oct = nullptr;
        int rc = devUpload(ctx, ctx->photon_allocs, &d_oct, oct, bytes);
        if (rc) return rc;
        float4* d_ph = nullptr;
        if ((rc = devAlloc(ctx, ctx->photon_allocs, &d_ph, (size_t)m.n_photons * 2))) return rc;
        if (m.n_photons)
        {
            CK(cudaMemcpyAsync(d_ph, m.photons, (size_t)m.n_photons * 32, cudaMemcpyHostToDevice, ctx->stream));
            bytes += m.n_photons * 32;
        }
        CK(cudaStreamSynchronize(ctx->stream)); // `oct` dies at scope exit
        ctx->photon_map[w].octants = d_oct;
        ctx->photon_map[w].photons = d_ph;
        ctx->photon_map[w].n_octants = m.n_octants;
        ctx->photon_map[w].n_photons = m.n_photons;
    }
    ctx->k_nearest = k_nearest;
    ctx->direct_visualization = direct_visualization;
    ctx->has_photons = true;
    if (h2d_bytes) *h2d_bytes = bytes;
    return MCRT_OK;
}


// Emission index space of PhotonMapper::PhotonMapper (photon-mapper.cpp:38-78): work item w = emission j of light l,
// offsets[l] <= w < offsets[l+1], emissions per light proportional to its flux. -> offsets, per-photon flux.
static int emissionPlan(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, std::vector<unsigned long long>& offsets,
                        std::vector<V4<double>>& flux64, std::vector<V4<float>>& flux32)
{
    if (!params || params->emissions == 0 || !(params->caustic_factor > 0.0) || params->max_photons_per_octree_leaf == 0 ||
        params->k_nearest_photons == 0)
    { ctx->error = "mcrt_photon_emit: invalid parameters"; return MCRT_ERR_INVALID; }
    if (params->k_nearest_photons > 1024) { ctx->error = "k_nearest_photons > 1024 unsupported"; return MCRT_ERR_UNSUPPORTED; }
    if (!ctx->has_scene) { ctx->error = "no scene uploaded"; return MCRT_ERR_NO_SCENE; }
    CK(cudaSetDevice(ctx->device));
    const DeviceScene<double>& sc = ctx->scene64;
    if (sc.n_lights == 0) { ctx->error = "scene has no emissive surfaces"; return MCRT_ERR_INVALID; }
    std::vector<Light<double>> lights(sc.n_lights);
    CK(cudaMemcpy(lights.data(), sc.lights, sizeof(Light<double>) * sc.n_lights, cudaMemcpyDeviceToHost));
    const size_t photon_emissions = (size_t)((double)params->emissions * params->caustic_factor);
    double total_add_flux = 0.0;
    for (const auto& l : lights) { V3<double> f = l.emittance * l.area; total_add_flux += (0.0 + f.x + f.y + f.z); }
    offsets.assign(sc.n_lights + 1, 0);
    flux64.resize(sc.n_lights); flux32.resize(sc.n_lights);
    for (uint32_t i = 0; i < sc.n_lights; i++)
    {
        const V3<double> light_flux = lights[i].emittance * lights[i].area;
        const double share = (0.0 + light_flux.x + light_flux.y + light_flux.z) / total_add_flux;   // glm::compAdd
        const size_t n_light = (size_t)((double)photon_emissions * share);
        const V3<double> pf = light_flux / (double)n_light;
        offsets[i + 1] = offsets[i] + n_light;
        flux64[i] = V4<double>(pf, 0.0);
        flux32[i] = V4<float>((float)pf.x, (float)pf.y, (float)pf.z, 0.0f);
    }
    if (offsets[sc.n_lights] == 0) { ctx->error = "no emissions"; return MCRT_ERR_INVALID; }
    return MCRT_OK;
}

static void freeEmission(mcrt_ctx* ctx)
{
    freeAll(ctx->emit_allocs);
    ctx->d_emit_offsets = nullptr; ctx->d_emit_flux = nullptr; ctx->d_emit_photons[0] = ctx->d_emit_photons[1] = nullptr;
    ctx->d_emit_lights[0] = ctx->d_emit_lights[1] = nullptr;
    ctx->d_emit_lpe_states[0] = ctx->d_emit_lpe_states[1] = nullptr;
    ctx->emit_stored[0] = ctx->emit_stored[1] = 0;
}

int mcrt_photon_emit_total(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, uint64_t* total_emissions)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!total_emissions) { ctx->error = "null output"; return MCRT_ERR_INVALID; }
    std::vector<unsigned long long> offsets; std::vector<V4<double>> f64; std::vector<V4<float>> f32;
    const int rc = emissionPlan(ctx, params, offsets, f64, f32);
    if (rc) return rc;
    *total_emissions = offsets.back();
    return MCRT_OK;
}

// Work items [work_first, work_first + work_count) of the emission plan; light l's emissions take the reference's
// emission indices pass * n_l + j, j < n_l (pass 0: the reference's own pass).
// lpe: the photons also record their reverse-DFA states when an LPE table the photon mapper takes is set.
static int emitRange(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, int precision, uint32_t pass, uint64_t work_first,
                     uint64_t work_count, const float** caustic_dev, uint64_t* n_caustic, const float** global_dev, uint64_t* n_global,
                     mcrt_stats* stats, bool lpe = false)
{
    std::vector<unsigned long long> offsets; std::vector<V4<double>> flux64; std::vector<V4<float>> flux32;
    int rc = emissionPlan(ctx, params, offsets, flux64, flux32);
    if (rc) return rc;
    const uint64_t total = offsets.back();
    if (work_first > total || work_count > total - work_first) { ctx->error = "mcrt_photon_emit_range: range outside the emission index space"; return MCRT_ERR_INVALID; }
    for (size_t l = 0; l + 1 < offsets.size(); l++)
        if (((unsigned long long)pass + 1ull) * (offsets[l + 1] - offsets[l]) > 0x100000000ull)
        { ctx->error = "mcrt_photon_emit_pass: the pass's emission indices do not fit 32 bits"; return MCRT_ERR_INVALID; }
    if (precision != MCRT_PRECISION_F64 && precision != MCRT_PRECISION_F32) { ctx->error = "unknown precision"; return MCRT_ERR_INVALID; }

    freeEmission(ctx);
    uint64_t bytes = 0;
    const unsigned long long* d_off = nullptr;
    if ((rc = devUpload(ctx, ctx->emit_allocs, &d_off, offsets, bytes))) { freeEmission(ctx); return rc; }
    const void* d_flux = nullptr;
    if (precision == MCRT_PRECISION_F64) { const V4<double>* q = nullptr; rc = devUpload(ctx, ctx->emit_allocs, &q, flux64, bytes); d_flux = q; }
    else { const V4<float>* q = nullptr; rc = devUpload(ctx, ctx->emit_allocs, &q, flux32, bytes); d_flux = q; }
    if (rc) { freeEmission(ctx); return rc; }
    // capacity: a path stores at most one photon per bounce; 4 photons per emission per map is far
    // above what any shipped scene produces (1.2 caustic per emission in water_caustics)
    for (int w = 0; w < 2; w++)
    {
        ctx->emit_capacity[w] = 4ull * work_count + 1024;
        if ((rc = devAlloc(ctx, ctx->emit_allocs, &ctx->d_emit_photons[w], (size_t)ctx->emit_capacity[w] * 2))) { freeEmission(ctx); return rc; }
        if ((rc = devAlloc(ctx, ctx->emit_allocs, &ctx->d_emit_lights[w], (size_t)ctx->emit_capacity[w]))) { freeEmission(ctx); return rc; }
        if (lpe && ctx->lpe_n && ctx->lpe_photon_error.empty() &&
            (rc = devAlloc(ctx, ctx->emit_allocs, &ctx->d_emit_lpe_states[w], (size_t)ctx->emit_capacity[w]))) { freeEmission(ctx); return rc; }
    }
    ctx->d_emit_offsets = d_off; ctx->d_emit_flux = d_flux;
    ctx->emit_non_caustic_reject = 1.0 / params->caustic_factor;
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) { freeEmission(ctx); ctx->error = "mcrt_photon_emit: upload failed"; return MCRT_ERR_CUDA; }

    if (work_count)
    {
        ctx->emit_work_first = work_first;
        ctx->emit_pass = pass;
        if (precision == MCRT_PRECISION_F64)
            rc = runWavefront<double>(ctx, nullptr, 0, 1, 0, 1, work_count, params->global_seed, MCRT_INTERNAL_EMIT, nullptr, nullptr, nullptr, 1, 1.0, nullptr, stats);
        else
            rc = runWavefront<float>(ctx, nullptr, 0, 1, 0, 1, work_count, params->global_seed, MCRT_INTERNAL_EMIT, nullptr, nullptr, nullptr, 1, 1.0, nullptr, stats);
        ctx->emit_work_first = 0;
        ctx->emit_pass = 0;
        if (rc) { freeEmission(ctx); return rc; }
        const Counters& c = ctx->h_counters[0];
        ctx->emit_stored[0] = c.n_photons[0]; ctx->emit_stored[1] = c.n_photons[1];
    }
    else if (stats) std::memset(stats, 0, sizeof(*stats));
    if (caustic_dev) *caustic_dev = reinterpret_cast<const float*>(ctx->d_emit_photons[0]);
    if (global_dev) *global_dev = reinterpret_cast<const float*>(ctx->d_emit_photons[1]);
    if (n_caustic) *n_caustic = ctx->emit_stored[0];
    if (n_global) *n_global = ctx->emit_stored[1];
    return MCRT_OK;
}

int mcrt_photon_emit_range(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, int precision, uint64_t work_first, uint64_t work_count,
                           const float** caustic_dev, uint64_t* n_caustic, const float** global_dev, uint64_t* n_global, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    return emitRange(ctx, params, precision, 0, work_first, work_count, caustic_dev, n_caustic, global_dev, n_global, stats);
}

// mcrt_photon_build_dev; lights_dev: null (the maps carry no light index), or the emitting light of each photon of the
// two arrays (mcrt_photon_emit_pass), reordered with the photons; lpe_states_dev likewise, each photon's reverse-DFA
// state; lpe_identity: null, or the identity of the LPE table the photons were emitted under
static int buildPhotonMaps(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, const float* caustic_dev, uint64_t n_caustic,
                           const float* global_dev, uint64_t n_global, const uint32_t* const lights_dev[2], double* build_ms,
                           const uint32_t* const lpe_states_dev[2] = nullptr, const std::string* lpe_identity = nullptr)
{
    if (!params || params->max_photons_per_octree_leaf == 0 || params->k_nearest_photons == 0 || params->k_nearest_photons > 1024 ||
        (n_caustic && !caustic_dev) || (n_global && !global_dev))
    { ctx->error = "mcrt_photon_build_dev: invalid arguments"; return MCRT_ERR_INVALID; }
    if (n_caustic >= 0xFFFFFFFFull || n_global >= 0xFFFFFFFFull) { ctx->error = "photon map with >= 2^32 photons unsupported"; return MCRT_ERR_UNSUPPORTED; }
    CK(cudaSetDevice(ctx->device));
    // Octree<Photon> + LinearOctree::compact on the device, straight from the photon arrays into
    // the layout k_knn walks: the photons never visit the host.
    ctx->built_valid = false;
    for (int w = 0; w < 2; w++) { ctx->built_dev[w] = PhotonOctreeDevice(); ctx->built_host_current[w] = false; ctx->photon_map[w] = DevicePhotonMap(); }
    freeAll(ctx->photon_allocs);
    ctx->has_photons = false;
    ctx->photon_lights = false;
    ctx->photon_lpe_identity.clear();
    ctx->photon_lpe_states = false;
    ctx->photon_build_ms = 0.0;
    const float4* src[2] = { reinterpret_cast<const float4*>(caustic_dev), reinterpret_cast<const float4*>(global_dev) };
    const uint64_t n[2] = { n_caustic, n_global };
    for (int w = 0; w < 2; w++)
    {
        const int rc = buildPhotonOctreeOnDevice(src[w], (uint32_t)n[w], params->scene_bounds, params->max_photons_per_octree_leaf,
                                                 ctx->sm_count, ctx->stream, ctx->photon_allocs, ctx->built_dev[w], ctx->error,
                                                 lights_dev ? lights_dev[w] : nullptr, lpe_states_dev ? lpe_states_dev[w] : nullptr);
        if (rc) return rc;
        ctx->photon_map[w].octants = ctx->built_dev[w].octants;
        ctx->photon_map[w].photons = ctx->built_dev[w].photons;
        ctx->photon_map[w].n_octants = ctx->built_dev[w].n_octants;
        ctx->photon_map[w].n_photons = ctx->built_dev[w].n_photons;
        ctx->photon_build_ms += ctx->built_dev[w].gpu_ms;
    }
    ctx->k_nearest = params->k_nearest_photons;
    ctx->direct_visualization = params->direct_visualization;
    ctx->has_photons = true;
    ctx->built_valid = true;
    ctx->photon_lights = lights_dev != nullptr;
    ctx->photon_lpe_identity = lpe_identity ? *lpe_identity : std::string();
    ctx->photon_lpe_states = lpe_states_dev != nullptr;
    if (build_ms) *build_ms = ctx->photon_build_ms;
    freeEmission(ctx);   // the raw emission buffers have been consumed (or superseded by the gathered arrays of a sharded pass)
    return MCRT_OK;
}

int mcrt_photon_build_dev(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, const float* caustic_dev, uint64_t n_caustic,
                          const float* global_dev, uint64_t n_global, double* build_ms)
{
    if (!ctx) return MCRT_ERR_INVALID;
    return buildPhotonMaps(ctx, params, caustic_dev, n_caustic, global_dev, n_global, nullptr, build_ms);
}

int mcrt_photon_emit(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, int precision, uint64_t* n_caustic,
                     uint64_t* n_global, mcrt_stats* stats)
{
    return mcrt_photon_emit_pass(ctx, params, precision, 0, n_caustic, n_global, stats);
}

int mcrt_photon_emit_pass(mcrt_ctx* ctx, const mcrt_photon_emit_params* params, int precision, uint32_t pass, uint64_t* n_caustic,
                          uint64_t* n_global, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    uint64_t total = 0;
    int rc = mcrt_photon_emit_total(ctx, params, &total);
    if (rc) return rc;
    const float* raw[2] = { nullptr, nullptr };
    uint64_t n[2] = { 0, 0 };
    if ((rc = emitRange(ctx, params, precision, pass, 0, total, &raw[0], &n[0], &raw[1], &n[1], stats, true))) return rc;
    if (n_caustic) *n_caustic = n[0];
    if (n_global) *n_global = n[1];
    double build_ms = 0.0;
    const uint32_t* const lights[2] = { ctx->d_emit_lights[0], ctx->d_emit_lights[1] };
    const uint32_t* const lpe_states[2] = { ctx->d_emit_lpe_states[0], ctx->d_emit_lpe_states[1] };
    const std::string identity = ctx->lpe_identity;   // the table the photons were emitted under
    rc = buildPhotonMaps(ctx, params, raw[0], n[0], raw[1], n[1], lights, &build_ms, lpe_states[0] ? lpe_states : nullptr,
                         ctx->lpe_n ? &identity : nullptr);
    freeEmission(ctx);
    if (rc) return rc;
    if (stats) stats->gpu_ms_knn = build_ms;   // emission pass: this field reports the octree build
    return MCRT_OK;
}

// host copy of a device-built map (mcrt_photon_download, mcrt_octree_build)
static int downloadBuiltMap(mcrt_ctx* ctx, const PhotonOctreeDevice& d, mcrt_ctx::HostPhotonMap& m)
{
    m = mcrt_ctx::HostPhotonMap();
    std::vector<DeviceOctant> oct(d.n_octants);
    m.octant_next.resize(d.n_octants);
    m.photons.resize((size_t)d.n_photons * 8);
    if (d.n_octants)
    {
        CK(cudaMemcpy(oct.data(), d.octants, oct.size() * sizeof(DeviceOctant), cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(m.octant_next.data(), d.next_sibling, (size_t)d.n_octants * 4, cudaMemcpyDeviceToHost));
    }
    if (d.n_photons) CK(cudaMemcpy(m.photons.data(), d.photons, (size_t)d.n_photons * 32, cudaMemcpyDeviceToHost));
    m.octant_bounds.resize(6 * (size_t)d.n_octants);
    m.octant_start.resize(d.n_octants); m.octant_count.resize(d.n_octants); m.octant_leaf.resize(d.n_octants);
    for (uint32_t i = 0; i < d.n_octants; i++)
    {
        for (int k = 0; k < 3; k++) { m.octant_bounds[6 * (size_t)i + k] = oct[i].bmin[k]; m.octant_bounds[6 * (size_t)i + 3 + k] = oct[i].bmax[k]; }
        m.octant_start[i] = oct[i].start; m.octant_count[i] = oct[i].count; m.octant_leaf[i] = (uint8_t)oct[i].leaf;
    }
    return MCRT_OK;
}

static void describeHostMap(const mcrt_ctx::HostPhotonMap& m, mcrt_photon_map_desc* out)
{
    std::memset(out, 0, sizeof(*out));
    out->n_octants = (uint32_t)m.octant_leaf.size();
    out->octant_bounds = m.octant_bounds.data();
    out->octant_start = m.octant_start.data();
    out->octant_count = m.octant_count.data();
    out->octant_next_sibling = m.octant_next.data();
    out->octant_leaf = m.octant_leaf.data();
    out->n_photons = m.photons.size() / 8;
    out->photons = m.photons.data();
}

int mcrt_octree_build(mcrt_ctx* ctx, const float* photons, uint64_t n, uint32_t max_photons_per_octree_leaf, const double* scene_bounds6,
                      void** handle, mcrt_photon_map_desc* out, double* gpu_ms)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!handle || !out || !scene_bounds6 || max_photons_per_octree_leaf == 0 || (n && !photons) || n >= 0xFFFFFFFFull)
    { ctx->error = "mcrt_octree_build: invalid arguments"; return MCRT_ERR_INVALID; }
    *handle = nullptr;
    CK(cudaSetDevice(ctx->device));
    std::vector<void*> keep;
    float4* d_in = nullptr;
    if (n)
    {
        CK(cudaMalloc((void**)&d_in, n * 32));
        keep.push_back(d_in);
        if (cudaMemcpyAsync(d_in, photons, n * 32, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) { freeAll(keep); ctx->error = "upload failed"; return MCRT_ERR_CUDA; }
    }
    PhotonOctreeDevice dev;
    int rc = buildPhotonOctreeOnDevice(d_in, (uint32_t)n, scene_bounds6, max_photons_per_octree_leaf, ctx->sm_count, ctx->stream, keep, dev, ctx->error);
    auto* m = new mcrt_ctx::HostPhotonMap();
    if (rc == MCRT_OK) rc = downloadBuiltMap(ctx, dev, *m);
    freeAll(keep);
    if (rc != MCRT_OK) { delete m; return rc; }
    describeHostMap(*m, out);
    if (gpu_ms) *gpu_ms = dev.gpu_ms;
    *handle = m;
    return MCRT_OK;
}

void mcrt_octree_free(void* handle)
{
    delete static_cast<mcrt_ctx::HostPhotonMap*>(handle);
}

int mcrt_photon_download(mcrt_ctx* ctx, int which, mcrt_photon_map_desc* out)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!out || (which != 0 && which != 1)) { ctx->error = "mcrt_photon_download: invalid arguments"; return MCRT_ERR_INVALID; }
    if (!ctx->built_valid) { ctx->error = "no maps built by mcrt_photon_emit"; return MCRT_ERR_NO_PHOTONS; }
    CK(cudaSetDevice(ctx->device));
    if (!ctx->built_host_current[which])
    {
        int rc = downloadBuiltMap(ctx, ctx->built_dev[which], ctx->built_map[which]);
        if (rc) return rc;
        ctx->built_host_current[which] = true;
    }
    describeHostMap(ctx->built_map[which], out);
    return MCRT_OK;
}

int mcrt_photon_download_lights(mcrt_ctx* ctx, int which, uint32_t* out, uint64_t n)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (which != 0 && which != 1) { ctx->error = "mcrt_photon_download_lights: invalid arguments"; return MCRT_ERR_INVALID; }
    if (!ctx->built_valid) { ctx->error = "no maps built by mcrt_photon_emit"; return MCRT_ERR_NO_PHOTONS; }
    if (!ctx->photon_lights)
    {
        ctx->error = "mcrt_photon_download_lights: the maps carry no light index (only maps emitted by mcrt_photon_emit / _emit_pass do)";
        return MCRT_ERR_UNSUPPORTED;
    }
    const PhotonOctreeDevice& d = ctx->built_dev[which];
    if (n != d.n_photons || (n && !out))
    {
        ctx->error = "mcrt_photon_download_lights: n " + std::to_string(n) + ", the map has " + std::to_string(d.n_photons) + " photons";
        return MCRT_ERR_INVALID;
    }
    CK(cudaSetDevice(ctx->device));
    if (n) CK(cudaMemcpy(out, d.lights, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return MCRT_OK;
}

int mcrt_photon_download_lpe_states(mcrt_ctx* ctx, int which, uint32_t* out, uint64_t n)
{
    if (!ctx) return MCRT_ERR_INVALID;
    const std::string name = "mcrt_photon_download_lpe_states";
    if (which != 0 && which != 1) { ctx->error = name + ": invalid arguments"; return MCRT_ERR_INVALID; }
    if (!ctx->built_valid) { ctx->error = "no maps built by mcrt_photon_emit"; return MCRT_ERR_NO_PHOTONS; }
    if (!ctx->photon_lpe_states)
    {
        ctx->error = name + ": the maps carry no LPE states (only maps emitted by mcrt_photon_emit / _emit_pass under an LPE "
                            "table the photon mapper takes do)";
        return MCRT_ERR_UNSUPPORTED;
    }
    const PhotonOctreeDevice& d = ctx->built_dev[which];
    if (n != d.n_photons || (n && !out))
    {
        ctx->error = name + ": n " + std::to_string(n) + ", the map has " + std::to_string(d.n_photons) + " photons";
        return MCRT_ERR_INVALID;
    }
    CK(cudaSetDevice(ctx->device));
    if (n) CK(cudaMemcpy(out, d.lpe_states, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return MCRT_OK;
}

int mcrt_render_rows_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y0, uint32_t y1, uint32_t sqrtspp,
                         uint32_t global_seed, int integrator_kind, int precision, double* out_rgb_dev, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!out_rgb_dev) { ctx->error = "null output"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    if (y1 <= y0) { ctx->error = "empty row range"; return MCRT_ERR_INVALID; }
    return renderFrame(ctx, camera, y0, 1, y1 - y0, sqrtspp, global_seed, integrator_kind, precision, out_rgb_dev, stats);
}

int mcrt_image_tonemap_dev(mcrt_ctx* ctx, const double* rgb_dev, uint32_t width, uint32_t height,
                           const mcrt_image_params* params, uint8_t* out_bgr_dev, double* exposure_factor, double* gain_factor)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!rgb_dev || !out_bgr_dev || !params || width == 0 || height == 0) { ctx->error = "mcrt_image_tonemap: invalid arguments"; return MCRT_ERR_INVALID; }
    if (params->tonemapper > MCRT_TONEMAP_ACES) { ctx->error = "mcrt_image_tonemap: unknown tonemapper"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    return imageTonemapOnDevice(rgb_dev, width, height, *params, out_bgr_dev, ctx->sm_count, ctx->stream, exposure_factor, gain_factor, ctx->error);
}

int mcrt_image_tonemap(mcrt_ctx* ctx, const double* rgb, uint32_t width, uint32_t height, const mcrt_image_params* params,
                       uint8_t* out_bgr, double* exposure_factor, double* gain_factor)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!rgb || !out_bgr || !params || width == 0 || height == 0) { ctx->error = "mcrt_image_tonemap: invalid arguments"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    const size_t n = (size_t)width * height;
    double* d_rgb = nullptr; uint8_t* d_out = nullptr;
    CK(cudaMalloc((void**)&d_rgb, n * 3 * sizeof(double)));
    if (cudaMalloc((void**)&d_out, n * 3) != cudaSuccess) { cudaFree(d_rgb); ctx->error = "cudaMalloc failed"; return MCRT_ERR_CUDA; }
    int rc = MCRT_OK;
    if (cudaMemcpyAsync(d_rgb, rgb, n * 3 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) { ctx->error = "upload failed"; rc = MCRT_ERR_CUDA; }
    if (rc == MCRT_OK) rc = mcrt_image_tonemap_dev(ctx, d_rgb, width, height, params, d_out, exposure_factor, gain_factor);
    if (rc == MCRT_OK && cudaMemcpy(out_bgr, d_out, n * 3, cudaMemcpyDeviceToHost) != cudaSuccess) { ctx->error = "copy back failed"; rc = MCRT_ERR_CUDA; }
    cudaFree(d_rgb); cudaFree(d_out);
    return rc;
}

int mcrt_bvh_build(mcrt_ctx* ctx, const double* prim_bounds, uint32_t n_prims, const double* scene_bounds6, int type,
                   int bins_per_axis, void** handle, mcrt_bvh_desc* out, double* gpu_ms)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!handle || !out) { ctx->error = "mcrt_bvh_build: null output"; return MCRT_ERR_INVALID; }
    *handle = nullptr;
    CK(cudaSetDevice(ctx->device));
    BvhBuildResult* r = new BvhBuildResult();
    const int rc = buildBvhOnDevice(prim_bounds, n_prims, scene_bounds6, type, bins_per_axis, ctx->sm_count, ctx->stream, *r, ctx->error);
    if (rc != MCRT_OK) { delete r; return rc; }
    out->n_nodes = (uint32_t)r->node_first_prim.size();
    out->n_prims = n_prims;
    out->node_bounds = r->node_bounds.data();
    out->node_first_prim = r->node_first_prim.data();
    out->node_prim_count = r->node_prim_count.data();
    out->node_next_sibling = r->node_next_sibling.data();
    out->prim_order = r->prim_order.data();
    out->build_rounds = r->iterations;
    out->kernel_launches = r->kernel_launches;
    if (gpu_ms) *gpu_ms = r->gpu_ms;
    *handle = r;
    return MCRT_OK;
}

void mcrt_bvh_free(void* handle)
{
    delete static_cast<BvhBuildResult*>(handle);
}

int mcrt_set_film(mcrt_ctx* ctx, const mcrt_film* film)
{
    if (!ctx) return MCRT_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    mcrt_film f = {MCRT_FILM_BOX, 0u, 0.5};
    if (film)
    {
        if (film->filter > MCRT_FILM_LANCZOS) { ctx->error = "mcrt_set_film: unknown filter"; return MCRT_ERR_INVALID; }
        if (film->cache_size == 1) { ctx->error = "mcrt_set_film: cache_size must be 0 or >= 2"; return MCRT_ERR_INVALID; }
        // default radii of Film::Film (film.cpp:32-45)
        static const double default_radius[7] = {0.5, 2.0, 2.0, 1.39, 1.0, 1.71, 2.0};
        f = *film;
        if (!(f.radius > 0.0)) f.radius = default_radius[f.filter];
    }
    if (ctx->d_film_cache) { cudaFree(ctx->d_film_cache); ctx->d_film_cache = nullptr; }
    if (f.cache_size)
    {
        // Film::filter_cache (film.cpp:50-58)
        std::vector<double> cache(f.cache_size);
        for (uint32_t i = 0; i < f.cache_size; i++)
            cache[i] = filmFilterFunction(f.filter, (2.0 * (double)(int)i) / (double)(f.cache_size - 1));
        CK(cudaMalloc((void**)&ctx->d_film_cache, cache.size() * sizeof(double)));
        CK(cudaMemcpy(ctx->d_film_cache, cache.data(), cache.size() * sizeof(double), cudaMemcpyHostToDevice));
    }
    ctx->film = f;
    ctx->film_default = f.filter == MCRT_FILM_BOX && f.radius == 0.5;
    return MCRT_OK;
}

int mcrt_render_rows_strided_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step,
                                 uint32_t n_rows, uint32_t sqrtspp, uint32_t global_seed, int integrator_kind,
                                 int precision, double* out_rgb_dev, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!out_rgb_dev) { ctx->error = "null output"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    return renderFrame(ctx, camera, y_first, y_step, n_rows, sqrtspp, global_seed, integrator_kind, precision, out_rgb_dev, stats);
}

int mcrt_render_rows_strided_peers(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step,
                                   uint32_t n_rows, uint32_t sqrtspp, uint32_t global_seed, int integrator_kind,
                                   int precision, void* const* frames, uint32_t n_frames, int frame_is_float32, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!frames || n_frames == 0 || n_frames > (uint32_t)MAX_FRAME_PEERS || !camera) { ctx->error = "mcrt_render_rows_strided_peers: 1..16 frames"; return MCRT_ERR_INVALID; }
    if (!ctx->film_default) { ctx->error = "a filtered film splats across rows: not available for row-sharded renders"; return MCRT_ERR_UNSUPPORTED; }
    CK(cudaSetDevice(ctx->device));
    PeerFrames pf{};
    for (uint32_t q = 0; q < n_frames; q++) { if (!frames[q]) { ctx->error = "null frame"; return MCRT_ERR_INVALID; } pf.frame[q] = frames[q]; }
    pf.n_frames = n_frames; pf.as_float = frame_is_float32 ? 1u : 0u;
    pf.y_first = y_first; pf.y_step = y_step; pf.row_values = camera->width * 3u;
    ctx->peer_out = pf;
    const int rc = renderFrame(ctx, camera, y_first, y_step, n_rows, sqrtspp, global_seed, integrator_kind, precision,
                                  static_cast<double*>(frames[0]), stats);
    ctx->peer_out.n_frames = 0;
    return rc;
}

int mcrt_render_film_sums_strided_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                                      uint32_t sqrtspp, uint32_t global_seed, int integrator_kind, int precision,
                                      double* rgb_sum_dev, double* weight_sum_dev, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!rgb_sum_dev || !weight_sum_dev) { ctx->error = "null output"; return MCRT_ERR_INVALID; }
    if (ctx->film_default) { ctx->error = "mcrt_render_film_sums_strided_dev is for reconstruction filters (mcrt_set_film); the default box film shards by rows directly"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    if (!camera) { ctx->error = "null camera"; return MCRT_ERR_INVALID; }
    const size_t film_pixels = (size_t)camera->width * camera->height;
    CK(cudaMemsetAsync(rgb_sum_dev, 0, film_pixels * 3 * sizeof(double), ctx->stream));
    CK(cudaMemsetAsync(weight_sum_dev, 0, film_pixels * sizeof(double), ctx->stream));
    const FilmSums sums = { rgb_sum_dev, weight_sum_dev };
    return renderFrame(ctx, camera, y_first, y_step, n_rows, sqrtspp, global_seed, integrator_kind, precision, nullptr, stats, &sums);
}

int mcrt_render_accumulate_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                               uint32_t sample_first, uint32_t sample_count, uint32_t global_seed, int integrator_kind,
                               int precision, double* rgb_sum_dev, double* weight_sum_dev, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    int rc;
    if ((rc = checkAccumulateSums(ctx, "mcrt_render_accumulate_dev", sample_count, rgb_sum_dev, weight_sum_dev))) return rc;
    CK(cudaSetDevice(ctx->device));
    const FilmSums sums = { rgb_sum_dev, weight_sum_dev };
    return renderDispatch(ctx, camera, y_first, y_step, n_rows, sample_first, sample_count, global_seed, integrator_kind,
                          precision, nullptr, stats, &sums);
}

namespace
{
    // The active-tile path of mcrt_render_accumulate_tiles_dev and of accumulatePlanes (the caller has checked the sums)
    int accumulateTiles(mcrt_ctx* ctx, const std::string& name, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step,
                        uint32_t n_rows, uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                        uint32_t global_seed, int integrator_kind, int precision, const FilmSums& sums, mcrt_stats* stats)
    {
        if (tile == 0) { ctx->error = name + ": tile is 0"; return MCRT_ERR_INVALID; }
        if (!active_tiles) { ctx->error = name + ": null tile mask"; return MCRT_ERR_INVALID; }
        // the mask's size follows from the row set: check it before reading the mask
        if (!camera || n_rows == 0 || y_step == 0 || camera->width == 0 ||
            (uint64_t)y_first + (uint64_t)(n_rows - 1) * y_step >= camera->height)
        {
            ctx->error = name + ": invalid camera / row range";
            return MCRT_ERR_INVALID;
        }
        if ((uint64_t)camera->width * n_rows > 0xFFFFFFFFull) { ctx->error = "row block too large"; return MCRT_ERR_INVALID; }
        if (!ctx->film_default && (y_first != 0 || y_step != 1 || n_rows != camera->height))
        {
            // a filter splats across tiles: the resolve's tiles span the whole frame, so the row set must be the whole frame
            ctx->error = name + ": with a reconstruction filter the row set must be the whole frame";
            return MCRT_ERR_UNSUPPORTED;
        }
        // tile-major, row-major inside a tile: adjacent lanes of k_generate take adjacent pixels of one tile
        const uint32_t width = camera->width;
        const uint32_t tiles_x = (width + tile - 1) / tile, tiles_y = (n_rows + tile - 1) / tile;
        std::vector<uint32_t>& list = ctx->h_pixel_list;
        list.clear();
        for (uint32_t ty = 0; ty < tiles_y; ty++)
            for (uint32_t tx = 0; tx < tiles_x; tx++)
            {
                if (!active_tiles[(size_t)ty * tiles_x + tx]) continue;
                const uint32_t y1 = std::min(n_rows, (ty + 1) * tile), x1 = std::min(width, (tx + 1) * tile);
                for (uint32_t y = ty * tile; y < y1; y++)
                    for (uint32_t x = tx * tile; x < x1; x++) list.push_back(y * width + x);
            }
        if (list.empty()) { ctx->error = name + ": no active tile"; return MCRT_ERR_INVALID; }
        CK(cudaSetDevice(ctx->device));
        if (ctx->pixel_list_values < list.size())
        {
            if (ctx->d_pixel_list) cudaFree(ctx->d_pixel_list);
            ctx->d_pixel_list = nullptr; ctx->pixel_list_values = 0;
            CK(cudaMalloc((void**)&ctx->d_pixel_list, list.size() * sizeof(uint32_t)));
            ctx->pixel_list_values = list.size();
        }
        CK(cudaMemcpyAsync(ctx->d_pixel_list, list.data(), list.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
        return renderDispatch(ctx, camera, y_first, y_step, n_rows, sample_first, sample_count, global_seed, integrator_kind,
                              precision, nullptr, stats, &sums, ctx->d_pixel_list, (uint32_t)list.size());
    }

    // The tail of mcrt_render_accumulate_groups_dev / _aovs_dev / _photon_components_dev, whose planes the caller has
    // checked: a uniform pass, or an active-tile pass when a mask is given
    int accumulatePlanes(mcrt_ctx* ctx, const std::string& name, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step,
                         uint32_t n_rows, uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                         uint32_t global_seed, int integrator_kind, int precision, const FilmSums& sums, mcrt_stats* stats)
    {
        int rc;
        if ((rc = checkAccumulateSums(ctx, name.c_str(), sample_count, sums.rgb, nullptr))) return rc;
        if (active_tiles)
            return accumulateTiles(ctx, name, camera, y_first, y_step, n_rows, tile, active_tiles, sample_first, sample_count, global_seed,
                                   integrator_kind, precision, sums, stats);
        CK(cudaSetDevice(ctx->device));
        return renderDispatch(ctx, camera, y_first, y_step, n_rows, sample_first, sample_count, global_seed, integrator_kind,
                              precision, nullptr, stats, &sums);
    }
}

int mcrt_render_accumulate_tiles_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                                     uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                                     uint32_t global_seed, int integrator_kind, int precision, double* rgb_sum_dev,
                                     double* weight_sum_dev, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    int rc;
    if ((rc = checkAccumulateSums(ctx, "mcrt_render_accumulate_tiles_dev", sample_count, rgb_sum_dev, weight_sum_dev))) return rc;
    const FilmSums sums = { rgb_sum_dev, weight_sum_dev };
    return accumulateTiles(ctx, "mcrt_render_accumulate_tiles_dev", camera, y_first, y_step, n_rows, tile, active_tiles, sample_first,
                           sample_count, global_seed, integrator_kind, precision, sums, stats);
}

int mcrt_set_light_groups(mcrt_ctx* ctx, const uint32_t* group_of_light, uint32_t n_lights, uint32_t n_groups)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!ctx->has_scene) { ctx->error = "mcrt_set_light_groups: no scene uploaded"; return MCRT_ERR_NO_SCENE; }
    if (!group_of_light)
    {
        if (n_lights || n_groups) { ctx->error = "mcrt_set_light_groups: a null table clears it; n_lights and n_groups must be 0"; return MCRT_ERR_INVALID; }
        ctx->has_light_groups = false;
        ctx->n_light_groups = 0;
        ctx->lpe_n = 0;   // its labels named groups of the old table
        return MCRT_OK;
    }
    if (n_lights != ctx->scene64.n_lights)
    {
        ctx->error = "mcrt_set_light_groups: n_lights " + std::to_string(n_lights) + ", the scene has " + std::to_string(ctx->scene64.n_lights);
        return MCRT_ERR_INVALID;
    }
    if (n_groups == 0xFFFFFFFFu) { ctx->error = "mcrt_set_light_groups: n_groups + 1 planes must fit 32 bits"; return MCRT_ERR_INVALID; }
    for (uint32_t l = 0; l < n_lights; l++)
        if (group_of_light[l] >= n_groups)
        {
            ctx->error = "mcrt_set_light_groups: light " + std::to_string(l) + " has group " + std::to_string(group_of_light[l]) +
                         ", n_groups is " + std::to_string(n_groups);
            return MCRT_ERR_INVALID;
        }
    if (ctx->emissive_unlit)
    {
        ctx->error = "mcrt_set_light_groups: the scene has an emissive primitive that is not one of its lights";
        return MCRT_ERR_UNSUPPORTED;
    }
    CK(cudaSetDevice(ctx->device));
    ctx->has_light_groups = false;
    ctx->lpe_n = 0;   // its labels named groups of the old table
    if (ctx->group_of_light_values < n_lights)
    {
        if (ctx->d_group_of_light) cudaFree(ctx->d_group_of_light);
        ctx->d_group_of_light = nullptr; ctx->group_of_light_values = 0;
        CK(cudaMalloc((void**)&ctx->d_group_of_light, n_lights * sizeof(uint32_t)));
        ctx->group_of_light_values = n_lights;
    }
    if (n_lights) CK(cudaMemcpyAsync(ctx->d_group_of_light, group_of_light, n_lights * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->h_group_of_light.assign(group_of_light, group_of_light + n_lights);
    ctx->n_light_groups = n_groups;
    ctx->has_light_groups = true;
    return MCRT_OK;
}

int mcrt_set_light_path_expressions(mcrt_ctx* ctx, const char* const* exprs, uint32_t n)
{
    if (!ctx) return MCRT_ERR_INVALID;
    const std::string name = "mcrt_set_light_path_expressions";
    if (!ctx->has_scene) { ctx->error = name + ": no scene uploaded"; return MCRT_ERR_NO_SCENE; }
    ctx->lpe_n = 0;
    if (!exprs)
    {
        if (n) { ctx->error = name + ": a null list clears the table; n must be 0"; return MCRT_ERR_INVALID; }
        return MCRT_OK;
    }
    LpeTable t;
    std::string why;
    const int rc = lpeCompile(exprs, n, ctx->has_light_groups ? ctx->n_light_groups : 0u, t, why);
    if (rc != MCRT_OK) { ctx->error = name + ": " + why; return rc; }
    // light l reads the symbol of its group's label, or the unlabelled L
    const uint32_t n_lights = ctx->scene64.n_lights;
    std::vector<uint8_t> light_symbol(std::max<uint32_t>(n_lights, 1u), (uint8_t)MCRT_LPE_SYM_L);
    if (ctx->has_light_groups)
        for (uint32_t l = 0; l < n_lights; l++)
        {
            auto it = std::lower_bound(t.labels.begin(), t.labels.end(), ctx->h_group_of_light[l]);
            if (it != t.labels.end() && *it == ctx->h_group_of_light[l])
                light_symbol[l] = (uint8_t)(MCRT_LPE_SYM_LABEL0 + (it - t.labels.begin()));
        }
    CK(cudaSetDevice(ctx->device));
    if (!ctx->d_lpe_next)
    {
        CK(cudaMalloc((void**)&ctx->d_lpe_next, (size_t)MCRT_LPE_MAX_STATES * MCRT_LPE_MAX_SYMBOLS));
        CK(cudaMalloc((void**)&ctx->d_lpe_accept, 256 * sizeof(uint32_t)));
    }
    if (ctx->lpe_light_values < light_symbol.size())
    {
        if (ctx->d_lpe_light_symbol) cudaFree(ctx->d_lpe_light_symbol);
        ctx->d_lpe_light_symbol = nullptr; ctx->lpe_light_values = 0;
        CK(cudaMalloc((void**)&ctx->d_lpe_light_symbol, light_symbol.size()));
        ctx->lpe_light_values = light_symbol.size();
    }
    CK(cudaMemcpyAsync(ctx->d_lpe_next, t.next.data(), t.next.size(), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_lpe_accept, t.accept.data(), 256 * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_lpe_light_symbol, light_symbol.data(), light_symbol.size(), cudaMemcpyHostToDevice, ctx->stream));
    if (t.photon_error.empty())
    {
        if (!ctx->d_lpe_rev_next)
        {
            CK(cudaMalloc((void**)&ctx->d_lpe_rev_next, (size_t)MCRT_LPE_MAX_STATES * MCRT_LPE_MAX_SYMBOLS));
            CK(cudaMalloc((void**)&ctx->d_lpe_join, (size_t)MCRT_LPE_MAX_STATES * MCRT_LPE_MAX_STATES * sizeof(uint32_t)));
            CK(cudaMalloc((void**)&ctx->d_lpe_join_any, 256));
        }
        CK(cudaMemcpyAsync(ctx->d_lpe_rev_next, t.rev_next.data(), t.rev_next.size(), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->d_lpe_join, t.join.data(), t.join.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->d_lpe_join_any, t.join_any.data(), 256, cudaMemcpyHostToDevice, ctx->stream));
    }
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->lpe_symbols = t.n_symbols;
    ctx->lpe_rev_states = t.rev_n_states;
    ctx->lpe_rev_start = t.rev_start;
    ctx->lpe_photon_error = t.photon_error;
    {
        std::string& id = ctx->lpe_identity;
        id.clear();
        auto put = [&](const void* data, size_t bytes) { id.append(static_cast<const char*>(data), bytes); };
        const uint32_t head[4] = { n, t.n_symbols, t.rev_n_states, t.rev_start };
        put(head, sizeof(head));
        put(t.next.data(), t.next.size());
        put(t.accept.data(), t.accept.size() * sizeof(uint32_t));
        put(light_symbol.data(), light_symbol.size());
        put(t.rev_next.data(), t.rev_next.size());
        put(t.join.data(), t.join.size() * sizeof(uint32_t));
        put(t.photon_error.data(), t.photon_error.size());
    }
    ctx->lpe_n = n;
    return MCRT_OK;
}

int mcrt_render_accumulate_lpe_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                                   uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                                   uint32_t global_seed, int integrator_kind, int precision, double* planes_dev,
                                   uint32_t n_planes, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    const std::string name = "mcrt_render_accumulate_lpe_dev";
    if (!ctx->film_default) { ctx->error = name + ": LPE planes take the box film only"; return MCRT_ERR_UNSUPPORTED; }
    if (integrator_kind == MCRT_INTEGRATOR_PHOTON)
    {
        // a photon term's string needs the photon's own events, which only maps emitted under this table record
        if (!ctx->has_photons || !ctx->lpe_n || ctx->photon_lpe_identity.empty() || ctx->photon_lpe_identity != ctx->lpe_identity)
        {
            ctx->error = name + ": the photon maps carry no LPE states for this table (only maps emitted by mcrt_photon_emit / "
                                "_emit_pass after mcrt_set_light_path_expressions with the same expressions do)";
            return MCRT_ERR_UNSUPPORTED;
        }
        if (!ctx->lpe_photon_error.empty())
        {
            ctx->error = name + ": the photon mapper cannot take this table: " + ctx->lpe_photon_error;
            return MCRT_ERR_UNSUPPORTED;
        }
    }
    if (!ctx->lpe_n) { ctx->error = name + ": no LPE table (mcrt_set_light_path_expressions)"; return MCRT_ERR_INVALID; }
    if (n_planes != ctx->lpe_n)
    {
        ctx->error = name + ": n_planes " + std::to_string(n_planes) + ", the table has " + std::to_string(ctx->lpe_n) + " expressions";
        return MCRT_ERR_INVALID;
    }
    return accumulatePlanes(ctx, name, camera, y_first, y_step, n_rows, tile, active_tiles, sample_first, sample_count, global_seed,
                            integrator_kind, precision, FilmSums{ planes_dev, nullptr, n_planes, FILM_MODE_LPE }, stats);
}

int mcrt_render_accumulate_groups_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                                      uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                                      uint32_t global_seed, int integrator_kind, int precision, double* planes_dev,
                                      uint32_t n_planes, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    const std::string name = "mcrt_render_accumulate_groups_dev";
    if (!ctx->film_default) { ctx->error = name + ": light-group planes take the box film only"; return MCRT_ERR_UNSUPPORTED; }
    if (integrator_kind == MCRT_INTEGRATOR_PHOTON && !(ctx->has_photons && ctx->photon_lights))
    {
        ctx->error = name + ": the photon maps carry no light index (only maps emitted by mcrt_photon_emit / _emit_pass do)";
        return MCRT_ERR_UNSUPPORTED;
    }
    if (!ctx->has_light_groups) { ctx->error = name + ": no light-group table (mcrt_set_light_groups)"; return MCRT_ERR_INVALID; }
    if (n_planes != ctx->n_light_groups + 1)
    {
        ctx->error = name + ": n_planes " + std::to_string(n_planes) + ", the table has " + std::to_string(ctx->n_light_groups) +
                     " groups + the sky";
        return MCRT_ERR_INVALID;
    }
    return accumulatePlanes(ctx, name, camera, y_first, y_step, n_rows, tile, active_tiles, sample_first, sample_count, global_seed,
                            integrator_kind, precision, FilmSums{ planes_dev, nullptr, n_planes, FILM_MODE_GROUPS }, stats);
}

int mcrt_render_accumulate_aovs_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step, uint32_t n_rows,
                                    uint32_t tile, const uint8_t* active_tiles, uint32_t sample_first, uint32_t sample_count,
                                    uint32_t global_seed, int integrator_kind, int precision, double* planes_dev,
                                    uint32_t n_planes, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    const std::string name = "mcrt_render_accumulate_aovs_dev";
    if (!ctx->film_default) { ctx->error = name + ": AOV planes take the box film only"; return MCRT_ERR_UNSUPPORTED; }
    if (integrator_kind == MCRT_INTEGRATOR_PHOTON)
    {
        ctx->error = name + ": the photon mapper has no light-path AOVs (its estimates are not split by first lobe)";
        return MCRT_ERR_UNSUPPORTED;
    }
    if (n_planes != MCRT_AOV_COUNT)
    {
        ctx->error = name + ": n_planes " + std::to_string(n_planes) + ", an AOV render has " + std::to_string(MCRT_AOV_COUNT);
        return MCRT_ERR_INVALID;
    }
    return accumulatePlanes(ctx, name, camera, y_first, y_step, n_rows, tile, active_tiles, sample_first, sample_count, global_seed,
                            integrator_kind, precision, FilmSums{ planes_dev, nullptr, n_planes, FILM_MODE_AOV }, stats);
}

int mcrt_render_accumulate_photon_components_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y_first, uint32_t y_step,
                                                 uint32_t n_rows, uint32_t tile, const uint8_t* active_tiles,
                                                 uint32_t sample_first, uint32_t sample_count, uint32_t global_seed,
                                                 int integrator_kind, int precision, double* planes_dev, uint32_t n_planes,
                                                 mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    const std::string name = "mcrt_render_accumulate_photon_components_dev";
    // an allowlist: every kind but the photon mapper would run the path tracer's AOV kernels, whose planes go up to 7
    if (integrator_kind == MCRT_INTEGRATOR_PATH)
    {
        ctx->error = name + ": the path tracer has no photon-mapper components (it has light-path AOVs)";
        return MCRT_ERR_UNSUPPORTED;
    }
    if (integrator_kind != MCRT_INTEGRATOR_PHOTON)
    {
        ctx->error = name + ": unknown integrator kind " + std::to_string(integrator_kind);
        return MCRT_ERR_INVALID;
    }
    if (!ctx->film_default) { ctx->error = name + ": component planes take the box film only"; return MCRT_ERR_UNSUPPORTED; }
    if (n_planes != MCRT_PM_COMPONENT_COUNT)
    {
        ctx->error = name + ": n_planes " + std::to_string(n_planes) + ", a component render has " +
                     std::to_string(MCRT_PM_COMPONENT_COUNT);
        return MCRT_ERR_INVALID;
    }
    // the kernels' FILM_MODE_AOV instantiations: each deposit site names its plane, here the MCRT_PM_* estimator planes
    return accumulatePlanes(ctx, name, camera, y_first, y_step, n_rows, tile, active_tiles, sample_first, sample_count, global_seed,
                            integrator_kind, precision, FilmSums{ planes_dev, nullptr, n_planes, FILM_MODE_AOV }, stats);
}

int mcrt_light_groups_combine_dev(mcrt_ctx* ctx, const double* planes_dev, uint32_t n_planes, uint64_t n_values,
                                  const double* weights, double* out_dev)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!planes_dev || !weights || !out_dev || n_planes == 0 || n_values % 3 != 0)
    {
        ctx->error = "mcrt_light_groups_combine_dev: null pointer, no plane or n_values not a multiple of 3";
        return MCRT_ERR_INVALID;
    }
    CK(cudaSetDevice(ctx->device));
    const size_t values = 3 * (size_t)n_planes;
    if (ctx->group_weight_values < values)
    {
        if (ctx->d_group_weights) cudaFree(ctx->d_group_weights);
        ctx->d_group_weights = nullptr; ctx->group_weight_values = 0;
        CK(cudaMalloc((void**)&ctx->d_group_weights, values * sizeof(double)));
        ctx->group_weight_values = values;
    }
    CK(cudaMemcpyAsync(ctx->d_group_weights, weights, values * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    if (n_values) launchLightGroupsCombine(planes_dev, n_planes, n_values, ctx->d_group_weights, out_dev, ctx->sm_count * ctx->blocks_per_sm, ctx->stream);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    return MCRT_OK;
}

namespace
{
    // Shared by mcrt_progressive_resolve_dev (tile_samples null: every pixel has a_samples / b_samples) and
    // mcrt_progressive_resolve_tiles_dev (tile_samples: HOST {nA, nB}[n_tiles]).
    int progressiveResolve(mcrt_ctx* ctx, const char* fn, const double* a_rgb_dev, const double* a_weight_dev, uint64_t a_samples,
                           const double* b_rgb_dev, const double* b_weight_dev, uint64_t b_samples, const uint32_t* tile_samples,
                           uint32_t width, uint32_t rows, uint32_t tile, double* out_rgb_dev, double* tile_error_dev,
                           double* tile_sums_dev, double* frame_error)
    {
        const std::string name(fn);
        if (!out_rgb_dev || width == 0 || rows == 0 || (uint64_t)width * rows > 0xFFFFFFFFull)
        {
            ctx->error = name + ": null output, empty frame or more than 2^32 pixels";
            return MCRT_ERR_INVALID;
        }
        if (tile == 0) { ctx->error = name + ": tile is 0"; return MCRT_ERR_INVALID; }
        const uint64_t tiles_x = (width + tile - 1) / tile, tiles_y = (rows + tile - 1) / tile;
        const uint64_t n_tiles = tiles_x * tiles_y;
        bool both = a_samples && b_samples;   // the frame error is finite only if every tile has both halves
        if (tile_samples)
        {
            both = true;
            for (uint64_t t = 0; t < n_tiles; t++)
            {
                a_samples += tile_samples[2 * t] != 0; b_samples += tile_samples[2 * t + 1] != 0;
                both = both && tile_samples[2 * t] != 0 && tile_samples[2 * t + 1] != 0;
            }
        }
        if (a_samples + b_samples == 0) { ctx->error = name + ": no samples to resolve"; return MCRT_ERR_INVALID; }
        if ((a_samples && !a_rgb_dev) || (b_samples && !b_rgb_dev))
        {
            ctx->error = name + ": null sums for a half with samples";
            return MCRT_ERR_INVALID;
        }
        const bool weighted = a_weight_dev || b_weight_dev;
        if (weighted && ((a_samples && !a_weight_dev) || (b_samples && !b_weight_dev)))
        {
            ctx->error = name + ": weight sums must be given for both halves or for neither";
            return MCRT_ERR_INVALID;
        }
        CK(cudaSetDevice(ctx->device));
        // scratch: {sum v, sum I^2} per tile, then the frame's; then the tiles' {nA, nB} when they are given
        const size_t sums_values = 2 * (n_tiles + 1);
        const size_t scratch_values = sums_values + (tile_samples ? 2 * n_tiles : 0);
        if (ctx->resolve_scratch_values < scratch_values)
        {
            if (ctx->d_resolve_scratch) cudaFree(ctx->d_resolve_scratch);
            ctx->d_resolve_scratch = nullptr; ctx->resolve_scratch_values = 0;
            CK(cudaMalloc((void**)&ctx->d_resolve_scratch, scratch_values * sizeof(double)));
            ctx->resolve_scratch_values = scratch_values;
        }
        double* d_counts = nullptr;
        std::vector<double> counts;
        if (tile_samples)
        {
            counts.assign(tile_samples, tile_samples + 2 * n_tiles);
            d_counts = ctx->d_resolve_scratch + sums_values;
            CK(cudaMemcpyAsync(d_counts, counts.data(), counts.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        }
        // with per-tile counts the halves' scalar counts are unused: only whether a half has samples anywhere matters
        ProgressiveHalf a = { a_samples ? a_rgb_dev : nullptr, a_samples ? a_weight_dev : nullptr, tile_samples ? 0.0 : (double)a_samples };
        ProgressiveHalf b = { b_samples ? b_rgb_dev : nullptr, b_samples ? b_weight_dev : nullptr, tile_samples ? 0.0 : (double)b_samples };
        CK(cudaMemsetAsync(ctx->d_resolve_scratch, 0, sums_values * sizeof(double), ctx->stream));
        launchProgressiveResolve(a, b, weighted, width, rows, tile, (uint32_t)tiles_x, out_rgb_dev, ctx->d_resolve_scratch, tile_error_dev,
                                 (uint32_t)n_tiles, ctx->sm_count * ctx->blocks_per_sm, ctx->stream, d_counts);
        if (tile_sums_dev)
            CK(cudaMemcpyAsync(tile_sums_dev, ctx->d_resolve_scratch, 2 * n_tiles * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
        double frame_sums[2] = { 0.0, 0.0 };
        CK(cudaMemcpyAsync(frame_sums, ctx->d_resolve_scratch + 2 * n_tiles, sizeof(frame_sums), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        CK(cudaGetLastError());
        if (frame_error) *frame_error = progressiveRelativeError(frame_sums[0], frame_sums[1], both);
        return MCRT_OK;
    }
}

int mcrt_progressive_resolve_dev(mcrt_ctx* ctx, const double* a_rgb_dev, const double* a_weight_dev, uint64_t a_samples,
                                 const double* b_rgb_dev, const double* b_weight_dev, uint64_t b_samples,
                                 uint32_t width, uint32_t rows, uint32_t tile, double* out_rgb_dev,
                                 double* tile_error_dev, double* frame_error)
{
    if (!ctx) return MCRT_ERR_INVALID;
    return progressiveResolve(ctx, "mcrt_progressive_resolve_dev", a_rgb_dev, a_weight_dev, a_samples, b_rgb_dev, b_weight_dev,
                              b_samples, nullptr, width, rows, tile, out_rgb_dev, tile_error_dev, nullptr, frame_error);
}

int mcrt_progressive_resolve_tiles_dev(mcrt_ctx* ctx, const double* a_rgb_dev, const double* a_weight_dev,
                                       const double* b_rgb_dev, const double* b_weight_dev, const uint32_t* tile_samples,
                                       uint32_t width, uint32_t rows, uint32_t tile, double* out_rgb_dev,
                                       double* tile_error_dev, double* tile_sums_dev, double* frame_error)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!tile_samples) { ctx->error = "mcrt_progressive_resolve_tiles_dev: null tile_samples"; return MCRT_ERR_INVALID; }
    return progressiveResolve(ctx, "mcrt_progressive_resolve_tiles_dev", a_rgb_dev, a_weight_dev, 0, b_rgb_dev, b_weight_dev, 0,
                              tile_samples, width, rows, tile, out_rgb_dev, tile_error_dev, tile_sums_dev, frame_error);
}

static_assert(MCRT_FEATURES_MAX_SPECULAR_DEPTH + 1 <= IOR_STACK_CAPACITY, "a guide chain must not overflow the IOR stack");

namespace
{
    // mcrt_render_features_dev (specular_depth 0: the first-hit kernel) and mcrt_render_features_chain_dev
    int renderFeatures(const char* fn, mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t sample_first, uint32_t sample_count,
                       uint32_t global_seed, int precision, uint32_t specular_depth, double* features_dev, mcrt_stats* stats)
    {
        if (!ctx) return MCRT_ERR_INVALID;
        const std::string f = fn;
        if (!camera || !features_dev) { ctx->error = f + ": null camera or buffer"; return MCRT_ERR_INVALID; }
        if (sample_count == 0) { ctx->error = f + ": sample_count is 0"; return MCRT_ERR_INVALID; }
        if ((uint64_t)sample_first + sample_count > 0x100000000ull)
        {
            ctx->error = f + ": sample range beyond 2^32 samples per pixel";
            return MCRT_ERR_INVALID;
        }
        const uint64_t n_pixels = (uint64_t)camera->width * camera->height;
        if (n_pixels == 0 || n_pixels > 0xFFFFFFFFull) { ctx->error = f + ": empty frame or more than 2^32 pixels"; return MCRT_ERR_INVALID; }
        if (precision != MCRT_PRECISION_F64 && precision != MCRT_PRECISION_F32) { ctx->error = "unknown precision"; return MCRT_ERR_INVALID; }
        if (specular_depth > MCRT_FEATURES_MAX_SPECULAR_DEPTH)
        {
            ctx->error = f + ": specular_depth above MCRT_FEATURES_MAX_SPECULAR_DEPTH";
            return MCRT_ERR_INVALID;
        }
        if (!ctx->has_scene) { ctx->error = "no scene uploaded"; return MCRT_ERR_NO_SCENE; }
        CK(cudaSetDevice(ctx->device));
        cudaStream_t s = ctx->stream;
        const int grid = ctx->sm_count * ctx->blocks_per_sm;
        CK(cudaMemsetAsync(ctx->d_counters, 0, sizeof(Counters), s));
        CK(cudaEventRecord(ctx->ev_start, s));
        if (precision == MCRT_PRECISION_F64)
        {
            DeviceScene<double> sc = ctx->scene64;
            if (ctx->exact_traversal) sc.bvh4 = nullptr;
            if (specular_depth == 0)
                Launch<double>::features(sc, deviceCamera<double>(*camera), global_seed, sample_first, sample_count, features_dev,
                                         ctx->d_counters, grid, s);
            else
                Launch<double>::featuresChain(sc, deviceCamera<double>(*camera), global_seed, sample_first, sample_count, specular_depth,
                                              rayEps<double>(ctx), features_dev, ctx->d_counters, grid, s);
        }
        else if (specular_depth == 0)
            Launch<float>::features(ctx->scene32, deviceCamera<float>(*camera), global_seed, sample_first, sample_count, features_dev,
                                    ctx->d_counters, grid, s);
        else
            Launch<float>::featuresChain(ctx->scene32, deviceCamera<float>(*camera), global_seed, sample_first, sample_count, specular_depth,
                                         rayEps<float>(ctx), features_dev, ctx->d_counters, grid, s);
        CK(cudaEventRecord(ctx->ev_stop, s));
        CK(cudaMemcpyAsync(&ctx->h_counters[0], ctx->d_counters, sizeof(Counters), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        CK(cudaGetLastError());
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop);
        fillStats(stats, ctx->h_counters[0], 0, 1, ms);
        if (ctx->h_counters[0].traversal_overflow) { ctx->error = "traversal stack/heap overflow"; return MCRT_ERR_UNSUPPORTED; }
        return MCRT_OK;
    }
}

int mcrt_render_features_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t sample_first, uint32_t sample_count,
                             uint32_t global_seed, int precision, double* features_dev, mcrt_stats* stats)
{
    return renderFeatures("mcrt_render_features_dev", ctx, camera, sample_first, sample_count, global_seed, precision, 0u,
                          features_dev, stats);
}

int mcrt_render_features_chain_dev(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t sample_first, uint32_t sample_count,
                                   uint32_t global_seed, int precision, uint32_t specular_depth, double* features_dev,
                                   mcrt_stats* stats)
{
    return renderFeatures("mcrt_render_features_chain_dev", ctx, camera, sample_first, sample_count, global_seed, precision,
                          specular_depth, features_dev, stats);
}

namespace
{
    // The arguments mcrt_denoise_dev and mcrt_denoise_planes_dev both check: frame size, tile, each tile's halves,
    // iterations and sigmas. -> MCRT_OK with the parameters in *pr and the tile count in *n_tiles.
    int denoiseCheck(mcrt_ctx* ctx, const char* fn, uint32_t width, uint32_t height, uint32_t tile, const uint32_t* tile_samples,
                     const mcrt_denoise_params* params, mcrt_denoise_params* pr, uint64_t* n_tiles)
    {
        const std::string name(fn);
        const uint64_t n_pixels = (uint64_t)width * height;
        if (n_pixels == 0 || n_pixels > 0xFFFFFFFFull) { ctx->error = name + ": empty frame or more than 2^32 pixels"; return MCRT_ERR_INVALID; }
        if (tile == 0) { ctx->error = name + ": tile is 0"; return MCRT_ERR_INVALID; }
        *pr = { MCRT_DENOISE_DEFAULT_ITERATIONS, 0u, MCRT_DENOISE_DEFAULT_SIGMA_COLOR, MCRT_DENOISE_DEFAULT_SIGMA_NORMAL,
                MCRT_DENOISE_DEFAULT_SIGMA_DEPTH, MCRT_DENOISE_DEFAULT_SIGMA_ALBEDO };
        if (params) *pr = *params;
        if (pr->iterations > MCRT_DENOISE_MAX_ITERATIONS) { ctx->error = name + ": more than MCRT_DENOISE_MAX_ITERATIONS iterations"; return MCRT_ERR_INVALID; }
        for (double sg : { pr->sigma_color, pr->sigma_normal, pr->sigma_depth, pr->sigma_albedo })
            if (!std::isfinite(sg) || sg < 0.0) { ctx->error = name + ": a sigma is negative or not finite"; return MCRT_ERR_INVALID; }
        const uint64_t tiles_x = (width + tile - 1) / tile, tiles_y = (height + tile - 1) / tile;
        *n_tiles = tiles_x * tiles_y;
        for (uint64_t t = 0; t < *n_tiles; t++)
            if (tile_samples[2 * t] == 0 || tile_samples[2 * t + 1] == 0)
            {
                ctx->error = name + ": a tile has no samples in one half";
                return MCRT_ERR_INVALID;
            }
        return MCRT_OK;
    }

    // Grows the context's denoiser scratch (the denoiser's, then the tiles' {nA, nB}, then {sum v', sum out^2}), uploads
    // the tile counts and zeroes the sums. -> MCRT_OK with the device counts and sums.
    int denoiseScratch(mcrt_ctx* ctx, uint64_t n_pixels, uint64_t n_tiles, const uint32_t* tile_samples, double** d_counts, double** d_sums)
    {
        const size_t dn_values = denoiseScratchValues((size_t)n_pixels);
        const size_t scratch_values = dn_values + 2 * n_tiles + 2;
        if (ctx->denoise_scratch_values < scratch_values)
        {
            if (ctx->d_denoise_scratch) cudaFree(ctx->d_denoise_scratch);
            ctx->d_denoise_scratch = nullptr; ctx->denoise_scratch_values = 0;
            CK(cudaMalloc((void**)&ctx->d_denoise_scratch, scratch_values * sizeof(double)));
            ctx->denoise_scratch_values = scratch_values;
        }
        *d_counts = ctx->d_denoise_scratch + dn_values;
        *d_sums = *d_counts + 2 * n_tiles;
        const std::vector<double> counts(tile_samples, tile_samples + 2 * n_tiles);
        CK(cudaMemcpyAsync(*d_counts, counts.data(), counts.size() * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemsetAsync(*d_sums, 0, 2 * sizeof(double), ctx->stream));
        return MCRT_OK;
    }
}

int mcrt_denoise_dev(mcrt_ctx* ctx, const double* a_rgb_dev, const double* a_weight_dev,
                     const double* b_rgb_dev, const double* b_weight_dev, const uint32_t* tile_samples,
                     uint32_t tile, const double* features_dev, uint32_t width, uint32_t height,
                     const mcrt_denoise_params* params, double* out_rgb_dev, double* frame_error)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!a_rgb_dev || !b_rgb_dev || !tile_samples || !features_dev || !out_rgb_dev || !frame_error)
    {
        ctx->error = "mcrt_denoise_dev: null buffer";
        return MCRT_ERR_INVALID;
    }
    const uint64_t n_pixels = (uint64_t)width * height;
    if (n_pixels == 0 || n_pixels > 0xFFFFFFFFull) { ctx->error = "mcrt_denoise_dev: empty frame or more than 2^32 pixels"; return MCRT_ERR_INVALID; }
    if (tile == 0) { ctx->error = "mcrt_denoise_dev: tile is 0"; return MCRT_ERR_INVALID; }
    if (!a_weight_dev != !b_weight_dev)
    {
        ctx->error = "mcrt_denoise_dev: weight sums must be given for both halves or for neither";
        return MCRT_ERR_INVALID;
    }
    mcrt_denoise_params pr;
    uint64_t n_tiles = 0;
    if (int rc = denoiseCheck(ctx, "mcrt_denoise_dev", width, height, tile, tile_samples, params, &pr, &n_tiles)) return rc;
    CK(cudaSetDevice(ctx->device));
    double *d_counts = nullptr, *d_sums = nullptr;
    if (int rc = denoiseScratch(ctx, n_pixels, n_tiles, tile_samples, &d_counts, &d_sums)) return rc;
    cudaStream_t s = ctx->stream;
    const uint32_t tiles_x = (width + tile - 1) / tile;
    const DenoiseInput in = { a_rgb_dev, a_weight_dev, b_rgb_dev, b_weight_dev, d_counts, features_dev, width, height, tile, tiles_x };
    const DenoiseSigmas sg = { pr.sigma_color, pr.sigma_normal, pr.sigma_depth, pr.sigma_albedo };
    launchDenoise(in, sg, pr.iterations, ctx->d_denoise_scratch, out_rgb_dev, d_sums, s);
    double sums[2] = { 0.0, 0.0 };
    CK(cudaMemcpyAsync(sums, d_sums, sizeof(sums), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    *frame_error = progressiveRelativeError(sums[0], sums[1], true);
    return MCRT_OK;
}

int mcrt_denoise_planes_dev(mcrt_ctx* ctx, const double* a_rgb_dev, const double* b_rgb_dev,
                            const double* a_planes_dev, const double* b_planes_dev, uint32_t n_planes,
                            const uint32_t* tile_samples, uint32_t tile, const double* features_dev,
                            uint32_t width, uint32_t height, const mcrt_denoise_params* params,
                            double* a_out_planes_dev, double* b_out_planes_dev,
                            double* out_rgb_dev, double* frame_error)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!a_rgb_dev || !b_rgb_dev || !a_planes_dev || !b_planes_dev || !tile_samples || !features_dev || !a_out_planes_dev ||
        !b_out_planes_dev)
    {
        ctx->error = "mcrt_denoise_planes_dev: null buffer";
        return MCRT_ERR_INVALID;
    }
    if (!out_rgb_dev != !frame_error)
    {
        ctx->error = "mcrt_denoise_planes_dev: out_rgb_dev and frame_error must be given together or not at all";
        return MCRT_ERR_INVALID;
    }
    if (n_planes == 0) { ctx->error = "mcrt_denoise_planes_dev: n_planes is 0"; return MCRT_ERR_INVALID; }
    mcrt_denoise_params pr;
    uint64_t n_tiles = 0;
    if (int rc = denoiseCheck(ctx, "mcrt_denoise_planes_dev", width, height, tile, tile_samples, params, &pr, &n_tiles)) return rc;
    const uint64_t n_pixels = (uint64_t)width * height;
    if (n_planes > (1ull << 40) / n_pixels)   // 48 TB of plane states: no device holds them, and the sizes below stay in range
    {
        ctx->error = "mcrt_denoise_planes_dev: more than 2^40 plane pixels";
        return MCRT_ERR_INVALID;
    }
    // the outputs are written while the inputs are still read, and the plane outputs also hold plane states
    const uintptr_t frame_bytes = 3 * sizeof(double) * n_pixels, planes_bytes = frame_bytes * n_planes;
    struct Range { const void* p; uintptr_t bytes; };
    const Range inputs[] = { { a_rgb_dev, frame_bytes }, { b_rgb_dev, frame_bytes }, { a_planes_dev, planes_bytes },
                             { b_planes_dev, planes_bytes }, { features_dev, 8 * sizeof(double) * n_pixels } };
    const Range outputs[] = { { a_out_planes_dev, planes_bytes }, { b_out_planes_dev, planes_bytes }, { out_rgb_dev, frame_bytes } };
    auto overlap = [](const Range& u, const Range& v) {
        const uintptr_t a = (uintptr_t)u.p, b = (uintptr_t)v.p;
        return u.p && v.p && a < b + v.bytes && b < a + u.bytes;
    };
    for (int o = 0; o < 3; o++)
    {
        for (const Range& r : inputs)
            if (overlap(outputs[o], r)) { ctx->error = "mcrt_denoise_planes_dev: an output buffer overlaps an input"; return MCRT_ERR_INVALID; }
        for (int p = o + 1; p < 3; p++)
            if (overlap(outputs[o], outputs[p])) { ctx->error = "mcrt_denoise_planes_dev: two output buffers overlap"; return MCRT_ERR_INVALID; }
    }
    CK(cudaSetDevice(ctx->device));
    const size_t planes_values = denoisePlanesScratchValues((size_t)n_pixels, n_planes);
    if (ctx->denoise_planes_scratch_values < planes_values)
    {
        if (ctx->d_denoise_planes_scratch) cudaFree(ctx->d_denoise_planes_scratch);
        ctx->d_denoise_planes_scratch = nullptr; ctx->denoise_planes_scratch_values = 0;
        CK(cudaMalloc((void**)&ctx->d_denoise_planes_scratch, planes_values * sizeof(double)));
        ctx->denoise_planes_scratch_values = planes_values;
    }
    double *d_counts = nullptr, *d_sums = nullptr;
    if (int rc = denoiseScratch(ctx, n_pixels, n_tiles, tile_samples, &d_counts, &d_sums)) return rc;
    cudaStream_t s = ctx->stream;
    const uint32_t tiles_x = (width + tile - 1) / tile;
    const DenoiseInput in = { a_rgb_dev, nullptr, b_rgb_dev, nullptr, d_counts, features_dev, width, height, tile, tiles_x };
    const DenoiseSigmas sg = { pr.sigma_color, pr.sigma_normal, pr.sigma_depth, pr.sigma_albedo };
    const DenoisePlanes planes = { a_planes_dev, b_planes_dev, a_out_planes_dev, b_out_planes_dev, n_planes };
    launchDenoisePlanes(in, planes, sg, pr.iterations, ctx->d_denoise_scratch, ctx->d_denoise_planes_scratch, out_rgb_dev, d_sums, s);
    double sums[2] = { 0.0, 0.0 };
    CK(cudaMemcpyAsync(sums, d_sums, sizeof(sums), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    if (frame_error) *frame_error = progressiveRelativeError(sums[0], sums[1], true);
    return MCRT_OK;
}

int mcrt_film_resolve_dev(mcrt_ctx* ctx, const double* rgb_sum_dev, const double* weight_sum_dev, uint64_t n_pixels, double* out_rgb_dev)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!rgb_sum_dev || !weight_sum_dev || !out_rgb_dev) { ctx->error = "null buffer"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    launchResolveFilmWeighted(rgb_sum_dev, weight_sum_dev, out_rgb_dev, n_pixels, ctx->sm_count * ctx->blocks_per_sm, ctx->stream);
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaGetLastError());
    return MCRT_OK;
}

int mcrt_bvh4_host(const mcrt_scene_desc* scene, uint32_t max_leaf, void** handle, const void** nodes128, uint32_t* n_nodes)
{
    if (!scene || !handle || !nodes128 || !n_nodes) return MCRT_ERR_INVALID;
    auto* v = new std::vector<Bvh4Node>();
    const int rc = buildBvh4(max_leaf, *scene, *v);
    if (rc) { delete v; return rc; }
    *handle = v; *nodes128 = v->data(); *n_nodes = (uint32_t)v->size();
    return MCRT_OK;
}

void mcrt_bvh4_host_free(void* handle)
{
    delete static_cast<std::vector<Bvh4Node>*>(handle);
}

namespace
{
    struct Bvh4SplitHost { std::vector<Bvh4Node> nodes; std::vector<uint32_t> refs; };
}

int mcrt_bvh4_split_host(const mcrt_scene_desc* scene, double node_cost, double ref_budget, void** handle, const void** nodes128,
                         uint32_t* n_nodes, const uint32_t** refs, uint32_t* n_refs)
{
    if (!scene || !handle || !nodes128 || !n_nodes || !refs || !n_refs || !(node_cost >= 0.0) || !(ref_budget >= 1.0)) return MCRT_ERR_INVALID;
    auto* v = new Bvh4SplitHost();
    const int rc = buildBvh4Split(*scene, node_cost, ref_budget, v->nodes, v->refs);
    if (rc) { delete v; return rc; }
    *handle = v; *nodes128 = v->nodes.data(); *n_nodes = (uint32_t)v->nodes.size(); *refs = v->refs.data(); *n_refs = (uint32_t)v->refs.size();
    return MCRT_OK;
}

void mcrt_bvh4_split_host_free(void* handle)
{
    delete static_cast<Bvh4SplitHost*>(handle);
}

int mcrt_lpe_compile_host(const char* const* exprs, uint32_t n, uint32_t n_groups, uint8_t* next, uint32_t* accept,
                          uint8_t* group_symbol, uint32_t* n_states, uint32_t* n_symbols, char* error, uint32_t error_capacity)
{
    if (!next || !accept || !n_states || !n_symbols || (n_groups && !group_symbol)) return MCRT_ERR_INVALID;
    LpeTable t;
    std::string why;
    const int rc = lpeCompile(exprs, n, n_groups, t, why);
    if (error && error_capacity)
    {
        const size_t len = std::min<size_t>(why.size(), error_capacity - 1);
        std::memcpy(error, why.data(), len);
        error[len] = '\0';
    }
    if (rc != MCRT_OK) return rc;
    std::memcpy(next, t.next.data(), t.next.size());
    std::memcpy(accept, t.accept.data(), 256 * sizeof(uint32_t));
    for (uint32_t g = 0; g < n_groups; g++)
    {
        auto it = std::lower_bound(t.labels.begin(), t.labels.end(), g);
        group_symbol[g] = (uint8_t)(it != t.labels.end() && *it == g ? MCRT_LPE_SYM_LABEL0 + (it - t.labels.begin()) : MCRT_LPE_SYM_L);
    }
    *n_states = t.n_states;
    *n_symbols = t.n_symbols;
    return MCRT_OK;
}

int mcrt_lpe_compile_photon_host(const char* const* exprs, uint32_t n, uint32_t n_groups, uint8_t* rev_next, uint32_t* rev_start,
                                 uint32_t* rev_n_states, uint32_t* join, char* error, uint32_t error_capacity)
{
    if (!rev_next || !rev_start || !rev_n_states || !join) return MCRT_ERR_INVALID;
    LpeTable t;
    std::string why;
    int rc = lpeCompile(exprs, n, n_groups, t, why);
    if (rc == MCRT_OK && !t.photon_error.empty()) { why = t.photon_error; rc = MCRT_ERR_UNSUPPORTED; }
    if (error && error_capacity)
    {
        const size_t len = std::min<size_t>(why.size(), error_capacity - 1);
        std::memcpy(error, why.data(), len);
        error[len] = '\0';
    }
    if (rc != MCRT_OK) return rc;
    std::memcpy(rev_next, t.rev_next.data(), t.rev_next.size());
    std::memcpy(join, t.join.data(), t.join.size() * sizeof(uint32_t));
    *rev_start = t.rev_start;
    *rev_n_states = t.rev_n_states;
    return MCRT_OK;
}

int mcrt_frame_alloc(mcrt_ctx* ctx, uint64_t bytes, void** dev_ptr, unsigned char ipc_handle[64])
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!dev_ptr || !ipc_handle || bytes == 0) { ctx->error = "mcrt_frame_alloc: invalid arguments"; return MCRT_ERR_INVALID; }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    CK(cudaSetDevice(ctx->device));
    void* p = nullptr;
    CK(cudaMalloc(&p, bytes));
    cudaIpcMemHandle_t h;
    if (cudaIpcGetMemHandle(&h, p) != cudaSuccess) { cudaFree(p); ctx->error = "cudaIpcGetMemHandle failed"; return MCRT_ERR_CUDA; }
    CK(cudaMemset(p, 0, bytes));
    std::memcpy(ipc_handle, &h, 64);
    *dev_ptr = p;
    return MCRT_OK;
}

int mcrt_frame_open(mcrt_ctx* ctx, const unsigned char ipc_handle[64], void** dev_ptr)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!dev_ptr || !ipc_handle) { ctx->error = "mcrt_frame_open: invalid arguments"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    std::memcpy(&h, ipc_handle, 64);
    void* p = nullptr;
    CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    *dev_ptr = p;
    return MCRT_OK;
}

int mcrt_frame_close(mcrt_ctx* ctx, void* peer_ptr)
{
    if (!ctx) return MCRT_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaIpcCloseMemHandle(peer_ptr));
    return MCRT_OK;
}

int mcrt_frame_free(mcrt_ctx* ctx, void* dev_ptr)
{
    if (!ctx) return MCRT_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaFree(dev_ptr));
    return MCRT_OK;
}

int mcrt_fp64_peak(mcrt_ctx* ctx, double* dfma_per_second)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!dfma_per_second) { ctx->error = "null output"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    const int grid = ctx->sm_count * 8, iterations = 2048;
    double best = 0.0;
    for (int rep = 0; rep < 4; rep++)   // first repetition warms up
    {
        CK(cudaEventRecord(ctx->ev_start, ctx->stream));
        launchFp64Peak(reinterpret_cast<double*>(ctx->d_counters), iterations, grid, ctx->stream);
        CK(cudaEventRecord(ctx->ev_stop, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop));
        const double rate = (double)grid * 256.0 * 8.0 * iterations / (ms * 1e-3);
        if (rep > 0 && rate > best) best = rate;
    }
    *dfma_per_second = best;
    return MCRT_OK;
}

int mcrt_render_rows(mcrt_ctx* ctx, const mcrt_camera* camera, uint32_t y0, uint32_t y1, uint32_t sqrtspp,
                     uint32_t global_seed, int integrator_kind, int precision, double* out_rgb, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (!out_rgb || !camera || y1 <= y0) { ctx->error = "mcrt_render_rows: invalid arguments"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    const size_t values = (size_t)camera->width * (y1 - y0) * 3;
    // device staging for the resolved frame: kept in the context (grow-only), so that a render call
    // costs no cudaMalloc / cudaFree (both synchronise the device)
    if (ctx->host_out_values < values)
    {
        if (ctx->d_host_out) cudaFree(ctx->d_host_out);
        ctx->d_host_out = nullptr; ctx->host_out_values = 0;
        CK(cudaMalloc((void**)&ctx->d_host_out, values * sizeof(double)));
        ctx->host_out_values = values;
    }
    int rc = renderFrame(ctx, camera, y0, 1, y1 - y0, sqrtspp, global_seed, integrator_kind, precision, ctx->d_host_out, stats);
    if (rc == MCRT_OK)
    {
        cudaError_t e = cudaMemcpyAsync(out_rgb, ctx->d_host_out, values * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { ctx->error = cudaGetErrorString(e); rc = MCRT_ERR_CUDA; }
    }
    return rc;
}

int mcrt_sample_rays(mcrt_ctx* ctx, const mcrt_ray* rays, const uint32_t* pixel, const uint32_t* sample, size_t n,
                     uint32_t global_seed, int integrator_kind, int precision, double* out_rgb, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (n == 0) return MCRT_OK;
    if (!rays || !pixel || !sample || !out_rgb || n > 0xFFFFFFFFull) { ctx->error = "mcrt_sample_rays: invalid arguments"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    double* d_rays = nullptr; uint32_t* d_pixel = nullptr; uint32_t* d_sample = nullptr; double* d_out = nullptr;
    int rc = MCRT_OK;
    auto cleanup = [&]() { cudaFree(d_rays); cudaFree(d_pixel); cudaFree(d_sample); cudaFree(d_out); };
    if (cudaMalloc((void**)&d_rays, n * 6 * sizeof(double)) != cudaSuccess || cudaMalloc((void**)&d_pixel, n * 4) != cudaSuccess ||
        cudaMalloc((void**)&d_sample, n * 4) != cudaSuccess || cudaMalloc((void**)&d_out, n * 3 * sizeof(double)) != cudaSuccess)
    { cleanup(); ctx->error = "cudaMalloc failed"; return MCRT_ERR_CUDA; }
    static_assert(sizeof(mcrt_ray) == 6 * sizeof(double), "mcrt_ray must be 6 doubles");
    cudaMemcpyAsync(d_rays, rays, n * 6 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream);
    cudaMemcpyAsync(d_pixel, pixel, n * 4, cudaMemcpyHostToDevice, ctx->stream);
    cudaMemcpyAsync(d_sample, sample, n * 4, cudaMemcpyHostToDevice, ctx->stream);
    if (precision == MCRT_PRECISION_F64)
        rc = runWavefront<double>(ctx, nullptr, 0, 1, 0, 1, n, global_seed, integrator_kind, d_rays, d_pixel, d_sample, n, 1.0, d_out, stats);
    else if (precision == MCRT_PRECISION_F32)
        rc = runWavefront<float>(ctx, nullptr, 0, 1, 0, 1, n, global_seed, integrator_kind, d_rays, d_pixel, d_sample, n, 1.0, d_out, stats);
    else { ctx->error = "unknown precision"; rc = MCRT_ERR_INVALID; }
    if (rc == MCRT_OK && cudaMemcpy(out_rgb, d_out, n * 3 * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess)
    { ctx->error = "copy back failed"; rc = MCRT_ERR_CUDA; }
    cleanup();
    return rc;
}

int mcrt_trace_closest(mcrt_ctx* ctx, const mcrt_ray* rays, size_t n, int precision, mcrt_hit* hits, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (n == 0) return MCRT_OK;
    if (!rays || !hits) { ctx->error = "mcrt_trace_closest: null buffer"; return MCRT_ERR_INVALID; }
    if (!ctx->has_scene) { ctx->error = "no scene uploaded"; return MCRT_ERR_NO_SCENE; }
    CK(cudaSetDevice(ctx->device));
    double* d_rays = nullptr; double* d_tuv = nullptr; uint32_t* d_prim = nullptr;
    auto cleanup = [&]() { cudaFree(d_rays); cudaFree(d_tuv); cudaFree(d_prim); };
    if (cudaMalloc((void**)&d_rays, n * 6 * sizeof(double)) != cudaSuccess || cudaMalloc((void**)&d_tuv, n * 3 * sizeof(double)) != cudaSuccess ||
        cudaMalloc((void**)&d_prim, n * 4) != cudaSuccess)
    { cleanup(); ctx->error = "cudaMalloc failed"; return MCRT_ERR_CUDA; }
    cudaStream_t s = ctx->stream;
    cudaMemcpyAsync(d_rays, rays, n * 6 * sizeof(double), cudaMemcpyHostToDevice, s);
    cudaMemsetAsync(ctx->d_counters, 0, sizeof(Counters), s);
    const int grid = ctx->sm_count * ctx->blocks_per_sm;
    cudaEventRecord(ctx->ev_start, s);
    if (precision == MCRT_PRECISION_F64)
    {
        DeviceScene<double> sc = ctx->scene64;
        if (ctx->exact_traversal) sc.bvh4 = nullptr;
        Launch<double>::traceUser(sc, d_rays, n, d_tuv, d_prim, ctx->d_counters, grid, s);
    }
    else if (precision == MCRT_PRECISION_F32) Launch<float>::traceUser(ctx->scene32, d_rays, n, d_tuv, d_prim, ctx->d_counters, grid, s);
    else { cleanup(); ctx->error = "unknown precision"; return MCRT_ERR_INVALID; }
    cudaEventRecord(ctx->ev_stop, s);
    std::vector<double> tuv(n * 3);
    std::vector<uint32_t> prim(n);
    cudaMemcpyAsync(tuv.data(), d_tuv, n * 3 * sizeof(double), cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(prim.data(), d_prim, n * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(&ctx->h_counters[0], ctx->d_counters, sizeof(Counters), cudaMemcpyDeviceToHost, s);
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    cleanup();
    if (e != cudaSuccess) { ctx->error = cudaGetErrorString(e); return MCRT_ERR_CUDA; }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop);
    fillStats(stats, ctx->h_counters[0], 0, 1, ms);
    for (size_t i = 0; i < n; i++)
    {
        // Intersection::uv is only set when the triangle has vertex normals (triangle.cpp:57-61)
        const bool interp = prim[i] != NO_PRIM && ctx->prim_interpolates[prim[i]];
        hits[i].t = tuv[3 * i];
        hits[i].u = interp ? tuv[3 * i + 1] : 0.0;
        hits[i].v = interp ? tuv[3 * i + 2] : 0.0;
        hits[i].prim = prim[i];
        hits[i].interpolate = interp ? 1u : 0u;
    }
    if (ctx->h_counters[0].traversal_overflow) { ctx->error = "traversal stack/heap overflow"; return MCRT_ERR_UNSUPPORTED; }
    return MCRT_OK;
}

int mcrt_sampler_stream(mcrt_ctx* ctx, const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t n_shuffles,
                        uint32_t global_seed, uint32_t* out_u32x7)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (n == 0) return MCRT_OK;
    if (!pixel || !sample || !out_u32x7) { ctx->error = "mcrt_sampler_stream: null buffer"; return MCRT_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    uint32_t* d_pixel = nullptr; uint32_t* d_sample = nullptr; uint32_t* d_out = nullptr;
    auto cleanup = [&]() { cudaFree(d_pixel); cudaFree(d_sample); cudaFree(d_out); };
    if (cudaMalloc((void**)&d_pixel, n * 4) != cudaSuccess || cudaMalloc((void**)&d_sample, n * 4) != cudaSuccess ||
        cudaMalloc((void**)&d_out, n * 28) != cudaSuccess)
    { cleanup(); ctx->error = "cudaMalloc failed"; return MCRT_ERR_CUDA; }
    cudaStream_t s = ctx->stream;
    cudaMemcpyAsync(d_pixel, pixel, n * 4, cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_sample, sample, n * 4, cudaMemcpyHostToDevice, s);
    launchSamplerStream(d_pixel, d_sample, n, n_shuffles, global_seed, d_out, s);
    cudaMemcpyAsync(out_u32x7, d_out, n * 28, cudaMemcpyDeviceToHost, s);
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    cleanup();
    if (e != cudaSuccess) { ctx->error = cudaGetErrorString(e); return MCRT_ERR_CUDA; }
    return MCRT_OK;
}

int mcrt_knn_search(mcrt_ctx* ctx, int which, const double* points_xyz, size_t n, uint32_t* out_index, double* out_dist2,
                    uint32_t* out_count, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (n == 0) return MCRT_OK;
    if (!points_xyz || !out_index || !out_dist2 || !out_count || (which != 0 && which != 1))
    { ctx->error = "mcrt_knn_search: invalid arguments"; return MCRT_ERR_INVALID; }
    if (!ctx->has_photons) { ctx->error = "no photon maps uploaded"; return MCRT_ERR_NO_PHOTONS; }
    CK(cudaSetDevice(ctx->device));
    const uint32_t k = ctx->k_nearest;
    double* d_pts = nullptr; uint32_t* d_idx = nullptr; double* d_d2 = nullptr; uint32_t* d_cnt = nullptr; uint32_t* d_flag = nullptr;
    auto cleanup = [&]() { cudaFree(d_pts); cudaFree(d_idx); cudaFree(d_d2); cudaFree(d_cnt); cudaFree(d_flag); };
    if (cudaMalloc((void**)&d_pts, n * 24) != cudaSuccess || cudaMalloc((void**)&d_idx, n * k * 4) != cudaSuccess ||
        cudaMalloc((void**)&d_d2, n * k * 8) != cudaSuccess || cudaMalloc((void**)&d_cnt, n * 4) != cudaSuccess ||
        cudaMalloc((void**)&d_flag, 4) != cudaSuccess)
    { cleanup(); ctx->error = "cudaMalloc failed"; return MCRT_ERR_CUDA; }
    cudaStream_t s = ctx->stream;
    cudaMemcpyAsync(d_pts, points_xyz, n * 24, cudaMemcpyHostToDevice, s);
    cudaMemsetAsync(d_flag, 0, 4, s);
    cudaEventRecord(ctx->ev_start, s);
    launchKnnUser(ctx->photon_map[which], k, d_pts, n, d_idx, d_d2, d_cnt, d_flag, ctx->sm_count * ctx->blocks_per_sm, s);
    cudaEventRecord(ctx->ev_stop, s);
    uint32_t flag = 0;
    cudaMemcpyAsync(out_index, d_idx, n * k * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(out_dist2, d_d2, n * k * 8, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(out_count, d_cnt, n * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(&flag, d_flag, 4, cudaMemcpyDeviceToHost, s);
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    cleanup();
    if (e != cudaSuccess) { ctx->error = cudaGetErrorString(e); return MCRT_ERR_CUDA; }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop);
    if (stats) { std::memset(stats, 0, sizeof(*stats)); stats->knn_queries = n; stats->gpu_ms_total = ms; stats->gpu_ms_knn = ms; }
    if (flag) { ctx->error = "k-NN frontier overflow"; return MCRT_ERR_UNSUPPORTED; }
    return MCRT_OK;
}

int mcrt_photon_gather_radius(mcrt_ctx* ctx, double r_caustic, double r_global)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if (r_caustic == 0.0 && r_global == 0.0) { ctx->gather_r2[0] = ctx->gather_r2[1] = 0.0; return MCRT_OK; }
    const double r[2] = { r_caustic, r_global };
    for (int w = 0; w < 2; w++)
        if (!(r[w] > 0.0) || !std::isfinite(r[w] * r[w]))
        { ctx->error = "mcrt_photon_gather_radius: radii must be (0, 0) or two positive finite numbers"; return MCRT_ERR_INVALID; }
    ctx->gather_r2[0] = r_caustic * r_caustic; ctx->gather_r2[1] = r_global * r_global;
    return MCRT_OK;
}

int mcrt_photon_gather_search(mcrt_ctx* ctx, int which, const double* points_xyz, size_t n, double radius, uint32_t* out_count,
                              double* out_flux_sum, double* out_cone_sum, mcrt_stats* stats)
{
    if (!ctx) return MCRT_ERR_INVALID;
    if ((which != 0 && which != 1) || !(radius > 0.0) || !std::isfinite(radius * radius))
    { ctx->error = "mcrt_photon_gather_search: invalid arguments"; return MCRT_ERR_INVALID; }
    if (n == 0) return MCRT_OK;
    if (!points_xyz || !out_count || !out_flux_sum || !out_cone_sum) { ctx->error = "mcrt_photon_gather_search: null buffer"; return MCRT_ERR_INVALID; }
    if (!ctx->has_photons) { ctx->error = "no photon maps uploaded"; return MCRT_ERR_NO_PHOTONS; }
    CK(cudaSetDevice(ctx->device));
    double* d_pts = nullptr; uint32_t* d_cnt = nullptr; double* d_flux = nullptr; double* d_cone = nullptr; uint32_t* d_flag = nullptr;
    auto cleanup = [&]() { cudaFree(d_pts); cudaFree(d_cnt); cudaFree(d_flux); cudaFree(d_cone); cudaFree(d_flag); };
    if (cudaMalloc((void**)&d_pts, n * 24) != cudaSuccess || cudaMalloc((void**)&d_cnt, n * 4) != cudaSuccess ||
        cudaMalloc((void**)&d_flux, n * 24) != cudaSuccess || cudaMalloc((void**)&d_cone, n * 24) != cudaSuccess ||
        cudaMalloc((void**)&d_flag, 4) != cudaSuccess)
    { cleanup(); ctx->error = "cudaMalloc failed"; return MCRT_ERR_CUDA; }
    cudaStream_t s = ctx->stream;
    cudaMemcpyAsync(d_pts, points_xyz, n * 24, cudaMemcpyHostToDevice, s);
    cudaMemsetAsync(d_flag, 0, 4, s);
    cudaEventRecord(ctx->ev_start, s);
    launchGatherUser(ctx->photon_map[which], d_pts, n, radius * radius, d_cnt, d_flux, d_cone, d_flag, ctx->sm_count * ctx->blocks_per_sm, s);
    cudaEventRecord(ctx->ev_stop, s);
    uint32_t flag = 0;
    cudaMemcpyAsync(out_count, d_cnt, n * 4, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(out_flux_sum, d_flux, n * 24, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(out_cone_sum, d_cone, n * 24, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(&flag, d_flag, 4, cudaMemcpyDeviceToHost, s);
    cudaError_t e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) e = cudaGetLastError();
    cleanup();
    if (e != cudaSuccess) { ctx->error = cudaGetErrorString(e); return MCRT_ERR_CUDA; }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop);
    if (stats) { std::memset(stats, 0, sizeof(*stats)); stats->knn_queries = n; stats->gpu_ms_total = ms; stats->gpu_ms_knn = ms; }
    if (flag) { ctx->error = "gather stack overflow"; return MCRT_ERR_UNSUPPORTED; }
    return MCRT_OK;
}

} // extern "C"
