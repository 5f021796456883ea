// Wavefront path tracer: one kernel per stage over compacted queues that live in HBM.
//
// Stage kernels (each a grid-stride "persistent" launch sized to the SM count; queue lengths are
// read from device memory so the host enqueues iterations without synchronising):
//   k_generate  Camera::samplePixel ray generation (source/camera/camera.cpp:66-99) for the next
//               (pixel, sample) work items, appended behind the survivors of the last bounce
//   k_extend    Scene::intersect for every live path            (source/scene/scene.cpp:151-176)
//   k_shade     one iteration of PathTracer::sampleRay's loop   (source/integrator/path-tracer/
//               path-tracer.cpp:21-50): miss/sky, Interaction, sampleEmissive, the light-sampling
//               half of sampleDirect, sampleBSDF, throughput, absorb (Russian roulette),
//               RefractionHistory::update; survivors are compacted into the other path buffer with
//               warp-aggregated appends, NEE candidates into the shadow queue
//   k_shadow    the visibility half of Integrator::sampleDirect (source/integrator/
//               integrator.cpp:68-86): closest-hit query, "hit that very light", MIS weight
//   k_advance   queue bookkeeping between iterations (one thread)
//
// Path state is ping-ponged between two compact buffers (no index indirection: every access is a
// coalesced 16/32-byte vector load/store). Radiance contributions are scattered straight into the
// float64 film with RED.ADD.F64, adjacent lanes hitting adjacent pixels.
#pragma once

#include "bsdf.cuh"
#include "intersect.cuh"
#include "bvh4.cuh"
#include "photon.cuh"
#include "film.cuh"
#include "mcrt_abi.h"

// launch-bound knobs (overridable at build time for tuning experiments)
// (float traversal runs at 64 registers / 32 warps per SM; double traversal keeps 128 registers, since it
// would spill at 64; shade runs 3 CTAs of 128 threads)
#ifndef MCRT_TRACE_MINBLOCKS_F64
#define MCRT_TRACE_MINBLOCKS_F64 2
#endif
#ifndef MCRT_TRACE_MINBLOCKS_F32
#define MCRT_TRACE_MINBLOCKS_F32 4
#endif
#ifndef MCRT_TRACE_MINBLOCKS_F64_PRUNED   // double traversal without quadric code needs ~100 registers instead of 128
#define MCRT_TRACE_MINBLOCKS_F64_PRUNED 4
#endif
#ifndef MCRT_TRACE_MINBLOCKS_FAST          // order-free search (bvh4.cuh). 2 CTAs of 256: no spills; measured on C2, H100, DESIGN §10.6
#define MCRT_TRACE_MINBLOCKS_FAST 2
#endif
#ifndef MCRT_TRACE_MINBLOCKS_DYN           // order-free search with dynamic fetch (measured on the spaceship: 64 registers beat 80)
#define MCRT_TRACE_MINBLOCKS_DYN 4
#endif
#ifndef MCRT_KNN_MINBLOCKS                 // CTAs of 4 query warps per SM for k_knn
#define MCRT_KNN_MINBLOCKS 8   // 64 registers: the dependent warp collectives of a query need many warps to hide behind
#endif
#ifndef MCRT_GATHER_MINBLOCKS              // CTAs of 4 query warps per SM for k_gather
#define MCRT_GATHER_MINBLOCKS 3   // no spills in any instantiation (float64: 164 registers at most; 4 CTAs spill, DESIGN §5)
#endif
#ifndef MCRT_SHADE_MINBLOCKS
#define MCRT_SHADE_MINBLOCKS 3
#endif
#ifndef MCRT_SHADE_MINBLOCKS_LITE   // k_shade without the GGX / Oren-Nayar / conductor code: 166 registers, so 3 CTAs
#define MCRT_SHADE_MINBLOCKS_LITE 3  // hold it without spills; on the H100 that beat 4, 5 and 6 CTAs, which spill (DESIGN.md §10)
#endif
#ifndef MCRT_SORT_ORIGIN_BITS
#define MCRT_SORT_ORIGIN_BITS 4
#endif
#ifndef MCRT_SORT_DIR_Q
#define MCRT_SORT_DIR_Q 1
#endif

namespace mcrt
{
    constexpr int IOR_STACK_CAPACITY = 8; // iors[0] is implicit (scene ior); 7 stored entries

    struct Counters
    {
        uint32_t n_cur, n_next, n_shadow, n_gen;
        unsigned long long next_work, total_work;
        // statistics
        unsigned long long paths, extension_rays, shadow_rays, box_tests, prim_tests, knn_queries;
        unsigned long long shadow_box_tests, shadow_prim_tests; // the k_shadow share of box/prim tests
        unsigned long long ior_stack_overflows;
        unsigned long long replayed_rays;   // rays re-traced in the reference's order (ambiguous closest hit)
        uint32_t fetch_extend, fetch_shadow; // dynamic-fetch cursors of k_extend / k_shadow (traceManyFast), reset by k_advance
        uint32_t traversal_overflow, max_depth;
        uint32_t n_knn, _pad;
        // diagnostics of k_extend: sum over rays of (box+prim tests) and sum over warps of 32*max
        unsigned long long work_sum, work_warpmax;
        // photon emission pass: photons stored so far in the caustic / global arrays
        unsigned long long n_photons[2];
        uint32_t photon_overflow, _pad2;
    };

    template <class R> struct PathBuffer
    {
        V4<R>* ray_o;    // start.xyz, medium_ior
        V4<R>* ray_d;    // direction.xyz, refraction_scale
        V4<R>* thr;      // throughput.xyz, ls.bsdf_pdf
        V4<R>* iors_a;   // iors[1..4]  (touched only while the path is inside nested media)
        V4<R>* iors_b;   // iors[5..7]
        uint4* meta;     // pixel, sample, depth | diffuse_depth<<16, refraction_level
        uint4* meta2;    // ls.light as light index, ior_count | dirac<<8 | first lobe<<9 (FILM_MODE_AOV), film_index, source prim (fast mode)
    };

    // One shadow ray. k_shadow reads the queue through the ray-coherence sort, i.e. at random positions,
    // so the fields it always needs (o, d, meta) share one line instead of being three scattered reads;
    // k comes last because it is read only when the light is visible. float64: one 128-byte line, with
    // 16 bytes of padding after meta; float: one 64-byte half-line.
    template <class R> struct alignas(16 * sizeof(R)) ShadowRecord
    {
        V4<R> o;         // start.xyz, bsdf_pdf
        V4<R> d;         // direction.xyz, area * cos_light
        uint4 meta;      // light prim, film_index, source prim, sample (FILM_MODE_AOV: the AOV plane)
        V4<R> k;         // bsdf_absIdotN * Le * throughput, select_probability
    };
    static_assert(sizeof(ShadowRecord<double>) == 128 && sizeof(ShadowRecord<float>) == 64, "one shadow record per line");
    static_assert(offsetof(ShadowRecord<double>, k) == 96, "the float64 padding is the 16-byte chunk 5 (k_shade writes it)");

    // Ray-coherence sort. Incoherent secondary rays run the traversal kernels at ~10 of 32 lanes
    // active (ncu, r1 baseline) while coherent primary rays reach 31; so every queue is re-ordered
    // each bounce by a 17-bit key = direction class (cube face + 2 sign bits) | Morton code of the
    // origin cell (16^3 grid over the scene bounds). It is a counting sort: the producer kernel takes
    // rank = atomicAdd(&hist[key], 1) when it appends an entry, k_sort_scan turns the histogram into
    // bin starts (and zeroes it), k_sort_scatter writes order[bin_start[key] + rank] = entry. The
    // consumers index their queue through `order`; state stays where it was written.
    constexpr uint32_t SORT_ORIGIN_BITS = MCRT_SORT_ORIGIN_BITS;          // per axis
    constexpr uint32_t SORT_DIR_Q = MCRT_SORT_DIR_Q;                      // bits per in-face coordinate
    constexpr uint32_t SORT_DIR_BITS = 3 + 2 * SORT_DIR_Q;
    constexpr uint32_t SORT_KEY_BITS = 3 * SORT_ORIGIN_BITS + SORT_DIR_BITS;
    constexpr uint32_t SORT_BINS = 1u << SORT_KEY_BITS;

    struct RaySort
    {
        uint32_t* path_key[2];   // per path buffer
        uint32_t* path_rank[2];
        uint32_t* path_order;    // permutation of the current path buffer (null: identity)
        uint32_t* shadow_key;
        uint32_t* shadow_rank;
        uint32_t* shadow_order;
        uint32_t* hist_path;     // [SORT_BINS]
        uint32_t* hist_shadow;   // [SORT_BINS]
        uint32_t* bin_start;     // [SORT_BINS] scratch: exclusive scan within each 1024-bin CTA segment
        uint32_t* block_offset;  // [2 * SORT_BINS / 1024]: segment offsets, then segment totals
        uint32_t* done_counter;  // last-CTA-done counter of k_sort_scan
        uint32_t shade_sorted;   // 1: k_shade also walks the queue in sorted order
        // shade-coherence sort: k_shade walks the paths grouped by the material class of the primitive they hit
        // (DeviceScene::shade_class), so that a warp runs one material branch instead of all of them
        uint32_t* shade_key;     // per path slot: class of the hit (k_shade_key)
        uint32_t* shade_rank;
        uint32_t* shade_order;   // null: disabled
        uint32_t* hist_shade;    // [SORT_BINS] (only SHADE_CLASS_BINS used; shares k_sort_scan)
        uint32_t prim_scale;     // != 0: the cell field of the key is the source primitive's position in
                                 // BVH order, (prim * prim_scale) >> 32 (large scenes: the BVH order is a
                                 // far finer spatial index than a 16^3 grid where the geometry is dense)
        float key_min[3], key_scale[3]; // origin -> cell: (o - key_min) * key_scale in [0, 2^SORT_ORIGIN_BITS)
    };

    MCRT_D uint32_t spreadBits3(uint32_t v) // bit k -> bit 3k (up to 10 bits)
    {
        v = (v | (v << 16)) & 0x030000FFu;
        v = (v | (v << 8)) & 0x0300F00Fu;
        v = (v | (v << 4)) & 0x030C30C3u;
        v = (v | (v << 2)) & 0x09249249u;
        return v;
    }

    // src_prim: ordered primitive the ray leaves from (NO_PRIM for camera rays)
    template <class R>
    MCRT_D uint32_t rayKey(const RaySort& rs, const V3<R>& o, const V3<R>& d, uint32_t src_prim)
    {
        uint32_t cell;
        if (rs.prim_scale && src_prim != NO_PRIM)
        {
            cell = (uint32_t)(((unsigned long long)src_prim * rs.prim_scale) >> 32);
        }
        else
        {
            constexpr float CELLS = (float)(1u << SORT_ORIGIN_BITS);
            float cx = ((float)o.x - rs.key_min[0]) * rs.key_scale[0];
            float cy = ((float)o.y - rs.key_min[1]) * rs.key_scale[1];
            float cz = ((float)o.z - rs.key_min[2]) * rs.key_scale[2];
            uint32_t ix = (uint32_t)fminf(fmaxf(cx, 0.0f), CELLS - 1.0f);
            uint32_t iy = (uint32_t)fminf(fmaxf(cy, 0.0f), CELLS - 1.0f);
            uint32_t iz = (uint32_t)fminf(fmaxf(cz, 0.0f), CELLS - 1.0f);
            cell = spreadBits3(ix) | (spreadBits3(iy) << 1) | (spreadBits3(iz) << 2);
        }
        float dx = (float)d.x, dy = (float)d.y, dz = (float)d.z;
        float ax = fabsf(dx), ay = fabsf(dy), az = fabsf(dz);
        uint32_t face; float u, v, m;
        if (ax >= ay && ax >= az) { face = dx < 0.0f ? 1u : 0u; u = dy; v = dz; m = ax; }
        else if (ay >= az)        { face = dy < 0.0f ? 3u : 2u; u = dx; v = dz; m = ay; }
        else                      { face = dz < 0.0f ? 5u : 4u; u = dx; v = dy; m = az; }
        // in-face coordinates in [-1,1] -> SORT_DIR_Q bits each
        constexpr float Q = (float)(1u << SORT_DIR_Q);
        float inv = m > 0.0f ? 0.5f * Q / m : 0.0f;
        uint32_t qu = (uint32_t)fminf(fmaxf(u * inv + 0.5f * Q, 0.0f), Q - 1.0f);
        uint32_t qv = (uint32_t)fminf(fmaxf(v * inv + 0.5f * Q, 0.0f), Q - 1.0f);
        uint32_t dir = (face << (2 * SORT_DIR_Q)) | (qu << SORT_DIR_Q) | qv;
        return (dir << (3 * SORT_ORIGIN_BITS)) | cell;
    }

    // rank = atomicAdd(&hist[key], 1) with the lanes of a warp that share a key aggregated into one
    // atomic (camera rays all fall into a handful of bins: un-aggregated that is ~0.5 M same-address
    // atomics per launch). Call with the warp converged; lanes with pred == false do not take part.
    MCRT_D uint32_t sortRank(uint32_t* hist, uint32_t key, bool pred)
    {
        const unsigned active = __ballot_sync(0xFFFFFFFFu, pred);
        uint32_t rank = 0;
        if (pred)
        {
            const unsigned peers = __match_any_sync(active, key);
            const unsigned lane = threadIdx.x & 31u;
            const int leader = __ffs(peers) - 1;
            uint32_t base = 0;
            if ((int)lane == leader) base = atomicAdd(&hist[key], (uint32_t)__popc(peers));
            base = __shfl_sync(peers, base, leader);
            rank = base + __popc(peers & ((1u << lane) - 1u));
        }
        return rank;
    }

    // Photon emission pass (PhotonMapper::PhotonMapper + emitPhoton, photon-mapper.cpp:24-277).
    // Work item w = emission j of light l: emit_offsets[l] <= w < emit_offsets[l+1].
    template <class R> struct EmitParams
    {
        const unsigned long long* emit_offsets;  // [n_lights + 1] prefix sums of num_light_emissions
        const V4<R>* photon_flux;                // [n_lights] light_flux / num_light_emissions
        float4* photons[2];                      // output: 2 float4 per photon {flux.xyz,pos.x | pos.yz,phi,theta}
        uint32_t* lights[2];                     // output: the index of the light that emitted each photon
        unsigned long long capacity[2];
        R non_caustic_reject;                    // 1 / caustic_factor
        uint32_t pass;                           // emissions of light l take the indices pass * n_l + j (mcrt_photon_emit_pass)
        // k_emit_*<R, true> (an LPE table is set): the reversed expressions' DFA (lpe.h; symbols of WaveParams::lpe_*),
        // its start state, and the output, the state of each photon before its storage vertex's event
        const uint8_t* lpe_rev_next;
        uint32_t lpe_rev_start;
        uint32_t* lpe_states[2];
    };

    template <class R> struct WaveParams
    {
        DeviceScene<R> scene;
        DeviceCamera<R> camera;
        PathBuffer<R> buf[2];
        ShadowRecord<R>* shadow;
        V4<R>* hits;           // t,u,v,prim
        Counters* counters;
        double* film;          // [n_film][3]
        // user-supplied rays (mcrt_sample_rays); null for camera rendering
        const double* user_rays;
        const uint32_t* user_pixel;
        const uint32_t* user_sample;
        // camera work over a subset of the pixels (k_generate<R, FILM, true>): the pixels' positions in the
        // n_rows x width grid, tile-major and row-major inside a tile; n_pixels is then the list's length
        const uint32_t* pixel_list;
        uint32_t capacity;
        uint32_t global_seed;
        uint32_t spp;
        uint32_t row_first;     // first image row of this render
        uint32_t row_step;      // distance between consecutive rendered rows (1 = contiguous block)
        uint32_t n_pixels;      // pixels in this render (rows * width)
        uint32_t integrator;    // MCRT_INTEGRATOR_*
        R ray_eps;              // C::EPSILON in parity mode; scale-aware in fast mode
        PhotonParams<R> pm;     // photon maps + k-NN query queue (photon-mapped renders only)
        RaySort sort;           // coherence sort of the path / shadow queues (null order = disabled)
        const uint32_t* sobol_bytes; // byte-sliced Sobol matrices [6][4][256] (makeSobolByteTable)
        EmitParams<R> emit;         // photon emission pass (mcrt_photon_emit) only
        FilmParams filmp;           // reconstruction filter (FILM_MODE_SPLAT only)
        // light-group render (mcrt_render_accumulate_groups_dev): `film` holds n_planes planes of plane_values values each;
        // a contribution of light l goes to plane group_of_light[l], the sky's to plane n_planes - 1. 0: one plane.
        // AOV render (mcrt_render_accumulate_aovs_dev, FILM_MODE_AOV): n_planes = MCRT_AOV_COUNT light-path planes instead;
        // photon-mapper components (mcrt_render_accumulate_photon_components_dev, FILM_MODE_AOV): MCRT_PM_COMPONENT_COUNT
        const uint32_t* group_of_light;
        size_t plane_values;
        uint32_t n_planes;
        uint32_t film_mode;     // FilmMode: which kernel instantiations the launchers pick (host only)
        // LPE render (mcrt_render_accumulate_lpe_dev, FILM_MODE_LPE): n_planes = the expressions; the DFA's
        // transitions [states][lpe_symbols], accept masks [256] and the symbol of each light (lpe.h)
        const uint8_t* lpe_next;
        const uint32_t* lpe_accept;
        const uint8_t* lpe_light_symbol;
        uint32_t lpe_symbols;
    };

    // ------------------------------------------------------------------------------------------
    template <class R> struct Mode;
    template <> struct Mode<double> { static constexpr bool parity = true; static constexpr int trace_minblocks = MCRT_TRACE_MINBLOCKS_F64; static constexpr int trace_minblocks_pruned = MCRT_TRACE_MINBLOCKS_F64_PRUNED; };
    template <> struct Mode<float> { static constexpr bool parity = false; static constexpr int trace_minblocks = MCRT_TRACE_MINBLOCKS_F32; static constexpr int trace_minblocks_pruned = MCRT_TRACE_MINBLOCKS_F32; };

    // FAST (parity mode only): order-free search over the 4-wide BVH with the reference-order replay as
    // fallback (bvh4.cuh); the launchers pick it whenever the scene has that BVH
    template <int PRIMS = PRIMS_ALL, bool FAST = false, class R>
    MCRT_D Hit<R> traceClosest(const DeviceScene<R>& sc, const V3<R>& o, const V3<R>& d, uint32_t skip_prim,
                               TraceCounters& cnt, uint32_t& overflow)
    {
        RayQ<R> rq;
        rq.o = o; rq.d = d;
        if constexpr (!(Mode<R>::parity && FAST) || PRIMS == PRIMS_ALL) rq.inv_d = R(1) / d;   // the order-free search needs it for quadrics only (clip-box test)
        if constexpr (Mode<R>::parity)
        {
            if constexpr (FAST)
            {
                // order-free search; the rare ray whose answer could depend on the visiting order is
                // replayed in the reference's order (bvh4.cuh)
                bool ambiguous;
                Hit<R> h = traverseFast<PRIMS>(sc, rq, cnt, ambiguous);
                if (ambiguous)
                {
                    const DeviceScene<R> sc_copy = sc;   // the out-of-line call takes addresses: keep those copies off the hot path
                    RayQ<R> rq_copy = rq;
                    rq_copy.inv_d = R(1) / d;            // only the replay's float64 slab test needs it
                    Hit<R> h2;
                    traceReferenceOrderOutOfLine<PRIMS>(&sc_copy, &rq_copy, &h2, &cnt.box_tests, &cnt.prim_tests, &overflow);
                    h = h2;
                    cnt.replayed++;
                }
                return h;
            }
            else
            {
                return traverseReferenceOrder<PRIMS>(sc, rq, cnt, overflow);
            }
        }
        else
        {
            return traverseWide<PRIMS>(sc, rq, skip_prim, cnt, overflow);
        }
    }

    // Occlusion query of next-event estimation for the order-free search (parity mode): the hit returned has
    // prim == target iff the target is what Scene::intersect would return (bvh4.cuh, FastSearch<PRIMS, true>)
    template <int PRIMS>
    MCRT_D Hit<double> traceVisible(const DeviceScene<double>& sc, const V3<double>& o, const V3<double>& d, uint32_t target,
                                    TraceCounters& cnt, uint32_t& overflow)
    {
        RayQ<double> rq;
        rq.o = o; rq.d = d;
        if constexpr (PRIMS == PRIMS_ALL) rq.inv_d = 1.0 / d;
        FastSearch<PRIMS, true> fs;
        if (!fs.beginOcclusion(sc, rq, target, cnt)) { Hit<double> miss = fs.best; miss.prim = NO_PRIM; return miss; }
        if (fs.verdict != 2u) { while (fs.step(sc, rq, cnt)) { } }     // 2 already: a degenerate ray goes straight to the replay
        Hit<double> h = fs.best;
        if (fs.verdict == 1u) h.prim = NO_PRIM;
        else if (fs.verdict == 2u)
        {
            const DeviceScene<double> sc_copy = sc;
            RayQ<double> rq_copy = rq;
            rq_copy.inv_d = 1.0 / d;
            Hit<double> h2;
            traceReferenceOrderOutOfLine<PRIMS>(&sc_copy, &rq_copy, &h2, &cnt.box_tests, &cnt.prim_tests, &overflow);
            h = h2;
            cnt.replayed++;
        }
        return h;
    }

    MCRT_D void filmAdd(double* film, uint32_t index, double r, double g, double b)
    {
        if (r != 0.0) atomicAdd(&film[3 * (size_t)index + 0], r);
        if (g != 0.0) atomicAdd(&film[3 * (size_t)index + 1], g);
        if (b != 0.0) atomicAdd(&film[3 * (size_t)index + 2], b);
    }

    template <class R>
    MCRT_D void filmAddV(double* film, uint32_t index, const V3<R>& v)
    {
        filmAdd(film, index, (double)v.x, (double)v.y, (double)v.z);
    }

    // image pixel of a film index (rows may be interleaved over ranks)
    template <class R>
    MCRT_D uint32_t pixelOfFilmIndex(const WaveParams<R>& p, uint32_t film_index)
    {
        const uint32_t row = film_index / p.camera.width, col = film_index - row * p.camera.width;
        return (p.row_first + row * p.row_step) * p.camera.width + col;
    }

    // Film modes of the depositing kernels. FILM_MODE_BOX: the default box film, the kernels every benchmark and parity
    // case runs; FILM_MODE_SPLAT: a reconstruction filter; FILM_MODE_GROUPS: the box film with one plane per light group;
    // FILM_MODE_AOV: the box film with one plane per class of contribution, the plane each deposit site names - the
    // light-path planes (MCRT_AOV_*) in the path tracer, the estimator planes (MCRT_PM_*) in the photon mapper;
    // FILM_MODE_LPE: the box film with one plane per light path expression, a deposit into every plane whose bit is set
    // in the accept mask of its event string (path tracer only)
    enum FilmMode : int { FILM_MODE_BOX = 0, FILM_MODE_SPLAT = 1, FILM_MODE_GROUPS = 2, FILM_MODE_AOV = 3, FILM_MODE_LPE = 4 };

    // FILM_MODE_LPE: the DFA of the expressions (lpe.h). Lanes of a warp sit in different states, so the few-KB tables are
    // read through the read-only data path rather than from constant memory.
    template <class R>
    MCRT_D uint32_t lpeNext(const WaveParams<R>& p, uint32_t state, uint32_t symbol)
    {
        return __ldg(&p.lpe_next[state * p.lpe_symbols + symbol]);
    }
    template <class R>
    MCRT_D uint32_t lpeAccept(const WaveParams<R>& p, uint32_t state) { return __ldg(&p.lpe_accept[state]); }
    // symbol of an emitter: its label's, or the unlabelled L (NO_PRIM: an emissive primitive that is not a light)
    template <class R>
    MCRT_D uint32_t lpeLightSymbol(const WaveParams<R>& p, uint32_t light)
    {
        return light == NO_PRIM ? (uint32_t)MCRT_LPE_SYM_L : (uint32_t)__ldg(&p.lpe_light_symbol[light]);
    }
    // event of a scattering vertex: the interaction type the reference selected, smooth (dirac_delta) or rough
    MCRT_D uint32_t lpeVertexSymbol(uint32_t type, bool dirac_delta)
    {
        if (type == IA_DIFFUSE) return MCRT_LPE_SYM_RD;
        if (type == IA_REFLECT) return dirac_delta ? MCRT_LPE_SYM_RS : MCRT_LPE_SYM_RG;
        return dirac_delta ? MCRT_LPE_SYM_TS : MCRT_LPE_SYM_TG;
    }

    // AOV plane of a contribution. lobe: interaction type + 1 of the path's first scattering vertex, 0 for the camera
    // ray's own miss (the sky: background) or emitter hit (emission); indirect: the light path has more than one
    // scattering vertex
    MCRT_D uint32_t aovPlane(uint32_t lobe, bool indirect, bool miss)
    {
        if (lobe == 0u) return miss ? MCRT_AOV_BACKGROUND : MCRT_AOV_EMISSION;
        const uint32_t direct = lobe == IA_DIFFUSE + 1u ? MCRT_AOV_DIFFUSE_DIRECT
                              : (lobe == IA_REFLECT + 1u ? MCRT_AOV_REFLECTION_DIRECT : MCRT_AOV_TRANSMISSION_DIRECT);
        return direct + (indirect ? 1u : 0u);
    }

    // Film::deposit of one radiance contribution of sample (pixel, sample). light: index of the emitter it comes from,
    // NO_PRIM for the sky (read by FILM_MODE_GROUPS only); plane: its AOV plane (FILM_MODE_AOV), or its accept mask, one
    // bit per plane (FILM_MODE_LPE)
    template <int FILM, class R>
    MCRT_D void depositRadiance(const WaveParams<R>& p, uint32_t film_index, uint32_t pixel, uint32_t sample, const V3<R>& v,
                                uint32_t light = NO_PRIM, uint32_t plane = 0u)
    {
        if constexpr (FILM == FILM_MODE_BOX)
        {
            filmAddV(p.film, film_index, v);
        }
        else if constexpr (FILM == FILM_MODE_GROUPS)
        {
            const uint32_t plane = light == NO_PRIM ? p.n_planes - 1u : p.group_of_light[light];
            filmAddV(p.film + plane * p.plane_values, film_index, v);
        }
        else if constexpr (FILM == FILM_MODE_AOV)
        {
            filmAddV(p.film + plane * p.plane_values, film_index, v);
        }
        else if constexpr (FILM == FILM_MODE_LPE)
        {
            for (uint32_t m = plane; m; m &= m - 1u) filmAddV(p.film + (uint32_t)(__ffs(m) - 1) * p.plane_values, film_index, v);
        }
        else
        {
            filmSplatSample(p.filmp, p.global_seed, pixel, sample, (double)v.x, (double)v.y, (double)v.z);
        }
    }

    // Warp-aggregated append: one atomic per warp, lanes get consecutive slots.
    MCRT_D uint32_t warpAppend(uint32_t* counter, bool pred)
    {
        const unsigned mask = __ballot_sync(0xFFFFFFFFu, pred); // callers keep the warp converged
        if (!pred) return 0xFFFFFFFFu;
        const unsigned lane = threadIdx.x & 31u;
        const unsigned leader = __ffs(mask) - 1;
        uint32_t base = 0;
        if (lane == leader) base = atomicAdd(counter, (uint32_t)__popc(mask));
        base = __shfl_sync(mask, base, leader);
        return base + __popc(mask & ((1u << lane) - 1u));
    }

    MCRT_D void flushStats(Counters* c, const TraceCounters& cnt, unsigned long long rays, bool shadow, uint32_t overflow)
    {
        // block-level reduction through warp shuffles, then one atomic per warp
        unsigned long long b = cnt.box_tests, p = cnt.prim_tests, r = rays;
        uint32_t a = cnt.replayed;
        for (int off = 16; off > 0; off >>= 1)
        {
            b += __shfl_down_sync(0xFFFFFFFFu, b, off);
            p += __shfl_down_sync(0xFFFFFFFFu, p, off);
            r += __shfl_down_sync(0xFFFFFFFFu, r, off);
            a += __shfl_down_sync(0xFFFFFFFFu, a, off);
        }
        if ((threadIdx.x & 31u) == 0)
        {
            if (a) atomicAdd(&c->replayed_rays, (unsigned long long)a);
            if (b) atomicAdd(&c->box_tests, b);
            if (p) atomicAdd(&c->prim_tests, p);
            if (shadow && b) atomicAdd(&c->shadow_box_tests, b);
            if (shadow && p) atomicAdd(&c->shadow_prim_tests, p);
            if (r) atomicAdd(shadow ? &c->shadow_rays : &c->extension_rays, r);
        }
        if (overflow) atomicOr(&c->traversal_overflow, 1u);
    }

    // ------------------------------------------------------------------------------------------
    // Camera ray for (pixel, sample): camera.cpp:66-95
    template <class R>
    MCRT_D void cameraRay(const DeviceCamera<R>& c, R scene_ior, uint32_t pixel, const SamplerState& smp,
                          V3<R>& start, V3<R>& direction)
    {
        const uint32_t x = pixel % c.width, y = pixel / c.width;
        R pixel_size = c.sensor_width / R(c.width);
        R half_w = R(c.width) * R(0.5), half_h = R(c.height) * R(0.5);
        R u[2];
        samplerGet<R, DIM_PIXEL, 2>(smp, u);
        R px = R(x) + u[0], py = R(y) + u[1];
        R lx = pixel_size * (half_w - px), ly = pixel_size * (half_h - py);
        direction = normalize(c.forward * c.focal_length + c.left * lx + c.up * ly);
        start = c.eye;
        if (c.thin_lens)
        {
            R ul[2];
            samplerGet<R, DIM_LENS, 2>(smp, ul);
            // Sampling::uniformDisk, sampling.hpp:30-34
            R azimuth = ul[1] * Consts<R>::TWO_PI;
            R sn, cs;
            msincos(azimuth, &sn, &cs);
            R su = msqrt(ul[0]);
            R ax = (cs * su) * c.aperture_radius, ay = (sn * su) * c.aperture_radius;
            V3<R> focus_point = start + direction * (c.focus_distance / dot(direction, c.forward));
            V3<R> s2 = c.eye + c.left * ax + c.up * ay;
            direction = normalize(focus_point - s2);
            start = s2;
        }
    }

    // LIST: camera work item w is sample w / n_pixels of pixel pixel_list[w % n_pixels] (adaptive sampling);
    // otherwise of pixel w % n_pixels
    template <class R, bool FILM, bool LIST>
    __global__ void __launch_bounds__(256) k_generate(WaveParams<R> p, int next)
    {
        Counters* c = p.counters;
        const uint32_t n_next = c->n_next;
        const unsigned long long remaining = c->total_work - c->next_work;
        const uint32_t room = p.capacity - n_next;
        const uint32_t count = remaining < (unsigned long long)room ? (uint32_t)remaining : room;
        if (blockIdx.x == 0 && threadIdx.x == 0) c->n_gen = count;
        const unsigned long long base_work = c->next_work;
        const PathBuffer<R>& out = p.buf[next];

        const uint32_t count_rounded = (count + 31u) & ~31u;
        for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < count_rounded; j += gridDim.x * blockDim.x)
        {
            const bool valid = j < count;
            uint32_t key = 0;
            const uint32_t slot = n_next + j;
            if (valid)
            {
            const unsigned long long w = base_work + j;
            uint32_t pixel, sample, film_index;
            V3<R> start, direction;
            if (p.user_rays)
            {
                pixel = p.user_pixel[w];
                sample = p.user_sample[w];
                film_index = (uint32_t)w;
                const double* r = p.user_rays + 6 * w;
                start = V3<R>((R)r[0], (R)r[1], (R)r[2]);
                direction = V3<R>((R)r[3], (R)r[4], (R)r[5]);
            }
            else
            {
                // sample-major over this rank's pixels: adjacent lanes = adjacent pixels
                uint32_t local = (uint32_t)(w % p.n_pixels);
                if constexpr (LIST) local = p.pixel_list[local];
                // a progressive pass starts at work item sample_first * n_pixels (runWavefront)
                sample = (uint32_t)(w / p.n_pixels);
                const uint32_t row = local / p.camera.width, col = local - row * p.camera.width;
                pixel = (p.row_first + row * p.row_step) * p.camera.width + col;
                film_index = local;
                SamplerState smp = SamplerState::make(p.global_seed, pixel, sample, 0u);
                cameraRay(p.camera, p.scene.scene_ior, pixel, smp, start, direction);
                if constexpr (FILM) filmSplatSampleWeight(p.filmp, p.global_seed, pixel, sample);
            }
            stStream(&out.ray_o[slot], V4<R>(start, p.scene.scene_ior));
            stStream(&out.ray_d[slot], V4<R>(direction, R(1)));
            stStream(&out.thr[slot], V4<R>(R(1), R(1), R(1), R(0)));
            stStream(&out.meta[slot], make_uint4(pixel, sample, 0u, 0u));
            stStream(&out.meta2[slot], make_uint4(NO_PRIM, 1u, film_index, NO_PRIM));
            if (p.sort.path_order) key = rayKey(p.sort, start, direction, NO_PRIM);
            }
            if (p.sort.path_order)
            {
                const uint32_t rank = sortRank(p.sort.hist_path, key, valid);
                if (valid) { p.sort.path_key[next][slot] = key; p.sort.path_rank[next][slot] = rank; }
            }
        }
    }

    static __global__ void k_advance(Counters* c)
    {
        c->n_cur = c->n_next + c->n_gen;
        c->next_work += c->n_gen;
        c->paths += c->n_gen;
        c->n_next = 0;
        c->n_gen = 0;
        c->n_shadow = 0;
        c->n_knn = 0;
        c->fetch_extend = 0;
        c->fetch_shadow = 0;
    }

    // FAST: 0 reference-order replay for every ray, 1 order-free search one ray per lane, 2 order-free search with
    // dynamic fetch (traceManyFast; big scenes, where ray lengths within a warp differ most)
    template <class R, int PRIMS, int FAST>
    __global__ void __launch_bounds__(256, FAST == 2 ? MCRT_TRACE_MINBLOCKS_DYN : (FAST == 1 ? MCRT_TRACE_MINBLOCKS_FAST : (PRIMS == PRIMS_ALL ? Mode<R>::trace_minblocks : Mode<R>::trace_minblocks_pruned))) k_extend(WaveParams<R> p, int cur)
    {
        const uint32_t n = p.counters->n_cur;
        const PathBuffer<R>& in = p.buf[cur];
        TraceCounters cnt = { 0u, 0u, 0u };
        uint32_t overflow = 0;
        unsigned long long rays = 0;
        const uint32_t* order = p.sort.path_order;
        if constexpr (Mode<R>::parity && FAST == 2)
        {
            traceManyFast<PRIMS>(p.scene, n, &p.counters->fetch_extend,
                [&](uint32_t ii, RayQ<R>& r)
                {
                    const uint32_t i = order ? order[ii] : ii;
                    const V4<R> ro = ldStream(&in.ray_o[i]), rd = ldStream(&in.ray_d[i]);
                    r.o = ro.xyz(); r.d = rd.xyz();
                    if constexpr (PRIMS == PRIMS_ALL) r.inv_d = R(1) / r.d;   // quadric clip-box test
                    return i;
                },
                [&](uint32_t i, const RayQ<R>&, const Hit<R>& h)
                {
                    stStream(&p.hits[i], V4<R>(h.t, h.u, h.v, h.prim == NO_PRIM ? R(-1) : R(h.prim)));
                    rays++;
                }, cnt, overflow);
            flushStats(p.counters, cnt, rays, false, overflow);
            return;
        }
        for (uint32_t ii = blockIdx.x * blockDim.x + threadIdx.x; ii < n; ii += gridDim.x * blockDim.x)
        {
            const uint32_t i = order ? order[ii] : ii;
            const V4<R> ro = ldStream(&in.ray_o[i]);
            const V4<R> rd = ldStream(&in.ray_d[i]);
            uint32_t skip = NO_PRIM;
            if constexpr (!Mode<R>::parity) skip = in.meta2[i].w;
#ifdef MCRT_TAIL_DIAGNOSTIC
            const uint32_t w0 = cnt.box_tests + cnt.prim_tests;
#endif
            Hit<R> h = traceClosest<PRIMS, FAST != 0>(p.scene, ro.xyz(), rd.xyz(), skip, cnt, overflow);
            stStream(&p.hits[i], V4<R>(h.t, h.u, h.v, h.prim == NO_PRIM ? R(-1) : R(h.prim)));
            rays++;
#ifdef MCRT_TAIL_DIAGNOSTIC
            // tuning builds only: how much of the warp's time (~ its slowest ray) the average ray uses
            const uint32_t w = cnt.box_tests + cnt.prim_tests - w0;
            const unsigned am = __activemask();
            const uint32_t wmax = __reduce_max_sync(am, w);
            atomicAdd(&p.counters->work_sum, (unsigned long long)w);
            if ((threadIdx.x & 31u) == (unsigned)(__ffs(am) - 1)) atomicAdd(&p.counters->work_warpmax, 32ull * wmax);
#endif
        }
        flushStats(p.counters, cnt, rays, false, overflow);
    }

    // Light sample: Surface::operator()(u,v) and Surface::normal (triangle.cpp:93-102,
    // sphere.cpp:37-49)
    template <class R>
    MCRT_D void sampleLightPoint(const Light<R>& l, R u, R v, V3<R>& pos, V3<R>& normal)
    {
        if (l.type == PRIM_TRIANGLE)
        {
            R su = msqrt(u);
            pos = (R(1) - su) * l.p0 + (R(1) - v) * su * l.p1 + v * su * l.p2;
            normal = l.normal;
        }
        else
        {
            R z = R(1) - R(2) * u;
            R r = msqrt(R(1) - pow2(z));
            R phi = Consts<R>::TWO_PI * v;
            R sn, cs;
            msincos(phi, &sn, &cs);
            pos = l.p0 + l.p1.x * V3<R>(r * cs, r * sn, z);
            normal = (pos - l.p0) / l.p1.x;
        }
    }

    template <class R> MCRT_D R powerHeuristic(R a_pdf, R b_pdf)
    {
        R a2 = a_pdf * a_pdf;
        return a2 / (a2 + b_pdf * b_pdf);
    }

    // Scene::skyColor, scene.cpp:219-223
    template <class R> MCRT_D V3<R> skyColor(const V3<R>& dir)
    {
        R d = R(0) * dir.x + R(1) * dir.y + R(0) * dir.z;
        // float32: a direction's y can round past +-1 (a refracted or reflected ray that is vertical to round-off), where
        // asin is NaN and the NaN would poison the pixel; its limit is the pole's colour
        if constexpr (sizeof(R) == 4) d = gclamp(d, R(-1), R(1));
        R fy = (R(1) + masin(d) / Consts<R>::PI) / R(2);
        return mix(V3<R>(R(1), R(0.5), R(0)), V3<R>(R(0), R(0.5), R(1)), fy);
    }

    // FEATS: material features present in the scene (mask over Material::flags): SHADE_FEATS_LITE drops
    // Oren-Nayar, GGX (evaluation, VNDF sampling) and the conductor Fresnel from the instantiation
    constexpr uint32_t SHADE_FEATS_ALL = 0xFFFFFFFFu;
    constexpr uint32_t SHADE_FEATS_LITE = ~(uint32_t)(MAT_ROUGH | MAT_ROUGH_SPECULAR | MAT_COMPLEX_IOR);

    template <class R, int KIND, int FILM, uint32_t FEATS>
    __global__ void __launch_bounds__(128, FEATS == 0xFFFFFFFFu ? MCRT_SHADE_MINBLOCKS : MCRT_SHADE_MINBLOCKS_LITE) k_shade(WaveParams<R> p, int cur)
    {
        __shared__ SobolByteTables sobol_tab;
        sobol_tab.fill(p.sobol_bytes);
        __syncthreads();
        Counters* c = p.counters;
        const uint32_t n = c->n_cur;
        const PathBuffer<R>& in = p.buf[cur];
        const PathBuffer<R>& out = p.buf[cur ^ 1];
        const DeviceScene<R>& sc = p.scene;
        uint32_t local_max_depth = 0;
        uint32_t stack_overflows = 0;

        const uint32_t n_rounded = (n + 31u) & ~31u; // keep warps converged for the ballots
        const uint32_t* order = p.sort.shade_order ? p.sort.shade_order : (p.sort.shade_sorted ? p.sort.path_order : nullptr);
        const bool sorting = p.sort.path_order != nullptr;
        for (uint32_t ii = blockIdx.x * blockDim.x + threadIdx.x; ii < n_rounded; ii += gridDim.x * blockDim.x)
        {
            bool alive = ii < n;
            const uint32_t i = (alive && order) ? order[ii] : ii;
            bool want_shadow = false;
            uint32_t want_knn = 0;   // 0 none, 1 caustic, 2 caustic + global
            KnnQuery<R> knn_q;

            PathRay<R> ray, nray;
            V3<R> throughput;
            uint4 meta, meta2;
            R ls_bsdf_pdf = R(0), ls_select = R(0);
            uint32_t ls_light = NO_PRIM, ior_count = 1, hit_prim = NO_PRIM;
            R iors[IOR_STACK_CAPACITY];
            // shadow candidate
            V3<R> sh_o, sh_d, sh_k;
            R sh_bsdf_pdf = R(0), sh_area_cos = R(0), sh_select = R(0);
            uint32_t sh_light = NO_PRIM;
            // FILM_MODE_AOV: interaction type + 1 of the path's first vertex (0 before it; path tracer only), the shadow
            // ray's plane
            uint32_t lobe = 0, sh_plane = 0;
            // FILM_MODE_LPE: the DFA state after the events so far (bits 16-23 of meta2.y; 0 after C); sh_plane then holds
            // the shadow ray's accept mask
            uint32_t lpe_state = 0;

            if (alive)
            {
                const V4<R> ro = ldStream(&in.ray_o[i]), rd = ldStream(&in.ray_d[i]), th = ldStream(&in.thr[i]), hv = ldStream(&p.hits[i]);
                meta = ldStream(&in.meta[i]); meta2 = ldStream(&in.meta2[i]);
                ray.start = ro.xyz(); ray.medium_ior = ro.w;
                ray.direction = rd.xyz(); ray.refraction_scale = rd.w;
                throughput = th.xyz(); ls_bsdf_pdf = th.w;
                ray.depth = meta.z & 0xFFFFu; ray.diffuse_depth = meta.z >> 16;
                ray.refraction_level = (int32_t)meta.w;
                ls_light = meta2.x;
                ior_count = meta2.y & 0xFFu;
                ray.dirac_delta = (meta2.y >> 8) & 1u;
                if constexpr (KIND == 0 && FILM == FILM_MODE_AOV) lobe = (meta2.y >> 9) & 3u;
                if constexpr (FILM == FILM_MODE_LPE) lpe_state = (meta2.y >> 16) & 0xFFu;
                ray.refraction = false;
                const uint32_t film_index = meta2.z;

                iors[0] = sc.scene_ior;
                if (ior_count > 1)
                {
                    const V4<R> ia_ = in.iors_a[i];
                    iors[1] = ia_.x; iors[2] = ia_.y; iors[3] = ia_.z; iors[4] = ia_.w;
                    if (ior_count > 5)
                    {
                        const V4<R> ib_ = in.iors_b[i];
                        iors[5] = ib_.x; iors[6] = ib_.y; iors[7] = ib_.z;
                    }
                }
                // LightSample::select_probability of the light picked at the previous bounce,
                // recomputed from the CDF exactly as Scene::selectLight does (scene.cpp:229-233)
                if (ls_light != NO_PRIM)
                {
                    ls_select = sc.lights[ls_light].cdf;
                    if (ls_light > 0) ls_select -= sc.lights[ls_light - 1].cdf;
                }

                if (ray.depth > local_max_depth) local_max_depth = ray.depth;

                Hit<R> hit;
                hit.t = hv.x; hit.u = hv.y; hit.v = hv.z;
                hit.prim = hv.w < R(0) ? NO_PRIM : (uint32_t)hv.w;
                hit_prim = hit.prim;

                if (hit.prim == NO_PRIM)
                {
                    // path-tracer.cpp:27-30; the photon mapper adds no sky (photon-mapper.cpp:292-295)
                    if constexpr (KIND == 0 && FILM == FILM_MODE_LPE)
                        depositRadiance<FILM>(p, film_index, meta.x, meta.y, skyColor(ray.direction) * throughput, NO_PRIM,
                                              lpeAccept(p, lpeNext(p, lpe_state, MCRT_LPE_SYM_B)));
                    else if constexpr (KIND == 0)
                        depositRadiance<FILM>(p, film_index, meta.x, meta.y, skyColor(ray.direction) * throughput, NO_PRIM,
                                              FILM == FILM_MODE_AOV ? aovPlane(lobe, ray.depth > 1u, true) : 0u);
                    alive = false;
                }
                else
                {
                    // Sampler::shuffle() was called depth+1 times (path-tracer.cpp:23)
                    SamplerState smp = SamplerState::make(p.global_seed, meta.x, meta.y, ray.depth + 1u);
                    smp.tab = &sobol_tab;

                    // RefractionHistory::externalIOR, ray.cpp:95-98
                    int ext_idx = ray.refraction_level - 1;
                    ext_idx = ext_idx < 0 ? 0 : (ext_idx > (int)ior_count - 1 ? (int)ior_count - 1 : ext_idx);
                    const R external_ior = iors[ext_idx];

                    Interaction<R> ia;
                    buildInteraction<FEATS>(ia, sc, hit, ray, external_ior, smp);
                    const Material<R>& m = *ia.material;
                    const PrimShade<R> ps = sc.shade[hit.prim];

                    // ---- Integrator::sampleEmissive, integrator.cpp:93-110
                    if ((m.flags & MAT_EMISSIVE) && !ia.inside)
                    {
                        if (ray.depth == 0 || ray.dirac_delta)
                        {
                            if constexpr (FILM == FILM_MODE_LPE)
                                depositRadiance<FILM>(p, film_index, meta.x, meta.y, m.emittance * throughput, ps.light,
                                                      lpeAccept(p, lpeNext(p, lpe_state, lpeLightSymbol(p, ps.light))));
                            else
                                depositRadiance<FILM>(p, film_index, meta.x, meta.y, m.emittance * throughput, ps.light,
                                                      FILM != FILM_MODE_AOV ? 0u : (KIND == 0 ? aovPlane(lobe, ray.depth > 1u, false)
                                                                                              : (uint32_t)MCRT_PM_EMISSION));
                        }
                        else if (ls_light != NO_PRIM && sc.lights[ls_light].prim == hit.prim)
                        {
                            R cos_light_theta = dot(ia.out, ia.normal);
                            R light_pdf = pow2(ia.t) / (ps.area * cos_light_theta);
                            R mis_weight = powerHeuristic(ls_bsdf_pdf, light_pdf);
                            if constexpr (FILM == FILM_MODE_LPE)
                                depositRadiance<FILM>(p, film_index, meta.x, meta.y, (mis_weight * m.emittance / ls_select) * throughput, ls_light,
                                                      lpeAccept(p, lpeNext(p, lpe_state, lpeLightSymbol(p, ls_light))));
                            else
                                depositRadiance<FILM>(p, film_index, meta.x, meta.y, (mis_weight * m.emittance / ls_select) * throughput, ls_light,
                                                      FILM != FILM_MODE_AOV ? 0u : (KIND == 0 ? aovPlane(lobe, ray.depth > 1u, false)
                                                                                              : (uint32_t)MCRT_PM_DIRECT));
                        }
                    }

                    // the camera ray's hit is the first vertex: its lobe is the path's, for NEE here and everything after
                    if constexpr (KIND == 0 && FILM == FILM_MODE_AOV) if (ray.depth == 0) lobe = ia.type + 1u;

                    // ---- PhotonMapper::sampleRay control flow, photon-mapper.cpp:299-332
                    bool do_direct = true, do_bsdf = true;
                    if constexpr (FILM == FILM_MODE_LPE)
                    {
                        // this vertex's event, for NEE here and everything after; once no expression can match, nothing
                        // the path could still add lands in a plane, and the sampler is a pure function of (pixel,
                        // sample, depth), so ending it here changes no plane
                        lpe_state = lpeNext(p, lpe_state, lpeVertexSymbol(ia.type, ia.dirac_delta));
                        if (lpe_state == MCRT_LPE_DEAD) { do_direct = false; do_bsdf = false; alive = false; }
                    }
                    if constexpr (KIND == 1)
                    {
                        if (ia.dirac_delta)
                        {
                            do_direct = false;
                            if (!ray.dirac_delta && ray.depth != 0) { do_bsdf = false; alive = false; }
                        }
                        else
                        {
                            want_knn = 1; // caustic estimate at every non-delta hit
                            if (!p.pm.direct_visualization && (ray.dirac_delta || ray.depth == 0))
                            {
                                // delay the global evaluation: direct light + one more bounce
                            }
                            else
                            {
                                want_knn = 2; // + global estimate, then the path ends
                                do_direct = false; do_bsdf = false; alive = false;
                            }
                        }
                        // a dead path, or one whose every photon term no expression accepts, queries no map (its
                        // estimates would land in no plane), as a zero mask traces no shadow ray
                        if constexpr (FILM == FILM_MODE_LPE)
                            if (lpe_state == MCRT_LPE_DEAD || !__ldg(&p.pm.lpe_join_any[lpe_state])) want_knn = 0;
                        if (want_knn)
                        {
                            knn_q.pos_n1 = V4<R>(ia.position, ia.n1);
                            knn_q.nrm_n2 = V4<R>(ia.shading_cs.c2, ia.n2);
                            knn_q.out_rf = V4<R>(ia.out, ia.Rf);
                            knn_q.weight_t = V4<R>(throughput, ia.T);
                            // FILM_MODE_LPE: the forward state after x's event in bits 16-23 (k_knn / k_gather join it
                            // with each photon's)
                            knn_q.meta = make_uint4(ps.material, film_index, (ia.inside ? 1u : 0u) |
                                                                             (FILM == FILM_MODE_LPE ? lpe_state << 16 : 0u), meta.y);
                        }
                    }

                    // ---- Integrator::sampleDirect up to the visibility query, integrator.cpp:31-66
                    if (!do_direct)
                    {
                    }
                    else if (sc.n_lights == 0 || (m.flags & MAT_DIRAC_DELTA))
                    {
                        ls_light = NO_PRIM;
                    }
                    else
                    {
                        R u[3];
                        samplerGet<R, DIM_LIGHT, 3>(smp, u);
                        // Sampling::weightedIdx, sampling.hpp:13-28
                        uint32_t left = 0, right = sc.n_lights - 1;
                        while (left < right)
                        {
                            uint32_t middle = (left + right) / 2;
                            if (sc.lights[middle].cdf < u[2]) left = middle + 1; else right = middle;
                        }
                        const Light<R>& L = sc.lights[left];
                        ls_select = L.cdf;
                        if (left > 0) ls_select -= sc.lights[left - 1].cdf;
                        ls_light = left;

                        V3<R> light_pos, light_normal;
                        sampleLightPoint(L, u[0], u[1], light_pos, light_normal);
                        V3<R> s_start = ia.position + ia.normal * p.ray_eps;
                        V3<R> s_dir = normalize(light_pos - s_start);
                        R cos_light_theta = dot(-s_dir, light_normal);
                        if (cos_light_theta > R(0))
                        {
                            bool ok = true;
                            R cos_theta = dot(s_dir, ia.normal);
                            if (cos_theta <= R(0))
                            {
                                if ((m.flags & MAT_OPAQUE) || cos_theta == R(0)) ok = false;
                                else
                                {
                                    s_start = ia.position - ia.normal * p.ray_eps;
                                    s_dir = normalize(light_pos - s_start);
                                }
                            }
                            if (ok)
                            {
                                V3<R> bsdf_absIdotN; R bsdf_pdf;
                                if (ia.bsdfWorld(bsdf_absIdotN, s_dir, bsdf_pdf))
                                {
                                    want_shadow = true;
                                    sh_o = s_start; sh_d = s_dir;
                                    sh_k = bsdf_absIdotN * L.emittance * throughput;
                                    sh_bsdf_pdf = bsdf_pdf;
                                    sh_area_cos = L.area * cos_light_theta;
                                    sh_select = ls_select;
                                    sh_light = L.prim;
                                    if constexpr (FILM == FILM_MODE_AOV) sh_plane = KIND == 0 ? aovPlane(lobe, ray.depth > 0u, false) : (uint32_t)MCRT_PM_DIRECT;
                                    if constexpr (FILM == FILM_MODE_LPE)
                                    {
                                        // a mask no expression sets traces no shadow ray, like a zero BSDF value
                                        sh_plane = lpeAccept(p, lpeNext(p, lpe_state, lpeLightSymbol(p, ls_light)));
                                        want_shadow = sh_plane != 0u;
                                    }
                                }
                            }
                        }
                    }

                    // ---- Interaction::sampleBSDF, throughput, absorb: path-tracer.cpp:37-47
                    V3<R> bsdf_absIdotN;
                    if (!do_bsdf)
                    {
                    }
                    else if (!sampleBSDF(ia, ray, smp, p.ray_eps, false, bsdf_absIdotN, ls_bsdf_pdf, nray))
                    {
                        alive = false;
                    }
                    else
                    {
                        throughput *= bsdf_absIdotN / ls_bsdf_pdf;
                        // Integrator::absorb, integrator.cpp:112-129
                        R survive = compMax(throughput) * nray.refraction_scale;
                        if (survive == R(0))
                        {
                            alive = false;
                        }
                        else if (nray.diffuse_depth > 3u || nray.depth > 16u)
                        {
                            survive = gmin(R(0.95), survive);
                            R ua;
                            samplerGet<R, DIM_ABSORB, 1>(smp, &ua);
                            if (survive <= ua) alive = false;
                            else throughput /= survive;
                        }
                    }

                    if (alive)
                    {
                        // RefractionHistory::update, ray.cpp:80-93
                        if (nray.refraction_level > 0)
                        {
                            if (nray.refraction_level == (int32_t)ior_count)
                            {
                                if (ior_count < (uint32_t)IOR_STACK_CAPACITY) iors[ior_count++] = nray.medium_ior;
                                else stack_overflows++;
                            }
                            else if (nray.refraction_level < (int32_t)ior_count - 1)
                            {
                                ior_count--;
                            }
                        }
                    }
                }
            }

            // ---- compaction: survivors → next path buffer, NEE candidates → shadow queue.
            // All four atomics (two queue appends, two sort ranks) are issued back to back so their
            // round trips overlap; the stores follow.
            const uint32_t slot = warpAppend(&c->n_next, alive);
            const uint32_t sslot = warpAppend(&c->n_shadow, want_shadow);
            uint32_t pkey = 0, prank = 0, skey = 0, srank = 0;
            if (sorting && alive)
            {
                // un-aggregated: lanes of an (unsorted) shade warp rarely share a bin
                pkey = rayKey(p.sort, nray.start, nray.direction, hit_prim);
                prank = atomicAdd(&p.sort.hist_path[pkey], 1u);
            }
            if (sorting && want_shadow)
            {
                skey = rayKey(p.sort, sh_o, sh_d, hit_prim);
                srank = atomicAdd(&p.sort.hist_shadow[skey], 1u);
            }
            if (alive)
            {
                stStream(&out.ray_o[slot], V4<R>(nray.start, nray.medium_ior));
                stStream(&out.ray_d[slot], V4<R>(nray.direction, nray.refraction_scale));
                stStream(&out.thr[slot], V4<R>(throughput, ls_bsdf_pdf));
                if (ior_count > 1)
                {
                    out.iors_a[slot] = V4<R>(iors[1], iors[2], iors[3], iors[4]);
                    if (ior_count > 5) out.iors_b[slot] = V4<R>(iors[5], iors[6], iors[7], R(0));
                }
                stStream(&out.meta[slot], make_uint4(meta.x, meta.y, (nray.depth & 0xFFFFu) | (nray.diffuse_depth << 16),
                                                     (uint32_t)nray.refraction_level));
                stStream(&out.meta2[slot], make_uint4(ls_light, ior_count | (nray.dirac_delta ? 256u : 0u) | (lobe << 9) |
                                                                    (FILM == FILM_MODE_LPE ? lpe_state << 16 : 0u), meta2.z,
                                                      sc.shade[hit_prim].type == PRIM_TRIANGLE ? hit_prim : NO_PRIM));
                if (sorting) { p.sort.path_key[cur ^ 1][slot] = pkey; p.sort.path_rank[cur ^ 1][slot] = prank; }
            }
            if (want_shadow)
            {
                ShadowRecord<R>& srec = p.shadow[sslot];
                stStream(&srec.o, V4<R>(sh_o, sh_bsdf_pdf));
                stStream(&srec.d, V4<R>(sh_d, sh_area_cos));
                stStream(&srec.meta, make_uint4(sh_light, meta2.z, sc.shade[hit_prim].type == PRIM_TRIANGLE ? hit_prim : NO_PRIM,
                                                FILM == FILM_MODE_AOV || FILM == FILM_MODE_LPE ? sh_plane : meta.y));
                // float64: also write the padding after meta, so that no 32-byte sector of the record is left half
                // written (without this store the C2 shade stage measured 930 instead of 744 ms per frame)
                if constexpr (sizeof(R) == 8) stStream(reinterpret_cast<uint4*>(&srec) + 5, make_uint4(0u, 0u, 0u, 0u));
                stStream(&srec.k, V4<R>(sh_k, sh_select));
                if (sorting) { p.sort.shadow_key[sslot] = skey; p.sort.shadow_rank[sslot] = srank; }
            }

            if constexpr (KIND == 1)
            {
                // k-NN queries: caustic map always, global map when the path ends here
                const uint32_t q0 = warpAppend(&c->n_knn, want_knn >= 1);
                if (want_knn >= 1 && q0 < p.pm.query_capacity) p.pm.queries[q0] = knn_q;
                const uint32_t q1 = warpAppend(&c->n_knn, want_knn == 2);
                if (want_knn == 2 && q1 < p.pm.query_capacity)
                {
                    knn_q.meta.z |= 2u;
                    p.pm.queries[q1] = knn_q;
                }
            }
        }

        if (local_max_depth) atomicMax(&c->max_depth, local_max_depth);
        if (stack_overflows) atomicAdd(&c->ior_stack_overflows, (unsigned long long)stack_overflows);
    }

    // FILM_MODE_GROUPS finds the sampled light's group through the light primitive's shading record (sm.x is L.prim);
    // FILM_MODE_AOV reads the AOV plane k_shade stored in place of the sample index (sm.w), FILM_MODE_LPE the accept mask
    template <class R, int FILM, int PRIMS, int FAST>
    __global__ void __launch_bounds__(256, FAST == 2 ? MCRT_TRACE_MINBLOCKS_DYN : (FAST == 1 ? MCRT_TRACE_MINBLOCKS_FAST : (PRIMS == PRIMS_ALL ? Mode<R>::trace_minblocks : Mode<R>::trace_minblocks_pruned))) k_shadow(WaveParams<R> p)
    {
        const uint32_t n = p.counters->n_shadow;
        TraceCounters cnt = { 0u, 0u, 0u };
        uint32_t overflow = 0;
        unsigned long long rays = 0;
        const uint32_t* order = p.sort.shadow_order;
        if constexpr (Mode<R>::parity && FAST == 2)
        {
            traceManyFast<PRIMS, true>(p.scene, n, &p.counters->fetch_shadow,
                [&](uint32_t ii, RayQ<R>& r, uint32_t& target)
                {
                    const uint32_t i = order ? order[ii] : ii;
                    const V4<R> so = ldStream(&p.shadow[i].o), sd = ldStream(&p.shadow[i].d);
                    r.o = so.xyz(); r.d = sd.xyz();
                    if constexpr (PRIMS == PRIMS_ALL) r.inv_d = R(1) / r.d;
                    target = p.shadow[i].meta.x;
                    return i;
                },
                [&](uint32_t i, const RayQ<R>&, const Hit<R>& h)
                {
                    rays++;
                    const ShadowRecord<R>& srec = p.shadow[i];
                    const uint4 sm = srec.meta;
                    if (h.prim == sm.x)   // integrator.cpp:70-86: visible iff the closest hit is that very light primitive
                    {
                        const V4<R> so = srec.o, sd = srec.d, sk = srec.k;
                        R light_pdf = pow2(h.t) / sd.w;
                        R mis_weight = powerHeuristic(light_pdf, so.w);
                        depositRadiance<FILM>(p, sm.y, pixelOfFilmIndex(p, sm.y), sm.w, sk.xyz() * (mis_weight / (light_pdf * sk.w)),
                                              FILM == FILM_MODE_GROUPS ? p.scene.shade[sm.x].light : NO_PRIM, sm.w);
                    }
                }, cnt, overflow);
            flushStats(p.counters, cnt, rays, true, overflow);
            return;
        }
        for (uint32_t ii = blockIdx.x * blockDim.x + threadIdx.x; ii < n; ii += gridDim.x * blockDim.x)
        {
            const uint32_t i = order ? order[ii] : ii;
            const ShadowRecord<R>& srec = p.shadow[i];
            const V4<R> so = ldStream(&srec.o), sd = ldStream(&srec.d);
            const uint4 sm = ldStream(&srec.meta);
            Hit<R> h;
            if constexpr (Mode<R>::parity && FAST != 0) h = traceVisible<PRIMS>(p.scene, so.xyz(), sd.xyz(), sm.x, cnt, overflow);
            else h = traceClosest<PRIMS, false>(p.scene, so.xyz(), sd.xyz(), sm.z, cnt, overflow);
            rays++;
            // integrator.cpp:70-86: visible iff the closest hit is that very light primitive
            if (h.prim == sm.x)
            {
                const V4<R> sk = srec.k;
                R light_pdf = pow2(h.t) / sd.w;
                R mis_weight = powerHeuristic(light_pdf, so.w);
                depositRadiance<FILM>(p, sm.y, pixelOfFilmIndex(p, sm.y), sm.w, sk.xyz() * (mis_weight / (light_pdf * sk.w)),
                                      FILM == FILM_MODE_GROUPS ? p.scene.shade[sm.x].light : NO_PRIM, sm.w);
            }
        }
        flushStats(p.counters, cnt, rays, true, overflow);
    }



    // ------------------------------------------------------------------------------------------
    // Shade-coherence key: class of the primitive each live path hit (misses: class 0), ranks from a
    // per-CTA shared-memory histogram + one global atomic per class per CTA chunk.
    constexpr uint32_t SHADE_CLASS_BINS = 64;

    template <class R>
    __global__ void __launch_bounds__(256) k_shade_key(WaveParams<R> p)
    {
        __shared__ uint32_t s_hist[SHADE_CLASS_BINS], s_base[SHADE_CLASS_BINS];
        const uint32_t n = p.counters->n_cur;
        const uint32_t chunks = (n + 255u) / 256u;
        for (uint32_t chunk = blockIdx.x; chunk < chunks; chunk += gridDim.x)
        {
            if (threadIdx.x < SHADE_CLASS_BINS) s_hist[threadIdx.x] = 0u;
            __syncthreads();
            const uint32_t i = chunk * 256u + threadIdx.x;
            uint32_t key = 0, local = 0;
            if (i < n)
            {
                const R w = p.hits[i].w;
                if (!(w < R(0))) key = p.scene.shade_class[(uint32_t)w];
                local = atomicAdd(&s_hist[key], 1u);
            }
            __syncthreads();
            if (threadIdx.x < SHADE_CLASS_BINS && s_hist[threadIdx.x]) s_base[threadIdx.x] = atomicAdd(&p.sort.hist_shade[threadIdx.x], s_hist[threadIdx.x]);
            __syncthreads();
            if (i < n) { p.sort.shade_key[i] = key; p.sort.shade_rank[i] = s_base[key] + local; }
            __syncthreads();
        }
    }

    // ------------------------------------------------------------------------------------------
    // Counting-sort helpers. k_sort_scan: exclusive prefix sum of the SORT_BINS-entry histogram into
    // bin_start, zeroing the histogram for the next bounce (one 1024-thread CTA: 128 bins per thread,
    // 512 KB read once). k_sort_scatter: order[bin_start[key] + rank] = entry.
    constexpr uint32_t SORT_SCAN_BLOCKS = SORT_BINS / 1024;   // 1024 bins per CTA

    static __global__ void __launch_bounds__(256) k_sort_scan(uint32_t* hist, uint32_t* bin_start, uint32_t* block_offset,
                                                              uint32_t* done_counter)
    {
        __shared__ uint32_t warp_sums[8];
        __shared__ uint32_t is_last;
        const uint32_t t = threadIdx.x, base = blockIdx.x * 1024u + t * 4u;
        const uint4 v = *reinterpret_cast<const uint4*>(hist + base);
        *reinterpret_cast<uint4*>(hist + base) = make_uint4(0u, 0u, 0u, 0u);
        const uint32_t sum = v.x + v.y + v.z + v.w;
        uint32_t incl = sum;
        for (int off = 1; off < 32; off <<= 1)
        {
            const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, off);
            if ((t & 31u) >= (uint32_t)off) incl += u;
        }
        if ((t & 31u) == 31u) warp_sums[t >> 5] = incl;
        __syncthreads();
        uint32_t warp_base = 0;
        for (uint32_t w = 0; w < (t >> 5); w++) warp_base += warp_sums[w];
        const uint32_t excl = warp_base + incl - sum;
        *reinterpret_cast<uint4*>(bin_start + base) = make_uint4(excl, excl + v.x, excl + v.x + v.y, excl + v.x + v.y + v.z);
        if (t == 255u)
        {
            block_offset[SORT_SCAN_BLOCKS + blockIdx.x] = excl + sum;   // this CTA's total
            __threadfence();
            is_last = atomicAdd(done_counter, 1u) == gridDim.x - 1u;
        }
        __syncthreads();
        if (is_last && t < 32u)
        {
            // exclusive scan of the CTA totals by one warp (SORT_SCAN_BLOCKS / 32 consecutive per lane)
            __threadfence();
            constexpr uint32_t PER_LANE = SORT_SCAN_BLOCKS / 32;
            uint32_t lane_sum = 0;
            for (uint32_t k = 0; k < PER_LANE; k++) lane_sum += block_offset[SORT_SCAN_BLOCKS + t * PER_LANE + k];
            uint32_t inc = lane_sum;
            for (int off = 1; off < 32; off <<= 1)
            {
                const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, inc, off);
                if (t >= (uint32_t)off) inc += u;
            }
            uint32_t run = inc - lane_sum;
            for (uint32_t k = 0; k < PER_LANE; k++)
            {
                const uint32_t tot = block_offset[SORT_SCAN_BLOCKS + t * PER_LANE + k];
                block_offset[t * PER_LANE + k] = run;
                run += tot;
            }
            if (t == 0) *done_counter = 0u;
        }
    }

    static __global__ void __launch_bounds__(256) k_sort_scatter(const uint32_t* key, const uint32_t* rank, const uint32_t* bin_start,
                                                                 const uint32_t* block_offset, uint32_t* order, const uint32_t* n_ptr)
    {
        const uint32_t n = *n_ptr;
        for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        {
            const uint32_t k = key[i];
            order[block_offset[k >> 10] + bin_start[k] + rank[i]] = i;
        }
    }

    // ------------------------------------------------------------------------------------------
    // The Interaction fields Interaction::BSDF reads, rebuilt from a photon-map query (k_knn, k_gather)
    template <uint32_t FEATS, class R>
    MCRT_D void queryInteraction(const WaveParams<R>& p, const KnnQuery<R>& qr, Interaction<R>& ia)
    {
        ia.type = IA_DIFFUSE;
        ia.n1 = qr.pos_n1.w; ia.n2 = qr.nrm_n2.w; ia.Rf = qr.out_rf.w; ia.T = qr.weight_t.w;
        ia.material = &p.scene.materials[qr.meta.x];
        ia.fmask = FEATS;   // the BSDF evaluations of the estimate (photon-mapper.cpp:343-391)
        ia.out = qr.out_rf.xyz();
        ia.shading_cs = Frame<R>(qr.nrm_n2.xyz());
        ia.inside = qr.meta.z & 1u;
    }

    // One photon's term of the radiance estimate (photon-mapper.cpp:343-391): flux f / pdf, in the caustic map (which 0)
    // weighted by the cone filter 1 - d/r (:383-386). false: the BSDF has no value in the photon's direction.
    template <class R>
    MCRT_D bool photonTerm(Interaction<R>& ia, uint32_t which, const float4& a, const float4& b, R d2, R inv_r2, V3<R>& term)
    {
        V3<R> bsdf_absIdotN; R bsdf_pdf;
        if (!ia.bsdfWorld(bsdf_absIdotN, photonDir<R>(b.z, b.w), bsdf_pdf)) return false;
        const V3<R> flux((R)a.x, (R)a.y, (R)a.z);
        if (which == 0)
        {
            const R wp = gmax(R(0), R(1) - msqrt(d2 * inv_r2));
            term = (flux * bsdf_absIdotN * wp) / bsdf_pdf;
        }
        else
        {
            term = flux * bsdf_absIdotN / bsdf_pdf;
        }
        return true;
    }

    // Light-group split of a photon estimate (FILM_MODE_GROUPS of k_knn / k_gather). Each lane keeps one run: the sum of
    // its photons' terms since its photons' light group last changed (plane: that group; NO_PRIM: no run). Every term of
    // a query shares the estimate's scale and the path weight, so the planes' deposits add up to the one-plane deposit up
    // to rounding, and no term is negative. depositGroupRuns adds up the runs of each plane present over the warp, and
    // the plane's lowest lane deposits scale(sum) * weight; with one group that is one deposit, as the one-plane kernel.
    template <class R, class Scale>
    MCRT_D void depositGroupRuns(const WaveParams<R>& p, uint32_t film_index, uint32_t plane, const V3<R>& sum, const V3<R>& weight,
                                 Scale&& scale)
    {
        const unsigned lane = threadIdx.x & 31u;
        unsigned pending = __ballot_sync(0xFFFFFFFFu, plane != NO_PRIM);
        while (pending)
        {
            const int leader = __ffs(pending) - 1;
            const uint32_t g = __shfl_sync(0xFFFFFFFFu, plane, leader);
            const bool mine = plane == g;
            V3<R> v = mine ? sum : V3<R>(R(0));
            for (int off = 16; off > 0; off >>= 1)
            {
                v.x += __shfl_xor_sync(0xFFFFFFFFu, v.x, off);
                v.y += __shfl_xor_sync(0xFFFFFFFFu, v.y, off);
                v.z += __shfl_xor_sync(0xFFFFFFFFu, v.z, off);
            }
            if ((int)lane == leader) filmAddV(p.film + g * p.plane_values, film_index, scale(v) * weight);
            pending &= ~__ballot_sync(0xFFFFFFFFu, mine);
        }
    }

    // One step of the split, on the whole warp: each lane adds its photon's term of group g (NO_PRIM: no photon) to its
    // run; the lanes whose photon belongs to another group than their run hand the run to the warp first.
    template <class R, class Scale>
    MCRT_D void groupRunStep(const WaveParams<R>& p, uint32_t film_index, const V3<R>& weight, Scale&& scale, uint32_t g,
                             const V3<R>& term, uint32_t& run, V3<R>& run_sum)
    {
        const bool flush = g != NO_PRIM && run != NO_PRIM && g != run;
        if (__any_sync(0xFFFFFFFFu, flush))
        {
            depositGroupRuns(p, film_index, flush ? run : NO_PRIM, run_sum, weight, scale);
            if (flush) { run = NO_PRIM; run_sum = V3<R>(R(0)); }
        }
        if (g != NO_PRIM) { run = g; run_sum += term; }
    }

    // The LPE split of a photon estimate (FILM_MODE_LPE of k_knn / k_gather): groupRunStep / depositGroupRuns with runs
    // keyed by the photon's accept mask, join[query state][photon state], and a run's sum deposited into every plane of
    // its mask. Every 32-bit value is a mask, so `has` marks a run; a mask of 0 starts none, so its photon adds nothing.
    template <class R, class Scale>
    MCRT_D void depositMaskRuns(const WaveParams<R>& p, uint32_t film_index, bool has, uint32_t mask, const V3<R>& sum,
                                const V3<R>& weight, Scale&& scale)
    {
        const unsigned lane = threadIdx.x & 31u;
        unsigned pending = __ballot_sync(0xFFFFFFFFu, has);
        while (pending)
        {
            const int leader = __ffs(pending) - 1;
            const uint32_t g = __shfl_sync(0xFFFFFFFFu, mask, leader);
            const bool mine = has && mask == g;
            V3<R> v = mine ? sum : V3<R>(R(0));
            for (int off = 16; off > 0; off >>= 1)
            {
                v.x += __shfl_xor_sync(0xFFFFFFFFu, v.x, off);
                v.y += __shfl_xor_sync(0xFFFFFFFFu, v.y, off);
                v.z += __shfl_xor_sync(0xFFFFFFFFu, v.z, off);
            }
            if ((int)lane == leader)
            {
                const V3<R> d = scale(v) * weight;
                for (uint32_t m = g; m; m &= m - 1u) filmAddV(p.film + (uint32_t)(__ffs(m) - 1) * p.plane_values, film_index, d);
            }
            pending &= ~__ballot_sync(0xFFFFFFFFu, mine);
        }
    }

    template <class R, class Scale>
    MCRT_D void maskRunStep(const WaveParams<R>& p, uint32_t film_index, const V3<R>& weight, Scale&& scale, uint32_t mask,
                            const V3<R>& term, bool& run_has, uint32_t& run, V3<R>& run_sum)
    {
        const bool flush = mask != 0u && run_has && mask != run;
        if (__any_sync(0xFFFFFFFFu, flush))
        {
            depositMaskRuns(p, film_index, flush, run, run_sum, weight, scale);
            if (flush) { run_has = false; run_sum = V3<R>(R(0)); }
        }
        if (mask != 0u) { run_has = true; run = mask; run_sum += term; }
    }

    // accept mask of a photon term: the query's forward state (KnnQuery::meta.z bits 16-23) joined with the photon's
    template <class R>
    MCRT_D uint32_t lpePhotonMask(const WaveParams<R>& p, uint32_t query_state, uint32_t which, unsigned long long idx)
    {
        const uint32_t r = __ldg(&p.pm.lpe_states[which][idx]);
        return r == MCRT_LPE_DEAD ? 0u : __ldg(&p.pm.lpe_join[query_state * p.pm.lpe_rev_states + r]);
    }

    // ------------------------------------------------------------------------------------------
    // k_knn: one warp per photon-map query emitted by k_shade<R,1>; search + radiance estimate.
    // FILM_MODE_GROUPS splits the estimate by the light group of each photon (depositGroupRuns); FILM_MODE_AOV deposits
    // the whole estimate into its map's component plane, MCRT_PM_CAUSTIC + which.
    template <class R, int SLOTS, int FILM, uint32_t FEATS>
    __global__ void __launch_bounds__(32 * KNN_WARPS_PER_BLOCK, MCRT_KNN_MINBLOCKS) k_knn(WaveParams<R> p)
    {
        extern __shared__ __align__(16) unsigned char knn_smem[];
        const uint32_t n = min(p.counters->n_knn, p.pm.query_capacity);
        const uint32_t k = p.pm.k_nearest;
        const KnnShared sh = knnSharedFor(knn_smem, (k + 31u) & ~31u);
        const unsigned lane = threadIdx.x & 31u;
        const uint32_t warps_total = gridDim.x * KNN_WARPS_PER_BLOCK;
        uint32_t overflow = 0;
        for (uint32_t q = blockIdx.x * KNN_WARPS_PER_BLOCK + (threadIdx.x >> 5); q < n; q += warps_total)
        {
            const KnnQuery<R> qr = p.pm.queries[q];
            const uint32_t which = (qr.meta.z >> 1) & 1u;
            const DevicePhotonMap& map = p.pm.map[which];
            double res_max;
            const uint32_t found = knnSearchWarpT<SLOTS>(map, k, (double)qr.pos_n1.x, (double)qr.pos_n1.y, (double)qr.pos_n1.z,
                                                         sh, &res_max, &overflow);
            if (found == 0) continue;

            Interaction<R> ia;
            queryInteraction<FEATS>(p, qr, ia);

            const R top_d2 = (R)res_max;
            const R inv_max_r2 = R(1) / top_d2;
            if constexpr (FILM == FILM_MODE_GROUPS)
            {
                const auto scale = [&](const V3<R>& v) { return which == 0 ? R(3) * v * inv_max_r2 * Consts<R>::INV_PI : v / (top_d2 * Consts<R>::PI); };
                const V3<R> weight = qr.weight_t.xyz();
                uint32_t run = NO_PRIM;
                V3<R> run_sum(R(0));
                // uniform steps of 32 results, so that every lane takes part in the hand-over of runs
                for (uint32_t base = 0; base < found; base += 32)
                {
                    const uint32_t s = base + lane;
                    uint32_t g = NO_PRIM;
                    V3<R> term(R(0));
                    if (s < found)
                    {
                        const uint32_t idx = sh.res_idx[s];
                        g = p.group_of_light[__ldg(&p.pm.lights[which][idx])];
                        const float4 a = __ldg(&map.photons[2 * (size_t)idx]);
                        const float4 b = __ldg(&map.photons[2 * (size_t)idx + 1]);
                        if (!photonTerm(ia, which, a, b, (R)sh.res_d2[s], inv_max_r2, term)) term = V3<R>(R(0));
                    }
                    groupRunStep(p, qr.meta.y, weight, scale, g, term, run, run_sum);
                }
                depositGroupRuns(p, qr.meta.y, run, run_sum, weight, scale);
                __syncwarp();
                continue;
            }
            if constexpr (FILM == FILM_MODE_LPE)
            {
                const auto scale = [&](const V3<R>& v) { return which == 0 ? R(3) * v * inv_max_r2 * Consts<R>::INV_PI : v / (top_d2 * Consts<R>::PI); };
                const V3<R> weight = qr.weight_t.xyz();
                const uint32_t state = (qr.meta.z >> 16) & 0xFFu;
                bool run_has = false;
                uint32_t run = 0;
                V3<R> run_sum(R(0));
                for (uint32_t base = 0; base < found; base += 32)
                {
                    const uint32_t s = base + lane;
                    uint32_t mask = 0;
                    V3<R> term(R(0));
                    if (s < found)
                    {
                        const uint32_t idx = sh.res_idx[s];
                        mask = lpePhotonMask(p, state, which, idx);
                        const float4 a = __ldg(&map.photons[2 * (size_t)idx]);
                        const float4 b = __ldg(&map.photons[2 * (size_t)idx + 1]);
                        if (!photonTerm(ia, which, a, b, (R)sh.res_d2[s], inv_max_r2, term)) term = V3<R>(R(0));
                    }
                    maskRunStep(p, qr.meta.y, weight, scale, mask, term, run_has, run, run_sum);
                }
                depositMaskRuns(p, qr.meta.y, run_has, run, run_sum, weight, scale);
                __syncwarp();
                continue;
            }
            V3<R> sum(R(0));
            for (uint32_t s = lane; s < found; s += 32)
            {
                const uint32_t idx = sh.res_idx[s];
                const float4 a = __ldg(&map.photons[2 * (size_t)idx]);
                const float4 b = __ldg(&map.photons[2 * (size_t)idx + 1]);
                V3<R> bsdf_absIdotN; R bsdf_pdf;
                if (ia.bsdfWorld(bsdf_absIdotN, photonDir<R>(b.z, b.w), bsdf_pdf))
                {
                    const V3<R> flux((R)a.x, (R)a.y, (R)a.z);
                    if (which == 0)
                    {
                        // cone filter, photon-mapper.cpp:383-386
                        R wp = gmax(R(0), R(1) - msqrt((R)sh.res_d2[s] * inv_max_r2));
                        sum += (flux * bsdf_absIdotN * wp) / bsdf_pdf;
                    }
                    else
                    {
                        sum += flux * bsdf_absIdotN / bsdf_pdf;
                    }
                }
            }
            for (int off = 16; off > 0; off >>= 1)
            {
                sum.x += __shfl_xor_sync(0xFFFFFFFFu, sum.x, off);
                sum.y += __shfl_xor_sync(0xFFFFFFFFu, sum.y, off);
                sum.z += __shfl_xor_sync(0xFFFFFFFFu, sum.z, off);
            }
            if (lane == 0)
            {
                V3<R> radiance = which == 0 ? R(3) * sum * inv_max_r2 * Consts<R>::INV_PI
                                            : sum / (top_d2 * Consts<R>::PI);
                depositRadiance<FILM>(p, qr.meta.y, pixelOfFilmIndex(p, qr.meta.y), qr.meta.w, radiance * qr.weight_t.xyz(), NO_PRIM,
                                      MCRT_PM_CAUSTIC + which);
            }
            __syncwarp();
        }
        if (lane == 0)
        {
            if (overflow) atomicOr(&p.counters->traversal_overflow, 1u);
        }
        if (threadIdx.x == 0 && blockIdx.x == 0) atomicAdd(&p.counters->knn_queries, (unsigned long long)n);
    }

    // Batched LinearOctree::knnSearch on caller points (mcrt_knn_search): results sorted by the host.
    template <int SLOTS>
    __global__ void __launch_bounds__(32 * KNN_WARPS_PER_BLOCK) k_knn_user(DevicePhotonMap map, uint32_t k, const double* points,
                                                                          size_t n, uint32_t* out_index, double* out_d2,
                                                                          uint32_t* out_count, uint32_t* overflow_flag)
    {
        extern __shared__ __align__(16) unsigned char knn_smem[];
        const KnnShared sh = knnSharedFor(knn_smem, (k + 31u) & ~31u);
        const unsigned lane = threadIdx.x & 31u;
        const size_t warps_total = (size_t)gridDim.x * KNN_WARPS_PER_BLOCK;
        uint32_t overflow = 0;
        for (size_t q = (size_t)blockIdx.x * KNN_WARPS_PER_BLOCK + (threadIdx.x >> 5); q < n; q += warps_total)
        {
            double res_max;
            const uint32_t found = knnSearchWarpT<SLOTS>(map, k, points[3 * q], points[3 * q + 1], points[3 * q + 2], sh, &res_max, &overflow);
            for (uint32_t s = lane; s < k; s += 32)
            {
                out_index[q * k + s] = s < found ? sh.res_idx[s] : 0xFFFFFFFFu;
                out_d2[q * k + s] = s < found ? sh.res_d2[s] : 1.7976931348623157e308;
            }
            if (lane == 0) out_count[q] = found;
            __syncwarp();
        }
        if (overflow && lane == 0) atomicOr(overflow_flag, 1u);
    }


    // k_gather: k_knn with a fixed radius per map (PhotonParams::gather_r2, mcrt_photon_gather_radius) instead of
    // the k nearest photons: every photon within r (gatherWarp) enters the estimate with k_knn's formulas, r^2 in
    // place of the k-th distance2 - caustic 3/(pi r^2) sum flux f/pdf (1 - d/r), global 1/(pi r^2) sum flux f/pdf.
    // The BSDF is evaluated on the lane that finds the photon, while the batch streams.
    // FILM_MODE_GROUPS splits the estimate by light group as k_knn does, one step per 32 photons streamed; FILM_MODE_AOV
    // deposits into the map's component plane as k_knn does.
    template <class R, int FILM, uint32_t FEATS>
    __global__ void __launch_bounds__(32 * KNN_WARPS_PER_BLOCK, MCRT_GATHER_MINBLOCKS) k_gather(WaveParams<R> p)
    {
        __shared__ uint32_t gather_stack[KNN_WARPS_PER_BLOCK][GATHER_STACK];
        uint32_t* const stack = gather_stack[threadIdx.x >> 5];
        const uint32_t n = min(p.counters->n_knn, p.pm.query_capacity);
        const unsigned lane = threadIdx.x & 31u;
        const uint32_t warps_total = gridDim.x * KNN_WARPS_PER_BLOCK;
        uint32_t overflow = 0;
        for (uint32_t q = blockIdx.x * KNN_WARPS_PER_BLOCK + (threadIdx.x >> 5); q < n; q += warps_total)
        {
            const KnnQuery<R> qr = p.pm.queries[q];
            const uint32_t which = (qr.meta.z >> 1) & 1u;
            const double r2 = p.pm.gather_r2[which];
            Interaction<R> ia;
            queryInteraction<FEATS>(p, qr, ia);
            const R inv_r2 = R(1) / (R)r2;
            if constexpr (FILM == FILM_MODE_GROUPS)
            {
                const auto scale = [&](const V3<R>& v) { return which == 0 ? R(3) * v * inv_r2 * Consts<R>::INV_PI : v / ((R)r2 * Consts<R>::PI); };
                const V3<R> weight = qr.weight_t.xyz();
                const uint32_t* const lights = p.pm.lights[which];
                uint32_t g = NO_PRIM, run = NO_PRIM;   // g: the group of this lane's photon of the current step
                V3<R> term(R(0)), run_sum(R(0));
                gatherWarp(p.pm.map[which], (double)qr.pos_n1.x, (double)qr.pos_n1.y, (double)qr.pos_n1.z, r2, stack, &overflow,
                           [&](unsigned long long idx, double d2, const float4& a, const float4& b)
                           {
                               g = p.group_of_light[__ldg(&lights[idx])];
                               if (!photonTerm(ia, which, a, b, (R)d2, inv_r2, term)) term = V3<R>(R(0));
                           },
                           [&]
                           {
                               groupRunStep(p, qr.meta.y, weight, scale, g, term, run, run_sum);
                               g = NO_PRIM;
                           });
                depositGroupRuns(p, qr.meta.y, run, run_sum, weight, scale);   // no photon: no run, no deposit
                __syncwarp();
                continue;
            }
            if constexpr (FILM == FILM_MODE_LPE)
            {
                const auto scale = [&](const V3<R>& v) { return which == 0 ? R(3) * v * inv_r2 * Consts<R>::INV_PI : v / ((R)r2 * Consts<R>::PI); };
                const V3<R> weight = qr.weight_t.xyz();
                const uint32_t state = (qr.meta.z >> 16) & 0xFFu;
                uint32_t mask = 0, run = 0;   // mask: the accept mask of this lane's photon of the current step
                bool run_has = false;
                V3<R> term(R(0)), run_sum(R(0));
                gatherWarp(p.pm.map[which], (double)qr.pos_n1.x, (double)qr.pos_n1.y, (double)qr.pos_n1.z, r2, stack, &overflow,
                           [&](unsigned long long idx, double d2, const float4& a, const float4& b)
                           {
                               mask = lpePhotonMask(p, state, which, idx);
                               if (!photonTerm(ia, which, a, b, (R)d2, inv_r2, term)) term = V3<R>(R(0));
                           },
                           [&]
                           {
                               maskRunStep(p, qr.meta.y, weight, scale, mask, term, run_has, run, run_sum);
                               mask = 0;
                           });
                depositMaskRuns(p, qr.meta.y, run_has, run, run_sum, weight, scale);
                __syncwarp();
                continue;
            }
            V3<R> sum(R(0));
            bool found = false;
            gatherWarp(p.pm.map[which], (double)qr.pos_n1.x, (double)qr.pos_n1.y, (double)qr.pos_n1.z, r2, stack, &overflow,
                       [&](unsigned long long, double d2, const float4& a, const float4& b)
                       {
                           found = true;
                           V3<R> bsdf_absIdotN; R bsdf_pdf;
                           if (ia.bsdfWorld(bsdf_absIdotN, photonDir<R>(b.z, b.w), bsdf_pdf))
                           {
                               const V3<R> flux((R)a.x, (R)a.y, (R)a.z);
                               if (which == 0)
                               {
                                   const R wp = gmax(R(0), R(1) - msqrt((R)d2 * inv_r2));   // cone filter, photon-mapper.cpp:383-386
                                   sum += (flux * bsdf_absIdotN * wp) / bsdf_pdf;
                               }
                               else
                               {
                                   sum += flux * bsdf_absIdotN / bsdf_pdf;
                               }
                           }
                       });
            if (!__any_sync(0xFFFFFFFFu, found)) continue;   // as k_knn: no photon, no deposit
            for (int off = 16; off > 0; off >>= 1)
            {
                sum.x += __shfl_xor_sync(0xFFFFFFFFu, sum.x, off);
                sum.y += __shfl_xor_sync(0xFFFFFFFFu, sum.y, off);
                sum.z += __shfl_xor_sync(0xFFFFFFFFu, sum.z, off);
            }
            if (lane == 0)
            {
                V3<R> radiance = which == 0 ? R(3) * sum * inv_r2 * Consts<R>::INV_PI : sum / ((R)r2 * Consts<R>::PI);
                depositRadiance<FILM>(p, qr.meta.y, pixelOfFilmIndex(p, qr.meta.y), qr.meta.w, radiance * qr.weight_t.xyz(), NO_PRIM,
                                      MCRT_PM_CAUSTIC + which);
            }
            __syncwarp();
        }
        if (lane == 0 && overflow) atomicOr(&p.counters->traversal_overflow, 1u);
        if (threadIdx.x == 0 && blockIdx.x == 0) atomicAdd(&p.counters->knn_queries, (unsigned long long)n);
    }


    // ------------------------------------------------------------------------------------------
    // Photon emission pass on the device (SURVEY.md §8f-1). Same wavefront as the camera paths:
    // k_emit_generate -> [sort] -> k_extend -> k_emit_shade -> ... ; photons are appended to the
    // caustic / global arrays with one atomic per warp per array.
    // LPE (an LPE table is set): the path carries its reverse-DFA state in bits 16-23 of meta2.y, as camera paths carry
    // theirs; every photon is traced and stored as without it, whatever its state, since it counts for the radius of
    // every estimate near it.
    template <class R, bool LPE>
    __global__ void __launch_bounds__(256) k_emit_generate(WaveParams<R> p, int next)
    {
        Counters* c = p.counters;
        const uint32_t n_next = c->n_next;
        const unsigned long long remaining = c->total_work - c->next_work;
        const uint32_t room = p.capacity - n_next;
        const uint32_t count = remaining < (unsigned long long)room ? (uint32_t)remaining : room;
        if (blockIdx.x == 0 && threadIdx.x == 0) c->n_gen = count;
        const unsigned long long base_work = c->next_work;
        const PathBuffer<R>& out = p.buf[next];
        const DeviceScene<R>& sc = p.scene;

        const uint32_t count_rounded = (count + 31u) & ~31u;
        for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < count_rounded; j += gridDim.x * blockDim.x)
        {
            const bool valid = j < count;
            uint32_t key = 0;
            const uint32_t slot = n_next + j;
            if (valid)
            {
                const unsigned long long w = base_work + j;
                // light of this emission: last l with emit_offsets[l] <= w
                uint32_t lo = 0, hi = sc.n_lights;
                while (hi - lo > 1) { const uint32_t mid = (lo + hi) / 2; if (p.emit.emit_offsets[mid] <= w) lo = mid; else hi = mid; }
                const uint32_t light = lo;
                // pass > 0 continues each light's sample sequence past the emissions of the earlier passes
                const unsigned long long n_light = p.emit.emit_offsets[light + 1] - p.emit.emit_offsets[light];
                const uint32_t index = (uint32_t)((unsigned long long)p.emit.pass * n_light + (w - p.emit.emit_offsets[light]));
                // photon-mapper.cpp:95-110: initiate(light_index), setIndex(offset + i), get<PM_LIGHT,4>
                SamplerState smp = SamplerState::make(p.global_seed, light, index, 0u);
                R u[4];
                samplerGet<R, DIM_PM_LIGHT, 4>(smp, u);
                V3<R> pos, normal;
                sampleLightPoint(sc.lights[light], u[0], u[1], pos, normal);
                const V3<R> dir = Frame<R>(normal).from(cosWeightedHemi(u[2], u[3]));
                pos += normal * p.ray_eps;   // photon-mapper.cpp:108 (C::EPSILON in parity mode)
                const V4<R> flux = p.emit.photon_flux[light];
                out.ray_o[slot] = V4<R>(pos, sc.scene_ior);
                out.ray_d[slot] = V4<R>(dir, R(1));
                out.thr[slot] = V4<R>(flux.x, flux.y, flux.z, R(0));
                out.meta[slot] = make_uint4(light, index, 0u, 0u);
                uint32_t lpe_state = 0;
                if constexpr (LPE)
                    lpe_state = p.emit.lpe_rev_start == MCRT_LPE_DEAD ? (uint32_t)MCRT_LPE_DEAD
                              : (uint32_t)__ldg(&p.emit.lpe_rev_next[p.emit.lpe_rev_start * p.lpe_symbols + lpeLightSymbol(p, light)]);
                out.meta2[slot] = make_uint4(NO_PRIM, 1u | (lpe_state << 16), 0u, sc.lights[light].type == PRIM_TRIANGLE ? sc.lights[light].prim : NO_PRIM);
                if (p.sort.path_order) key = rayKey(p.sort, pos, dir, sc.lights[light].prim);
            }
            if (p.sort.path_order)
            {
                const uint32_t rank = sortRank(p.sort.hist_path, key, valid);
                if (valid) { p.sort.path_key[next][slot] = key; p.sort.path_rank[next][slot] = rank; }
            }
        }
    }

    MCRT_D void storePhoton(float4* arr, unsigned long long idx, const V3<double>& flux, const V3<double>& pos, const V3<double>& dir)
    {
        // Photon::Photon, photon.hpp:7-12: float flux/position, polar angles of the direction
        const float theta = (float)atan2(sqrt(dir.x * dir.x + dir.y * dir.y), dir.z);
        const float phi = (float)atan2(dir.y, dir.x);
        arr[2 * idx] = make_float4((float)flux.x, (float)flux.y, (float)flux.z, (float)pos.x);
        arr[2 * idx + 1] = make_float4((float)pos.y, (float)pos.z, phi, theta);
    }

    template <class R, bool LPE>
    __global__ void __launch_bounds__(128, MCRT_SHADE_MINBLOCKS) k_emit_shade(WaveParams<R> p, int cur)
    {
        __shared__ SobolByteTables sobol_tab;
        sobol_tab.fill(p.sobol_bytes);
        __syncthreads();
        Counters* c = p.counters;
        const uint32_t n = c->n_cur;
        const PathBuffer<R>& in = p.buf[cur];
        const PathBuffer<R>& out = p.buf[cur ^ 1];
        const DeviceScene<R>& sc = p.scene;
        const bool sorting = p.sort.path_order != nullptr;
        uint32_t local_max_depth = 0, stack_overflows = 0;

        const uint32_t n_rounded = (n + 31u) & ~31u;
        for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_rounded; i += gridDim.x * blockDim.x)
        {
            bool alive = i < n;
            int store = -1;              // 0 caustic, 1 global
            V3<R> ph_flux, ph_pos, ph_dir;
            PathRay<R> ray, nray;
            V3<R> flux;
            uint4 meta, meta2;
            uint32_t ior_count = 1, hit_prim = NO_PRIM;
            R iors[IOR_STACK_CAPACITY];
            // LPE: the state before this vertex's event (stored with its photon) and after it (for the next bounce)
            uint32_t lpe_state = 0, lpe_next = 0;

            if (alive)
            {
                const V4<R> ro = ldStream(&in.ray_o[i]), rd = ldStream(&in.ray_d[i]), th = ldStream(&in.thr[i]), hv = ldStream(&p.hits[i]);
                meta = ldStream(&in.meta[i]); meta2 = ldStream(&in.meta2[i]);
                if constexpr (LPE) lpe_state = (meta2.y >> 16) & 0xFFu;
                ray.start = ro.xyz(); ray.medium_ior = ro.w;
                ray.direction = rd.xyz(); ray.refraction_scale = rd.w;
                flux = th.xyz();
                ray.depth = meta.z & 0xFFFFu; ray.diffuse_depth = meta.z >> 16;
                ray.refraction_level = (int32_t)meta.w;
                ior_count = meta2.y & 0xFFu;
                ray.dirac_delta = (meta2.y >> 8) & 1u;
                ray.refraction = false;
                iors[0] = sc.scene_ior;
                if (ior_count > 1)
                {
                    const V4<R> ia_ = in.iors_a[i];
                    iors[1] = ia_.x; iors[2] = ia_.y; iors[3] = ia_.z; iors[4] = ia_.w;
                    if (ior_count > 5) { const V4<R> ib_ = in.iors_b[i]; iors[5] = ib_.x; iors[6] = ib_.y; iors[7] = ib_.z; }
                }
                if (ray.depth > local_max_depth) local_max_depth = ray.depth;

                Hit<R> hit;
                hit.t = hv.x; hit.u = hv.y; hit.v = hv.z;
                hit.prim = hv.w < R(0) ? NO_PRIM : (uint32_t)hv.w;
                hit_prim = hit.prim;
                if (hit.prim == NO_PRIM)
                {
                    alive = false;  // photon-mapper.cpp:238-241
                }
                else
                {
                    SamplerState smp = SamplerState::make(p.global_seed, meta.x, meta.y, ray.depth + 1u);
                    smp.tab = &sobol_tab;
                    int ext_idx = ray.refraction_level - 1;
                    ext_idx = ext_idx < 0 ? 0 : (ext_idx > (int)ior_count - 1 ? (int)ior_count - 1 : ext_idx);
                    Interaction<R> ia;
                    buildInteraction(ia, sc, hit, ray, iors[ext_idx], smp);
                    const Material<R>& m = *ia.material;
                    if constexpr (LPE)
                        lpe_next = lpe_state == MCRT_LPE_DEAD ? (uint32_t)MCRT_LPE_DEAD
                                 : (uint32_t)__ldg(&p.emit.lpe_rev_next[lpe_state * p.lpe_symbols + lpeVertexSymbol(ia.type, ia.dirac_delta)]);

                    // photon-mapper.cpp:245-256: store only where non-delta interactions are possible
                    if (!(m.flags & MAT_DIRAC_DELTA))
                    {
                        if (ray.dirac_delta)
                        {
                            store = 0; ph_flux = flux;
                        }
                        else
                        {
                            R ur;
                            samplerGet<R, DIM_PM_REJECT, 1>(smp, &ur);
                            if (p.emit.non_caustic_reject > ur) { store = 1; ph_flux = flux / p.emit.non_caustic_reject; }
                        }
                        ph_pos = ia.position; ph_dir = -ray.direction;
                    }

                    V3<R> bsdf_absIdotN; R bsdf_pdf;
                    if (!sampleBSDF(ia, ray, smp, p.ray_eps, true, bsdf_absIdotN, bsdf_pdf, nray))
                    {
                        alive = false;
                    }
                    else
                    {
                        bsdf_absIdotN /= bsdf_pdf;
                        // photon-mapper.cpp:265-272: survival probability instead of flux scaling
                        R survive = gmin(compMax(bsdf_absIdotN), R(0.95));
                        R ua;
                        samplerGet<R, DIM_ABSORB, 1>(smp, &ua);
                        if (survive == R(0) || survive <= ua) alive = false;
                        else
                        {
                            flux *= bsdf_absIdotN / survive;
                            if (nray.refraction_level > 0)   // RefractionHistory::update
                            {
                                if (nray.refraction_level == (int32_t)ior_count)
                                {
                                    if (ior_count < (uint32_t)IOR_STACK_CAPACITY) iors[ior_count++] = nray.medium_ior;
                                    else stack_overflows++;
                                }
                                else if (nray.refraction_level < (int32_t)ior_count - 1) ior_count--;
                            }
                        }
                    }
                }
            }

            // photons: warp-aggregated append per array
            for (int which = 0; which < 2; which++)
            {
                const bool mine = store == which;
                const unsigned mask = __ballot_sync(0xFFFFFFFFu, mine);
                if (mask)
                {
                    const unsigned lane = threadIdx.x & 31u;
                    const int leader = __ffs(mask) - 1;
                    unsigned long long base = 0;
                    if ((int)lane == leader) base = atomicAdd(&c->n_photons[which], (unsigned long long)__popc(mask));
                    base = __shfl_sync(0xFFFFFFFFu, base, leader);
                    if (mine)
                    {
                        const unsigned long long idx = base + __popc(mask & ((1u << lane) - 1u));
                        if (idx < p.emit.capacity[which])
                        {
                            storePhoton(p.emit.photons[which], idx, V3<double>((double)ph_flux.x, (double)ph_flux.y, (double)ph_flux.z),
                                        V3<double>((double)ph_pos.x, (double)ph_pos.y, (double)ph_pos.z),
                                        V3<double>((double)ph_dir.x, (double)ph_dir.y, (double)ph_dir.z));
                            p.emit.lights[which][idx] = meta.x;   // the light k_emit_generate emitted the path from
                            if constexpr (LPE) p.emit.lpe_states[which][idx] = lpe_state;
                        }
                        else c->photon_overflow = 1u;
                    }
                }
            }

            const uint32_t slot = warpAppend(&c->n_next, alive);
            uint32_t pkey = 0, prank = 0;
            if (sorting && alive)
            {
                pkey = rayKey(p.sort, nray.start, nray.direction, hit_prim);
                prank = atomicAdd(&p.sort.hist_path[pkey], 1u);
            }
            if (alive)
            {
                out.ray_o[slot] = V4<R>(nray.start, nray.medium_ior);
                out.ray_d[slot] = V4<R>(nray.direction, nray.refraction_scale);
                out.thr[slot] = V4<R>(flux, R(0));
                if (ior_count > 1)
                {
                    out.iors_a[slot] = V4<R>(iors[1], iors[2], iors[3], iors[4]);
                    if (ior_count > 5) out.iors_b[slot] = V4<R>(iors[5], iors[6], iors[7], R(0));
                }
                out.meta[slot] = make_uint4(meta.x, meta.y, (nray.depth & 0xFFFFu) | (nray.diffuse_depth << 16), (uint32_t)nray.refraction_level);
                out.meta2[slot] = make_uint4(NO_PRIM, ior_count | (nray.dirac_delta ? 256u : 0u) | (lpe_next << 16), 0u,
                                             sc.shade[hit_prim].type == PRIM_TRIANGLE ? hit_prim : NO_PRIM);
                if (sorting) { p.sort.path_key[cur ^ 1][slot] = pkey; p.sort.path_rank[cur ^ 1][slot] = prank; }
            }
        }
        if (local_max_depth) atomicMax(&c->max_depth, local_max_depth);
        if (stack_overflows) atomicAdd(&c->ior_stack_overflows, (unsigned long long)stack_overflows);
    }

    // ------------------------------------------------------------------------------------------
    // Batched Scene::intersect on caller rays (mcrt_trace_closest)
    template <class R, bool FAST>
    __global__ void __launch_bounds__(256) k_trace_user(DeviceScene<R> sc, const double* rays6, size_t n, double* out_tuv,
                                                        uint32_t* out_prim, Counters* c)
    {
        TraceCounters cnt = { 0u, 0u, 0u };
        uint32_t overflow = 0;
        unsigned long long rays = 0;
        for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        {
            const double* r = rays6 + 6 * i;
            Hit<R> h = traceClosest<PRIMS_ALL, FAST>(sc, V3<R>((R)r[0], (R)r[1], (R)r[2]), V3<R>((R)r[3], (R)r[4], (R)r[5]), NO_PRIM, cnt, overflow);
            out_tuv[3 * i + 0] = (double)h.t; out_tuv[3 * i + 1] = (double)h.u; out_tuv[3 * i + 2] = (double)h.v;
            out_prim[i] = h.prim;
            rays++;
        }
        flushStats(c, cnt, rays, false, overflow);
    }

    // ------------------------------------------------------------------------------------------
    // First-hit guides of the denoiser (mcrt_render_features_dev). For samples [sample_first, sample_first +
    // sample_count) of each pixel, in increasing order, the closest hit of the sample's camera ray adds
    // {albedo.rgb, shading normal.xyz, t, 1} to out[pixel][8]; a miss adds nothing. Albedo is the specular
    // reflectance of mirrors and conductors and the reflectance of everything else. One thread owns a pixel and
    // adds its samples in order, so accumulating consecutive ranges is bit-identical to accumulating their union.
    template <class R, bool FAST>
    __global__ void __launch_bounds__(256) k_features(DeviceScene<R> sc, DeviceCamera<R> cam, uint32_t global_seed,
                                                      uint32_t sample_first, uint32_t sample_count, double* out, Counters* c)
    {
        TraceCounters cnt = { 0u, 0u, 0u };
        uint32_t overflow = 0;
        unsigned long long rays = 0;
        const uint32_t n = cam.width * cam.height;
        for (uint32_t pixel = blockIdx.x * blockDim.x + threadIdx.x; pixel < n; pixel += gridDim.x * blockDim.x)
        {
            double* f = out + 8 * (size_t)pixel;
            double sum[8];
            for (int k = 0; k < 8; k++) sum[k] = f[k];
            for (uint32_t k = 0; k < sample_count; k++)
            {
                const SamplerState smp = SamplerState::make(global_seed, pixel, sample_first + k, 0u);
                V3<R> start, direction;
                cameraRay(cam, sc.scene_ior, pixel, smp, start, direction);
                const Hit<R> h = traceClosest<PRIMS_ALL, FAST>(sc, start, direction, NO_PRIM, cnt, overflow);
                rays++;
                if (h.prim == NO_PRIM) continue;
                const PrimShade<R> ps = sc.shade[h.prim];
                const Material<R>& m = sc.materials[ps.material];
                const V3<R> albedo = (m.flags & (MAT_PERFECT_MIRROR | MAT_COMPLEX_IOR)) ? m.specular_reflectance : m.reflectance;
                V3<R> normal, shading_normal;
                surfaceNormals(sc, ps, h, start + direction * h.t, direction, normal, shading_normal);
                sum[0] += (double)albedo.x; sum[1] += (double)albedo.y; sum[2] += (double)albedo.z;
                sum[3] += (double)shading_normal.x; sum[4] += (double)shading_normal.y; sum[5] += (double)shading_normal.z;
                sum[6] += (double)h.t;
                sum[7] += 1.0;
            }
            for (int k = 0; k < 8; k++) f[k] = sum[k];
        }
        flushStats(c, cnt, rays, false, overflow);
    }

    // Guides after perfectly specular bounces (mcrt_render_features_chain_dev). Each sample follows its own path,
    // exactly as k_generate / k_shade trace it, through at most `specular_depth` hits on MAT_DIRAC_DELTA materials,
    // with throughput T = prod f/pdf and distance L = sum t. The first hit on any other material, the hit at the
    // depth cap, or a hit whose sampleBSDF rejects the direction or leaves T at 0, is the end vertex: it adds
    // {T * albedo, shading normal, L + t, 1}, with k_features' albedo and normal. A miss adds nothing. At depth 0 this
    // is k_features' sum bit for bit. A pure delta chain has diffuse_depth 0 and depth < 16, so the path would not
    // roulette there. Each continued vertex pushes at most one IOR, so a depth of at most IOR_STACK_CAPACITY - 1
    // (MCRT_FEATURES_MAX_SPECULAR_DEPTH, checked in abi.cu) cannot overflow the IOR stack.

    template <class R, bool FAST>
    __global__ void __launch_bounds__(256) k_features_chain(DeviceScene<R> sc, DeviceCamera<R> cam, uint32_t global_seed,
                                                            uint32_t sample_first, uint32_t sample_count, uint32_t specular_depth,
                                                            R ray_eps, double* out, Counters* c)
    {
        TraceCounters cnt = { 0u, 0u, 0u };
        uint32_t overflow = 0;
        unsigned long long rays = 0;
        const uint32_t n = cam.width * cam.height;
        for (uint32_t pixel = blockIdx.x * blockDim.x + threadIdx.x; pixel < n; pixel += gridDim.x * blockDim.x)
        {
            double* f = out + 8 * (size_t)pixel;
            double sum[8];
            for (int k = 0; k < 8; k++) sum[k] = f[k];
            for (uint32_t k = 0; k < sample_count; k++)
            {
                const uint32_t sample = sample_first + k;
                PathRay<R> ray;
                cameraRay(cam, sc.scene_ior, pixel, SamplerState::make(global_seed, pixel, sample, 0u), ray.start, ray.direction);
                ray.medium_ior = sc.scene_ior; ray.refraction_scale = R(1);
                ray.depth = 0u; ray.diffuse_depth = 0u; ray.refraction_level = 0;
                ray.dirac_delta = false; ray.refraction = false;
                R iors[IOR_STACK_CAPACITY];
                iors[0] = sc.scene_ior;
                uint32_t ior_count = 1, skip = NO_PRIM;
                V3<R> throughput(R(1), R(1), R(1));
                R distance = R(0);
                for (uint32_t depth = 0;; depth++)
                {
                    const Hit<R> h = traceClosest<PRIMS_ALL, FAST>(sc, ray.start, ray.direction, skip, cnt, overflow);
                    rays++;
                    if (h.prim == NO_PRIM) break;
                    const PrimShade<R> ps = sc.shade[h.prim];
                    const Material<R>& m = sc.materials[ps.material];
                    if (depth < specular_depth && (m.flags & MAT_DIRAC_DELTA))
                    {
                        // k_shade's bounce at this depth: RefractionHistory::externalIOR, Interaction, sampleBSDF
                        const SamplerState smp = SamplerState::make(global_seed, pixel, sample, depth + 1u);
                        int ext_idx = ray.refraction_level - 1;
                        ext_idx = ext_idx < 0 ? 0 : (ext_idx > (int)ior_count - 1 ? (int)ior_count - 1 : ext_idx);
                        Interaction<R> ia;
                        buildInteraction<SHADE_FEATS_ALL>(ia, sc, h, ray, iors[ext_idx], smp);
                        PathRay<R> nray;
                        V3<R> bsdf_absIdotN;
                        R pdf;
                        if (sampleBSDF(ia, ray, smp, ray_eps, false, bsdf_absIdotN, pdf, nray))
                        {
                            const V3<R> next_throughput = throughput * (bsdf_absIdotN / pdf);
                            if (compMax(next_throughput) != R(0))
                            {
                                throughput = next_throughput;
                                distance += h.t;
                                // RefractionHistory::update, ray.cpp:80-93
                                if (nray.refraction_level > 0)
                                {
                                    if (nray.refraction_level == (int32_t)ior_count)
                                    {
                                        if (ior_count < (uint32_t)IOR_STACK_CAPACITY) iors[ior_count++] = nray.medium_ior;
                                    }
                                    else if (nray.refraction_level < (int32_t)ior_count - 1)
                                    {
                                        ior_count--;
                                    }
                                }
                                skip = ps.type == PRIM_TRIANGLE ? h.prim : NO_PRIM;   // the source primitive (fast mode)
                                ray = nray;
                                ray.refraction = false;
                                continue;
                            }
                        }
                    }
                    const V3<R> albedo = throughput * ((m.flags & (MAT_PERFECT_MIRROR | MAT_COMPLEX_IOR)) ? m.specular_reflectance : m.reflectance);
                    V3<R> normal, shading_normal;
                    surfaceNormals(sc, ps, h, ray.start + ray.direction * h.t, ray.direction, normal, shading_normal);
                    sum[0] += (double)albedo.x; sum[1] += (double)albedo.y; sum[2] += (double)albedo.z;
                    sum[3] += (double)shading_normal.x; sum[4] += (double)shading_normal.y; sum[5] += (double)shading_normal.z;
                    sum[6] += (double)(distance + h.t);
                    sum[7] += 1.0;
                    break;
                }
            }
            for (int k = 0; k < 8; k++) f[k] = sum[k];
        }
        flushStats(c, cnt, rays, false, overflow);
    }

    // Film::Splat::get for the box filter: mean of the samples, clamped at 0 (film.cpp:106-113)
    // Film::Splat::get with accumulated weights (film.cpp:106-113)
    static __global__ void k_resolve_film_weighted(const double* film, const double* wsum, double* out, size_t n_pixels)
    {
        for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < 3 * n_pixels; i += (size_t)gridDim.x * blockDim.x)
        {
            const double w = wsum[i / 3];
            const double v = w == 0.0 ? 0.0 : film[i] / w;
            out[i] = (v < 0.0) ? 0.0 : v;
        }
    }

    // Film resolve fused with the frame exchange of a row-sharded multi-GPU render: this rank's rows
    // (y_first + k * y_step) go straight into the full-frame buffer of EVERY rank - peer memory mapped
    // through CUDA IPC, stores travel over NVLink - at their final position, as the float3 framebuffer
    // (or float64). No staging buffer, no all-gather, no re-interleaving copy.
    constexpr int MAX_FRAME_PEERS = 16;
    struct PeerFrames
    {
        void* frame[MAX_FRAME_PEERS];
        uint32_t n_frames, as_float;
        uint32_t y_first, y_step, row_values;   // row_values = width * 3
    };

    static __global__ void __launch_bounds__(256) k_resolve_film_peers(const double* film, PeerFrames pf, size_t n_values, double weight)
    {
        for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_values; i += (size_t)gridDim.x * blockDim.x)
        {
            double v = film[i] / weight;
            v = (v < 0.0) ? 0.0 : v;
            const size_t row = i / pf.row_values, col = i - row * pf.row_values;
            const size_t at = ((size_t)pf.y_first + row * pf.y_step) * pf.row_values + col;
            if (pf.as_float)
            {
                const float f = (float)v;
                for (uint32_t q = 0; q < pf.n_frames; q++) static_cast<float*>(pf.frame[q])[at] = f;
            }
            else
            {
                for (uint32_t q = 0; q < pf.n_frames; q++) static_cast<double*>(pf.frame[q])[at] = v;
            }
        }
    }

    // FP64 issue-rate probe for bench.py's roofline: 8 independent DFMA chains per thread
    static __global__ void __launch_bounds__(256) k_fp64_peak(double* sink, int iterations)
    {
        double a0 = threadIdx.x * 1e-9, a1 = a0 + 1.0, a2 = a0 + 2.0, a3 = a0 + 3.0, a4 = a0 + 4.0, a5 = a0 + 5.0, a6 = a0 + 6.0, a7 = a0 + 7.0;
        const double m = 1.0000001, c = 1e-9;
        for (int i = 0; i < iterations; i++)
        {
            a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
            a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
        }
        const double r = ((a0 + a1) + (a2 + a3)) + ((a4 + a5) + (a6 + a7));
        if (r == 12345.678) sink[0] = r;   // never true: keeps the chains alive
    }

    // One half of a progressive render (mcrt_progressive_resolve_dev): unresolved sums over a set of sample passes.
    struct ProgressiveHalf
    {
        const double* rgb;    // [pixels][3]; null when the half has no samples
        const double* wsum;   // [pixels] weight sums of a reconstruction filter; null with the box film
        double samples;       // samples per pixel in this half (the box film's weight)
    };

    // Relative error sqrt(sum v / sum I^2) of a region. +inf while one half has no samples; 0 where the halves agree
    // exactly (a region that is black in both halves included).
    MCRT_HD double progressiveRelativeError(double sum_v, double sum_i2, bool both_halves)
    {
        if (!both_halves) return HUGE_VAL;
        if (sum_v == 0.0) return 0.0;
        return sum_i2 > 0.0 ? sqrt(sum_v / sum_i2) : HUGE_VAL;
    }

    static __global__ void k_resolve_film(const double* film, double* out, size_t n_values, double weight)
    {
        for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_values; i += (size_t)gridDim.x * blockDim.x)
        {
            // res / w with w = spp (every sample deposits weight 1), then glm::max(., 0.0)
            double v = film[i] / weight;
            out[i] = (v < 0.0) ? 0.0 : v;
        }
    }
}
