// Photon-map lookup on the device: LinearOctree<Photon>::knnSearch
// (source/octree/linear-octree.cpp:24-117) as a warp-cooperative kernel, and the radiance estimates
// of PhotonMapper::estimateGlobalRadiance / estimateCausticRadiance
// (source/integrator/photon-mapper/photon-mapper.cpp:343-391).
//
// One warp per query. The k nearest photons are unique (distances are float64 of float32 positions),
// so any exact search returns the reference's set; the estimate then only differs by summation
// order. The warp keeps
//   * the k current results (distance2, photon index) in shared memory, unsorted, with the running
//     maximum found by a warp reduction (the reference's bounded max-heap, linear-octree.cpp:60-84);
//   * the best-first frontier of octants (the reference's `to_visit` heap, :39-46) as an unsorted
//     array popped by a warp-parallel arg-min;
//   * the pruning radius max_distance2 with the reference's two tightening rules (:82, :96-100).
// Leaves (and inner octants holding <= k photons, :51-54) stream their contiguous photon range 32
// photons = 1 KB per step, coalesced; children of an inner octant are tested by lanes 0..7 at once.
#pragma once

#include "bsdf.cuh"

namespace mcrt
{
    constexpr uint32_t OCTANT_NULL = 0xFFFFFFFFu;
    constexpr int KNN_FRONTIER = 256;
    constexpr int KNN_WARPS_PER_BLOCK = 4;

    struct alignas(16) DeviceOctant
    {
        double bmin[3], bmax[3];
        unsigned long long start, count;
        uint32_t children[8];   // OCTANT_NULL padded (derived from the next_sibling chain at upload)
        uint32_t n_children, leaf;
    };

    struct DevicePhotonMap
    {
        const DeviceOctant* octants;
        const float4* photons;  // 2 per photon: {flux.xyz, pos.x}, {pos.y, pos.z, phi, theta}
        uint32_t n_octants, _pad;
        unsigned long long n_photons;
    };

    // What k_shade hands to k_knn: the Interaction fields Interaction::BSDF needs, the weight
    // (path throughput) and where to deposit.
    template <class R> struct KnnQuery
    {
        V4<R> pos_n1;        // position.xyz, n1
        V4<R> nrm_n2;        // shading normal.xyz, n2
        V4<R> out_rf;        // out.xyz, R (specular reflect probability)
        V4<R> weight_t;      // throughput.xyz, T (transparency)
        uint4 meta;          // material, film_index, flags (bit0 inside, bit1 map: 0 caustic 1 global), -
    };

    template <class R> struct PhotonParams
    {
        DevicePhotonMap map[2];
        KnnQuery<R>* queries;
        uint32_t k_nearest, direct_visualization, query_capacity, _pad;
        double gather_r2[2];     // fixed gather radius^2 per map (k_gather); 0: the k-NN estimate (k_knn)
        // per map, the index of the light that emitted each photon, in map order (maps emitted on the device; read by the
        // light-group estimates only). Kept out of DevicePhotonMap so that the search kernels' parameters keep their layout.
        const uint32_t* lights[2];
        // FILM_MODE_LPE: per map, the reverse-DFA state of each photon in map order (lpe_states), and the join of the
        // forward states with those states, [forward][lpe_rev_states] accept masks; lpe_join_any[s]: some photon history
        // completes forward state s, so k_shade queries the maps there (lpe.h)
        const uint32_t* lpe_states[2];
        const uint32_t* lpe_join;
        const uint8_t* lpe_join_any;
        uint32_t lpe_rev_states;
    };

    MCRT_D double octantDistance2(const DeviceOctant& o, double px, double py, double pz)
    {
        // BoundingBox::distance2, bounding-box.cpp:43-47
        double dx = gmax(gmax(o.bmin[0] - px, px - o.bmax[0]), 0.0);
        double dy = gmax(gmax(o.bmin[1] - py, py - o.bmax[1]), 0.0);
        double dz = gmax(gmax(o.bmin[2] - pz, pz - o.bmax[2]), 0.0);
        return dx * dx + dy * dy + dz * dz;
    }

    MCRT_D double octantMaxDistance2(const DeviceOctant& o, double px, double py, double pz)
    {
        // BoundingBox::max_distance2, bounding-box.cpp:50-54
        double dx = gmax(o.bmax[0] - px, px - o.bmin[0]);
        double dy = gmax(o.bmax[1] - py, py - o.bmin[1]);
        double dz = gmax(o.bmax[2] - pz, pz - o.bmin[2]);
        return dx * dx + dy * dy + dz * dz;
    }

    constexpr int KNN_HIST_BINS = 256;

    struct KnnShared
    {
        double* res_d2;       // [k_pad]
        uint32_t* res_idx;    // [k_pad]
        double* fr_d2;        // [KNN_FRONTIER]
        uint32_t* fr_node;    // [KNN_FRONTIER]
        uint32_t* hist;       // [KNN_HIST_BINS] distance histogram of one leaf (radius estimate before the result set is full)
    };

    // warp maximum of non-negative doubles: their bit patterns order like the values, so two
    // hardware integer reductions (REDUX) replace five 64-bit shuffle steps
    MCRT_D double warpMaxD(double v)
    {
        const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
        const unsigned hi = (unsigned)(bits >> 32), lo = (unsigned)bits;
        const unsigned mhi = __reduce_max_sync(0xFFFFFFFFu, hi);
        const unsigned mlo = __reduce_max_sync(0xFFFFFFFFu, hi == mhi ? lo : 0u);
        return __longlong_as_double((long long)(((unsigned long long)mhi << 32) | mlo));
    }

    // warp minimum of non-negative doubles (same trick, inverted)
    MCRT_D double warpMinD(double v)
    {
        const unsigned long long bits = (unsigned long long)__double_as_longlong(v);
        const unsigned hi = (unsigned)(bits >> 32), lo = (unsigned)bits;
        const unsigned mhi = __reduce_min_sync(0xFFFFFFFFu, hi);
        const unsigned mlo = __reduce_min_sync(0xFFFFFFFFu, hi == mhi ? lo : 0xFFFFFFFFu);
        return __longlong_as_double((long long)(((unsigned long long)mhi << 32) | mlo));
    }

    // Warp-cooperative search. Distances are always float64, as in the reference
    // (glm::distance2(data.pos(), p) on dvec3). Returns the number of results (<= k); the results
    // are left in sh.res_*; *res_max is the largest distance2 among them.
    // SLOTS = ceil(k / 32) when that is 1, 2, 4 or 8: once the result set is full it moves from
    // shared memory into SLOTS registers per lane (slot s lives in lane s % 32), so replacing the
    // farthest result and re-deriving the maximum are register operations + two REDUX (ncu on the
    // shared-memory version: 37 % of all instructions were those two loops). SLOTS = 0: any k.
    template <int SLOTS>
    MCRT_D uint32_t knnSearchWarpT(const DevicePhotonMap& map, uint32_t k, double px, double py, double pz,
                                   const KnnShared& sh, double* res_max, uint32_t* overflow)
    {
        constexpr int NS = SLOTS > 0 ? SLOTS : 1;
        double r_d2[NS]; uint32_t r_idx[NS];
        bool in_regs = false;
        const unsigned lane = threadIdx.x & 31u;
        *res_max = 0.0;
        if (map.n_octants == 0 || map.n_photons == 0) return 0;
        if ((unsigned long long)k > map.n_photons) k = (uint32_t)map.n_photons;

        uint32_t n_found = 0;
        double max_d2 = 1.7976931348623157e308;
        double cur_max = 0.0;        // max distance2 among stored results (valid once n_found == k)
        uint32_t n_frontier = 0;
        uint32_t cur = 0;
        double cur_d2 = octantDistance2(map.octants[0], px, py, pz);
        (void)cur_d2;

        while (true)
        {
            const DeviceOctant* node = &map.octants[cur];
            const unsigned long long count = node->count;
            if (node->leaf || count <= (unsigned long long)k)
            {
                const unsigned long long start = node->start, end = start + count;
                if (n_found < k && count >= (unsigned long long)k && count <= 8ull * 32ull)
                {
                    // Radius estimate before the fill. Filling the result set with the first k photons of the leaf
                    // and then replacing the farthest one photon at a time costs ~k ln(count/k) replacements of ~55
                    // dependent warp instructions each (70 % of the kernel, ncu). Instead: one pass histograms the
                    // photons' distances (256 bins between the nearest and the farthest point of the octant's box),
                    // the bin where the running count reaches k gives an upper bound of the k-th distance - the same
                    // kind of bound as the reference's farthest-corner rule (linear-octree.cpp:98-101), only tighter -
                    // and the fill below then accepts k photons plus the few that share the last bin.
                    const double lo = octantDistance2(*node, px, py, pz), hi = octantMaxDistance2(*node, px, py, pz);
                    if (hi > lo)
                    {
                        const double scale = (double)(KNN_HIST_BINS - 1) / (hi - lo);
                        for (uint32_t b = lane; b < (uint32_t)KNN_HIST_BINS; b += 32) sh.hist[b] = 0u;
                        __syncwarp();
                        for (unsigned long long idx = start + lane; idx < end; idx += 32)
                        {
                            const float4 a = __ldg(&map.photons[2 * idx]);
                            const float4 b = __ldg(&map.photons[2 * idx + 1]);
                            const double dx = px - (double)a.w, dy = py - (double)b.x, dz = pz - (double)b.y;
                            const double d2 = dx * dx + dy * dy + dz * dz;
                            if (d2 <= max_d2)
                            {
                                const double q = (d2 - lo) * scale;   // monotone in d2
                                const uint32_t bin = q <= 0.0 ? 0u : (q >= (double)(KNN_HIST_BINS - 1) ? (uint32_t)(KNN_HIST_BINS - 1) : (uint32_t)q);
                                atomicAdd(&sh.hist[bin], 1u);
                            }
                        }
                        __syncwarp();
                        uint32_t mine = 0;
#pragma unroll
                        for (int b = 0; b < KNN_HIST_BINS / 32; b++) mine += sh.hist[lane * (KNN_HIST_BINS / 32) + b];
                        uint32_t incl = mine;
                        for (int off = 1; off < 32; off <<= 1)
                        {
                            const uint32_t up = __shfl_up_sync(0xFFFFFFFFu, incl, off);
                            if (lane >= (unsigned)off) incl += up;
                        }
                        const unsigned reach = __ballot_sync(0xFFFFFFFFu, incl >= k);
                        if (reach)   // else: fewer than k photons of this leaf lie inside the current bound
                        {
                            const int owner = __ffs(reach) - 1;
                            uint32_t bsel = 0;
                            if ((int)lane == owner)
                            {
                                uint32_t running = incl - mine;
                                for (int b = 0; b < KNN_HIST_BINS / 32; b++)
                                {
                                    running += sh.hist[lane * (KNN_HIST_BINS / 32) + b];
                                    if (running >= k) { bsel = lane * (KNN_HIST_BINS / 32) + b; break; }
                                }
                            }
                            bsel = __shfl_sync(0xFFFFFFFFu, bsel, owner);
                            // every photon counted up to bin bsel has d2 < upper edge of that bin (the mapping is monotone)
                            const double bound = (lo + (double)(bsel + 1u) / scale) * (1.0 + 1e-9);
                            if (bound < max_d2) max_d2 = bound;
                        }
                        __syncwarp();
                    }
                }
                for (unsigned long long base = start; base < end; base += 32)
                {
                    const unsigned long long idx = base + lane;
                    double d2 = 0.0;
                    bool cand = false;
                    if (idx < end)
                    {
                        const float4 a = __ldg(&map.photons[2 * idx]);
                        const float4 b = __ldg(&map.photons[2 * idx + 1]);
                        // distance2(data.pos(), p) = length2(p - pos)
                        double dx = px - (double)a.w, dy = py - (double)b.x, dz = pz - (double)b.y;
                        d2 = dx * dx + dy * dy + dz * dz;
                        cand = d2 <= max_d2;
                    }
                    unsigned ballot = __ballot_sync(0xFFFFFFFFu, cand);
                    // fill phase: while the result set has room, the candidates of a batch are appended
                    // in parallel (the reference's push_unordered, linear-octree.cpp:63-66)
                    if (ballot && n_found < k)
                    {
                        const uint32_t room = k - n_found;
                        const uint32_t my = (uint32_t)__popc(ballot & ((1u << lane) - 1u));
                        if (cand && my < room) { sh.res_d2[n_found + my] = d2; sh.res_idx[n_found + my] = (uint32_t)(base + lane); }
                        const uint32_t taken = min(room, (uint32_t)__popc(ballot));
                        n_found += taken;
                        // drop the lanes that were stored from the ballot
                        unsigned rest = ballot;
                        for (uint32_t t = 0; t < taken; t++) rest &= rest - 1;
                        ballot = rest;
                        __syncwarp();
                        if (n_found == k)
                        {
                            double m = 0.0;
                            if constexpr (SLOTS > 0)
                            {
#pragma unroll
                                for (int j = 0; j < NS; j++)
                                {
                                    const uint32_t s = lane + 32u * j;
                                    r_d2[j] = s < k ? sh.res_d2[s] : -1.0;
                                    r_idx[j] = s < k ? sh.res_idx[s] : 0xFFFFFFFFu;
                                    m = fmax(m, r_d2[j]);
                                }
                                in_regs = true;
                            }
                            else
                            {
                                for (uint32_t s = lane; s < k; s += 32) m = fmax(m, sh.res_d2[s]);
                            }
                            cur_max = warpMaxD(m);
                            if (cur_max < max_d2) max_d2 = cur_max;
                        }
                    }
                    // replace phase: candidates in ascending distance order against the current farthest
                    // result; as soon as the nearest remaining candidate is beyond the radius all the
                    // others are too (the outcome - the k smallest - does not depend on the order)
                    bool pending = (ballot >> lane) & 1u;
                    while (ballot)
                    {
                        const double cd2 = warpMinD(pending ? d2 : 1.7976931348623157e308);
                        if (!(cd2 <= max_d2)) break;
                        const unsigned who = __ballot_sync(0xFFFFFFFFu, pending && d2 == cd2);
                        const int src = __ffs(who) - 1;
                        ballot &= ~(1u << src);
                        if ((int)lane == src) pending = false;
                        const uint32_t cidx = (uint32_t)(base + src);
                        {
                            // pop_push: replace the farthest of the k results (linear-octree.cpp:79)
                            double m = 0.0;
                            if constexpr (SLOTS > 0)
                            {
                                int mine = -1;
#pragma unroll
                                for (int j = NS - 1; j >= 0; j--) if (r_d2[j] == cur_max) mine = j;
                                const unsigned has = __ballot_sync(0xFFFFFFFFu, mine >= 0);
                                const int owner = __ffs(has) - 1;
#pragma unroll
                                for (int j = 0; j < NS; j++)
                                {
                                    if ((int)lane == owner && j == mine) { r_d2[j] = cd2; r_idx[j] = cidx; }
                                    m = fmax(m, r_d2[j]);
                                }
                            }
                            else
                            {
                                uint32_t slot = 0xFFFFFFFFu;
                                for (uint32_t s = lane; s < k; s += 32) if (sh.res_d2[s] == cur_max) slot = s;
                                const unsigned has = __ballot_sync(0xFFFFFFFFu, slot != 0xFFFFFFFFu);
                                const int owner = __ffs(has) - 1;
                                if ((int)lane == owner) { sh.res_d2[slot] = cd2; sh.res_idx[slot] = cidx; }
                                __syncwarp();
                                for (uint32_t s = lane; s < k; s += 32) m = fmax(m, sh.res_d2[s]);
                            }
                            cur_max = warpMaxD(m);
                            if (cur_max < max_d2) max_d2 = cur_max;
                        }
                    }
                }
            }
            else
            {
                // children: lanes 0..7 each take one (linear-octree.cpp:88-103)
                const uint32_t nc = node->n_children;
                uint32_t child = OCTANT_NULL;
                double d2 = 0.0, md2 = 1.7976931348623157e308;
                bool push = false;
                if (lane < nc)
                {
                    child = node->children[lane];
                    const DeviceOctant& cn = map.octants[child];
                    d2 = octantDistance2(cn, px, py, pz);
                    push = d2 <= max_d2;
                    if (push && cn.count >= (unsigned long long)k) md2 = octantMaxDistance2(cn, px, py, pz);
                }
                const unsigned ballot = __ballot_sync(0xFFFFFFFFu, push);
                if (push)
                {
                    const uint32_t slot = n_frontier + __popc(ballot & ((1u << lane) - 1u));
                    if (slot < (uint32_t)KNN_FRONTIER) { sh.fr_d2[slot] = d2; sh.fr_node[slot] = child; }
                }
                n_frontier += __popc(ballot);
                // set in every lane: the callers report lane 0's flag, and the dropped children may be any lanes'
                if (n_frontier > (uint32_t)KNN_FRONTIER) { *overflow = 1; n_frontier = KNN_FRONTIER; }
                // tighten with the farthest corner of any accepted child holding >= k photons
                double m = md2;
                for (int off = 4; off > 0; off >>= 1) m = fmin(m, __shfl_xor_sync(0xFFFFFFFFu, m, off));
                m = __shfl_sync(0xFFFFFFFFu, m, 0);
                if (m < max_d2) max_d2 = m;
                __syncwarp();
            }

            if (n_frontier == 0) break;
            // pop the nearest octant: warp arg-min over the unsorted frontier
            double mine_best = 1.7976931348623157e308;
            uint32_t mine_slot = 0xFFFFFFFFu;
            for (uint32_t s = lane; s < n_frontier; s += 32)
            {
                const double v = sh.fr_d2[s];
                if (v < mine_best || mine_slot == 0xFFFFFFFFu) { mine_best = v; mine_slot = s; }
            }
            const double best = warpMinD(mine_best);
            const unsigned holders = __ballot_sync(0xFFFFFFFFu, mine_slot != 0xFFFFFFFFu && mine_best == best);
            const uint32_t best_slot = __shfl_sync(0xFFFFFFFFu, mine_slot, __ffs(holders) - 1);
            if (best > max_d2) break; // linear-octree.cpp:113
            cur = sh.fr_node[best_slot];
            __syncwarp();
            if (lane == 0)
            {
                sh.fr_d2[best_slot] = sh.fr_d2[n_frontier - 1];
                sh.fr_node[best_slot] = sh.fr_node[n_frontier - 1];
            }
            n_frontier--;
            __syncwarp();
        }

        if (n_found < k)
        {
            double m = 0.0;
            for (uint32_t s = lane; s < n_found; s += 32) m = fmax(m, sh.res_d2[s]);
            cur_max = warpMaxD(m);
        }
        if constexpr (SLOTS > 0)
        {
            if (in_regs)
            {
                // hand the results back through shared memory (what the callers read)
#pragma unroll
                for (int j = 0; j < NS; j++)
                {
                    const uint32_t s = lane + 32u * j;
                    if (s < k) { sh.res_d2[s] = r_d2[j]; sh.res_idx[s] = r_idx[j]; }
                }
                __syncwarp();
            }
        }
        *res_max = cur_max;
        return n_found;
    }

    // register slots for a given k (0 = shared-memory fallback)
    inline int knnSlotsFor(uint32_t k)
    {
        return k <= 32 ? 1 : k <= 64 ? 2 : k <= 128 ? 4 : k <= 256 ? 8 : 0;
    }

    MCRT_D KnnShared knnSharedFor(unsigned char* smem, uint32_t k_pad)
    {
        const unsigned warp = threadIdx.x >> 5;
        const size_t per_warp = (size_t)k_pad * 12 + (size_t)KNN_FRONTIER * 12 + (size_t)KNN_HIST_BINS * 4;
        unsigned char* base = smem + warp * ((per_warp + 15) & ~(size_t)15);
        KnnShared sh;
        sh.res_d2 = reinterpret_cast<double*>(base);
        sh.fr_d2 = sh.res_d2 + k_pad;
        sh.res_idx = reinterpret_cast<uint32_t*>(sh.fr_d2 + KNN_FRONTIER);
        sh.fr_node = sh.res_idx + k_pad;
        sh.hist = sh.fr_node + KNN_FRONTIER;
        return sh;
    }

    inline size_t knnSharedBytes(uint32_t k)
    {
        const uint32_t k_pad = (k + 31u) & ~31u;
        const size_t per_warp = (size_t)k_pad * 12 + (size_t)KNN_FRONTIER * 12 + (size_t)KNN_HIST_BINS * 4;
        return KNN_WARPS_PER_BLOCK * ((per_warp + 15) & ~(size_t)15);
    }

    // Fixed-radius search (progressive photon mapping, Knaus & Zwicker 2011): every photon whose float64
    // distance2 to p is <= r2, the same inclusive test as knnSearchWarpT. One warp per query, depth first:
    // the children of an inner octant within r (octantDistance2 <= r2) are tested by lanes 0..7 and pushed
    // through a ballot onto the warp's stack in shared memory. A leaf - or an inner octant whose whole box
    // lies within r (octantMaxDistance2 <= r2) - streams its contiguous photon range 32 photons = 1 KB per
    // step, coalesced; every photon is still tested, so rounding at the box's corners cannot admit one
    // beyond r. visit(idx, d2, a, b) runs on each lane that holds an accepted photon (a, b: its two float4);
    // batch_end() runs on the whole warp, converged, after each step of 32 photons.
    // There is no result set, so the number of photons found is unbounded. A stack overflow drops octants
    // and sets *overflow (the callers fail the call, as for the k-NN frontier); a depth-first walk holds at
    // most 7 per level + 1, and the octree builder caps the depth at 64, so GATHER_STACK = 512 suffices.
    constexpr int GATHER_STACK = 512;

    template <class Visit, class BatchEnd>
    MCRT_D void gatherWarp(const DevicePhotonMap& map, double px, double py, double pz, double r2, uint32_t* stack,
                           uint32_t* overflow, Visit&& visit, BatchEnd&& batch_end)
    {
        const unsigned lane = threadIdx.x & 31u;
        if (map.n_octants == 0 || map.n_photons == 0) return;
        if (!(octantDistance2(map.octants[0], px, py, pz) <= r2)) return;
        uint32_t n_stack = 0, cur = 0;
        while (true)
        {
            const DeviceOctant* node = &map.octants[cur];
            if (node->leaf || octantMaxDistance2(*node, px, py, pz) <= r2)
            {
                const unsigned long long start = node->start, end = start + node->count;
                for (unsigned long long base = start; base < end; base += 32)
                {
                    const unsigned long long idx = base + lane;
                    if (idx < end)
                    {
                        const float4 a = __ldg(&map.photons[2 * idx]);
                        const float4 b = __ldg(&map.photons[2 * idx + 1]);
                        const double dx = px - (double)a.w, dy = py - (double)b.x, dz = pz - (double)b.y;
                        const double d2 = dx * dx + dy * dy + dz * dz;
                        if (d2 <= r2) visit(idx, d2, a, b);
                    }
                    batch_end();
                }
            }
            else
            {
                uint32_t child = OCTANT_NULL;
                bool push = false;
                if (lane < node->n_children)
                {
                    child = node->children[lane];
                    push = octantDistance2(map.octants[child], px, py, pz) <= r2;
                }
                const unsigned ballot = __ballot_sync(0xFFFFFFFFu, push);
                if (push)
                {
                    const uint32_t slot = n_stack + __popc(ballot & ((1u << lane) - 1u));
                    if (slot < (uint32_t)GATHER_STACK) stack[slot] = child;
                }
                n_stack += __popc(ballot);
                if (n_stack > (uint32_t)GATHER_STACK) { *overflow = 1; n_stack = GATHER_STACK; }
            }
            __syncwarp();
            if (n_stack == 0) break;
            cur = stack[--n_stack];
            __syncwarp();   // the slot just read is the next push's
        }
    }

    template <class Visit>
    MCRT_D void gatherWarp(const DevicePhotonMap& map, double px, double py, double pz, double r2, uint32_t* stack,
                           uint32_t* overflow, Visit&& visit)
    {
        gatherWarp(map, px, py, pz, r2, stack, overflow, visit, [] {});
    }

    // Photon::dir(), photon.hpp:19-27: std::sin/std::cos of the *float* angles (float overloads),
    // products in double. The float results are obtained by rounding the double functions, which is
    // what glibc's sinf/cosf return in all but vanishingly rare double-rounding cases.
    MCRT_D V3<float> photonDirFast(float phi, float theta)
    {
        float st, ct, sp, cp;
        sincosf(theta, &st, &ct);
        sincosf(phi, &sp, &cp);
        return V3<float>(st * cp, st * sp, ct);
    }

    template <class R>
    MCRT_D V3<R> photonDir(float phi, float theta)
    {
        if constexpr (sizeof(R) == 4) return photonDirFast(phi, theta);   // fast mode: float sincosf
        float st = (float)sin((double)theta), ct = (float)cos((double)theta);
        float sp = (float)sin((double)phi), cp = (float)cos((double)phi);
        double sin_theta = (double)st;
        return V3<R>((R)(sin_theta * (double)cp), (R)(sin_theta * (double)sp), (R)(double)ct);
    }
}
