// BVH construction on the device (widened scope, SURVEY.md §8f-2): the reference's three builders
//   BVH::recursiveBuildBinarySAH      source/bvh/bvh.cpp:165-283
//   BVH::recursiveBuildQuaternarySAH  source/bvh/bvh.cpp:285-432
//   BVH::recursiveBuildFromOctree     source/bvh/bvh.cpp:130-163 (+ Octree::insert, octree.cpp:34-81)
//   BVH::arbitrarySplit / compact     source/bvh/bvh.cpp:434-474
// rebuilt breadth-first. The result is the SAME tree, node for node: every decision of those
// builders is a function of bin counts and of min/max unions of primitive boxes, which are exact
// and order independent, and the few floating-point expressions (centroid, bin index, box area,
// SAH cost) are evaluated here in the reference's operation order with FMA contraction off (this
// file is compiled with --fmad=false). Every node's primitive list in the reference is ordered by
// original primitive index (partitions are stable), so primitives are moved with unordered
// warp-aggregated atomics during the build and each leaf is sorted by index at the end.
//
// One build round handles all nodes that are still open:
//   k_extent   centroid extent per node (warp-aggregated 64-bit integer min/max on sortable keys)
//   k_plan     per node: split axes / fall-backs / leaf decision
//   k_bin      per primitive: bin index, bin count and bin box (shared-memory bins when a whole
//              block sits in one node, global atomics otherwise)
//   k_arb_bin  arbitrarySplit: child = rank of the primitive in its node modulo N
//   k_split    one warp per node: evaluates every split candidate from the bins, picks the
//              reference's minimum (first one in loop order), creates the child nodes
//   k_scatter  moves primitive indices into their child's range
// then subtree sizes (bottom-up over rounds), depth-first numbering (top-down), emission of
// BVH::LinearNode arrays. Memory: bins are 56 B x bins_per_node x open nodes (at most n/9 nodes).
#include "bvh_build.h"

#include <algorithm>
#include <cfloat>
#include <cstring>

#include "../../include/mcrt_abi.h"

namespace mcrt
{
namespace
{
    constexpr uint32_t LEAF_SURFACES = 8;        // bvh.hpp:91
    constexpr uint32_t MAX_LEAF_SURFACES = 0xFF; // bvh.hpp:92
    constexpr double BUILD_EPS = 1e-9;           // C::EPSILON
    constexpr uint32_t NONE = 0xFFFFFFFFu;
    constexpr unsigned FULL = 0xFFFFFFFFu;

    enum Kind : uint32_t { KIND_QUAT = 0, KIND_BIN = 1, KIND_OCT = 2 };
    enum State : uint32_t { ST_LEAF = 0, ST_ACTIVE = 1, ST_ARB = 2, ST_INNER = 3 };
    enum Plan : uint32_t { PLAN_NONE = 0, PLAN_BIN2 = 1, PLAN_BIN4 = 2, PLAN_ARB = 3, PLAN_OCT = 4 };

    // order-preserving map double -> int64 (an involution), so that min/max run as integer atomics
    __host__ __device__ inline long long dkey(double d)
    {
#ifdef __CUDA_ARCH__
        long long b = __double_as_longlong(d);
#else
        long long b; std::memcpy(&b, &d, 8);
#endif
        return b >= 0 ? b : (b ^ 0x7FFFFFFFFFFFFFFFLL);
    }
    __host__ __device__ inline double keyd(long long k)
    {
        long long b = k >= 0 ? k : (k ^ 0x7FFFFFFFFFFFFFFFLL);
#ifdef __CUDA_ARCH__
        return __longlong_as_double(b);
#else
        double d; std::memcpy(&d, &b, 8); return d;
#endif
    }
    #define KEY_EMPTY_MIN 0x7FEFFFFFFFFFFFFFLL                              /* dkey(DBL_MAX) */
    #define KEY_EMPTY_MAX ((long long)(0xFFEFFFFFFFFFFFFFULL ^ 0x7FFFFFFFFFFFFFFFULL)) /* dkey(-DBL_MAX) */

    struct Bin
    {
        long long mn[3], mx[3];
        unsigned long long count;
    };

    struct BNode
    {
        long long bb[6];      // node box (keys): BuildNode::BB
        long long cext[6];    // centroid extent of its primitives
        double cube[6];       // octree cell (KIND_OCT)
        double pmin[2], pdim[2];
        uint32_t begin, end;  // range in the primitive index array
        uint32_t kind, state;
        uint32_t plan, axis[2], arb_n;
        uint32_t slot, split[2], split_round;
        uint32_t n_children, first_child;
        uint32_t vchild[8];   // bin group -> child node
        uint32_t cursor;      // scatter cursor into [begin, end)
        uint32_t subtree, df, next_sibling, depth;
    };

    // where a primitive's box comes from: [n][6] doubles, or photons (2 float4 each, position in
    // {p0.w, p1.x, p1.y}) whose box is the point itself
    struct BoxSource
    {
        const double* bounds;
        const float4* points;
    };

    __device__ inline void loadBox(const BoxSource& src, uint32_t prim, double b[6])
    {
        if (src.points)
        {
            const float4 p0 = src.points[2 * (size_t)prim], p1 = src.points[2 * (size_t)prim + 1];
            b[0] = b[3] = (double)p0.w; b[1] = b[4] = (double)p1.x; b[2] = b[5] = (double)p1.y;
        }
        else
        {
            const double* q = src.bounds + 6 * (size_t)prim;
            for (int k = 0; k < 6; k++) b[k] = q[k];
        }
    }

    struct BuildCounters
    {
        uint32_t n_nodes, n_active_next, _a, _b;
    };

    __device__ inline void initNode(BNode& c)
    {
        for (int k = 0; k < 3; k++) { c.bb[k] = KEY_EMPTY_MIN; c.bb[3 + k] = KEY_EMPTY_MAX; c.cext[k] = KEY_EMPTY_MIN; c.cext[3 + k] = KEY_EMPTY_MAX; }
        for (int k = 0; k < 6; k++) c.cube[k] = 0.0;
        c.pmin[0] = c.pmin[1] = c.pdim[0] = c.pdim[1] = 0.0;
        c.plan = PLAN_NONE; c.axis[0] = c.axis[1] = 0; c.arb_n = 0; c.slot = 0; c.split[0] = c.split[1] = 0; c.split_round = NONE;
        c.n_children = 0; c.first_child = NONE;
        for (int k = 0; k < 8; k++) c.vchild[k] = NONE;
        c.subtree = 1; c.df = 0; c.next_sibling = 0; c.depth = 0;
    }

    // BoundingBox::area (bounding-box.cpp:35-40) of a box held as keys
    __device__ inline double keyArea(const long long* mn, const long long* mx)
    {
        if (mn[0] > mx[0] || mn[1] > mx[1] || mn[2] > mx[2]) return 0.0;
        const double dx = keyd(mx[0]) - keyd(mn[0]), dy = keyd(mx[1]) - keyd(mn[1]), dz = keyd(mx[2]) - keyd(mn[2]);
        return 2.0 * (dx * dy + dx * dz + dy * dz);
    }

    __global__ void k_init(uint32_t* idx, uint32_t* node_of, uint32_t n)
    {
        for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) { idx[p] = p; node_of[p] = 0; }
    }

    __global__ void k_init_bins(Bin* bins, size_t n_bins)
    {
        for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_bins; i += (size_t)gridDim.x * blockDim.x)
        {
            Bin b;
            for (int k = 0; k < 3; k++) { b.mn[k] = KEY_EMPTY_MIN; b.mx[k] = KEY_EMPTY_MAX; }
            b.count = 0;
            bins[i] = b;
        }
    }

    __device__ inline long long warpMinLL(long long v)
    {
        for (int o = 16; o > 0; o >>= 1) { const long long w = __shfl_xor_sync(FULL, v, o); v = w < v ? w : v; }
        return v;
    }
    __device__ inline long long warpMaxLL(long long v)
    {
        for (int o = 16; o > 0; o >>= 1) { const long long w = __shfl_xor_sync(FULL, v, o); v = w > v ? w : v; }
        return v;
    }

    // centroid_extent.merge(s->BB().centroid()) over the node's primitives (bvh.cpp:175-180, 297-302)
    __global__ void __launch_bounds__(256) k_extent(BNode* nodes, const uint32_t* idx, const uint32_t* node_of, BoxSource src, uint32_t n)
    {
        const uint32_t stride = gridDim.x * blockDim.x;
        for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += stride)
        {
            const uint32_t p = base + threadIdx.x;
            const bool valid = p < n;
            const uint32_t nd = valid ? node_of[p] : NONE;
            bool need = false;
            if (valid) { const BNode& N = nodes[nd]; need = N.state == ST_ACTIVE && N.kind != KIND_OCT; }
            long long c[3] = {0, 0, 0};
            if (need)
            {
                double b[6];
                loadBox(src, idx[p], b);
                for (int k = 0; k < 3; k++) c[k] = dkey((b[3 + k] + b[k]) / 2.0);   // BoundingBox::centroid
            }
            const uint32_t nd0 = __shfl_sync(FULL, nd, 0);
            if (__all_sync(FULL, need && nd == nd0))
            {
                long long lo[3], hi[3];
                for (int k = 0; k < 3; k++) { lo[k] = warpMinLL(c[k]); hi[k] = warpMaxLL(c[k]); }
                if ((threadIdx.x & 31) == 0)
                    for (int k = 0; k < 3; k++) { atomicMin(&nodes[nd].cext[k], lo[k]); atomicMax(&nodes[nd].cext[3 + k], hi[k]); }
            }
            else if (need)
            {
                for (int k = 0; k < 3; k++) { atomicMin(&nodes[nd].cext[k], c[k]); atomicMax(&nodes[nd].cext[3 + k], c[k]); }
            }
        }
    }

    __global__ void k_plan(BNode* nodes, const uint32_t* active, uint32_t n_active, int bins_per_axis)
    {
        const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
        if (a >= n_active) return;
        BNode& N = nodes[active[a]];
        N.slot = a;
        const uint32_t size = N.end - N.begin;
        if (N.state == ST_ARB)
        {
            // min_cost > S.size() in the previous round: arbitrarySplit(node, 2 | 4) (bvh.cpp:237-245, 385-393)
            N.plan = PLAN_ARB; N.arb_n = N.kind == KIND_BIN ? 2u : 4u;
            return;
        }
        if (N.kind == KIND_OCT) { N.plan = PLAN_OCT; return; }
        double lo[3], dims[3];
        for (int k = 0; k < 3; k++) { lo[k] = keyd(N.cext[k]); dims[k] = keyd(N.cext[3 + k]) - lo[k]; }
        if (N.kind == KIND_QUAT)
        {
            // bvh.cpp:304-306
            int a0, a1;
            if (dims[0] > dims[1]) { a0 = 0; a1 = dims[1] > dims[2] ? 1 : 2; }
            else if (dims[0] > dims[2]) { a0 = 0; a1 = 1; }
            else { a0 = 1; a1 = 2; }
            if (dims[a0] < BUILD_EPS || dims[a1] < BUILD_EPS)
            {
                N.kind = KIND_BIN;   // recursiveBuildBinarySAH on this node and below (bvh.cpp:308-313)
            }
            else
            {
                N.plan = PLAN_BIN4; N.axis[0] = a0; N.axis[1] = a1;
                N.pmin[0] = lo[a0]; N.pmin[1] = lo[a1]; N.pdim[0] = dims[a0]; N.pdim[1] = dims[a1];
                return;
            }
        }
        // bvh.cpp:182-184
        const int axis = dims[0] > dims[1] ? (dims[0] > dims[2] ? 0 : 2) : (dims[1] > dims[2] ? 1 : 2);
        if (dims[axis] < BUILD_EPS)
        {
            if (size > MAX_LEAF_SURFACES) { N.plan = PLAN_ARB; N.arb_n = 2; }
            else { N.state = ST_LEAF; N.plan = PLAN_NONE; }
            return;
        }
        N.plan = PLAN_BIN2; N.axis[0] = axis; N.axis[1] = axis;
        N.pmin[0] = lo[axis]; N.pdim[0] = dims[axis];
        (void)bins_per_axis;
    }

    __device__ inline uint32_t binOf(const BNode& N, const double* b, int B)
    {
        double c[3];
        for (int k = 0; k < 3; k++) c[k] = (b[3 + k] + b[k]) / 2.0;
        if (N.plan == PLAN_BIN2)
        {
            // getIdx, bvh.cpp:196-201
            const double f = (c[N.axis[0]] - N.pmin[0]) / N.pdim[0];
            int i = (int)floor(f * (double)B);
            return (uint32_t)(i < B - 1 ? i : B - 1);
        }
        if (N.plan == PLAN_BIN4)
        {
            // getIdx, bvh.cpp:318-323; bins[idx.x][idx.y]
            const double f0 = (c[N.axis[0]] - N.pmin[0]) / N.pdim[0], f1 = (c[N.axis[1]] - N.pmin[1]) / N.pdim[1];
            int i0 = (int)floor(f0 * (double)B), i1 = (int)floor(f1 * (double)B);
            i0 = i0 < B - 1 ? i0 : B - 1; i1 = i1 < B - 1 ? i1 : B - 1;
            return (uint32_t)(i0 * B + i1);
        }
        // PLAN_OCT: Octree::insertInOctant (octree.cpp:70-80): x -> 4, y -> 2, z -> 1
        uint32_t oct = 0;
        for (int k = 0; k < 3; k++)
        {
            const double origin = (N.cube[3 + k] + N.cube[k]) / 2.0;
            if (c[k] >= origin) oct |= (4u >> k);
        }
        return oct;
    }

    template <class BinT>
    __device__ inline void binAccumulate(BinT* bin, const double* b)
    {
        atomicAdd(&bin->count, 1ull);
        for (int k = 0; k < 3; k++) { atomicMin(&bin->mn[k], dkey(b[k])); atomicMax(&bin->mx[k], dkey(b[3 + k])); }
    }

    // bins[idx].first++; bins[idx].second.merge(s->BB()) (bvh.cpp:203-209, 325-335)
    __global__ void __launch_bounds__(256) k_bin(const BNode* nodes, const uint32_t* idx, const uint32_t* node_of, BoxSource src,
                                                  uint32_t n, Bin* bins, uint32_t bin_stride, uint32_t* bin_of, int B, uint32_t chunk)
    {
        extern __shared__ unsigned char smem_raw[];
        Bin* sbins = reinterpret_cast<Bin*>(smem_raw);
        for (uint32_t c0 = blockIdx.x * chunk; c0 < n; c0 += gridDim.x * chunk)
        {
            const uint32_t c1 = min(c0 + chunk, n);
            const uint32_t nd_first = node_of[c0], nd_last = node_of[c1 - 1];
            // nodes are contiguous ranges: same node at both ends = one node for the whole chunk
            const bool one_node = nd_first == nd_last;
            if (one_node)
            {
                const BNode& N = nodes[nd_first];
                const bool open = (N.state == ST_ACTIVE) && (N.plan == PLAN_BIN2 || N.plan == PLAN_BIN4 || N.plan == PLAN_OCT);
                if (!open) continue;   // block-uniform; bin_of is only read for nodes split in this round
                const uint32_t nb = N.plan == PLAN_BIN2 ? (uint32_t)B : (N.plan == PLAN_BIN4 ? (uint32_t)(B * B) : 8u);
                for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x)
                {
                    for (int k = 0; k < 3; k++) { sbins[i].mn[k] = KEY_EMPTY_MIN; sbins[i].mx[k] = KEY_EMPTY_MAX; }
                    sbins[i].count = 0;
                }
                __syncthreads();
                for (uint32_t p = c0 + threadIdx.x; p < c1; p += blockDim.x)
                {
                    double b[6];
                    loadBox(src, idx[p], b);
                    const uint32_t bin = binOf(N, b, B);
                    bin_of[p] = bin;
                    binAccumulate(&sbins[bin], b);
                }
                __syncthreads();
                Bin* g = bins + (size_t)N.slot * bin_stride;
                for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x)
                {
                    if (sbins[i].count == 0) continue;
                    atomicAdd(&g[i].count, sbins[i].count);
                    for (int k = 0; k < 3; k++) { atomicMin(&g[i].mn[k], sbins[i].mn[k]); atomicMax(&g[i].mx[k], sbins[i].mx[k]); }
                }
                __syncthreads();
            }
            else
            {
                for (uint32_t p = c0 + threadIdx.x; p < c1; p += blockDim.x)
                {
                    const BNode& N = nodes[node_of[p]];
                    const bool open = (N.state == ST_ACTIVE) && (N.plan == PLAN_BIN2 || N.plan == PLAN_BIN4 || N.plan == PLAN_OCT);
                    if (!open) continue;
                    double b[6];
                    loadBox(src, idx[p], b);
                    const uint32_t bin = binOf(N, b, B);
                    bin_of[p] = bin;
                    binAccumulate(&bins[(size_t)N.slot * bin_stride + bin], b);
                }
            }
        }
    }

    // BVH::arbitrarySplit (bvh.cpp:434-474): child = (position in S) % N; S is ordered by original
    // primitive index, so the position is the rank of the index inside the node. One block per node.
    __global__ void __launch_bounds__(256) k_arb_bin(const BNode* nodes, const uint32_t* active, const uint32_t* idx, BoxSource src,
                                                      Bin* bins, uint32_t bin_stride, uint32_t* bin_of)
    {
        const BNode& N = nodes[active[blockIdx.x]];
        if (N.plan != PLAN_ARB) return;
        __shared__ uint32_t tile[256];
        const uint32_t begin = N.begin, end = N.end;
        for (uint32_t p0 = begin; p0 < end; p0 += blockDim.x)
        {
            const uint32_t p = p0 + threadIdx.x;
            const uint32_t mine = p < end ? idx[p] : 0u;
            uint32_t rank = 0;
            for (uint32_t q0 = begin; q0 < end; q0 += blockDim.x)
            {
                __syncthreads();
                tile[threadIdx.x] = q0 + threadIdx.x < end ? idx[q0 + threadIdx.x] : NONE;
                __syncthreads();
                const uint32_t m = min(blockDim.x, end - q0);
                for (uint32_t t = 0; t < m; t++) rank += tile[t] < mine ? 1u : 0u;
            }
            if (p < end)
            {
                const uint32_t bin = rank % N.arb_n;
                bin_of[p] = bin;
                double b[6];
                loadBox(src, mine, b);
                binAccumulate(&bins[(size_t)N.slot * bin_stride + bin], b);
            }
        }
    }

    struct Group
    {
        long long mn[3], mx[3];
        unsigned long long count;
        __device__ void clear() { for (int k = 0; k < 3; k++) { mn[k] = KEY_EMPTY_MIN; mx[k] = KEY_EMPTY_MAX; } count = 0; }
        __device__ void add(const Bin& b)
        {
            count += b.count;
            for (int k = 0; k < 3; k++) { mn[k] = b.mn[k] < mn[k] ? b.mn[k] : mn[k]; mx[k] = b.mx[k] > mx[k] ? b.mx[k] : mx[k]; }
        }
    };

    __device__ inline void quadGroups(const Bin* sb, int B, int i, int j, Group g[4])
    {
        for (int v = 0; v < 4; v++) g[v].clear();
        for (int x = 0; x < B; x++)
            for (int y = 0; y < B; y++)
            {
                const Bin& b = sb[x * B + y];
                if (b.count == 0) continue;   // merging an empty box and adding 0 changes nothing
                g[(x > i ? 1 : 0) | (y > j ? 2 : 0)].add(b);
            }
    }

    __device__ inline void halfGroups(const Bin* sb, int B, int i, Group g[2])
    {
        g[0].clear(); g[1].clear();
        for (int x = 0; x < B; x++) if (sb[x].count) g[x > i ? 1 : 0].add(sb[x]);
    }

    // One warp per open node: SAH sweep over the bins + child creation.
    constexpr int SPLIT_WARPS = 4;
    __global__ void __launch_bounds__(32 * SPLIT_WARPS) k_split(BNode* nodes, const uint32_t* active, uint32_t n_active, const Bin* bins,
                                                                uint32_t bin_stride, int B, uint32_t round, BuildCounters* counters,
                                                                uint32_t* active_next, uint32_t node_capacity, uint32_t leaf_max,
                                                                uint32_t depth_cap)
    {
        extern __shared__ unsigned char smem_raw[];
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        Bin* sb = reinterpret_cast<Bin*>(smem_raw) + (size_t)warp * bin_stride;
        const uint32_t a = blockIdx.x * SPLIT_WARPS + warp;
        if (a >= n_active) return;
        const uint32_t nd = active[a];
        BNode& N = nodes[nd];
        const uint32_t plan = N.plan;
        if (plan == PLAN_NONE) return;   // became a leaf in k_plan
        const uint32_t nb = plan == PLAN_BIN2 ? (uint32_t)B : (plan == PLAN_BIN4 ? (uint32_t)(B * B) : (plan == PLAN_OCT ? 8u : N.arb_n));
        const Bin* gb = bins + (size_t)N.slot * bin_stride;
        for (uint32_t i = lane; i < nb; i += 32) sb[i] = gb[i];
        __syncwarp();
        const uint32_t size = N.end - N.begin;

        uint32_t n_groups = 0;
        Group g[8];
        if (plan == PLAN_BIN2 || plan == PLAN_BIN4)
        {
            const double node_area = keyArea(N.bb, N.bb + 3);
            const int cands = plan == PLAN_BIN2 ? B - 1 : (B - 1) * (B - 1);
            double best = DBL_MAX;      // min_cost, bvh.cpp:214, 337
            int best_c = 0;             // split_bin = 0
            for (int c = lane; c < cands; c += 32)
            {
                double cost;
                if (plan == PLAN_BIN2)
                {
                    Group h[2];
                    halfGroups(sb, B, c, h);
                    // bvh.cpp:233
                    cost = 1.0 + ((double)h[0].count * keyArea(h[0].mn, h[0].mx) + (double)h[1].count * keyArea(h[1].mn, h[1].mx)) / node_area;
                }
                else
                {
                    Group q[4];
                    quadGroups(sb, B, c / (B - 1), c % (B - 1), q);
                    // bvh.cpp:368-374
                    cost = 0.0;
                    for (int v = 0; v < 4; v++) cost += keyArea(q[v].mn, q[v].mx) * (double)q[v].count;
                    cost = 1.0 + cost / node_area;
                }
                if (cost < best) { best = cost; best_c = c; }
            }
            // first minimum in loop order
            for (int o = 16; o > 0; o >>= 1)
            {
                const double oc = __shfl_xor_sync(FULL, best, o);
                const int oi = __shfl_xor_sync(FULL, best_c, o);
                if (oc < best || (oc == best && oi < best_c)) { best = oc; best_c = oi; }
            }
            if (best > (double)size)
            {
                // bvh.cpp:237-245, 385-393
                if (lane == 0)
                {
                    if (size > MAX_LEAF_SURFACES)
                    {
                        N.state = ST_ARB;
                        active_next[atomicAdd(&counters->n_active_next, 1u)] = nd;
                    }
                    else N.state = ST_LEAF;
                    N.plan = PLAN_NONE;
                }
                return;
            }
            if (plan == PLAN_BIN2)
            {
                halfGroups(sb, B, best_c, g); n_groups = 2;
                if (lane == 0) { N.split[0] = best_c; N.split[1] = 0; }
            }
            else
            {
                quadGroups(sb, B, best_c / (B - 1), best_c % (B - 1), g); n_groups = 4;
                if (lane == 0) { N.split[0] = best_c / (B - 1); N.split[1] = best_c % (B - 1); }
            }
        }
        else
        {
            n_groups = nb;
            for (uint32_t v = 0; v < nb; v++) { g[v].clear(); g[v].add(sb[v]); }
        }

        if (lane != 0) return;
        uint32_t k = 0;
        for (uint32_t v = 0; v < n_groups; v++) k += g[v].count ? 1u : 0u;
        const uint32_t first = atomicAdd(&counters->n_nodes, k);
        if (first + k > node_capacity) { N.state = ST_LEAF; N.plan = PLAN_NONE; return; }   // cannot happen (capacity 2n); keeps memory safe
        if (plan == PLAN_OCT)
        {
            // bvh_node->BB = union of the children's boxes (bvh.cpp:134-162)
            for (int d = 0; d < 3; d++) { N.bb[d] = KEY_EMPTY_MIN; N.bb[3 + d] = KEY_EMPTY_MAX; }
            for (uint32_t v = 0; v < n_groups; v++)
                if (g[v].count)
                    for (int d = 0; d < 3; d++) { N.bb[d] = g[v].mn[d] < N.bb[d] ? g[v].mn[d] : N.bb[d]; N.bb[3 + d] = g[v].mx[d] > N.bb[3 + d] ? g[v].mx[d] : N.bb[3 + d]; }
        }
        uint32_t offset = N.begin, t = 0;
        for (uint32_t v = 0; v < n_groups; v++)
        {
            if (!g[v].count) { N.vchild[v] = NONE; continue; }
            const uint32_t id = first + t;
            BNode& C = nodes[id];
            initNode(C);
            for (int d = 0; d < 3; d++) { C.bb[d] = g[v].mn[d]; C.bb[3 + d] = g[v].mx[d]; }
            C.begin = offset; C.end = offset + (uint32_t)g[v].count; C.cursor = offset;
            C.kind = N.kind;
            C.depth = N.depth + 1;
            C.state = ((C.end - C.begin) <= leaf_max || C.depth >= depth_cap) ? ST_LEAF : ST_ACTIVE;
            if (plan == PLAN_OCT)
            {
                // Octree::insert, octree.cpp:50-60
                for (int d = 0; d < 3; d++)
                {
                    const double centroid = (N.cube[3 + d] + N.cube[d]) / 2.0;
                    const double half = (N.cube[3 + d] - N.cube[d]) / 2.0;
                    const double origin = centroid + half * ((v & (4u >> d)) ? 0.5 : -0.5);
                    const double h = half * 0.5;
                    C.cube[d] = origin - h; C.cube[3 + d] = origin + h;
                }
            }
            if (C.state == ST_ACTIVE) active_next[atomicAdd(&counters->n_active_next, 1u)] = id;
            N.vchild[v] = id;
            offset = C.end; t++;
        }
        N.first_child = first; N.n_children = k;
        N.state = ST_INNER; N.split_round = round;
    }

    __global__ void __launch_bounds__(256) k_scatter(BNode* nodes, const uint32_t* idx, const uint32_t* node_of, const uint32_t* bin_of,
                                                      uint32_t n, uint32_t round, int B, uint32_t* idx_out, uint32_t* node_out)
    {
        const uint32_t stride = gridDim.x * blockDim.x;
        for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += stride)
        {
            const uint32_t p = base + threadIdx.x;
            const bool valid = p < n;
            uint32_t child = NONE, nd = NONE, prim = 0;
            if (valid)
            {
                nd = node_of[p]; prim = idx[p];
                const BNode& N = nodes[nd];
                if (N.state == ST_INNER && N.split_round == round)
                {
                    const uint32_t bin = bin_of[p];
                    uint32_t v;
                    if (N.plan == PLAN_BIN2) v = bin > N.split[0] ? 1u : 0u;                                   // bvh.cpp:250-262
                    else if (N.plan == PLAN_BIN4) v = ((bin / B) > N.split[0] ? 1u : 0u) | ((bin % B) > N.split[1] ? 2u : 0u); // bvh.cpp:401-405
                    else v = bin;
                    child = N.vchild[v];
                }
            }
            const unsigned peers = __match_any_sync(FULL, child);
            if (child != NONE)
            {
                const int leader = __ffs(peers) - 1;
                uint32_t at = 0;
                if ((int)(threadIdx.x & 31) == leader) at = atomicAdd(&nodes[child].cursor, (uint32_t)__popc(peers));
                at = __shfl_sync(peers, at, leader);
                at += __popc(peers & ((1u << (threadIdx.x & 31)) - 1u));
                idx_out[at] = prim; node_out[at] = child;
            }
            else if (valid)
            {
                idx_out[p] = prim; node_out[p] = nd;
            }
        }
    }

    // every node's surface list is in original order: rank-sort each leaf, one warp per node
    __global__ void __launch_bounds__(128) k_sort_leaves(const BNode* nodes, uint32_t n_nodes, const uint32_t* idx, uint32_t* idx_out)
    {
        const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
        if (i >= n_nodes) return;
        const BNode& N = nodes[i];
        if (N.state != ST_LEAF) return;
        const uint32_t begin = N.begin, end = N.end;
        for (uint32_t a = begin + lane; a < end; a += 32)
        {
            const uint32_t v = idx[a];
            uint32_t rank = 0;
            for (uint32_t b = begin; b < end; b++) rank += idx[b] < v ? 1u : 0u;   // indices are unique
            idx_out[begin + rank] = v;
        }
    }

    __global__ void k_subtree(BNode* nodes, uint32_t g0, uint32_t g1)
    {
        const uint32_t i = g0 + blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= g1) return;
        BNode& N = nodes[i];
        uint32_t s = 1;
        if (N.state == ST_INNER) for (uint32_t k = 0; k < N.n_children; k++) s += nodes[N.first_child + k].subtree;
        N.subtree = s;
    }

    // df_idx of BVH::recursiveBuild* (pre-order) and next_sibling of BVH::compact (bvh.cpp:434-456)
    __global__ void k_number(BNode* nodes, uint32_t g0, uint32_t g1)
    {
        const uint32_t i = g0 + blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= g1) return;
        const BNode& N = nodes[i];
        if (N.state != ST_INNER) return;
        uint32_t d = N.df + 1;
        for (uint32_t k = 0; k < N.n_children; k++)
        {
            BNode& C = nodes[N.first_child + k];
            C.df = d;
            d += C.subtree;
            C.next_sibling = k + 1 < N.n_children ? d : 0u;
        }
    }

    __global__ void k_emit(const BNode* nodes, uint32_t n_nodes, double* out_bounds, uint32_t* out_first, uint32_t* out_count, uint32_t* out_next)
    {
        const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= n_nodes) return;
        const BNode& N = nodes[i];
        const uint32_t d = N.df;
        for (int k = 0; k < 6; k++) out_bounds[6 * (size_t)d + k] = keyd(N.bb[k]);
        out_first[d] = N.begin;
        out_count[d] = N.state == ST_LEAF ? N.end - N.begin : 0u;
        out_next[d] = N.next_sibling;
    }

    // LinearOctree<Photon> in the layout k_knn walks (photon.cuh: DeviceOctant), depth-first order:
    // tight box of the contained photons, [start, start+count) = all photons below the octant
    // (LinearOctant::contained_data), children in octant order (linear-octree.cpp:201-244)
    __global__ void k_emit_octants(const BNode* nodes, uint32_t n_nodes, DeviceOctant* out, uint32_t* out_next)
    {
        const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= n_nodes) return;
        const BNode& N = nodes[i];
        DeviceOctant o;
        for (int k = 0; k < 3; k++) { o.bmin[k] = keyd(N.bb[k]); o.bmax[k] = keyd(N.bb[3 + k]); }
        o.start = N.begin; o.count = N.end - N.begin;
        o.leaf = N.state == ST_LEAF ? 1u : 0u;
        o.n_children = N.state == ST_INNER ? N.n_children : 0u;
        for (uint32_t k = 0; k < 8; k++) o.children[k] = k < o.n_children ? nodes[N.first_child + k].df : OCTANT_NULL;
        out[N.df] = o;
        out_next[N.df] = N.next_sibling ? N.next_sibling : OCTANT_NULL;
    }

    __global__ void k_gather_points(const uint32_t* idx, const float4* in, float4* out, uint32_t n)
    {
        for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x)
        {
            const uint32_t src = idx[p];
            out[2 * (size_t)p] = in[2 * (size_t)src]; out[2 * (size_t)p + 1] = in[2 * (size_t)src + 1];
        }
    }

    __global__ void k_gather_lights(const uint32_t* idx, const uint32_t* in, uint32_t* out, uint32_t n)
    {
        for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) out[p] = in[idx[p]];
    }

    // a leaf octant's box is the box of its own photons; for a single-leaf tree nobody has binned them
    __global__ void k_root_leaf_box(BNode* nodes, const float4* points, uint32_t n)
    {
        if (blockIdx.x || threadIdx.x) return;
        BNode& N = nodes[0];
        for (int k = 0; k < 3; k++) { N.bb[k] = KEY_EMPTY_MIN; N.bb[3 + k] = KEY_EMPTY_MAX; }
        for (uint32_t i = 0; i < n; i++)
        {
            const float4 p0 = points[2 * (size_t)i], p1 = points[2 * (size_t)i + 1];
            const long long k3[3] = {dkey((double)p0.w), dkey((double)p1.x), dkey((double)p1.y)};
            for (int k = 0; k < 3; k++) { N.bb[k] = k3[k] < N.bb[k] ? k3[k] : N.bb[k]; N.bb[3 + k] = k3[k] > N.bb[3 + k] ? k3[k] : N.bb[3 + k]; }
        }
    }

    struct DeviceBuffers
    {
        std::vector<void*> allocs;
        ~DeviceBuffers() { for (void* p : allocs) cudaFree(p); }
        template <class T> T* get(size_t count)
        {
            void* p = nullptr;
            if (cudaMalloc(&p, count * sizeof(T) + 16) != cudaSuccess) return nullptr;
            allocs.push_back(p);
            return static_cast<T*>(p);
        }
    };

    struct CoreResult
    {
        BNode* d_nodes = nullptr;
        uint32_t* d_idx = nullptr;     // final primitive order
        uint32_t n_nodes = 0, rounds = 0, launches = 0;
    };
}

#define BK(call)                                                                      \
    do {                                                                              \
        cudaError_t e_ = (call);                                                      \
        if (e_ != cudaSuccess) { error = std::string(#call) + ": " + cudaGetErrorString(e_); return MCRT_ERR_CUDA; } \
    } while (0)

// The build rounds + leaf sort + depth-first numbering shared by the BVH and the photon octree.
static int buildCore(DeviceBuffers& mem, BoxSource src, uint32_t n, const BNode& root, bool octree, int B, uint32_t bin_stride,
                     uint32_t leaf_max, uint32_t depth_cap, uint32_t node_capacity, int sm_count, cudaStream_t s, cudaEvent_t ev_start,
                     CoreResult& res, std::string& error)
{
    const uint32_t max_active = n / (leaf_max + 1) + 2;
    uint32_t* d_idx[2] = {mem.get<uint32_t>(n), mem.get<uint32_t>(n)};
    uint32_t* d_node_of[2] = {mem.get<uint32_t>(n), mem.get<uint32_t>(n)};
    uint32_t* d_bin_of = mem.get<uint32_t>(n);
    BNode* d_nodes = mem.get<BNode>(node_capacity);
    uint32_t* d_active[2] = {mem.get<uint32_t>(max_active), mem.get<uint32_t>(max_active)};
    Bin* d_bins = mem.get<Bin>((size_t)max_active * bin_stride);
    BuildCounters* d_counters = mem.get<BuildCounters>(1);
    if (!d_idx[0] || !d_idx[1] || !d_node_of[0] || !d_node_of[1] || !d_bin_of || !d_nodes || !d_active[0] || !d_active[1] || !d_bins || !d_counters)
    { error = "hierarchy build: out of device memory"; return MCRT_ERR_CUDA; }

    BK(cudaMemcpyAsync(d_nodes, &root, sizeof(root), cudaMemcpyHostToDevice, s));
    const int grid = sm_count * 8;
    uint32_t launches = 0;
    BK(cudaEventRecord(ev_start, s));   // allocations and the input copy stay outside the reported build time
    k_init<<<grid, 256, 0, s>>>(d_idx[0], d_node_of[0], n); launches++;

    const uint32_t zero_active = 0;
    BuildCounters hc; hc.n_nodes = 1; hc.n_active_next = 0; hc._a = hc._b = 0;
    BK(cudaMemcpyAsync(d_counters, &hc, sizeof(hc), cudaMemcpyHostToDevice, s));
    BK(cudaMemcpyAsync(d_active[0], &zero_active, sizeof(uint32_t), cudaMemcpyHostToDevice, s));

    const size_t split_smem = (size_t)SPLIT_WARPS * bin_stride * sizeof(Bin);
    const size_t bin_smem = (size_t)bin_stride * sizeof(Bin);
    if (split_smem > 48 * 1024) BK(cudaFuncSetAttribute(k_split, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)split_smem));
    // k_bin chunk: every block handles contiguous chunks, large enough to amortise the shared bins
    const uint32_t chunk = 4096;

    std::vector<uint32_t> gen;   // node id boundaries per round
    gen.push_back(0); gen.push_back(1);
    uint32_t n_active = root.state == ST_ACTIVE ? 1u : 0u, round = 0;
    int cur = 0;
    while (n_active > 0)
    {
        if (n_active > max_active) { error = "hierarchy build: internal error (open node list overflow)"; return MCRT_ERR_CUDA; }
        const size_t n_bins = (size_t)n_active * bin_stride;
        k_init_bins<<<(unsigned)std::min<size_t>((n_bins + 255) / 256, (size_t)grid), 256, 0, s>>>(d_bins, n_bins); launches++;
        if (!octree) { k_extent<<<grid, 256, 0, s>>>(d_nodes, d_idx[cur], d_node_of[cur], src, n); launches++; }
        k_plan<<<(n_active + 127) / 128, 128, 0, s>>>(d_nodes, d_active[cur], n_active, B);
        k_bin<<<grid, 256, bin_smem, s>>>(d_nodes, d_idx[cur], d_node_of[cur], src, n, d_bins, bin_stride, d_bin_of, B, chunk);
        if (!octree) { k_arb_bin<<<n_active, 256, 0, s>>>(d_nodes, d_active[cur], d_idx[cur], src, d_bins, bin_stride, d_bin_of); launches++; }
        k_split<<<(n_active + SPLIT_WARPS - 1) / SPLIT_WARPS, 32 * SPLIT_WARPS, split_smem, s>>>(
            d_nodes, d_active[cur], n_active, d_bins, bin_stride, B, round, d_counters, d_active[cur ^ 1], node_capacity, leaf_max, depth_cap);
        k_scatter<<<grid, 256, 0, s>>>(d_nodes, d_idx[cur], d_node_of[cur], d_bin_of, n, round, B, d_idx[cur ^ 1], d_node_of[cur ^ 1]);
        launches += 4;
        BK(cudaMemcpyAsync(&hc, d_counters, sizeof(hc), cudaMemcpyDeviceToHost, s));
        BK(cudaStreamSynchronize(s));
        BK(cudaGetLastError());
        if (hc.n_nodes > node_capacity) { error = "hierarchy build: node pool overflow (degenerate input: coincident points?)"; return MCRT_ERR_UNSUPPORTED; }
        n_active = hc.n_active_next;
        gen.push_back(hc.n_nodes);
        hc.n_active_next = 0;
        BK(cudaMemcpyAsync(d_counters, &hc, sizeof(hc), cudaMemcpyHostToDevice, s));
        cur ^= 1;
        round++;
        if (round > 4096) { error = "hierarchy build does not terminate (coincident centroids?)"; return MCRT_ERR_UNSUPPORTED; }
    }
    const uint32_t n_nodes = hc.n_nodes;

    k_sort_leaves<<<(unsigned)(((size_t)n_nodes * 32 + 127) / 128), 128, 0, s>>>(d_nodes, n_nodes, d_idx[cur], d_idx[cur ^ 1]); launches++;
    cur ^= 1;
    for (size_t g = gen.size() - 1; g-- > 0;)
        if (gen[g + 1] > gen[g]) { k_subtree<<<(gen[g + 1] - gen[g] + 127) / 128, 128, 0, s>>>(d_nodes, gen[g], gen[g + 1]); launches++; }
    for (size_t g = 0; g + 1 < gen.size(); g++)
        if (gen[g + 1] > gen[g]) { k_number<<<(gen[g + 1] - gen[g] + 127) / 128, 128, 0, s>>>(d_nodes, gen[g], gen[g + 1]); launches++; }
    res.d_nodes = d_nodes; res.d_idx = d_idx[cur]; res.n_nodes = n_nodes; res.rounds = round; res.launches = launches;
    return MCRT_OK;
}

static void initRoot(BNode& root, uint32_t n, uint32_t kind, uint32_t leaf_max)
{
    std::memset(&root, 0, sizeof(root));
    for (int k = 0; k < 3; k++) { root.bb[k] = KEY_EMPTY_MIN; root.bb[3 + k] = KEY_EMPTY_MAX; root.cext[k] = KEY_EMPTY_MIN; root.cext[3 + k] = KEY_EMPTY_MAX; }
    root.begin = 0; root.end = n; root.cursor = 0;
    root.kind = kind;
    root.state = n <= leaf_max ? ST_LEAF : ST_ACTIVE;
    root.split_round = NONE; root.first_child = NONE; root.subtree = 1;
    for (int k = 0; k < 8; k++) root.vchild[k] = NONE;
}

int buildBvhOnDevice(const double* prim_bounds_host, uint32_t n, const double scene_bounds[6], int type, int bins_per_axis,
                     int sm_count, cudaStream_t s, BvhBuildResult& out, std::string& error)
{
    if (!prim_bounds_host || n == 0 || !scene_bounds) { error = "mcrt_bvh_build: no primitives"; return MCRT_ERR_INVALID; }
    if (type != MCRT_BVH_OCTREE && type != MCRT_BVH_BINARY_SAH && type != MCRT_BVH_QUATERNARY_SAH) { error = "mcrt_bvh_build: unknown type"; return MCRT_ERR_INVALID; }
    int B = bins_per_axis;
    if (B <= 0) B = type == MCRT_BVH_BINARY_SAH ? 16 : 8;   // bvh.cpp:29,36
    uint32_t bin_stride = type == MCRT_BVH_OCTREE ? 8u : (type == MCRT_BVH_BINARY_SAH ? (uint32_t)B : (uint32_t)(B * B));
    if (type == MCRT_BVH_QUATERNARY_SAH && bin_stride < (uint32_t)B) bin_stride = B;   // binary fall-back inside a quaternary build
    if (bin_stride < 4) bin_stride = 4;                                                 // arbitrarySplit(4)
    if (B < 2 || bin_stride > 256) { error = "mcrt_bvh_build: bins_per_axis out of range (2..256 binary, 2..16 quaternary)"; return MCRT_ERR_UNSUPPORTED; }

    DeviceBuffers mem;
    // SAH splits always have two non-empty sides (<= 2n-1 nodes); octree cells can chain single children
    const uint32_t node_capacity = (type == MCRT_BVH_OCTREE ? 4u : 2u) * n + 64u;
    double* d_bounds = mem.get<double>(6 * (size_t)n);
    if (!d_bounds) { error = "mcrt_bvh_build: out of device memory"; return MCRT_ERR_CUDA; }
    BK(cudaMemcpyAsync(d_bounds, prim_bounds_host, 6 * (size_t)n * sizeof(double), cudaMemcpyHostToDevice, s));

    // root (bvh.cpp:19-20, 31-32, 38-39, 46-49)
    BNode root;
    initRoot(root, n, type == MCRT_BVH_OCTREE ? KIND_OCT : (type == MCRT_BVH_BINARY_SAH ? KIND_BIN : KIND_QUAT), LEAF_SURFACES);
    for (int k = 0; k < 3; k++) { root.bb[k] = dkey(scene_bounds[k]); root.bb[3 + k] = dkey(scene_bounds[3 + k]); }
    if (type == MCRT_BVH_OCTREE)
    {
        const double dims[3] = {scene_bounds[3] - scene_bounds[0], scene_bounds[4] - scene_bounds[1], scene_bounds[5] - scene_bounds[2]};
        double m = dims[0] > dims[1] ? dims[0] : dims[1]; m = m > dims[2] ? m : dims[2];   // compMax
        const double half_max = m / 2.0;
        for (int k = 0; k < 3; k++)
        {
            const double c = (scene_bounds[3 + k] + scene_bounds[k]) / 2.0;
            root.cube[k] = c - half_max; root.cube[3 + k] = c + half_max;
        }
        if (root.state == ST_LEAF)
        {
            // a single leaf: its box is the union of the primitive boxes
            for (int k = 0; k < 3; k++) { root.bb[k] = KEY_EMPTY_MIN; root.bb[3 + k] = KEY_EMPTY_MAX; }
            for (uint32_t i = 0; i < n; i++)
                for (int k = 0; k < 3; k++)
                {
                    const long long lo = dkey(prim_bounds_host[6 * (size_t)i + k]), hi = dkey(prim_bounds_host[6 * (size_t)i + 3 + k]);
                    if (lo < root.bb[k]) root.bb[k] = lo;
                    if (hi > root.bb[3 + k]) root.bb[3 + k] = hi;
                }
        }
    }

    cudaEvent_t ev0, ev1;
    BK(cudaEventCreate(&ev0)); BK(cudaEventCreate(&ev1));
    struct EventGuard { cudaEvent_t a, b; ~EventGuard() { cudaEventDestroy(a); cudaEventDestroy(b); } } guard{ev0, ev1};
    double* d_out_bounds = mem.get<double>(6 * (size_t)node_capacity);
    uint32_t* d_out_first = mem.get<uint32_t>(node_capacity);
    uint32_t* d_out_count = mem.get<uint32_t>(node_capacity);
    uint32_t* d_out_next = mem.get<uint32_t>(node_capacity);
    if (!d_out_bounds || !d_out_first || !d_out_count || !d_out_next) { error = "mcrt_bvh_build: out of device memory"; return MCRT_ERR_CUDA; }
    CoreResult core;
    BoxSource src; src.bounds = d_bounds; src.points = nullptr;
    const int rc = buildCore(mem, src, n, root, type == MCRT_BVH_OCTREE, B, bin_stride, LEAF_SURFACES, 0xFFFFFFFFu, node_capacity, sm_count, s, ev0, core, error);
    if (rc != MCRT_OK) return rc;
    const uint32_t n_nodes = core.n_nodes;

    k_emit<<<(n_nodes + 127) / 128, 128, 0, s>>>(core.d_nodes, n_nodes, d_out_bounds, d_out_first, d_out_count, d_out_next);
    BK(cudaEventRecord(ev1, s));

    out.node_bounds.resize(6 * (size_t)n_nodes);
    out.node_first_prim.resize(n_nodes); out.node_prim_count.resize(n_nodes); out.node_next_sibling.resize(n_nodes);
    out.prim_order.resize(n);
    BK(cudaMemcpyAsync(out.node_bounds.data(), d_out_bounds, out.node_bounds.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    BK(cudaMemcpyAsync(out.node_first_prim.data(), d_out_first, n_nodes * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    BK(cudaMemcpyAsync(out.node_prim_count.data(), d_out_count, n_nodes * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    BK(cudaMemcpyAsync(out.node_next_sibling.data(), d_out_next, n_nodes * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    BK(cudaMemcpyAsync(out.prim_order.data(), core.d_idx, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    BK(cudaStreamSynchronize(s));
    BK(cudaGetLastError());
    float ms = 0.f;
    BK(cudaEventElapsedTime(&ms, ev0, ev1));
    out.gpu_ms = ms;
    out.iterations = core.rounds;
    out.kernel_launches = core.launches + 1;
    return MCRT_OK;
}

// Octree<Photon> insertion + LinearOctree::compact (octree.cpp:34-81, linear-octree.cpp:201-244) on
// photons already in device memory: the same rounds with 8 bins = octants of the node's cell, a
// node is internal iff it holds more than max_node_data photons (and sits above level 64, the
// guard against coincident photons; the reference would recurse forever), boxes = tight boxes of the
// contained photons.
int buildPhotonOctreeOnDevice(const float4* d_photons, uint32_t n, const double cell[6], uint32_t max_node_data, int sm_count,
                              cudaStream_t s, std::vector<void*>& keep, PhotonOctreeDevice& out, std::string& error,
                              const uint32_t* d_lights, const uint32_t* d_lpe_states)
{
    out = PhotonOctreeDevice();
    if (n == 0) return MCRT_OK;
    if (!d_photons || !cell || max_node_data == 0) { error = "photon octree: invalid arguments"; return MCRT_ERR_INVALID; }
    DeviceBuffers mem;
    // Node pool: real maps have ~n / (max_node_data / 4) octants (water_caustics: 12.3 M photons, 186 k
    // octants at 200 per leaf); 16x that plus slack, never more than the 4n + 64 of the BVH octree.
    // Exhausting it (adversarial input) fails the build with an error, it does not corrupt memory.
    const uint64_t cap64 = std::min<uint64_t>(4ull * n + 64, 16ull * n / std::max<uint32_t>(1u, max_node_data / 4u) + 65536ull);
    const uint32_t node_capacity = (uint32_t)std::min<uint64_t>(cap64, 0x7FFFFFFFull);
    BNode root;
    initRoot(root, n, KIND_OCT, max_node_data);
    for (int k = 0; k < 6; k++) root.cube[k] = cell[k];

    cudaEvent_t ev0, ev1;
    BK(cudaEventCreate(&ev0)); BK(cudaEventCreate(&ev1));
    struct EventGuard { cudaEvent_t a, b; ~EventGuard() { cudaEventDestroy(a); cudaEventDestroy(b); } } guard{ev0, ev1};
    CoreResult core;
    BoxSource src; src.bounds = nullptr; src.points = d_photons;
    const int rc = buildCore(mem, src, n, root, true, 8, 8, max_node_data, 64, node_capacity, sm_count, s, ev0, core, error);
    if (rc != MCRT_OK) return rc;
    if (core.n_nodes == 1) k_root_leaf_box<<<1, 32, 0, s>>>(core.d_nodes, d_photons, n);

    DeviceOctant* d_oct = nullptr; uint32_t* d_next = nullptr; float4* d_sorted = nullptr;
    if (cudaMalloc((void**)&d_oct, (size_t)core.n_nodes * sizeof(DeviceOctant)) != cudaSuccess ||
        cudaMalloc((void**)&d_next, (size_t)core.n_nodes * sizeof(uint32_t)) != cudaSuccess ||
        cudaMalloc((void**)&d_sorted, (size_t)n * 2 * sizeof(float4)) != cudaSuccess)
    {
        cudaFree(d_oct); cudaFree(d_next); cudaFree(d_sorted);
        error = "photon octree: out of device memory"; return MCRT_ERR_CUDA;
    }
    keep.push_back(d_oct); keep.push_back(d_next); keep.push_back(d_sorted);
    uint32_t* d_sorted_lights = nullptr;
    if (d_lights)
    {
        if (cudaMalloc((void**)&d_sorted_lights, (size_t)n * sizeof(uint32_t)) != cudaSuccess)
        { error = "photon octree: out of device memory"; return MCRT_ERR_CUDA; }
        keep.push_back(d_sorted_lights);
    }
    uint32_t* d_sorted_states = nullptr;
    if (d_lpe_states)
    {
        if (cudaMalloc((void**)&d_sorted_states, (size_t)n * sizeof(uint32_t)) != cudaSuccess)
        { error = "photon octree: out of device memory"; return MCRT_ERR_CUDA; }
        keep.push_back(d_sorted_states);
    }
    k_emit_octants<<<(core.n_nodes + 127) / 128, 128, 0, s>>>(core.d_nodes, core.n_nodes, d_oct, d_next);
    k_gather_points<<<sm_count * 8, 256, 0, s>>>(core.d_idx, d_photons, d_sorted, n);
    if (d_lights) k_gather_lights<<<sm_count * 8, 256, 0, s>>>(core.d_idx, d_lights, d_sorted_lights, n);
    if (d_lpe_states) k_gather_lights<<<sm_count * 8, 256, 0, s>>>(core.d_idx, d_lpe_states, d_sorted_states, n);
    BK(cudaEventRecord(ev1, s));
    BK(cudaStreamSynchronize(s));
    BK(cudaGetLastError());
    float ms = 0.f;
    BK(cudaEventElapsedTime(&ms, ev0, ev1));
    out.octants = d_oct; out.next_sibling = d_next; out.photons = d_sorted; out.lights = d_sorted_lights; out.lpe_states = d_sorted_states;
    out.n_octants = core.n_nodes; out.n_photons = n; out.gpu_ms = ms; out.rounds = core.rounds;
    return MCRT_OK;
}
}
