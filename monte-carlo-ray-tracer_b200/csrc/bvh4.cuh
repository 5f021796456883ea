// Closest-hit traversal of parity mode: order-free search + exact-order fallback.
//
// What has to be reproduced is the *result* of Scene::intersect (source/scene/scene.cpp:151-176,
// source/bvh/bvh.cpp:80-129): the primitive with the smallest t, t/u/v computed by the reference's
// float64 primitive tests. Which primitive that is depends on the order in which the reference walks
// its tree only when two candidates compete within rounding distance of each other (ties on shared
// edges / coincident geometry, or a node whose entry distance rounds across the current best t).
// So the hot path does not replay the reference's priority queue:
//
//   1. traverseFast walks a 4-wide BVH (the reference's tree collapsed to <= 4 children per node by
//      mcrt_scene_upload; one 128-byte node = one cache line: 6 float4 of child planes + 4 child
//      references) depth-first, nearest child first, with a short (reference, entry distance) stack.
//      Boxes are float32, rounded outwards, and tested with margins that make the test conservative
//      for the float64 ray (FastRay below) - the boxes only decide which primitives get *tested*.
//      Primitives are tested with exactly the reference's float64 arithmetic (intersectTriangle /
//      intersectSphere / intersectQuadric, compiled with --fmad=false), so t, u, v of the winner are
//      bit-identical to the reference's.
//   2. Nodes are pruned only when their (lower-bounded) entry distance exceeds best.t + 2*delta, and
//      the search records the second-smallest hit distance. If that is within delta of the smallest
//      (delta = 1e-6 * t + 1e-12 * scene scale), the ray is *ambiguous*: the answer may depend on the
//      visiting order, and the ray is re-traced by traverseReferenceOrder (intersect.cuh), the
//      replay of the reference's best-first order with its binary-heap discipline. Otherwise the
//      smallest hit is separated from every other candidate by far more than the rounding of the
//      reference's slab and primitive tests, and the reference returns the same primitive whatever
//      its order.
//   mcrt_set_option("exact_traversal", 1) sends every ray down the replay; the parity tests compare
//   the two paths ray by ray (tests/test_gpu_parity.py::test_fast_traversal_equals_reference_order).
#pragma once

#include "intersect.cuh"

#ifndef MCRT_FAST_STACK
#define MCRT_FAST_STACK 40
#endif
#ifndef MCRT_SPECULATIVE              // 1: a lane holding a leaf keeps walking inner nodes until its warp-mates hold one too
#define MCRT_SPECULATIVE 0
#endif
#ifndef MCRT_FAST_SMEM_STACK          // entries of the search stack kept in shared memory (per thread); the rest is local memory.
#define MCRT_FAST_SMEM_STACK 0       // 0: the all-local stack (the L1 keeps the hot top of the local stacks, and the shared-memory form adds
#endif                               // address arithmetic and a branch per push / pop). Kept as a knob.

namespace mcrt
{
    constexpr uint32_t BVH4_LEAF = 0x80000000u;
    constexpr uint32_t BVH4_MAX_PRIMS = 1u << 23;     // leaf reference: 23 bits first primitive, 8 bits count
    constexpr int FAST_STACK = MCRT_FAST_STACK;
    constexpr int FAST_SMEM_STACK = MCRT_FAST_SMEM_STACK;
    constexpr int FAST_LOCAL_STACK = FAST_STACK - FAST_SMEM_STACK;
    // dynamic shared memory of a kernel that runs the search: FAST_SMEM_STACK entries of 8 bytes per thread, entry e of
    // thread t at [e * blockDim.x + t] (conflict-free); 0 by default (see above)
    inline size_t fastStackSharedBytes(int block_threads) { return (size_t)FAST_SMEM_STACK * block_threads * sizeof(uint2); }

    // children c = 0..3: box [lo[k][c], hi[k][c]] on axis k; child[c] = 0 (empty), inner node index
    // (>= 1: the root is node 0 and nobody's child) or BVH4_LEAF | first_prim << 8 | count
    struct alignas(16) Bvh4Node
    {
        float lo[3][4];
        float hi[3][4];
        uint32_t child[4];
        uint32_t _pad[4];
    };
    static_assert(sizeof(Bvh4Node) == 128, "one cache line per node");

    // float32 view of a float64 ray for the box tests. t_k = b * inv_d_k - o_k * inv_d_k with
    // inv_d = 1/d in float (|d_k| clamped away from 0 so that no inf/NaN arises). Rounding o, d to
    // float and evaluating in float moves each plane distance by at most a few 2^-24 of |o_k inv_d_k|
    // + |t|; the near-plane term is therefore lowered and the far-plane term raised by 2^-19 |o_k
    // inv_d_k|, and the interval ends are scaled by (1 -+ 2^-18) in the comparison: a box the exact
    // ray touches is never missed.
    struct FastRay
    {
        float idx, idy, idz;          // 1 / d
        float onx, ony, onz;          // o * inv_d raised  (subtracted on the near planes)
        float ofx, ofy, ofz;          // o * inv_d lowered (subtracted on the far planes)
        uint32_t near_row[3];         // float4 row offset of the near plane inside the node: lo (0) or hi (3)
    };

    MCRT_D FastRay makeFastRay(const V3<double>& o, const V3<double>& d)
    {
        FastRay r;
        auto inv = [](double v) { float f = (float)v; if (!(fabsf(f) >= 1e-18f)) f = copysignf(1e-18f, f); return 1.0f / f; };
        r.idx = inv(d.x); r.idy = inv(d.y); r.idz = inv(d.z);
        const float ox = (float)o.x * r.idx, oy = (float)o.y * r.idy, oz = (float)o.z * r.idz;
        const float mx = fabsf(ox) * 1.9073486e-6f, my = fabsf(oy) * 1.9073486e-6f, mz = fabsf(oz) * 1.9073486e-6f; // 2^-19
        r.onx = ox + mx; r.ony = oy + my; r.onz = oz + mz;
        r.ofx = ox - mx; r.ofy = oy - my; r.ofz = oz - mz;
        r.near_row[0] = r.idx < 0.0f ? 3u : 0u;
        r.near_row[1] = r.idy < 0.0f ? 3u : 0u;
        r.near_row[2] = r.idz < 0.0f ? 3u : 0u;
        return r;
    }

    // One primitive record of `geom` (sc.geom: ordered primitives, sc.bvh4_geom: leaf references) against the ray with the
    // reference's float64 arithmetic (no acceptance rule)
    template <int PRIMS, class R>
    MCRT_D bool intersectPrim(const DeviceScene<R>& sc, const V4<R>* __restrict__ geom, uint32_t prim, const RayQ<R>& ray, R& t, R& u, R& v, bool& is_triangle)
    {
        const V4<R> g0 = geom[3 * prim + 0];
        const uint32_t type = PRIMS == PRIMS_TRI ? (uint32_t)PRIM_TRIANGLE : (uint32_t)g0.w;
        u = R(0); v = R(0);
        is_triangle = type == PRIM_TRIANGLE;
        if (type == PRIM_TRIANGLE)
        {
            const V4<R> g1 = geom[3 * prim + 1];
            const V4<R> g2 = geom[3 * prim + 2];
            return intersectTriangle(g0, g1, g2, ray, t, u, v);
        }
        else if (PRIMS == PRIMS_TRI_SPHERE || type == PRIM_SPHERE)
        {
            const V4<R> g1 = geom[3 * prim + 1];
            return intersectSphere(g0, g1, ray, t);
        }
        else
        {
            return intersectQuadric(sc.quadrics[(uint32_t)g0.x], ray, t);
        }
    }

    // distance below which two hits count as competing (see the header)
    MCRT_D double ambiguityDelta(double t, double scene_scale) { return 1e-6 * t + 1e-12 * scene_scale; }

    // Degenerate rays. Where a ray runs exactly along a box plane, through a vertex or along an edge, the reference's float64 slab test
    // decides by rounding - or by NaN: 0 * inf for a zero direction component - whether a box, and with it a primitive the ray does
    // touch, is reached at all; the conservative float boxes of the search never miss such a primitive, so there the two can differ
    // although no second candidate is near. Such rays are handed to the replay as well: a direction component of (nearly) zero, or a
    // triangle hit within 1e-9 (scaled with distance) of the triangle's boundary. Measure-zero for rays a renderer generates, but
    // mcrt_trace_closest takes the caller's rays. tests/test_fast_search_cpu.py::test_degenerate_rays_* (CPU restatement, 1.25 M
    // adversarial rays: no unflagged answer differs from the reference-order answer).
    MCRT_D bool degenerateDirection(const V3<double>& d)
    {
        return fabs(d.x) < 1e-12 || fabs(d.y) < 1e-12 || fabs(d.z) < 1e-12;
    }
    MCRT_D bool onTriangleBoundary(double u, double v, double t, double scene_scale)
    {
        const double e = 1e-9 * fmax(1.0, t / scene_scale);
        return u < e || v < e || u + v > 1.0 - e;
    }

    // The search as a resumable state: begin(), then step() until it returns false. One step = walk down
    // through inner nodes to the next leaf, test its primitives, pop the next pending subtree.
    // OCC (occlusion query of next-event estimation, integrator.cpp:68-86): the caller only needs to know
    // whether `target` (the sampled light primitive) is the closest hit. The target is tested directly -
    // same float64 test, same t as the reference computes for it - and the tree is searched only for
    // something *in front* of it: the limit is known from the start and the search stops at the first
    // occluder. A hit within delta of the target's t (either side) is a tie the reference's visiting order
    // decides: such rays are replayed like ambiguous closest hits.
    template <int PRIMS, bool OCC = false> struct FastSearch
    {
        Hit<double> best;
        double second_t;       // second-smallest hit distance seen (competitor of best.t)
        float limit;           // prune subtrees that start beyond this: best.t + 2 delta, rounded up
        int sp;
        uint32_t cur;          // node index or leaf reference being visited
        FastRay fr;
        uint2 lstack[FAST_LOCAL_STACK > 0 ? FAST_LOCAL_STACK : 1];   // (child reference, lower bound of its entry distance as float bits)
        uint2* sstack;         // this thread's column of the shared-memory part of the stack
        uint32_t target;       // OCC: the primitive whose visibility is asked
        uint32_t verdict;      // OCC: 0 target visible so far, 1 occluded, 2 tie -> replay
        bool degenerate;       // the ray or its winning hit is degenerate (see degenerateDirection / onTriangleBoundary): replay

        // -> false: the ray does not hit the target at all (nothing to search)
        MCRT_D bool beginOcclusion(const DeviceScene<double>& sc, const RayQ<double>& ray, uint32_t target_prim, TraceCounters& cnt)
        {
            best.u = 0.0; best.v = 0.0; best.interpolate = 0; best.prim = NO_PRIM; best.t = Consts<double>::MAXV;
            second_t = Consts<double>::MAXV;
            target = target_prim; verdict = 0u;
            sp = 0; cur = 0;
            attach();
            double t, u, v;
            bool is_tri;
            cnt.prim_tests++;
            if (!intersectPrim<PRIMS>(sc, sc.geom, target_prim, ray, t, u, v, is_tri)) return false;
            best.t = t; best.u = u; best.v = v; best.prim = target_prim;
            degenerate = degenerateDirection(ray.d) || (is_tri && onTriangleBoundary(u, v, t, (double)sc.scene_scale));
            if (degenerate) { verdict = 2u; return true; }     // step() is not entered: see traceManyFast / traceVisible
            limit = __double2float_ru(t + 2.0 * ambiguityDelta(t, (double)sc.scene_scale));
            fr = makeFastRay(ray.o, ray.d);
            return true;
        }

        MCRT_D void begin(const RayQ<double>& ray)
        {
            best.t = Consts<double>::MAXV; best.u = 0.0; best.v = 0.0; best.prim = NO_PRIM; best.interpolate = 0;
            second_t = Consts<double>::MAXV;
            limit = __int_as_float(0x7f800000);   // +inf until something is hit
            sp = 0;
            cur = 0;                              // node 0 = root
            degenerate = degenerateDirection(ray.d);
            attach();
            fr = makeFastRay(ray.o, ray.d);
        }

        MCRT_D void attach()
        {
            extern __shared__ uint2 fast_stack_smem[];
            sstack = fast_stack_smem + threadIdx.x;
        }

        // A full stack drops the entry and hands the ray to the replay, which answers in the reference's order with a heap of its own:
        // the closest hit is marked degenerate, the occlusion query a tie unless it still finds an occluder (which answers it anyway).
        MCRT_D void push(uint32_t ref, uint32_t tn_bits)
        {
            if (sp < FAST_SMEM_STACK) sstack[sp * blockDim.x] = make_uint2(ref, tn_bits);
            else if (sp < FAST_STACK) lstack[sp - FAST_SMEM_STACK] = make_uint2(ref, tn_bits);
            else { if constexpr (OCC) verdict = 2u; else degenerate = true; return; }
            sp++;
        }

        MCRT_D bool pop()
        {
            while (sp > 0)
            {
                --sp;
                const uint2 e = sp < FAST_SMEM_STACK ? sstack[sp * blockDim.x] : lstack[sp - FAST_SMEM_STACK];
                if (__uint_as_float(e.y) <= limit) { cur = e.x; return true; }
            }
            return false;
        }

        // One inner node: tests its four child boxes, pushes the far hits, continues with the nearest (or with the next
        // pending entry when nothing is hit). -> false: nothing left to visit.
        MCRT_D bool visitNode(const DeviceScene<double>& sc, TraceCounters& cnt)
        {
            const float4* __restrict__ n = reinterpret_cast<const float4*>(sc.bvh4) + 8 * (size_t)cur;
            // float4 rows of a node: lo.x lo.y lo.z hi.x hi.y hi.z; the near plane of axis k is lo for d_k >= 0
            const float4 bnx = __ldg(n + 0 + fr.near_row[0]), bny = __ldg(n + 1 + fr.near_row[1]), bnz = __ldg(n + 2 + fr.near_row[2]);
            const float4 bfx = __ldg(n + 3 - fr.near_row[0]), bfy = __ldg(n + 4 - fr.near_row[1]), bfz = __ldg(n + 5 - fr.near_row[2]);
            const uint4 ch = __ldg(reinterpret_cast<const uint4*>(n + 6));
            cnt.box_tests += 4;

            #define MCRT_SLAB(C, REF, SLOT)                                                                   \
                uint32_t key##SLOT;                                                                           \
                {                                                                                             \
                    const float tn = fmaxf(fmaxf(__fmaf_rn(bnx.C, fr.idx, -fr.onx), __fmaf_rn(bny.C, fr.idy, -fr.ony)), \
                                           fmaxf(__fmaf_rn(bnz.C, fr.idz, -fr.onz), 0.0f)) * 0.99999619f;    \
                    const float tf = fminf(fminf(__fmaf_rn(bfx.C, fr.idx, -fr.ofx), __fmaf_rn(bfy.C, fr.idy, -fr.ofy)), \
                                           __fmaf_rn(bfz.C, fr.idz, -fr.ofz)) * 1.00000381f;                  \
                    const bool hit = (REF) != 0u && tn <= tf && tn <= limit;                                   \
                    key##SLOT = hit ? ((__float_as_uint(tn) & 0x7FFFFFFCu) | SLOT##u) : 0xFFFFFFFFu;           \
                }
            MCRT_SLAB(x, ch.x, 0)
            MCRT_SLAB(y, ch.y, 1)
            MCRT_SLAB(z, ch.z, 2)
            MCRT_SLAB(w, ch.w, 3)
            #undef MCRT_SLAB

            // sort the four keys ascending (entry distance in the high 30 bits, slot in the low 2)
            #define MCRT_CE(A, B) { const uint32_t lo_ = min(A, B); B = max(A, B); A = lo_; }
            MCRT_CE(key0, key1) MCRT_CE(key2, key3) MCRT_CE(key0, key2) MCRT_CE(key1, key3) MCRT_CE(key1, key2)
            #undef MCRT_CE
            auto refOf = [&](uint32_t key) { const uint32_t s = key & 3u; return s == 0u ? ch.x : (s == 1u ? ch.y : (s == 2u ? ch.z : ch.w)); };

            if (key0 == 0xFFFFFFFFu) return pop();     // nothing hit: next pending entry, if any
            // far children first, so the nearest pending one is on top
            if (key3 != 0xFFFFFFFFu) push(refOf(key3), key3 & ~3u);
            if (key2 != 0xFFFFFFFFu) push(refOf(key2), key2 & ~3u);
            if (key1 != 0xFFFFFFFFu) push(refOf(key1), key1 & ~3u);
            cur = refOf(key0);
            return true;
        }

        // The primitives of one leaf: references i into sc.bvh4_geom / sc.bvh4_prim. A primitive cut by a spatial split has a
        // reference in several leaves, and each test of it gives a bit-identical t: such a repeat is not a competitor of the best
        // hit, and the target of an occlusion query is skipped by its ordered id. -> false: the search is over (OCC only: an
        // occluder or a tie was found).
        MCRT_D bool testLeaf(uint32_t leaf, const DeviceScene<double>& sc, const RayQ<double>& ray, TraceCounters& cnt)
        {
            const uint32_t first = (leaf >> 8) & (BVH4_MAX_PRIMS - 1u), count = leaf & 0xFFu;
            for (uint32_t i = first; i < first + count; i++)
            {
                double t, u, v;
                bool is_tri;
                if constexpr (OCC)
                {
                    if (__ldg(sc.bvh4_prim + i) == target) continue;
                    if (intersectPrim<PRIMS>(sc, sc.bvh4_geom, i, ray, t, u, v, is_tri))
                    {
                        const double delta = ambiguityDelta(best.t, (double)sc.scene_scale);
                        // an occluder hit on its own boundary may be one the reference never reaches: replay
                        if (t <= best.t + delta && is_tri && onTriangleBoundary(u, v, t, (double)sc.scene_scale)) { verdict = 2u; cnt.prim_tests += i - first + 1; return false; }
                        if (t < best.t - delta) { verdict = 1u; cnt.prim_tests += i - first + 1; return false; }   // occluder: done
                        if (t <= best.t + delta) { verdict = 2u; cnt.prim_tests += i - first + 1; return false; }  // tie: replay
                    }
                    continue;
                }
                if (intersectPrim<PRIMS>(sc, sc.bvh4_geom, i, ray, t, u, v, is_tri))
                {
                    if (t < best.t)
                    {
                        second_t = best.t;
                        best.t = t; best.u = u; best.v = v; best.prim = __ldg(sc.bvh4_prim + i);
                        best.interpolate = (is_tri && onTriangleBoundary(u, v, t, (double)sc.scene_scale)) ? 1u : 0u;   // scratch use: winner on its boundary
                        limit = __double2float_ru(t + 2.0 * ambiguityDelta(t, (double)sc.scene_scale));
                    }
                    else if (t < second_t && !(t == best.t && __ldg(sc.bvh4_prim + i) == best.prim))
                    {
                        second_t = t;
                    }
                }
            }
            cnt.prim_tests += count;
            return true;
        }

        MCRT_D bool step(const DeviceScene<double>& sc, const RayQ<double>& ray, TraceCounters& cnt)
        {
#if MCRT_SPECULATIVE
            // Speculative form (Aila & Laine): a lane that reaches a leaf stashes it and keeps walking inner nodes until every
            // lane walking with it holds a leaf too; then all test their leaves together. Visits a superset of the nodes
            // (the stashed leaf could have shortened the ray first), never a different answer.
            uint32_t stashed = 0u;
            bool have_cur = true;
            while (true)
            {
                if (cur & BVH4_LEAF)
                {
                    if (stashed) break;                       // a second leaf: test the first one now
                    stashed = cur;
                    have_cur = pop();
                    if (!have_cur) break;
                }
                else
                {
                    have_cur = visitNode(sc, cnt);
                    if (!have_cur) break;
                }
                if (stashed && !__any_sync(__activemask(), stashed == 0u)) break;
            }
            if (stashed && !testLeaf(stashed, sc, ray, cnt)) return false;
            return have_cur;
#else
            while (!(cur & BVH4_LEAF))
            {
                if (!visitNode(sc, cnt)) return false;
            }
            if (!testLeaf(cur, sc, ray, cnt)) return false;
            return pop();
#endif
        }

        // another hit within delta of the closest: the answer may depend on the visiting order
        MCRT_D bool ambiguous(const DeviceScene<double>& sc) const
        {
            if (degenerate) return true;
            return best.prim != NO_PRIM && (best.interpolate != 0u || second_t <= best.t + ambiguityDelta(best.t, (double)sc.scene_scale));
        }
    };

    // -> closest hit; `ambiguous` set when another hit lies within delta of it
    template <int PRIMS>
    MCRT_D Hit<double> traverseFast(const DeviceScene<double>& sc, const RayQ<double>& ray, TraceCounters& cnt, bool& ambiguous)
    {
        FastSearch<PRIMS> fs;
        fs.begin(ray);
        while (fs.step(sc, ray, cnt)) { }
        ambiguous = fs.ambiguous(sc);
        return fs.best;
    }

    // Out of line: the replay only runs for the rare ambiguous ray, and inlining it would make every
    // ray pay its registers.
    template <int PRIMS>
    __device__ __noinline__ void traceReferenceOrderOutOfLine(const DeviceScene<double>* sc, const RayQ<double>* ray, Hit<double>* out,
                                                              uint32_t* box_tests, uint32_t* prim_tests, uint32_t* overflow)
    {
        TraceCounters c = { 0u, 0u };
        uint32_t ov = 0;
        *out = traverseReferenceOrder<PRIMS>(*sc, *ray, c, ov);
        *box_tests += c.box_tests; *prim_tests += c.prim_tests;
        if (ov) *overflow = 1;
    }

    // Many rays per warp with dynamic fetch. Rays of one warp need very different numbers of steps (on
    // big scenes the plain one-ray-per-lane loop leaves most lanes of a warp idle),
    // so a lane whose ray is finished does not wait for the warp's longest ray: when fewer than
    // MCRT_FETCH_THRESHOLD lanes are still searching, the warp takes the next rays of the (sorted) queue
    // for its idle lanes from a global counter. load(ii, ray) -> item id, done(item, ray, hit).
#ifndef MCRT_FETCH_THRESHOLD
#define MCRT_FETCH_THRESHOLD 22
#endif
    // OCC: load(ii, ray, target) also names the primitive whose visibility is asked; done() gets a hit whose
    // prim is the target iff it is the closest hit
    template <int PRIMS, bool OCC = false, class Load, class Done>
    MCRT_D void traceManyFast(const DeviceScene<double>& sc, uint32_t n, uint32_t* fetch_counter, Load load, Done done,
                              TraceCounters& cnt, uint32_t& overflow)
    {
        FastSearch<PRIMS, OCC> fs;
        RayQ<double> ray;
        uint32_t item = 0;
        bool active = false;
        bool more = true;        // warp-uniform: the queue may still hold rays
        const unsigned lane = threadIdx.x & 31u;
        while (true)
        {
            const unsigned need = __ballot_sync(0xFFFFFFFFu, !active);
            if (need && more)
            {
                uint32_t base = 0;
                const int leader = __ffs(need) - 1;
                if ((int)lane == leader) base = atomicAdd(fetch_counter, (uint32_t)__popc(need));
                base = __shfl_sync(0xFFFFFFFFu, base, leader);
                more = base < n;
                if (!active)
                {
                    const uint32_t ii = base + (uint32_t)__popc(need & ((1u << lane) - 1u));
                    if (ii < n)
                    {
                        if constexpr (OCC)
                        {
                            uint32_t target;
                            item = load(ii, ray, target);
                            if (fs.beginOcclusion(sc, ray, target, cnt)) { active = true; if (fs.verdict == 2u) fs.sp = 0, fs.cur = BVH4_LEAF; }   // degenerate: an empty leaf ends the search at once
                            else { Hit<double> miss = fs.best; miss.prim = NO_PRIM; done(item, ray, miss); }   // the ray misses the light itself
                        }
                        else
                        {
                            item = load(ii, ray);
                            fs.begin(ray);
                            active = true;
                        }
                    }
                }
            }
            if (__ballot_sync(0xFFFFFFFFu, active) == 0u)
            {
                if (!more) break;
                continue;        // every fetched ray was resolved at once (it misses its light): fetch again
            }
            while (active)
            {
                if (!fs.step(sc, ray, cnt))
                {
                    Hit<double> h = fs.best;
                    bool replay;
                    if constexpr (OCC) { replay = fs.verdict == 2u; if (fs.verdict == 1u) h.prim = NO_PRIM; }
                    else replay = fs.ambiguous(sc);
                    if (replay)
                    {
                        const DeviceScene<double> sc_copy = sc;
                        RayQ<double> rq_copy = ray;
                        rq_copy.inv_d = 1.0 / ray.d;          // only the replay's float64 slab test needs it
                        Hit<double> h2;
                        traceReferenceOrderOutOfLine<PRIMS>(&sc_copy, &rq_copy, &h2, &cnt.box_tests, &cnt.prim_tests, &overflow);
                        h = h2;
                        cnt.replayed++;
                    }
                    done(item, ray, h);
                    active = false;
                    break;
                }
                if (__popc(__activemask()) < MCRT_FETCH_THRESHOLD) break;
            }
        }
    }
}
