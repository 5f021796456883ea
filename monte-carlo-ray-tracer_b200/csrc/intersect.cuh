// Ray / primitive / BVH intersection on the device.
//
// Primitive tests follow the reference's formulas and rejection rules:
//   slab test     source/common/bounding-box.cpp:9-17
//   triangle      source/surface/triangle.cpp:23-63   (Möller–Trumbore, |det| < 1e-9 cull, u,v in
//                 [0,1] inclusive, t <= 0 rejected)
//   sphere        source/surface/sphere.cpp:13-26 + solveQuadratic source/common/util.hpp:60-83
//   quadric       source/surface/quadric.cpp:69-100 (clipped to its own box)
// Two traversals of the flattened BVH (source/bvh/bvh.cpp:80-129):
//   traverseReferenceOrder  parity mode. Best-first with the same binary heap discipline as
//       source/common/priority-queue.hpp:19-46,107-126, so that equal-t ties resolve to the same
//       primitive as on the CPU. The heap lives in per-thread local memory.
//   traverseWide            fast mode (float). Depth-first over the child-record layout with a
//       near-to-far ordered push; visits a superset of the nodes the best-first order visits and
//       returns the same closest t.
// A scene without a BVH takes the linear scan of source/scene/scene.cpp:159-173.
#pragma once

#include "scene.cuh"

namespace mcrt
{
    template <class R> struct RayQ
    {
        V3<R> o, d, inv_d;
    };

    struct TraceCounters
    {
        uint32_t box_tests;
        uint32_t prim_tests;
        uint32_t replayed;   // rays the order-free search handed to the reference-order replay (bvh4.cuh)
    };

    // BoundingBox::intersect
    template <class R>
    MCRT_D bool slabTest(const R* bmin, const R* bmax, const RayQ<R>& ray, R& t)
    {
        V3<R> t0 = (V3<R>(bmin[0], bmin[1], bmin[2]) - ray.o) * ray.inv_d;
        V3<R> t1 = (V3<R>(bmax[0], bmax[1], bmax[2]) - ray.o) * ray.inv_d;
        t = gmax(compMax(vmin(t0, t1)), R(0));
        return compMin(vmax(t0, t1)) >= t;
    }

    template <class R>
    MCRT_D bool boxContains(const R* bmin, const R* bmax, const V3<R>& p)
    {
        return p.x >= bmin[0] && p.y >= bmin[1] && p.z >= bmin[2] &&
               p.x <= bmax[0] && p.y <= bmax[1] && p.z <= bmax[2];
    }

    // solveQuadratic, util.hpp:60-83
    template <class R>
    MCRT_D bool solveQuadratic(R a, R b, R c, R& t_min, R& t_max)
    {
        if (a != R(0))
        {
            R d = b * b - R(4) * a * c;
            if (d < R(0)) return false;
            R t = R(-0.5) * (b + (b < R(0) ? -msqrt(d) : msqrt(d)));
            t_min = t / a;
            t_max = c / t;
            if (t_min > t_max) { R tmp = t_min; t_min = t_max; t_max = tmp; }
            return true;
        }
        if (b != R(0))
        {
            t_min = t_max = -c / b;
            return true;
        }
        return false;
    }

    template <class R>
    MCRT_D bool intersectTriangle(const V4<R>& g0, const V4<R>& g1, const V4<R>& g2, const RayQ<R>& ray,
                                  R& t_out, R& u_out, R& v_out)
    {
        const V3<R> v0 = g0.xyz(), E1 = g1.xyz(), E2 = g2.xyz();
        V3<R> P = cross(ray.d, E2);
        R determinant = dot(P, E1);
        if (determinant < Consts<R>::EPSILON && determinant > -Consts<R>::EPSILON) return false;
        R inv_determinant = R(1) / determinant;
        V3<R> T = ray.o - v0;
        R u = dot(P, T) * inv_determinant;
        if (u > R(1) || u < R(0)) return false;
        V3<R> Q = cross(T, E1);
        R v = dot(Q, ray.d) * inv_determinant;
        if (v > R(1) || v < R(0) || u + v > R(1)) return false;
        R t = dot(Q, E2) * inv_determinant;
        if (t <= R(0)) return false;
        t_out = t; u_out = u; v_out = v;
        return true;
    }

    template <class R>
    MCRT_D bool intersectSphere(const V4<R>& g0, const V4<R>& g1, const RayQ<R>& ray, R& t_out)
    {
        V3<R> so = ray.o - g0.xyz();
        if constexpr (sizeof(R) == 4)
        {
            // float32: b^2 - 4c cancels for a sphere seen from many radii away, and the error of the hit point can then exceed
            // the ray offset, so paths leaving the sphere hit it again. The discriminant from the squared distance between the
            // centre and the ray does not cancel (Haines et al., Ray Tracing Gems ch. 7); d is unit length, as a = 1 assumes.
            const R bh = dot(ray.d, so);
            const V3<R> f = so - ray.d * bh;
            const R r = g1.x, fl = msqrt(dot(f, f));
            const R disc = (r - fl) * (r + fl);
            if (disc < R(0)) return false;
            const R q = -(bh + (bh < R(0) ? -msqrt(disc) : msqrt(disc)));
            R t_min = (dot(so, so) - pow2(r)) / q, t_max = q;
            if (t_min > t_max) { const R tmp = t_min; t_min = t_max; t_max = tmp; }
            if (t_max < R(0)) return false;
            t_out = t_min < R(0) ? t_max : t_min;
            return true;
        }
        R b = R(2) * dot(ray.d, so);
        R c = dot(so, so) - pow2(g1.x);
        R t_min, t_max;
        if (solveQuadratic(R(1), b, c, t_min, t_max) && t_max >= R(0))
        {
            t_out = t_min < R(0) ? t_max : t_min;
            return true;
        }
        return false;
    }

    // glm mat4 * vec4: (m0*v0 + m1*v1) + (m2*v2 + m3*v3), type_mat4x4.inl:560-571
    template <class R>
    MCRT_D void mat4MulVec4(const R* M, const R* v, R* out)
    {
#pragma unroll
        for (int r = 0; r < 4; r++)
        {
            out[r] = (M[0 + r] * v[0] + M[4 + r] * v[1]) + (M[8 + r] * v[2] + M[12 + r] * v[3]);
        }
    }

    template <class R>
    MCRT_D R dot4(const R* a, const R* b)
    {
        return (a[0] * b[0] + a[1] * b[1]) + (a[2] * b[2] + a[3] * b[3]);
    }

    template <class R>
    MCRT_D bool intersectQuadric(const Quadric<R>& q, const RayQ<R>& ray, R& t_out)
    {
        R t_bb = R(0);
        if (!slabTest(q.bmin, q.bmax, ray, t_bb)) return false;
        V3<R> p = ray.o + ray.d * t_bb;
        R o[4] = { p.x, p.y, p.z, R(1) };
        R d[4] = { ray.d.x, ray.d.y, ray.d.z, R(0) };
        R Qo[4], Qd[4];
        mat4MulVec4(q.Q, o, Qo);
        mat4MulVec4(q.Q, d, Qd);
        R a = dot4(d, Qd);
        R b = dot4(d, Qo) * R(2);
        R c = dot4(o, Qo);
        R t_min, t_max;
        if (solveQuadratic(a, b, c, t_min, t_max) && t_max >= R(0))
        {
            R t = t_bb + (t_min < R(0) ? t_max : t_min);
            if (!boxContains(q.bmin, q.bmax, ray.o + ray.d * t)) return false;
            t_out = t;
            return true;
        }
        return false;
    }

    enum { PRIMS_ALL = 0, PRIMS_TRI_SPHERE = 1, PRIMS_TRI = 2 };

    // One ordered primitive against the ray; strict `t < best.t` acceptance (bvh.cpp:100).
    // PRIMS: instantiations for scenes made of triangles only (every OBJ scene: no type dispatch at all)
    // or of triangles and spheres (no quadric code) - the pruned branches are unreachable for them.
    template <int PRIMS = PRIMS_ALL, class R>
    MCRT_D void testPrim(const DeviceScene<R>& sc, uint32_t prim, const RayQ<R>& ray, Hit<R>& best)
    {
        const V4<R> g0 = sc.geom[3 * prim + 0];
        const uint32_t type = PRIMS == PRIMS_TRI ? (uint32_t)PRIM_TRIANGLE : (uint32_t)g0.w;
        R t, u = R(0), v = R(0);
        bool hit;
        if (type == PRIM_TRIANGLE)
        {
            const V4<R> g1 = sc.geom[3 * prim + 1];
            const V4<R> g2 = sc.geom[3 * prim + 2];
            hit = intersectTriangle(g0, g1, g2, ray, t, u, v);
        }
        else if (PRIMS == PRIMS_TRI_SPHERE || type == PRIM_SPHERE)
        {
            const V4<R> g1 = sc.geom[3 * prim + 1];
            hit = intersectSphere(g0, g1, ray, t);
        }
        else
        {
            hit = intersectQuadric(sc.quadrics[(uint32_t)g0.x], ray, t);
        }
        if (hit && t < best.t)
        {
            best.t = t; best.u = u; best.v = v; best.prim = prim;
        }
    }

    // ------------------------------------------------------------------------------------------
    // Parity traversal: same visiting order as BVH::intersect.
    constexpr int REF_HEAP_CAPACITY = 96; // reference max observed: 35 (SURVEY.md §3.2)

    template <class R>
    struct RefHeap
    {
        R t[REF_HEAP_CAPACITY];
        uint2 node[REF_HEAP_CAPACITY];   // (a, b) of the child record: no dependent load after a pop
        int size;

        // NodeIntersection::operator< is inverted (bvh.hpp:78): a < b  <=>  b.t < a.t
        MCRT_D void push(R vt, uint2 vn)
        {
            int index = size++;
            while (index > 0)
            {
                int parent = (index - 1) / 2;
                if (!(vt < t[parent])) break;
                t[index] = t[parent]; node[index] = node[parent];
                index = parent;
            }
            t[index] = vt; node[index] = vn;
        }

        MCRT_D void pop()
        {
            if (size > 1)
            {
                R vt = t[size - 1]; uint2 vn = node[size - 1];
                size--;
                int index = 0;
                while (true)
                {
                    int left = 2 * index + 1, right = left + 1, max_child;
                    if (right < size) max_child = left + ((t[right] < t[left]) ? 1 : 0);
                    else if (left < size) max_child = left;
                    else break;
                    if (!(t[max_child] < vt)) break;
                    t[index] = t[max_child]; node[index] = node[max_child];
                    index = max_child;
                }
                t[index] = vt; node[index] = vn;
            }
            else
            {
                size--;
            }
        }
    };

    template <int PRIMS = PRIMS_ALL, class R>
    MCRT_D Hit<R> traverseReferenceOrder(const DeviceScene<R>& sc, const RayQ<R>& ray, TraceCounters& cnt, uint32_t& overflow)
    {
        Hit<R> best;
        best.t = Consts<R>::MAXV; best.u = R(0); best.v = R(0); best.prim = NO_PRIM; best.interpolate = 0;

        if (sc.n_nodes == 0)
        {
            // Scene::intersect without a bvh object: every surface in order
            for (uint32_t i = 0; i < sc.n_prims; i++) testPrim<PRIMS>(sc, i, ray, best);
            cnt.prim_tests += sc.n_prims;
            return best;
        }

        RefHeap<R> heap;
        heap.size = 0;
        R t;
        cnt.box_tests++;
        if (!slabTest(sc.root_bmin, sc.root_bmax, ray, t)) return best;

        // (a, b) of the node being visited; the heap holds the (a, b) of pending children.
        // "while-while" control flow: every lane first walks down through inner nodes (all lanes of
        // the warp do box tests together), then all lanes test leaf primitives together. The order
        // of operations per ray is exactly the reference's; only the SIMT schedule changes.
        uint32_t cur_a, cur_b;
        if (sc.root_is_leaf) { cur_a = sc.root_first_prim; cur_b = sc.root_prim_count | WIDE_LEAF; }
        else { cur_a = 0; cur_b = sc.n_wide_root; }

        bool done = false;
        while (!done)
        {
            while (!(cur_b & WIDE_LEAF))
            {
                // children in next_sibling order; the loads are independent of each other
                for (uint32_t c = cur_a; c < cur_a + cur_b; c++)
                {
                    const WideChild<R>& cn = sc.wide[c];
                    if (slabTest(cn.bmin, cn.bmax, ray, t) && t < best.t)
                    {
                        if (heap.size < REF_HEAP_CAPACITY) heap.push(t, make_uint2(cn.a, cn.b));
                        else overflow = 1;
                    }
                }
                cnt.box_tests += cur_b;
                if (heap.size == 0 || heap.t[0] >= best.t) { done = true; break; }
                cur_a = heap.node[0].x; cur_b = heap.node[0].y;
                heap.pop();
            }
            if (done) break;
            {
                const uint32_t count = cur_b & ~WIDE_LEAF;
                for (uint32_t i = cur_a; i < cur_a + count; i++) testPrim<PRIMS>(sc, i, ray, best);
                cnt.prim_tests += count;
            }
            if (heap.size == 0 || heap.t[0] >= best.t) break;
            cur_a = heap.node[0].x; cur_b = heap.node[0].y;
            heap.pop();
        }
        return best;
    }

    // ------------------------------------------------------------------------------------------
    // Fast traversal (float): wide child records, depth-first, nearest child first.
    constexpr int WIDE_STACK = 48;

    MCRT_D bool slabTestWide(const float4& lo, const float4& hi, const RayQ<float>& ray, float best, float& t)
    {
        // lo = (min.x, min.y, min.z, max.x), hi = (max.y, max.z, a, b)
        float tx0 = (lo.x - ray.o.x) * ray.inv_d.x, tx1 = (lo.w - ray.o.x) * ray.inv_d.x;
        float ty0 = (lo.y - ray.o.y) * ray.inv_d.y, ty1 = (hi.x - ray.o.y) * ray.inv_d.y;
        float tz0 = (lo.z - ray.o.z) * ray.inv_d.z, tz1 = (hi.y - ray.o.z) * ray.inv_d.z;
        float tn = fmaxf(fmaxf(fminf(tx0, tx1), fminf(ty0, ty1)), fmaxf(fminf(tz0, tz1), 0.0f));
        float tf = fminf(fminf(fmaxf(tx0, tx1), fmaxf(ty0, ty1)), fmaxf(tz0, tz1));
        t = tn;
        return tf >= tn && tn < best;
    }

    // skip_prim: ordered-primitive id the ray starts on when that primitive is planar (a ray
    // leaving a triangle cannot hit it again; float has no room for the reference's 1e-9 offset).
    template <int PRIMS = PRIMS_ALL>
    MCRT_D Hit<float> traverseWide(const DeviceScene<float>& sc, const RayQ<float>& ray, uint32_t skip_prim,
                                   TraceCounters& cnt, uint32_t& overflow)
    {
        Hit<float> best;
        best.t = Consts<float>::MAXV; best.u = 0.0f; best.v = 0.0f; best.prim = NO_PRIM; best.interpolate = 0;

        if (sc.n_nodes == 0)
        {
            for (uint32_t i = 0; i < sc.n_prims; i++)
            {
                if (i != skip_prim) testPrim<PRIMS>(sc, i, ray, best);
            }
            cnt.prim_tests += sc.n_prims;
            return best;
        }

        float t;
        cnt.box_tests++;
        if (!slabTest(sc.root_bmin, sc.root_bmax, ray, t)) return best;

        // stack entries: (a, b) of a child record + its entry distance (culled against best.t on pop)
        uint32_t stack_a[WIDE_STACK], stack_b[WIDE_STACK];
        float stack_t[WIDE_STACK];
        int sp = 0;
        uint32_t cur_a, cur_b;
        if (sc.root_is_leaf) { cur_a = sc.root_first_prim; cur_b = sc.root_prim_count | WIDE_LEAF; }
        else { cur_a = 0; cur_b = sc.n_wide_root; }

        const float4* wide = reinterpret_cast<const float4*>(sc.wide);
        bool done = false;
        while (!done)
        {
            // "while-while": inner nodes first (all lanes doing box tests), then leaf primitives
            while (!(cur_b & WIDE_LEAF))
            {
                // the nearest hit child is visited next, the others are pushed; the stack is not kept
                // sorted: entries carry their entry distance and are culled against best.t on pop
                float near_t = Consts<float>::MAXV; uint32_t near_a = 0, near_b = 0; bool have = false;
                for (uint32_t c = 0; c < cur_b; c++)
                {
                    const float4 lo = __ldg(&wide[2 * (cur_a + c)]);
                    const float4 hi = __ldg(&wide[2 * (cur_a + c) + 1]);
                    float tc;
                    if (slabTestWide(lo, hi, ray, best.t, tc))
                    {
                        uint32_t a = __float_as_uint(hi.z), b = __float_as_uint(hi.w);
                        if (!have) { near_t = tc; near_a = a; near_b = b; have = true; continue; }
                        if (tc < near_t)
                        {
                            const float tt = near_t; const uint32_t ta = near_a, tb = near_b;
                            near_t = tc; near_a = a; near_b = b;
                            tc = tt; a = ta; b = tb;
                        }
                        if (sp < WIDE_STACK) { stack_a[sp] = a; stack_b[sp] = b; stack_t[sp] = tc; sp++; }
                        else overflow = 1;
                    }
                }
                cnt.box_tests += cur_b;
                if (have) { cur_a = near_a; cur_b = near_b; continue; }
                bool found = false;
                while (sp > 0)
                {
                    sp--;
                    if (stack_t[sp] < best.t) { cur_a = stack_a[sp]; cur_b = stack_b[sp]; found = true; break; }
                }
                if (!found) { done = true; break; }
            }
            if (done) break;
            {
                const uint32_t count = cur_b & ~WIDE_LEAF;
                for (uint32_t i = cur_a; i < cur_a + count; i++)
                {
                    if (i != skip_prim) testPrim<PRIMS>(sc, i, ray, best);
                }
                cnt.prim_tests += count;
            }
            bool found = false;
            while (sp > 0)
            {
                sp--;
                if (stack_t[sp] < best.t) { cur_a = stack_a[sp]; cur_b = stack_b[sp]; found = true; break; }
            }
            if (!found) break;
        }
        return best;
    }
}
