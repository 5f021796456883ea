// ORACLE / TEST INFRASTRUCTURE — never linked into or imported by the product (libmcrt_b200.so).
//
// Scalar float64 CPU restatement of the reference's path-tracing hot path, operating on the
// flattened scene description of include/mcrt_abi.h. One path at a time, the way the reference
// runs it; no SIMD, no threads. Build: g++ -O2 -ffp-contract=off (oracle/build_oracle.py).
// Pinned against the unmodified reference through tests/golden/*.npz (tests/test_oracle_cpu.py):
// sampler streams bit-exact, Scene::intersect same primitive and t, per-sample radiance and images
// to 1e-9. Each function cites the reference lines it restates (paths relative to /root/reference).
//
// The photon mapper (photon-mapper.cpp:24-391) is restated too: the emission pass photon by photon in emission order, the
// octree by the restated builder below, and PhotonMapper::sampleRay with a brute-force k-NN search in place of the octree
// search. Pinned by tests/test_photon_mapper_oracle_cpu.py to pm_hexagon_room_64: maps bit-exact, per-sample radiance and
// image to 1e-12, ray counts and k-NN results exact; tests/test_gpu_photon_mapper.py holds the device to it.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <limits>
#include <memory>
#include <thread>
#include <vector>

#include "mcrt_abi.h"

namespace
{
    struct D3
    {
        double x, y, z;
        D3() : x(0), y(0), z(0) {}
        D3(double a, double b, double c) : x(a), y(b), z(c) {}
        explicit D3(const double* p) : x(p[0]), y(p[1]), z(p[2]) {}
    };
    inline D3 operator+(D3 a, D3 b) { return D3(a.x + b.x, a.y + b.y, a.z + b.z); }
    inline D3 operator-(D3 a, D3 b) { return D3(a.x - b.x, a.y - b.y, a.z - b.z); }
    inline D3 operator*(D3 a, D3 b) { return D3(a.x * b.x, a.y * b.y, a.z * b.z); }
    inline D3 operator/(D3 a, D3 b) { return D3(a.x / b.x, a.y / b.y, a.z / b.z); }
    inline D3 operator*(D3 a, double s) { return D3(a.x * s, a.y * s, a.z * s); }
    inline D3 operator*(double s, D3 a) { return D3(s * a.x, s * a.y, s * a.z); }
    inline D3 operator/(D3 a, double s) { return D3(a.x / s, a.y / s, a.z / s); }
    inline D3 operator-(D3 a) { return D3(-a.x, -a.y, -a.z); }
    // GLM evaluation orders: lib/glm/glm/detail/func_geometric.inl:48-55,66-78,88,104-108
    inline double dot(D3 a, D3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
    inline D3 cross(D3 a, D3 b) { return D3(a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y); }
    inline D3 normalize(D3 v) { return v * (1.0 / std::sqrt(dot(v, v))); }
    inline double gmin(double x, double y) { return (y < x) ? y : x; }   // func_common.inl:17-30
    inline double gmax(double x, double y) { return (x < y) ? y : x; }
    inline double sq(double x) { return x * x; }
    inline double mixd(double x, double y, double a) { return x * (1.0 - a) + y * a; }
    inline D3 mix3(D3 x, D3 y, double a) { return x * (1.0 - a) + y * a; }
    inline double compMax(D3 v) { return gmax(gmax(v.x, v.y), v.z); }
    inline double compMin(D3 v) { return gmin(gmin(v.x, v.y), v.z); }

    const double PI = 3.14159265358979323846, INV_PI = 0.31830988618379067154, TWO_PI = 6.283185307179586476925;
    const double EPS = 1e-9; // source/common/constants.hpp:5-9

    // ---------------------------------------------------------------- sampler (sampler.hpp, sobol.hpp)
    uint32_t reverseBits(uint32_t x) // sobol.hpp:9-16
    {
        x = ((x & 0xaaaaaaaau) >> 1) | ((x & 0x55555555u) << 1);
        x = ((x & 0xccccccccu) >> 2) | ((x & 0x33333333u) << 2);
        x = ((x & 0xf0f0f0f0u) >> 4) | ((x & 0x0f0f0f0fu) << 4);
        x = ((x & 0xff00ff00u) >> 8) | ((x & 0x00ff00ffu) << 8);
        return (x >> 16) | (x << 16);
    }

    struct Directions
    {
        uint32_t v[6][32];
        Directions() // sobol.hpp:18-56 with the Joe-Kuo (s, a, m) rows for dimensions 2..7
        {
            const uint32_t s[6] = { 1, 2, 3, 3, 4, 4 }, a[6] = { 0, 1, 1, 2, 1, 4 };
            const uint32_t m[6][4] = { { 1, 0, 0, 0 }, { 1, 3, 0, 0 }, { 1, 3, 1, 0 }, { 1, 1, 1, 0 }, { 1, 1, 3, 3 }, { 1, 3, 5, 13 } };
            for (int d = 0; d < 6; d++)
            {
                uint32_t V[32];
                for (uint32_t b = 0; b < 32; b++)
                {
                    if (b < s[d]) V[b] = m[d][b] << (31 - b);
                    else
                    {
                        V[b] = V[b - s[d]] ^ (V[b - s[d]] >> s[d]);
                        for (uint32_t k = 1; k < s[d]; k++) V[b] ^= (((a[d] >> (s[d] - 1 - k)) & 1u) * V[b - k]);
                    }
                }
                for (int b = 0; b < 32; b++) v[d][b] = reverseBits(V[b]);
            }
        }
    };
    const Directions DIRS;

    uint32_t hash32(uint32_t x) { x ^= x >> 15; x *= 0xd168aaadu; x ^= x >> 15; x *= 0xaf723597u; x ^= x >> 15; return x; } // sampler.hpp:78-86
    uint32_t combine(uint32_t seed, uint32_t v) { return seed ^ (v + 0x9e3779b9u + (seed << 6) + (seed >> 2)); }            // :89-92
    uint32_t scramble(uint32_t x, uint32_t seed)                                                                           // :61-73
    {
        x ^= x * 0x3d20adeau; x += seed; x *= (seed >> 16) | 1u; x ^= x * 0x05526c56u; x ^= x * 0x53a22864u;
        return reverseBits(x);
    }

    struct Sampler // the thread_local registers of sampler.hpp:55-56
    {
        uint32_t global_seed, base_seed = 0, seed = 0, sequence = 0, bit_reversed_index = 0, shuffled_index = 0;
        explicit Sampler(uint32_t g) : global_seed(g) {}
        void initiate(uint32_t start) { base_seed = combine(global_seed, hash32(start)); }
        void setIndex(uint32_t i) { sequence = 0; seed = base_seed; bit_reversed_index = reverseBits(i); shuffled_index = i; }
        void shuffle() { seed = combine(base_seed, hash32(++sequence)); shuffled_index = scramble(bit_reversed_index, seed); }
        uint32_t raw(int dim) const
        {
            uint32_t x = shuffled_index;
            if (dim > 0)
            {
                x = 0;
                uint32_t index = shuffled_index;
                for (int bit = 0; index; index >>= 1, bit++) x ^= (index & 1u) * DIRS.v[dim - 1][bit];
            }
            return scramble(x, combine(seed, hash32((uint32_t)dim)));
        }
        double get(int dim) const { return raw(dim) * 0x1p-32; }
    };
    enum { PIXEL = 0, LENS = 2, LIGHT = 0, BSDF = 3, INTERACTION = 5, ABSORB = 6 }; // sampling.hpp:59-76

    // ---------------------------------------------------------------- scene
    struct Scene
    {
        mcrt_scene_desc d;
        std::vector<double> node_bounds, prim_area, tri_v0, tri_v1, tri_v2, tri_e1, tri_e2, tri_n, vn, sph, qQ, qG, qB, light_cdf;
        std::vector<uint32_t> node_first, node_count, node_next, prim_index, prim_material, light_prim;
        std::vector<uint8_t> prim_type;
        std::vector<int32_t> tri_vn;
        std::vector<mcrt_material> materials;
    };

    template <class T> void copyv(std::vector<T>& dst, const T* src, size_t n) { dst.assign(src, src + (src ? n : 0)); }

    struct Ray
    {
        D3 start, direction, inv_direction;
        double medium_ior = 1.0, refraction_scale = 1.0;
        bool dirac_delta = false, refraction = false;
        uint32_t depth = 0, diffuse_depth = 0;
        int refraction_level = 0;
        D3 at(double t) const { return start + direction * t; }
    };
    Ray makeRay(D3 start, D3 dir, double ior) // ray.cpp:13-14
    {
        Ray r; r.start = start; r.direction = dir; r.inv_direction = D3(1.0 / dir.x, 1.0 / dir.y, 1.0 / dir.z); r.medium_ior = ior;
        return r;
    }
    Ray rayTo(D3 start, D3 end) { return makeRay(start, normalize(end - start), 1.0); } // ray.cpp:10-11

    struct Isect { double t = std::numeric_limits<double>::max(); double u = 0, v = 0; uint32_t prim = 0xFFFFFFFFu; bool interpolate = false; };

    bool slab(const double* b, const Ray& r, double& t) // bounding-box.cpp:9-17
    {
        D3 t0 = (D3(b) - r.start) * r.inv_direction, t1 = (D3(b + 3) - r.start) * r.inv_direction;
        D3 lo(gmin(t0.x, t1.x), gmin(t0.y, t1.y), gmin(t0.z, t1.z)), hi(gmax(t0.x, t1.x), gmax(t0.y, t1.y), gmax(t0.z, t1.z));
        t = gmax(compMax(lo), 0.0);
        return compMin(hi) >= t;
    }

    bool solveQuadratic(double a, double b, double c, double& t_min, double& t_max) // util.hpp:60-83
    {
        if (a != 0.0)
        {
            double d = b * b - 4.0 * a * c;
            if (d < 0.0) return false;
            double t = -0.5 * (b + (b < 0.0 ? -std::sqrt(d) : std::sqrt(d)));
            t_min = t / a; t_max = c / t;
            if (t_min > t_max) std::swap(t_min, t_max);
            return true;
        }
        if (b != 0.0) { t_min = t_max = -c / b; return true; }
        return false;
    }

    bool hitPrim(const Scene& s, uint32_t prim, const Ray& r, Isect& out)
    {
        const uint32_t idx = s.prim_index[prim];
        if (s.prim_type[prim] == MCRT_PRIM_TRIANGLE) // triangle.cpp:23-63
        {
            D3 v0(&s.tri_v0[3 * idx]), E1(&s.tri_e1[3 * idx]), E2(&s.tri_e2[3 * idx]);
            D3 P = cross(r.direction, E2);
            double det = dot(P, E1);
            if (det < EPS && det > -EPS) return false;
            double inv = 1.0 / det;
            D3 T = r.start - v0;
            double u = dot(P, T) * inv;
            if (u > 1.0 || u < 0.0) return false;
            D3 Q = cross(T, E1);
            double v = dot(Q, r.direction) * inv;
            if (v > 1.0 || v < 0.0 || u + v > 1.0) return false;
            double t = dot(Q, E2) * inv;
            if (t <= 0.0) return false;
            out = Isect(); out.t = t;
            if (s.tri_vn[idx] >= 0) { out.u = u; out.v = v; out.interpolate = true; }
            return true;
        }
        if (s.prim_type[prim] == MCRT_PRIM_SPHERE) // sphere.cpp:13-26
        {
            const double* sp = &s.sph[4 * idx];
            D3 so = r.start - D3(sp);
            double b = 2.0 * dot(r.direction, so), c = dot(so, so) - sq(sp[3]);
            double t_min, t_max;
            if (solveQuadratic(1.0, b, c, t_min, t_max) && t_max >= 0.0) { out = Isect(); out.t = t_min < 0.0 ? t_max : t_min; return true; }
            return false;
        }
        // quadric.cpp:69-100
        const double* Q = &s.qQ[16 * idx]; const double* B = &s.qB[6 * idx];
        double t_bb = 0.0;
        if (!slab(B, r, t_bb)) return false;
        D3 p = r.at(t_bb);
        double o[4] = { p.x, p.y, p.z, 1.0 }, d[4] = { r.direction.x, r.direction.y, r.direction.z, 0.0 }, Qo[4], Qd[4];
        for (int k = 0; k < 4; k++) // glm mat4*vec4: (m0 v0 + m1 v1) + (m2 v2 + m3 v3)
        {
            Qo[k] = (Q[k] * o[0] + Q[4 + k] * o[1]) + (Q[8 + k] * o[2] + Q[12 + k] * o[3]);
            Qd[k] = (Q[k] * d[0] + Q[4 + k] * d[1]) + (Q[8 + k] * d[2] + Q[12 + k] * d[3]);
        }
        auto dot4 = [](const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + (a[2] * b[2] + a[3] * b[3]); };
        double a = dot4(d, Qd), b = dot4(d, Qo) * 2.0, c = dot4(o, Qo), t_min, t_max;
        if (solveQuadratic(a, b, c, t_min, t_max) && t_max >= 0.0)
        {
            double t = t_bb + (t_min < 0.0 ? t_max : t_min);
            D3 q = r.at(t);
            if (!(q.x >= B[0] && q.y >= B[1] && q.z >= B[2] && q.x <= B[3] && q.y <= B[4] && q.z <= B[5])) return false;
            out = Isect(); out.t = t;
            return true;
        }
        return false;
    }

    // Scene::intersect + BVH::intersect (scene.cpp:151-176, bvh.cpp:80-129) with the reference's
    // PriorityQueue push/pop (priority-queue.hpp:19-46,107-126)
    struct NodeHit { double t; uint32_t node; };
    struct Heap
    {
        std::vector<NodeHit> H;
        static bool less(const NodeHit& a, const NodeHit& b) { return b.t < a.t; } // bvh.hpp:78
        void push(NodeHit v)
        {
            H.push_back(v);
            size_t i = H.size() - 1;
            while (i > 0) { size_t p = (i - 1) / 2; if (!less(H[p], v)) break; H[i] = H[p]; i = p; }
            H[i] = v;
        }
        void shiftDown(NodeHit v, size_t i)
        {
            while (true)
            {
                size_t l = 2 * i + 1, r = l + 1, m;
                if (r < H.size()) m = l + (less(H[l], H[r]) ? 1 : 0);
                else if (l < H.size()) m = l;
                else break;
                if (!less(v, H[m])) break;
                H[i] = H[m]; i = m;
            }
            H[i] = v;
        }
        void pop() { if (H.size() > 1) { NodeHit v = H.back(); H.pop_back(); shiftDown(v, 0); } else H.pop_back(); }
    };

    // optional cross-check of every Scene::intersect call of a render against the order-free search (oracle_render_rows_checked)
    struct SearchCheck { const void* nodes; const uint32_t* refs; double scale; uint64_t calls, flagged, mismatches; };
    SearchCheck* g_search_check = nullptr;
    Isect intersectReferenceOrder(const Scene& s, const Ray& r, uint64_t* counter, size_t* peak = nullptr);
    void (*g_cross_fn)(const Scene& s, const Ray& r, const Isect& ref) = nullptr;

    Isect intersect(const Scene& s, const Ray& r, uint64_t* counter)
    {
        Isect is = intersectReferenceOrder(s, r, counter);
        if (g_search_check && g_cross_fn) g_cross_fn(s, r, is);
        return is;
    }

    // peak: largest number of entries the heap held (the device's replay heap has REF_HEAP_CAPACITY of them, intersect.cuh)
    Isect intersectReferenceOrder(const Scene& s, const Ray& r, uint64_t* counter, size_t* peak)
    {
        if (counter) (*counter)++;
        Isect best;
        const uint32_t n_prims = (uint32_t)s.prim_type.size();
        if (s.node_first.empty())
        {
            for (uint32_t i = 0; i < n_prims; i++) { Isect c; if (hitPrim(s, i, r, c) && c.t < best.t) { best = c; best.prim = i; } }
            return best;
        }
        Heap heap;
        double t;
        if (!slab(&s.node_bounds[0], r, t)) return best;
        uint32_t node = 0;
        while (true)
        {
            if (s.node_count[node])
            {
                for (uint32_t i = s.node_first[node]; i < s.node_first[node] + s.node_count[node]; i++)
                {
                    Isect c;
                    if (hitPrim(s, i, r, c) && c.t < best.t) { best = c; best.prim = i; }
                }
            }
            else
            {
                uint32_t child = node + 1;
                while (child != 0)
                {
                    if (slab(&s.node_bounds[6 * child], r, t) && t < best.t) heap.push({ t, child });
                    child = s.node_next[child];
                }
                if (peak) *peak = std::max(*peak, heap.H.size());
            }
            if (heap.H.empty() || heap.H.front().t >= best.t) break;
            node = heap.H.front().node;
            heap.pop();
        }
        return best;
    }

    // ---------------------------------------------------------------- materials (fresnel.cpp, ggx.cpp, material.cpp)
    double fresnelDielectric(double n1, double n2, double c) // fresnel.cpp:16-27
    {
        double g2 = sq(n2 / n1) + sq(c) - 1.0;
        if (g2 < 0.0) return 1.0;
        double g = std::sqrt(g2), gp = g + c, gm = g - c;
        return 0.5 * sq(gm / gp) * (1.0 + sq((gp * c - 1.0) / (gm * c + 1.0)));
    }
    D3 vsqrt(D3 v) { return D3(std::sqrt(v.x), std::sqrt(v.y), std::sqrt(v.z)); }
    D3 adds(D3 v, double s) { return D3(v.x + s, v.y + s, v.z + s); }
    D3 fresnelConductor(double n1, D3 re, D3 im, double c) // fresnel.cpp:30-49
    {
        double c2 = sq(c), s2 = 1.0 - c2;
        D3 er = re / n1, ei = im / n1, eta2 = er * er, etak2 = ei * ei;
        D3 t0 = adds(eta2 - etak2, -s2);
        D3 a2b2 = vsqrt(t0 * t0 + 4.0 * eta2 * etak2);
        D3 t1 = adds(a2b2, c2);
        D3 t2 = (2.0 * c) * vsqrt(0.5 * (a2b2 + t0));
        D3 rs = (t1 - t2) / (t1 + t2);
        D3 t3 = adds(c2 * a2b2, sq(s2)), t4 = t2 * s2;
        D3 rp = rs * (t3 - t4) / (t3 + t4);
        return (rp + rs) * 0.5;
    }
    double ggxD(D3 m, double ax, double ay) { return 1.0 / (PI * ax * ay * sq(sq(m.x / ax) + sq(m.y / ay) + sq(m.z))); }          // ggx.cpp:21-24
    double ggxLambda(D3 w, double ax, double ay) { return (-1.0 + std::sqrt(1.0 + (sq(ax * w.x) + sq(ay * w.y)) / (sq(w.z)))) / 2.0; } // :31-34
    double ggxG1(D3 w, double ax, double ay) { return 1.0 / (1.0 + ggxLambda(w, ax, ay)); }
    double ggxG2(D3 wi, D3 wo, double ax, double ay) { return 1.0 / (1.0 + ggxLambda(wo, ax, ay) + ggxLambda(wi, ax, ay)); }
    double ggxDV(D3 m, D3 wo, double ax, double ay) { return ggxG1(wo, ax, ay) * dot(wo, m) * ggxD(m, ax, ay) / wo.z; }
    double ggxReflection(D3 wi, D3 wo, double ax, double ay, double& pdf) // :46-52
    {
        D3 m = normalize(wo + wi);
        pdf = ggxDV(m, wo, ax, ay) / (4.0 * dot(m, wo));
        return ggxD(m, ax, ay) * ggxG2(wi, wo, ax, ay) / (4.0 * wo.z * wi.z);
    }
    double ggxTransmission(D3 wi, D3 wo, double n1, double n2, double ax, double ay, double& pdf) // :54-65
    {
        D3 m = wo * n1 + wi * n2;
        double l2 = dot(m, m);
        m = m / std::sqrt(l2);
        if (n1 < n2) m = -m;
        double dm = sq(n2) * std::abs(dot(wi, m)) / l2;
        pdf = ggxDV(m, wo, ax, ay) * dm;
        return std::abs(ggxG2(wi, wo, ax, ay) * ggxD(m, ax, ay) * dot(wo, m) * dm / (wo.z * wi.z));
    }
    D3 ggxVisibleMicrofacet(double u, double v, D3 wo, double ax, double ay) // :67-89
    {
        D3 Vh = normalize(D3(ax * wo.x, ay * wo.y, wo.z));
        double len2 = sq(Vh.x) + sq(Vh.y);
        D3 T1 = len2 > 0.0 ? D3(-Vh.y, Vh.x, 0.0) * (1.0 / std::sqrt(len2)) : D3(1.0, 0.0, 0.0);
        D3 T2 = cross(Vh, T1);
        double r = std::sqrt(u), phi = v * TWO_PI;
        double t1 = r * std::cos(phi), t2 = r * std::sin(phi);
        double s = 0.5 * (1.0 + Vh.z);
        t2 = (1.0 - s) * std::sqrt(1.0 - sq(t1)) + s * t2;
        D3 Nh = t1 * T1 + t2 * T2 + std::sqrt(std::max(0.0, 1.0 - sq(t1) - sq(t2))) * Vh;
        return normalize(D3(ax * Nh.x, ay * Nh.y, std::max(0.0, Nh.z)));
    }

    D3 diffuseReflection(const mcrt_material& m, D3 wi, D3 wo, double& pdf) // material.cpp:17-27,76-95
    {
        if (wi.z < 0.0) { pdf = 0.0; return D3(); }
        pdf = wi.z * INV_PI;
        D3 lambert = D3(m.reflectance) * INV_PI;
        if (!m.rough) return lambert;
        double cdp = gmin(gmax((wi.x * wo.x + wi.y * wo.y) / std::sqrt((sq(wi.x) + sq(wi.y)) * (sq(wo.x) + sq(wo.y))), 0.0), 1.0);
        double Dd = std::sqrt((1.0 - sq(wi.z)) * (1.0 - sq(wo.z))) / std::max(wi.z, wo.z);
        return lambert * (m.A + m.B * cdp * Dd);
    }
    D3 specularReflection(const mcrt_material& m, D3 wi, D3 wo, double& pdf) // material.cpp:29-45
    {
        if (wi.z < 0.0) { pdf = 0.0; return D3(); }
        if (m.rough_specular) return D3(m.specular_reflectance) * ggxReflection(wi, wo, m.a[0], m.a[1], pdf);
        pdf = 1.0;
        return D3(m.specular_reflectance) / std::abs(wi.z);
    }
    D3 specularTransmission(const mcrt_material& m, D3 wi, D3 wo, double n1, double n2, double& pdf, bool inside, bool flux) // :47-69
    {
        if (wi.z > 0.0) { pdf = 0.0; return D3(); }
        D3 btdf = !inside ? D3(m.transmittance) : D3(1, 1, 1);
        if (m.rough_specular)
        {
            btdf = btdf * ggxTransmission(wi, wo, n1, n2, m.a[0], m.a[1], pdf);
            if (flux) btdf = btdf * sq(n2 / n1);
        }
        else
        {
            pdf = 1.0;
            btdf = btdf * (D3(m.transmittance) / std::abs(wi.z));
            if (!flux) btdf = btdf * sq(n1 / n2);
        }
        return btdf;
    }

    // ---------------------------------------------------------------- coordinate system (coordinate-system.cpp:7-40)
    struct Frame
    {
        D3 c0, c1, c2;
        Frame() {}
        explicit Frame(D3 N)
        {
            double sign = std::copysign(1.0, N.z), a = -1.0 / (sign + N.z), b = N.x * N.y * a;
            c0 = D3(1.0 + sign * N.x * N.x * a, sign * b, -sign * N.x);
            c1 = D3(b, sign + N.y * N.y * a, -N.y);
            c2 = N;
        }
        D3 from(D3 v) const { return D3(c0.x * v.x + c1.x * v.y + c2.x * v.z, c0.y * v.x + c1.y * v.y + c2.y * v.z, c0.z * v.x + c1.z * v.y + c2.z * v.z); }
        D3 to(D3 v) const { return D3(c0.x * v.x + c0.y * v.y + c0.z * v.z, c1.x * v.x + c1.y * v.y + c1.z * v.z, c2.x * v.x + c2.y * v.y + c2.z * v.z); }
    };

    // ---------------------------------------------------------------- Interaction (interaction.cpp)
    enum { REFLECT, REFRACT, DIFFUSE };
    struct Interaction
    {
        int type; double t, n1, n2, T, R;
        const mcrt_material* material; uint32_t prim;
        D3 position, normal, out; Frame cs; bool inside, dirac_delta; Ray ray;

        D3 bsdfLocal(D3 wo, D3 wi, double& pdf, bool flux, bool wi_dirac) const // interaction.cpp:84-153
        {
            const mcrt_material& m = *material;
            double cos_theta = wo.z;
            if (m.rough_specular)
            {
                if (wi.z > 0.0) cos_theta = dot(wo, normalize(wo + wi));
                else { D3 h = normalize(wo * n1 + wi * n2); cos_theta = dot(wo, h); if (n1 < n2) cos_theta = -cos_theta; }
            }
            if (m.perfect_mirror || m.has_complex_ior)
            {
                D3 brdf = specularReflection(m, wi, wo, pdf);
                if (m.has_complex_ior) brdf = brdf * fresnelConductor(n1, D3(m.complex_ior_real), D3(m.complex_ior_imag), cos_theta);
                return brdf;
            }
            if (n2 < 1.0) return diffuseReflection(m, wi, wo, pdf);
            double F = fresnelDielectric(n1, n2, cos_theta), pdf_s, pdf_d;
            D3 brdf_s = specularReflection(m, wi, wo, pdf_s), brdf_d = diffuseReflection(m, wi, wo, pdf_d);
            double pdf_t = pdf_s; D3 btdf = brdf_s;
            if (F < 1.0) btdf = specularTransmission(m, wi, wo, n1, n2, pdf_t, inside, flux);
            if (wi_dirac)
            {
                if (type == REFLECT) { pdf = R; return brdf_s * F; }
                pdf = T * (1.0 - R); return btdf * T * (1.0 - F);
            }
            else if (!m.rough_specular) { pdf = pdf_d * (1.0 - R) * (1.0 - T); return brdf_d * (1.0 - F) * (1.0 - T); }
            pdf = mixd(mixd(pdf_d, pdf_t, T), pdf_s, R);
            return mix3(mix3(brdf_d, btdf, T), brdf_s, F);
        }
        bool bsdfWorld(D3& f, D3 world_wi, double& pdf) const // interaction.cpp:74-82
        {
            D3 wi = cs.to(world_wi), wo = cs.to(out);
            f = bsdfLocal(wo, wi, pdf, false, false) * std::abs(wi.z);
            return pdf > 0.0;
        }
    };

    D3 primNormal(const Scene& s, uint32_t prim, D3 pos)
    {
        const uint32_t idx = s.prim_index[prim];
        if (s.prim_type[prim] == MCRT_PRIM_TRIANGLE) return D3(&s.tri_n[3 * idx]);
        if (s.prim_type[prim] == MCRT_PRIM_SPHERE) return (pos - D3(&s.sph[4 * idx])) / s.sph[4 * idx + 3];
        const double* G = &s.qG[12 * idx]; // quadric.cpp:129-132, type_mat4x3.inl:474-477
        return normalize(D3(G[0] * pos.x + G[3] * pos.y + G[6] * pos.z + G[9] * 1.0, G[1] * pos.x + G[4] * pos.y + G[7] * pos.z + G[10] * 1.0,
                            G[2] * pos.x + G[5] * pos.y + G[8] * pos.z + G[11] * 1.0));
    }

    Interaction makeInteraction(const Scene& s, const Isect& is, const Ray& ray, double external_ior, const Sampler& smp) // interaction.cpp:12-54,156-183
    {
        Interaction ia;
        ia.t = is.t; ia.ray = ray; ia.out = -ray.direction; ia.n1 = ray.medium_ior; ia.prim = is.prim;
        ia.material = &s.materials[s.prim_material[is.prim]];
        const mcrt_material& m = *ia.material;
        ia.position = ray.at(is.t);
        D3 normal = primNormal(s, is.prim, ia.position);
        double cos_theta = dot(ray.direction, normal);
        ia.inside = cos_theta > 0.0;
        ia.n2 = (ia.inside && !m.opaque) ? external_ior : m.ior;
        D3 sn = normal;
        if (is.interpolate)
        {
            const double* N = &s.vn[9 * s.tri_vn[s.prim_index[is.prim]]];
            sn = normalize((1.0 - is.u - is.v) * D3(N) + is.u * D3(N + 3) + is.v * D3(N + 6)); // triangle.cpp:109-113
            if ((cos_theta < 0.0) != (dot(ray.direction, sn) < 0.0)) sn = normal;
        }
        if (cos_theta > 0.0) { normal = -normal; sn = -sn; }
        ia.normal = normal;
        ia.cs = Frame(sn);
        ia.R = fresnelDielectric(ia.n1, ia.n2, dot(sn, ia.out));
        ia.T = m.transparency;
        if (m.rough_specular) ia.R = gmin(gmax(ia.R, 0.1), 0.9);
        if (m.perfect_mirror || m.has_complex_ior) ia.type = REFLECT;
        else if (ia.n2 < 1.0) ia.type = DIFFUSE;
        else
        {
            double p = smp.get(INTERACTION);
            if (ia.R > p) ia.type = REFLECT;
            else if (ia.R + (1.0 - ia.R) * ia.T > p) ia.type = REFRACT;
            else ia.type = DIFFUSE;
        }
        ia.dirac_delta = ia.type != DIFFUSE && !m.rough_specular;
        return ia;
    }

    Ray spawn(const Interaction& ia, const Sampler& smp) // ray.cpp:16-67
    {
        const mcrt_material& m = *ia.material;
        Ray r;
        r.depth = ia.ray.depth + 1; r.diffuse_depth = ia.ray.diffuse_depth; r.refraction_scale = ia.ray.refraction_scale;
        r.start = ia.position; r.refraction_level = ia.ray.refraction_level; r.dirac_delta = ia.dirac_delta;
        auto specularNormal = [&]() // interaction.cpp:185-193
        {
            if (m.rough_specular) return ia.cs.from(ggxVisibleMicrofacet(smp.get(BSDF), smp.get(BSDF + 1), ia.cs.to(ia.out), m.a[0], m.a[1]));
            return ia.cs.c2;
        };
        if (ia.type == REFLECT)
        {
            D3 n = specularNormal();
            r.direction = ia.ray.direction - n * dot(n, ia.ray.direction) * 2.0; // glm::reflect
            r.medium_ior = ia.n1; r.start = r.start + ia.normal * EPS;
        }
        else if (ia.type == REFRACT)
        {
            D3 n = specularNormal();
            double inv_eta = ia.n1 / ia.n2, c = dot(n, ia.ray.direction), k = 1.0 - sq(inv_eta) * (1.0 - sq(c));
            if (k >= 0.0)
            {
                r.direction = inv_eta * ia.ray.direction - (inv_eta * c + std::sqrt(k)) * n;
                r.medium_ior = ia.n2; r.start = r.start - ia.normal * EPS;
                if (ia.inside) r.refraction_level--; else r.refraction_level++;
                r.refraction_scale *= sq(1.0 / inv_eta);
                r.refraction = true;
            }
            else
            {
                r.direction = ia.ray.direction - n * c * 2.0;
                r.medium_ior = ia.n1; r.start = r.start + ia.normal * EPS;
            }
        }
        else
        {
            r.diffuse_depth++;
            double u = smp.get(BSDF), v = smp.get(BSDF + 1); // Sampling::cosWeightedHemi, sampling.hpp:36-44
            double rr = std::sqrt(u), az = v * TWO_PI;
            r.direction = ia.cs.from(D3(rr * std::cos(az), rr * std::sin(az), std::sqrt(1 - u)));
            r.medium_ior = ia.n1; r.start = r.start + ia.normal * EPS;
        }
        r.inv_direction = D3(1.0 / r.direction.x, 1.0 / r.direction.y, 1.0 / r.direction.z);
        return r;
    }

    // flux: the photon pass's adjoint BSDF (photon-mapper.cpp:259), which keeps the (n2/n1)^2 of rough transmission
    bool sampleBSDF(const Interaction& ia, const Sampler& smp, D3& f, double& pdf, Ray& nr, bool flux = false) // interaction.cpp:56-72
    {
        nr = spawn(ia, smp);
        D3 wi = ia.cs.to(nr.direction);
        if ((nr.refraction && wi.z >= 0.0) || (!nr.refraction && wi.z <= 0.0)) return false;
        D3 wo = ia.cs.to(ia.out);
        f = ia.bsdfLocal(wo, wi, pdf, flux, nr.dirac_delta) * std::abs(wi.z);
        return pdf > 0.0;
    }

    // ---------------------------------------------------------------- integrator (integrator.cpp, path-tracer.cpp)
    struct LightSample { double bsdf_pdf = 0.0, select_probability = 0.0; uint32_t light = 0xFFFFFFFFu; };

    D3 lightPoint(const Scene& s, uint32_t prim, double u, double v)
    {
        const uint32_t idx = s.prim_index[prim];
        if (s.prim_type[prim] == MCRT_PRIM_TRIANGLE) // triangle.cpp:93-97
        {
            double su = std::sqrt(u);
            return (1 - su) * D3(&s.tri_v0[3 * idx]) + (1 - v) * su * D3(&s.tri_v1[3 * idx]) + v * su * D3(&s.tri_v2[3 * idx]);
        }
        const double* sp = &s.sph[4 * idx]; // sphere.cpp:37-44
        double z = 1.0 - 2.0 * u, r = std::sqrt(1.0 - sq(z)), phi = TWO_PI * v;
        return D3(sp) + sp[3] * D3(r * std::cos(phi), r * std::sin(phi), z);
    }

    double powerHeuristic(double a, double b) { double a2 = a * a; return a2 / (a2 + b * b); } // util.hpp:85-89

    D3 sampleDirect(const Scene& s, const Interaction& ia, LightSample& ls, const Sampler& smp, uint64_t* rays) // integrator.cpp:31-87
    {
        if (s.light_prim.empty() || ia.material->dirac_delta) { ls.light = 0xFFFFFFFFu; return D3(); }
        double u0 = smp.get(LIGHT), u1 = smp.get(LIGHT + 1), u2 = smp.get(LIGHT + 2);
        size_t left = 0, right = s.light_cdf.size() - 1; // sampling.hpp:13-28
        while (left < right) { size_t mid = (left + right) / 2; if (s.light_cdf[mid] < u2) left = mid + 1; else right = mid; }
        ls.select_probability = s.light_cdf[left];
        if (left > 0) ls.select_probability -= s.light_cdf[left - 1];
        ls.light = s.light_prim[left];
        D3 light_pos = lightPoint(s, ls.light, u0, u1);
        Ray shadow = rayTo(ia.position + ia.normal * EPS, light_pos);
        double cos_light = dot(-shadow.direction, primNormal(s, ls.light, light_pos));
        if (cos_light <= 0.0) return D3();
        double cos_theta = dot(shadow.direction, ia.normal);
        if (cos_theta <= 0.0)
        {
            if (ia.material->opaque || cos_theta == 0.0) return D3();
            shadow = rayTo(ia.position - ia.normal * EPS, light_pos);
        }
        Isect si = intersect(s, shadow, rays);
        if (si.prim == 0xFFFFFFFFu || si.prim != ls.light) return D3();
        double light_pdf = sq(si.t) / (s.prim_area[ls.light] * cos_light);
        double bsdf_pdf; D3 f;
        if (!ia.bsdfWorld(f, shadow.direction, bsdf_pdf)) return D3();
        double w = powerHeuristic(light_pdf, bsdf_pdf);
        return w * f * D3(s.materials[s.prim_material[ls.light]].emittance) / (light_pdf * ls.select_probability);
    }

    D3 sampleEmissive(const Scene& s, const Interaction& ia, const LightSample& ls) // integrator.cpp:93-110
    {
        if (ia.material->emissive && !ia.inside)
        {
            if (ia.ray.depth == 0 || ia.ray.dirac_delta) return D3(ia.material->emittance);
            if (ls.light == ia.prim)
            {
                double cos_light = dot(ia.out, ia.normal);
                double light_pdf = sq(ia.t) / (s.prim_area[ia.prim] * cos_light);
                double w = powerHeuristic(ls.bsdf_pdf, light_pdf);
                return w * D3(ia.material->emittance) / ls.select_probability;
            }
        }
        return D3();
    }

    D3 skyColor(const Ray& r) // scene.cpp:219-223
    {
        double fy = (1.0 + std::asin(0.0 * r.direction.x + 1.0 * r.direction.y + 0.0 * r.direction.z) / PI) / 2.0;
        return mix3(D3(1.0, 0.5, 0.0), D3(0.0, 0.5, 1.0), fy);
    }

    D3 sampleRay(const Scene& s, Ray ray, Sampler& smp, uint64_t* rays) // path-tracer.cpp:14-51
    {
        D3 radiance, throughput(1, 1, 1);
        std::vector<double> iors(1, ray.medium_ior); // RefractionHistory, ray.cpp:74-98
        LightSample ls;
        while (true)
        {
            smp.shuffle();
            Isect is = intersect(s, ray, rays);
            if (is.prim == 0xFFFFFFFFu) return radiance + skyColor(ray) * throughput;
            int ext = std::min(std::max(ray.refraction_level - 1, 0), (int)iors.size() - 1);
            Interaction ia = makeInteraction(s, is, ray, iors[ext], smp);
            radiance = radiance + sampleEmissive(s, ia, ls) * throughput;
            radiance = radiance + sampleDirect(s, ia, ls, smp, rays) * throughput;
            D3 f;
            if (!sampleBSDF(ia, smp, f, ls.bsdf_pdf, ray)) return radiance;
            throughput = throughput * (f / ls.bsdf_pdf);
            // Integrator::absorb, integrator.cpp:112-129
            double survive = compMax(throughput) * ray.refraction_scale;
            if (survive == 0.0) return radiance;
            if (ray.diffuse_depth > 3 || ray.depth > 16)
            {
                survive = std::min(0.95, survive);
                if (survive <= smp.get(ABSORB)) return radiance;
                throughput = throughput / survive;
            }
            if (ray.refraction_level > 0) // RefractionHistory::update
            {
                if (ray.refraction_level == (int)iors.size()) iors.push_back(ray.medium_ior);
                else if (ray.refraction_level < (int)iors.size() - 1) iors.pop_back();
            }
        }
    }

    Ray cameraRay(const mcrt_camera& c, double scene_ior, uint32_t pixel, const Sampler& smp) // camera.cpp:66-95
    {
        const size_t x = pixel % c.width, y = pixel / c.width;
        double pixel_size = c.sensor_width / c.width;
        double px = x + smp.get(PIXEL), py = y + smp.get(PIXEL + 1);
        double lx = pixel_size * (c.width * 0.5 - px), ly = pixel_size * (c.height * 0.5 - py);
        D3 dir = normalize(D3(c.forward) * c.focal_length + D3(c.left) * lx + D3(c.up) * ly);
        Ray ray = makeRay(D3(c.eye), dir, scene_ior);
        if (c.thin_lens)
        {
            double u = smp.get(LENS), v = smp.get(LENS + 1), az = v * TWO_PI;
            double ax = (std::cos(az) * std::sqrt(u)) * c.aperture_radius, ay = (std::sin(az) * std::sqrt(u)) * c.aperture_radius;
            D3 focus = ray.at(c.focus_distance / dot(ray.direction, D3(c.forward)));
            D3 start = D3(c.eye) + D3(c.left) * ax + D3(c.up) * ay;
            ray = makeRay(start, normalize(focus - start), scene_ior);
        }
        return ray;
    }
}

extern "C"
{

void* oracle_scene_create(const mcrt_scene_desc* d)
{
    Scene* s = new Scene();
    s->d = *d;
    copyv(s->node_bounds, d->node_bounds, 6 * (size_t)d->n_nodes);
    copyv(s->node_first, d->node_first_prim, d->n_nodes); copyv(s->node_count, d->node_prim_count, d->n_nodes);
    copyv(s->node_next, d->node_next_sibling, d->n_nodes);
    copyv(s->prim_type, d->prim_type, d->n_prims); copyv(s->prim_index, d->prim_index, d->n_prims);
    copyv(s->prim_material, d->prim_material, d->n_prims); copyv(s->prim_area, d->prim_area, d->n_prims);
    copyv(s->tri_v0, d->tri_v0, 3 * (size_t)d->n_tris); copyv(s->tri_v1, d->tri_v1, 3 * (size_t)d->n_tris);
    copyv(s->tri_v2, d->tri_v2, 3 * (size_t)d->n_tris); copyv(s->tri_e1, d->tri_e1, 3 * (size_t)d->n_tris);
    copyv(s->tri_e2, d->tri_e2, 3 * (size_t)d->n_tris); copyv(s->tri_n, d->tri_normal, 3 * (size_t)d->n_tris);
    copyv(s->tri_vn, d->tri_vn_index, d->n_tris); copyv(s->vn, d->vertex_normals, 9 * (size_t)d->n_vertex_normals);
    copyv(s->sph, d->sphere_origin_radius, 4 * (size_t)d->n_spheres);
    copyv(s->qQ, d->quadric_Q, 16 * (size_t)d->n_quadrics); copyv(s->qG, d->quadric_G, 12 * (size_t)d->n_quadrics);
    copyv(s->qB, d->quadric_bounds, 6 * (size_t)d->n_quadrics);
    copyv(s->materials, d->materials, d->n_materials);
    copyv(s->light_prim, d->light_prim, d->n_lights); copyv(s->light_cdf, d->light_cdf, d->n_lights);
    return s;
}

void oracle_scene_destroy(void* h) { delete static_cast<Scene*>(h); }

void oracle_sampler_stream(const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t n_shuffles, uint32_t seed, uint32_t* out)
{
    Sampler smp(seed);
    for (size_t i = 0; i < n; i++)
    {
        smp.initiate(pixel[i]); smp.setIndex(sample[i]);
        for (uint32_t k = 0; k < n_shuffles; k++) smp.shuffle();
        for (int d = 0; d < 7; d++) out[7 * i + d] = smp.raw(d);
    }
}

void oracle_trace(void* h, const mcrt_ray* rays, size_t n, mcrt_hit* hits)
{
    const Scene& s = *static_cast<Scene*>(h);
    for (size_t i = 0; i < n; i++)
    {
        Isect is = intersect(s, makeRay(D3(rays[i].origin), D3(rays[i].direction), s.d.scene_ior), nullptr);
        hits[i].t = is.t; hits[i].u = is.u; hits[i].v = is.v; hits[i].prim = is.prim; hits[i].interpolate = is.interpolate;
    }
}

// CPU restatement of the product's order-free closest-hit search (monte-carlo-ray-tracer_b200/csrc/bvh4.cuh: FastRay, FastSearch,
// ambiguityDelta) over the 4-wide float-box BVH the product derives from the scene (passed in: mcrt_bvh4_host). Same float32 slab
// arithmetic - fmaf and single multiplications are IEEE operations on both sides -, same margins, same pruning limit, the oracle's own
// float64 primitive tests (which equal the reference's). flags[i]: 1 = the search declares the ray ambiguous (the product then replays it
// in the reference's order), 0 = the search's answer is final. tests/test_fast_search_cpu.py: final answers == reference-order answers.
namespace
{
    struct Node4 { float lo[3][4], hi[3][4]; uint32_t child[4], pad[4]; };

    double ambiguityDelta(double t, double scale) { return 1e-6 * t + 1e-12 * scale; }

    float roundUpToFloat(double v) { float f = (float)v; if ((double)f < v) f = std::nextafterf(f, INFINITY); return f; }   // __double2float_ru

    // barycentrics of a triangle hit whatever the triangle's shading mode (hitPrim reports them for smooth triangles only)
    bool hitPrimUV(const Scene& s, uint32_t prim, const Ray& r, Isect& out, double& u, double& v)
    {
        if (!hitPrim(s, prim, r, out)) return false;
        if (s.prim_type[prim] == MCRT_PRIM_TRIANGLE)
        {
            const uint32_t idx = s.prim_index[prim];
            D3 v0(&s.tri_v0[3 * idx]), E1(&s.tri_e1[3 * idx]), E2(&s.tri_e2[3 * idx]);
            D3 P = cross(r.direction, E2);
            double inv = 1.0 / dot(P, E1);
            D3 T = r.start - v0;
            u = dot(P, T) * inv;
            v = dot(cross(T, E1), r.direction) * inv;
        }
        return true;
    }
    bool onBoundary(double u, double v, double t, double scale) { const double e = 1e-9 * std::fmax(1.0, t / scale); return u < e || v < e || u + v > 1.0 - e; }
    bool degenerateDirection(const Ray& r)
    {
        const double e = 1e-12;
        return std::fabs(r.direction.x) < e || std::fabs(r.direction.y) < e || std::fabs(r.direction.z) < e;
    }

    // FastRay (bvh4.cuh) restated: 1 / d and o / d raised and lowered for the near and far planes
    struct FastRay4 { float id[3], on[3], of[3]; };
    // MCRT_FAST_STACK (bvh4.cuh) of the default build: a ray that needs more entries is replayed. The peaks below are those of the
    // default walk (MCRT_SPECULATIVE = 0); the speculative form visits more nodes and can hold more entries.
    constexpr size_t kFastStack = 40;
    FastRay4 fastRay(const Ray& r)
    {
        auto inv = [](double v) { float f = (float)v; if (!(std::fabs(f) >= 1e-18f)) f = std::copysign(1e-18f, f); return 1.0f / f; };
        FastRay4 f;
        f.id[0] = inv(r.direction.x); f.id[1] = inv(r.direction.y); f.id[2] = inv(r.direction.z);
        const float od[3] = { (float)r.start.x * f.id[0], (float)r.start.y * f.id[1], (float)r.start.z * f.id[2] };
        for (int k = 0; k < 3; k++) { const float m = std::fabs(od[k]) * 1.9073486e-6f; f.on[k] = od[k] + m; f.of[k] = od[k] - m; }
        return f;
    }

    // FastSearch::step / visitNode / pop (bvh4.cuh) restated with an unbounded stack: depth first, nearest child next, the other hit
    // children pushed farthest first, entries culled against `limit` on pop. leaf(ref) tests a leaf and may lower `limit`; it returns
    // false to end the search. peak: the largest number of pending entries (the device's stack holds FAST_STACK of them).
    extern "C++" template <class Leaf>
    void walkFast(const Node4* nodes, const FastRay4& f, const float& limit, Leaf leaf, uint64_t& box_tests, size_t& peak)
    {
        struct Entry { uint32_t ref; float tn; };
        std::vector<Entry> stack;
        uint32_t cur = 0;
        auto pop = [&]() { while (!stack.empty()) { Entry e = stack.back(); stack.pop_back(); if (e.tn <= limit) { cur = e.ref; return true; } } return false; };
        while (true)
        {
            bool have = true;
            while (!(cur & 0x80000000u))
            {
                const Node4& n = nodes[cur];
                box_tests += 4;
                uint32_t key[4];
                for (int c = 0; c < 4; c++)
                {
                    float tn = 0.0f, tf = INFINITY;
                    for (int k = 0; k < 3; k++)
                    {
                        const float bn = f.id[k] < 0.0f ? n.hi[k][c] : n.lo[k][c], bf = f.id[k] < 0.0f ? n.lo[k][c] : n.hi[k][c];
                        tn = std::fmax(tn, std::fmaf(bn, f.id[k], -f.on[k]));
                        tf = std::fmin(tf, std::fmaf(bf, f.id[k], -f.of[k]));
                    }
                    tn *= 0.99999619f; tf *= 1.00000381f;
                    const bool hit = n.child[c] != 0u && tn <= tf && tn <= limit;
                    uint32_t bits; std::memcpy(&bits, &tn, 4);
                    key[c] = hit ? ((bits & 0x7FFFFFFCu) | (uint32_t)c) : 0xFFFFFFFFu;
                }
                std::sort(key, key + 4);
                if (key[0] == 0xFFFFFFFFu) { if (!pop()) { have = false; break; } continue; }
                for (int j = 3; j >= 1; j--)
                    if (key[j] != 0xFFFFFFFFu) { const uint32_t b = key[j] & ~3u; float tn; std::memcpy(&tn, &b, 4); stack.push_back({ n.child[key[j] & 3u], tn }); }
                peak = std::max(peak, stack.size());
                cur = n.child[key[0] & 3u];
            }
            if (!have) break;
            if (!leaf(cur)) break;
            if (!pop()) break;
        }
    }

    // refs: the ordered primitive of each leaf reference (a tree with spatial splits, mcrt_bvh4_split_host); null: leaves index ordered
    // primitives. A primitive with several references gives the same t at each: a repeat of the best primitive is not its competitor
    // (FastSearch::testLeaf).
    Isect searchFast(const Scene& s, const Node4* nodes, const uint32_t* refs, const Ray& r, double scene_scale, bool& ambiguous, uint64_t& box_tests,
                     uint64_t& prim_tests, size_t* peak = nullptr)
    {
        const FastRay4 f = fastRay(r);
        Isect best;
        bool best_edge = false;
        double second_t = std::numeric_limits<double>::max();
        float limit = INFINITY;
        size_t stack_peak = 0;
        walkFast(nodes, f, limit, [&](uint32_t cur)
        {
            const uint32_t first = (cur >> 8) & 0x7FFFFFu, count = cur & 0xFFu;
            for (uint32_t i = first; i < first + count; i++)
            {
                const uint32_t prim = refs ? refs[i] : i;
                Isect c;
                prim_tests++;
                double eu = 0.5, ev = 0.25;
                if (hitPrimUV(s, prim, r, c, eu, ev))
                {
                    if (c.t < best.t) { second_t = best.t; best = c; best.prim = prim; best_edge = onBoundary(eu, ev, c.t, scene_scale); limit = roundUpToFloat(c.t + 2.0 * ambiguityDelta(c.t, scene_scale)); }
                    else if (c.t < second_t && !(c.t == best.t && prim == best.prim)) second_t = c.t;
                }
            }
            return true;
        }, box_tests, stack_peak);
        if (peak) *peak = stack_peak;
        ambiguous = best.prim != 0xFFFFFFFFu && second_t <= best.t + ambiguityDelta(best.t, scene_scale);
        if (best.prim != 0xFFFFFFFFu && best_edge) ambiguous = true;      // R2: the winner is hit on its boundary
        if (degenerateDirection(r)) ambiguous = true;                     // R1: a direction component is (nearly) zero
        if (stack_peak > kFastStack) ambiguous = true;                    // R3: the device's stack is full (FastSearch::push)
        return best;
    }
}

// FastSearch<PRIMS, true> (csrc/bvh4.cuh): occlusion query of next-event estimation. verdict 0: the target is the closest hit (t in *t),
// 1: something lies in front of it (or the ray misses the target itself), 2: a tie within delta -> the product replays the ray.
namespace
{
    int searchVisible(const Scene& s, const Node4* nodes, const uint32_t* refs, const Ray& r, double scene_scale, uint32_t target, double& t_target)
    {
        Isect tgt;
        double tu = 0.5, tv = 0.25;
        if (!hitPrimUV(s, target, r, tgt, tu, tv)) return 1;
        t_target = tgt.t;
        if (degenerateDirection(r) || onBoundary(tu, tv, tgt.t, scene_scale)) return 2;
        auto inv = [](double v) { float f = (float)v; if (!(std::fabs(f) >= 1e-18f)) f = std::copysign(1e-18f, f); return 1.0f / f; };
        const float id[3] = { inv(r.direction.x), inv(r.direction.y), inv(r.direction.z) };
        const float od[3] = { (float)r.start.x * id[0], (float)r.start.y * id[1], (float)r.start.z * id[2] };
        float on[3], of[3];
        for (int k = 0; k < 3; k++) { const float m = std::fabs(od[k]) * 1.9073486e-6f; on[k] = od[k] + m; of[k] = od[k] - m; }
        const double delta = ambiguityDelta(tgt.t, scene_scale);
        const float limit = roundUpToFloat(tgt.t + 2.0 * delta);
        std::vector<uint32_t> stack(1, 0u);
        while (!stack.empty())
        {
            const uint32_t cur = stack.back(); stack.pop_back();
            if (cur & 0x80000000u)
            {
                const uint32_t first = (cur >> 8) & 0x7FFFFFu, count = cur & 0xFFu;
                for (uint32_t i = first; i < first + count; i++)
                {
                    const uint32_t prim = refs ? refs[i] : i;
                    if (prim == target) continue;      // every reference of the target, by its ordered id
                    Isect c;
                    double cu = 0.5, cv = 0.25;
                    if (hitPrimUV(s, prim, r, c, cu, cv))
                    {
                        if (c.t <= tgt.t + delta && onBoundary(cu, cv, c.t, scene_scale)) return 2;   // an occluder hit on its edge: the reference may have missed it
                        if (c.t < tgt.t - delta) return 1;
                        if (c.t <= tgt.t + delta) return 2;
                    }
                }
                continue;
            }
            const Node4& n = nodes[cur];
            for (int c = 0; c < 4; c++)
            {
                float tn = 0.0f, tf = INFINITY;
                for (int k = 0; k < 3; k++)
                {
                    const float bn = id[k] < 0.0f ? n.hi[k][c] : n.lo[k][c], bf = id[k] < 0.0f ? n.lo[k][c] : n.hi[k][c];
                    tn = std::fmax(tn, std::fmaf(bn, id[k], -on[k]));
                    tf = std::fmin(tf, std::fmaf(bf, id[k], -of[k]));
                }
                tn *= 0.99999619f; tf *= 1.00000381f;
                if (n.child[c] != 0u && tn <= tf && tn <= limit) stack.push_back(n.child[c]);   // the verdict does not depend on the visiting order
            }
        }
        return 0;
    }
}

// FastSearch<PRIMS, true> in the device's visiting order (walkFast): the verdict and the largest number of pending stack entries. The
// verdict equals searchVisible's unless a ray holds both an occluder and a tie (either is a correct verdict: both keep the reference's answer).
namespace
{
    int searchVisibleOrdered(const Scene& s, const Node4* nodes, const uint32_t* refs, const Ray& r, double scene_scale, uint32_t target, double& t_target,
                             size_t& peak)
    {
        Isect tgt;
        double tu = 0.5, tv = 0.25;
        peak = 0;
        if (!hitPrimUV(s, target, r, tgt, tu, tv)) return 1;
        t_target = tgt.t;
        if (degenerateDirection(r) || onBoundary(tu, tv, tgt.t, scene_scale)) return 2;
        const double delta = ambiguityDelta(tgt.t, scene_scale);
        const float limit = roundUpToFloat(tgt.t + 2.0 * delta);
        int verdict = 0;
        uint64_t box_tests = 0;
        walkFast(nodes, fastRay(r), limit, [&](uint32_t cur)
        {
            const uint32_t first = (cur >> 8) & 0x7FFFFFu, count = cur & 0xFFu;
            for (uint32_t i = first; i < first + count; i++)
            {
                const uint32_t prim = refs ? refs[i] : i;
                if (prim == target) continue;
                Isect c;
                double cu = 0.5, cv = 0.25;
                if (hitPrimUV(s, prim, r, c, cu, cv))
                {
                    if (c.t <= tgt.t + delta && onBoundary(cu, cv, c.t, scene_scale)) { verdict = 2; return false; }
                    if (c.t < tgt.t - delta) { verdict = 1; return false; }
                    if (c.t <= tgt.t + delta) { verdict = 2; return false; }
                }
            }
            return true;
        }, box_tests, peak);
        return verdict == 0 && peak > kFastStack ? 2 : verdict;     // a full stack hands the ray to the replay unless an occluder was found
    }
}

void oracle_trace_visible(void* h, const void* nodes128, const uint32_t* refs, double scene_scale, const mcrt_ray* rays, const uint32_t* target,
                          size_t n, uint8_t* verdict, double* t_target)
{
    const Scene& s = *static_cast<Scene*>(h);
    for (size_t i = 0; i < n; i++)
    {
        double t = 0.0;
        verdict[i] = (uint8_t)searchVisible(s, static_cast<const Node4*>(nodes128), refs, makeRay(D3(rays[i].origin), D3(rays[i].direction), s.d.scene_ior), scene_scale, target[i], t);
        t_target[i] = t;
    }
}

namespace
{
    void crossCheckImpl(const Scene& s, const Ray& r, const Isect& ref)
    {
        SearchCheck& c = *g_search_check;
        bool amb = false; uint64_t bt = 0, pt = 0;
        Isect f = searchFast(s, static_cast<const Node4*>(c.nodes), c.refs, r, c.scale, amb, bt, pt);
        c.calls++;
        if (amb) { c.flagged++; return; }
        if (f.prim != ref.prim || (ref.prim != 0xFFFFFFFFu && (f.t != ref.t || f.u != ref.u || f.v != ref.v))) c.mismatches++;
    }
}

// A whole render (rows [y0, y1)) by the restated path tracer, with EVERY Scene::intersect call - camera, bounce and shadow rays - also
// answered by the order-free search over `nodes128`: counts[0] calls, counts[1] flagged (would be replayed), counts[2] unflagged answers
// that differ from the reference-order answer (must be 0).
void oracle_render_rows(void* h, const mcrt_camera* cam, uint32_t y0, uint32_t y1, uint32_t sqrtspp, uint32_t seed, double* out, uint64_t* rays);
void oracle_render_rows_checked(void* h, const void* nodes128, const uint32_t* refs, double scene_scale, const mcrt_camera* cam, uint32_t y0,
                                uint32_t y1, uint32_t sqrtspp, uint32_t seed, double* out, uint64_t* counts)
{
    SearchCheck c{ nodes128, refs, scene_scale, 0, 0, 0 };
    g_search_check = &c;
    g_cross_fn = crossCheckImpl;
    uint64_t rays = 0;
    oracle_render_rows(h, cam, y0, y1, sqrtspp, seed, out, &rays);
    g_search_check = nullptr;
    counts[0] = c.calls; counts[1] = c.flagged; counts[2] = c.mismatches;
}

void oracle_trace_fast(void* h, const void* nodes128, uint32_t n_nodes, const uint32_t* refs, double scene_scale, const mcrt_ray* rays, size_t n,
                       mcrt_hit* hits, uint8_t* flags, uint64_t* box_tests, uint64_t* prim_tests)
{
    const Scene& s = *static_cast<Scene*>(h);
    (void)n_nodes;
    uint64_t bt = 0, pt = 0;
    for (size_t i = 0; i < n; i++)
    {
        bool amb = false;
        Isect is = searchFast(s, static_cast<const Node4*>(nodes128), refs, makeRay(D3(rays[i].origin), D3(rays[i].direction), s.d.scene_ior), scene_scale, amb, bt, pt);
        hits[i].t = is.t; hits[i].u = is.u; hits[i].v = is.v; hits[i].prim = is.prim; hits[i].interpolate = is.interpolate;
        flags[i] = amb ? 1 : 0;
    }
    if (box_tests) *box_tests = bt;
    if (prim_tests) *prim_tests = pt;
}

// Peaks of the traversal structures per ray. oracle_trace_peaks: the reference-order traversal (hits as oracle_trace) and the largest
// size of its heap. oracle_trace_fast_peaks: the order-free search (hits and flags as oracle_trace_fast) and the largest size of its
// stack. oracle_trace_visible_peaks: the occlusion query in the device's visiting order (verdict, t of the target, largest stack size).
void oracle_trace_peaks(void* h, const mcrt_ray* rays, size_t n, mcrt_hit* hits, uint32_t* heap_peak)
{
    const Scene& s = *static_cast<Scene*>(h);
    for (size_t i = 0; i < n; i++)
    {
        size_t peak = 0;
        Isect is = intersectReferenceOrder(s, makeRay(D3(rays[i].origin), D3(rays[i].direction), s.d.scene_ior), nullptr, &peak);
        hits[i].t = is.t; hits[i].u = is.u; hits[i].v = is.v; hits[i].prim = is.prim; hits[i].interpolate = is.interpolate;
        heap_peak[i] = (uint32_t)peak;
    }
}

void oracle_trace_fast_peaks(void* h, const void* nodes128, const uint32_t* refs, double scene_scale, const mcrt_ray* rays, size_t n, mcrt_hit* hits,
                             uint8_t* flags, uint32_t* stack_peak)
{
    const Scene& s = *static_cast<Scene*>(h);
    uint64_t bt = 0, pt = 0;
    for (size_t i = 0; i < n; i++)
    {
        bool amb = false;
        size_t peak = 0;
        Isect is = searchFast(s, static_cast<const Node4*>(nodes128), refs, makeRay(D3(rays[i].origin), D3(rays[i].direction), s.d.scene_ior), scene_scale, amb, bt, pt,
                             &peak);
        hits[i].t = is.t; hits[i].u = is.u; hits[i].v = is.v; hits[i].prim = is.prim; hits[i].interpolate = is.interpolate;
        flags[i] = amb ? 1 : 0;
        stack_peak[i] = (uint32_t)peak;
    }
}

// An upper bound, per ray, on the entries of fast mode's depth-first stack (traverseWide, intersect.cuh). That walk pushes every hit
// child of a visited node but the nearest, so its stack never holds more than the largest sum of (hit children - 1) over the nodes of
// one path of boxes the ray hits. Fast mode rounds the ray and the boxes to float and prunes by its best hit; boxes grown by `margin` on
// every side cover the rounding, and pruning only removes entries. The bound does not depend on the visiting order.
namespace
{
    uint32_t widePathBound(const Scene& s, const Ray& r, double margin, uint32_t node)
    {
        if (s.node_count[node]) return 0;
        uint32_t hits = 0, deepest = 0;
        for (uint32_t child = node + 1; child != 0; child = s.node_next[child])
        {
            const double* b = &s.node_bounds[6 * child];
            double tn = 0.0, tf = INFINITY;
            for (int k = 0; k < 3; k++)
            {
                const double o = k == 0 ? r.start.x : k == 1 ? r.start.y : r.start.z, d = k == 0 ? r.direction.x : k == 1 ? r.direction.y : r.direction.z;
                const double t0 = (b[k] - margin - o) / d, t1 = (b[3 + k] + margin - o) / d;
                tn = std::fmax(tn, std::fmin(t0, t1)); tf = std::fmin(tf, std::fmax(t0, t1));
            }
            if (tn > tf) continue;       // NaN (a zero direction component on a plane) counts as a hit
            hits++;
            deepest = std::max(deepest, widePathBound(s, r, margin, child));
        }
        return hits ? hits - 1 + deepest : 0;
    }
}

void oracle_wide_stack_bound(void* h, const mcrt_ray* rays, size_t n, double margin, uint32_t* bound)
{
    const Scene& s = *static_cast<Scene*>(h);
    for (size_t i = 0; i < n; i++)
        bound[i] = s.node_first.empty() ? 0u : widePathBound(s, makeRay(D3(rays[i].origin), D3(rays[i].direction), s.d.scene_ior), margin, 0);
}

void oracle_trace_visible_peaks(void* h, const void* nodes128, const uint32_t* refs, double scene_scale, const mcrt_ray* rays, const uint32_t* target,
                                size_t n, uint8_t* verdict, double* t_target, uint32_t* stack_peak)
{
    const Scene& s = *static_cast<Scene*>(h);
    for (size_t i = 0; i < n; i++)
    {
        double t = 0.0;
        size_t peak = 0;
        verdict[i] = (uint8_t)searchVisibleOrdered(s, static_cast<const Node4*>(nodes128), refs, makeRay(D3(rays[i].origin), D3(rays[i].direction), s.d.scene_ior),
                                                   scene_scale, target[i], t, peak);
        t_target[i] = t;
        stack_peak[i] = (uint32_t)peak;
    }
}

void oracle_sample_rays(void* h, const mcrt_ray* rays, const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t seed, double* out)
{
    const Scene& s = *static_cast<Scene*>(h);
    Sampler smp(seed);
    for (size_t i = 0; i < n; i++)
    {
        smp.initiate(pixel[i]); smp.setIndex(sample[i]);
        D3 r = sampleRay(s, makeRay(D3(rays[i].origin), D3(rays[i].direction), s.d.scene_ior), smp, nullptr);
        out[3 * i] = r.x; out[3 * i + 1] = r.y; out[3 * i + 2] = r.z;
    }
}

// Camera::samplePixel over rows [y0,y1) with the default box film (film.cpp:106-113)
void oracle_render_rows(void* h, const mcrt_camera* cam, uint32_t y0, uint32_t y1, uint32_t sqrtspp, uint32_t seed, double* out, uint64_t* rays)
{
    const Scene& s = *static_cast<Scene*>(h);
    Sampler smp(seed);
    uint64_t count = 0;
    const uint32_t spp = sqrtspp * sqrtspp;
    for (uint32_t y = y0; y < y1; y++)
        for (uint32_t x = 0; x < cam->width; x++)
        {
            const uint32_t pixel = y * cam->width + x;
            smp.initiate(pixel);
            double sum[3] = { 0, 0, 0 };
            for (uint32_t i = 0; i < spp; i++)
            {
                smp.setIndex(i);
                D3 r = sampleRay(s, cameraRay(*cam, s.d.scene_ior, pixel, smp), smp, &count);
                sum[0] += r.x * 1.0; sum[1] += r.y * 1.0; sum[2] += r.z * 1.0; // Film::Splat::update, weight 1
            }
            double* o = out + ((size_t)(y - y0) * cam->width + x) * 3;
            for (int k = 0; k < 3; k++) { double v = sum[k] / (double)spp; o[k] = (v < 0.0) ? 0.0 : v; }
        }
    if (rays) *rays = count;
}

// Camera::samplePixel's body for individual (pixel, sample) pairs: the camera ray and the radiance
// Integrator::sampleRay returns for it (what oracle/ref.py's sample_pixels asks of the reference)
void oracle_sample_pixels(void* h, const mcrt_camera* cam, const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t seed,
                          double* out_rgb, double* out_rays6)
{
    const Scene& s = *static_cast<Scene*>(h);
    Sampler smp(seed);
    for (size_t i = 0; i < n; i++)
    {
        smp.initiate(pixel[i]);
        smp.setIndex(sample[i]);
        const Ray ray = cameraRay(*cam, s.d.scene_ior, pixel[i], smp);
        if (out_rays6)
        {
            out_rays6[6 * i + 0] = ray.start.x; out_rays6[6 * i + 1] = ray.start.y; out_rays6[6 * i + 2] = ray.start.z;
            out_rays6[6 * i + 3] = ray.direction.x; out_rays6[6 * i + 4] = ray.direction.y; out_rays6[6 * i + 5] = ray.direction.z;
        }
        const D3 r = sampleRay(s, ray, smp, nullptr);
        out_rgb[3 * i + 0] = r.x; out_rgb[3 * i + 1] = r.y; out_rgb[3 * i + 2] = r.z;
    }
}

// Film with a reconstruction filter (film.cpp:19-113, filter.hpp:8-66), whole frame. `film` is the
// camera's "film" object after Film::Film resolved the default radius.
namespace
{
    double mitchell(double B, double Cc, double x) // filter.hpp:15-38
    {
        const double k = 6.0 / (6.0 - 2.0 * B);
        if (x < 1.0)
        {
            const double a = k * (12.0 - 9.0 * B - 6.0 * Cc) / 6.0;
            const double b = k * (-18.0 + 12.0 * B + 6.0 * Cc) / 6.0;
            const double d = k * (6.0 - 2.0 * B) / 6.0;
            return d + (b + a * x) * x * x;
        }
        const double a = k * (-B - 6.0 * Cc) / 6.0;
        const double b = k * (6.0 * B + 30.0 * Cc) / 6.0;
        const double c = k * (-12.0 * B - 48.0 * Cc) / 6.0;
        const double d = k * (8.0 * B + 24.0 * Cc) / 6.0;
        return d + (c + (b + a * x) * x) * x;
    }

    double filterFunction(uint32_t filter, double x) // film.cpp:32-45
    {
        switch (filter)
        {
            case MCRT_FILM_MITCHELL_NETRAVALI: return mitchell(1.0 / 3.0, 1.0 / 3.0, x);
            case MCRT_FILM_CATMULL_ROM: return mitchell(0.0, 0.5, x);
            case MCRT_FILM_B_SPLINE: return mitchell(1.0, 0.0, x);
            case MCRT_FILM_HERMITE: return mitchell(0.0, 0.0, x * 0.5);
            case MCRT_FILM_GAUSSIAN: return std::exp(-2.0 * x * x) - std::exp(-2.0 * 2.0 * 2.0);
            case MCRT_FILM_LANCZOS:
                if (x == 0.0) return 1.0;
                return 2.0 * std::sin(PI * x) * std::sin(PI * x / 2.0) / (PI * PI * x * x);
            default: return 1.0;
        }
    }
}

void oracle_render_film(void* h, const mcrt_camera* cam, const mcrt_film* film, uint32_t sqrtspp, uint32_t seed, double* out)
{
    const Scene& s = *static_cast<Scene*>(h);
    Sampler smp(seed);
    const uint32_t spp = sqrtspp * sqrtspp;
    const int64_t W = cam->width, H = cam->height;
    const double radius = film->radius;
    std::vector<double> cache(film->cache_size);
    for (uint32_t i = 0; i < film->cache_size; i++) cache[i] = filterFunction(film->filter, (2.0 * (int)i) / (film->cache_size - 1));
    const double inv_dx = film->cache_size ? (film->cache_size - 1) / radius : 0.0, two_inv_radius = 2.0 / radius;
    auto filter = [&](double x)
    {
        if (cache.empty()) return filterFunction(film->filter, two_inv_radius * std::abs(x));
        return cache[static_cast<size_t>(inv_dx * std::abs(x) + 0.5)];
    };
    std::vector<double> rgb((size_t)W * H * 3, 0.0), wsum((size_t)W * H, 0.0);
    for (uint32_t pixel = 0; pixel < (uint32_t)(W * H); pixel++)
    {
        smp.initiate(pixel);
        for (uint32_t i = 0; i < spp; i++)
        {
            smp.setIndex(i);
            const double px = (double)(pixel % W) + smp.get(PIXEL), py = (double)(pixel / W) + smp.get(PIXEL + 1);
            D3 v = sampleRay(s, cameraRay(*cam, s.d.scene_ior, pixel, smp), smp, nullptr);
            const int64_t x0 = std::max((int64_t)(px + 0.5 - radius), (int64_t)0), y0 = std::max((int64_t)(py + 0.5 - radius), (int64_t)0);
            const int64_t x1 = std::min((int64_t)(px - 0.5 + radius), W - 1), y1 = std::min((int64_t)(py - 0.5 + radius), H - 1);
            for (int64_t y = y0; y <= y1; y++)
            {
                const double wy = filter(y + 0.5 - py);
                for (int64_t x = x0; x <= x1; x++)
                {
                    const double w = wy * filter(x + 0.5 - px);
                    double* o = &rgb[(size_t)(y * W + x) * 3];
                    o[0] += v.x * w; o[1] += v.y * w; o[2] += v.z * w;
                    wsum[(size_t)(y * W + x)] += w;
                }
            }
        }
    }
    for (size_t i = 0; i < (size_t)W * H; i++)
        for (int k = 0; k < 3; k++)
        {
            const double v = wsum[i] == 0.0 ? 0.0 : rgb[3 * i + k] / wsum[i];
            out[3 * i + k] = v < 0.0 ? 0.0 : v;
        }
}

// BVH::BVH (bvh.cpp:13-78): the three hierarchy builders restated recursively, exactly in the
// reference's order of operations, over primitive boxes (Surface::Base::BB()) instead of surfaces.
namespace
{
    struct Box
    {
        double mn[3] = { 1.7976931348623157e308, 1.7976931348623157e308, 1.7976931348623157e308 };
        double mx[3] = { -1.7976931348623157e308, -1.7976931348623157e308, -1.7976931348623157e308 };
        void merge(const Box& b) { for (int i = 0; i < 3; i++) { if (mn[i] > b.mn[i]) mn[i] = b.mn[i]; if (mx[i] < b.mx[i]) mx[i] = b.mx[i]; } }
        void mergePoint(const double* p) { for (int i = 0; i < 3; i++) { if (mn[i] > p[i]) mn[i] = p[i]; if (mx[i] < p[i]) mx[i] = p[i]; } }
        bool valid() const { for (int i = 0; i < 3; i++) if (mn[i] > mx[i]) return false; return true; }
        double area() const   // bounding-box.cpp:35-40
        {
            if (!valid()) return 0.0;
            const double dx = mx[0] - mn[0], dy = mx[1] - mn[1], dz = mx[2] - mn[2];
            return 2.0 * (dx * dy + dx * dz + dy * dz);
        }
        void centroid(double* c) const { for (int i = 0; i < 3; i++) c[i] = (mx[i] + mn[i]) / 2.0; }
    };

    struct BuildNode
    {
        Box BB;
        std::vector<uint32_t> surfaces;      // primitive indices (BuildNode::surfaces)
        std::vector<std::unique_ptr<BuildNode>> children;
        uint32_t df_idx = 0;
    };

    struct BvhBuilder
    {
        const double* bounds;      // [n][6]
        int bins_per_axis;
        uint32_t df_idx = 0;
        static constexpr size_t leaf_surfaces = 8, max_leaf_surfaces = 0xFF;   // bvh.hpp:91-92
        static constexpr double EPS = 1e-9;

        Box boxOf(uint32_t s) const { Box b; for (int i = 0; i < 3; i++) { b.mn[i] = bounds[6 * (size_t)s + i]; b.mx[i] = bounds[6 * (size_t)s + 3 + i]; } return b; }

        void arbitrarySplit(BuildNode* node, size_t N)   // bvh.cpp:458-474
        {
            auto& S = node->surfaces;
            N = std::min(N, S.size());
            for (size_t i = 0; i < N; i++) node->children.push_back(std::make_unique<BuildNode>());
            for (size_t i = 0; i < S.size(); i++)
            {
                BuildNode* c = node->children[i % N].get();
                c->surfaces.push_back(S[i]);
                c->BB.merge(boxOf(S[i]));
            }
            S.clear();
        }

        void binary(BuildNode* node)   // recursiveBuildBinarySAH, bvh.cpp:165-283
        {
            node->df_idx = df_idx++;
            auto& S = node->surfaces;
            if (S.size() <= leaf_surfaces) return;
            Box extent;
            double c[3];
            for (uint32_t s : S) { boxOf(s).centroid(c); extent.mergePoint(c); }
            const double dims[3] = { extent.mx[0] - extent.mn[0], extent.mx[1] - extent.mn[1], extent.mx[2] - extent.mn[2] };
            const int axis = dims[0] > dims[1] ? (dims[0] > dims[2] ? 0 : 2) : (dims[1] > dims[2] ? 1 : 2);
            if (dims[axis] < EPS)
            {
                if (S.size() > max_leaf_surfaces) { arbitrarySplit(node, 2); for (auto& ch : node->children) binary(ch.get()); }
                return;
            }
            auto getIdx = [&](const double* cc)
            {
                const double f = (cc[axis] - extent.mn[axis]) / dims[axis];
                const int idx = (int)std::floor(f * bins_per_axis);
                return std::min(idx, bins_per_axis - 1);
            };
            std::vector<std::pair<size_t, Box>> bins(bins_per_axis);
            for (auto& b : bins) b.first = 0;
            for (uint32_t s : S) { const Box b = boxOf(s); b.centroid(c); const int idx = getIdx(c); bins[idx].first++; bins[idx].second.merge(b); }
            double min_cost = std::numeric_limits<double>::max();
            size_t split_bin = 0;
            for (size_t i = 0; i + 1 < (size_t)bins_per_axis; i++)
            {
                size_t A_count = 0, B_count = 0;
                Box A, B;
                for (size_t j = 0; j < i + 1; j++) { A_count += bins[j].first; A.merge(bins[j].second); }
                for (size_t j = i + 1; j < (size_t)bins_per_axis; j++) { B_count += bins[j].first; B.merge(bins[j].second); }
                const double cost = 1.0 + (A_count * A.area() + B_count * B.area()) / node->BB.area();
                if (cost < min_cost) { split_bin = i; min_cost = cost; }
            }
            if (min_cost > S.size())
            {
                if (S.size() > max_leaf_surfaces) { arbitrarySplit(node, 2); for (auto& ch : node->children) binary(ch.get()); }
                return;
            }
            auto A = std::make_unique<BuildNode>(), B = std::make_unique<BuildNode>();
            for (uint32_t s : S)
            {
                const Box b = boxOf(s); b.centroid(c);
                BuildNode* t = (size_t)getIdx(c) <= split_bin ? A.get() : B.get();
                t->surfaces.push_back(s); t->BB.merge(b);
            }
            S.clear();
            if (!A->surfaces.empty()) { node->children.push_back(std::move(A)); binary(node->children.back().get()); }
            if (!B->surfaces.empty()) { node->children.push_back(std::move(B)); binary(node->children.back().get()); }
        }

        void quaternary(BuildNode* node)   // recursiveBuildQuaternarySAH, bvh.cpp:285-432
        {
            node->df_idx = df_idx++;
            const int nb = bins_per_axis;
            auto& S = node->surfaces;
            if (S.size() <= leaf_surfaces) return;
            Box extent;
            double c[3];
            for (uint32_t s : S) { boxOf(s).centroid(c); extent.mergePoint(c); }
            const double dims[3] = { extent.mx[0] - extent.mn[0], extent.mx[1] - extent.mn[1], extent.mx[2] - extent.mn[2] };
            int ax, ay;
            if (dims[0] > dims[1]) { ax = 0; ay = dims[1] > dims[2] ? 1 : 2; }
            else if (dims[0] > dims[2]) { ax = 0; ay = 1; }
            else { ax = 1; ay = 2; }
            if (dims[ax] < EPS || dims[ay] < EPS) { df_idx--; binary(node); return; }
            auto getIdx = [&](const double* cc, int& ix, int& iy)
            {
                const double fx = (cc[ax] - extent.mn[ax]) / dims[ax], fy = (cc[ay] - extent.mn[ay]) / dims[ay];
                ix = std::min((int)std::floor(fx * (double)nb), nb - 1);
                iy = std::min((int)std::floor(fy * (double)nb), nb - 1);
            };
            std::vector<std::pair<size_t, Box>> bins((size_t)nb * nb);
            for (auto& b : bins) b.first = 0;
            for (uint32_t s : S) { const Box b = boxOf(s); b.centroid(c); int ix, iy; getIdx(c, ix, iy); bins[(size_t)ix * nb + iy].first++; bins[(size_t)ix * nb + iy].second.merge(b); }
            double min_cost = std::numeric_limits<double>::max();
            int split_x = 0, split_y = 0;
            for (int i = 0; i < nb - 1; i++)
                for (int j = 0; j < nb - 1; j++)
                {
                    Box BBs[4]; size_t counts[4] = { 0, 0, 0, 0 };
                    for (int v = 0; v < 4; v++)
                    {
                        const int x0 = (v & 1) ? i + 1 : 0, x1 = (v & 1) ? nb : i + 1;
                        const int y0 = (v & 2) ? j + 1 : 0, y1 = (v & 2) ? nb : j + 1;
                        for (int x = x0; x < x1; x++) for (int y = y0; y < y1; y++) { counts[v] += bins[(size_t)x * nb + y].first; BBs[v].merge(bins[(size_t)x * nb + y].second); }
                    }
                    double cost = 0.0;
                    for (int v = 0; v < 4; v++) cost += BBs[v].area() * counts[v];
                    cost = 1.0 + cost / node->BB.area();
                    if (cost < min_cost) { split_x = i; split_y = j; min_cost = cost; }
                }
            if (min_cost > S.size())
            {
                if (S.size() > max_leaf_surfaces) { arbitrarySplit(node, 4); for (auto& ch : node->children) quaternary(ch.get()); }
                return;
            }
            std::unique_ptr<BuildNode> fresh[4];
            for (uint32_t s : S)
            {
                const Box b = boxOf(s); b.centroid(c);
                int ix, iy; getIdx(c, ix, iy);
                const int child = (ix > split_x ? 1 : 0) | (iy > split_y ? 2 : 0);
                if (!fresh[child]) fresh[child] = std::make_unique<BuildNode>();
                fresh[child]->surfaces.push_back(s); fresh[child]->BB.merge(b);
            }
            S.clear();
            for (auto& ch : fresh) if (ch) { node->children.push_back(std::move(ch)); quaternary(node->children.back().get()); }
        }

        // Octree<SurfaceCentroid> insertion (octree.cpp:34-81) + recursiveBuildFromOctree (bvh.cpp:130-163);
        // `cell` is the octree node's box. A cell splits when it holds more than leaf_surfaces centroids.
        void octree(BuildNode* node, const Box& cell)
        {
            node->df_idx = df_idx++;
            auto S = std::move(node->surfaces);
            node->surfaces.clear();
            Box BB;
            if (S.size() <= leaf_surfaces)
            {
                node->surfaces = S;
                for (uint32_t s : S) BB.merge(boxOf(s));
            }
            else
            {
                double origin[3], half[3], c[3];
                cell.centroid(origin);
                for (int i = 0; i < 3; i++) half[i] = (cell.mx[i] - cell.mn[i]) / 2.0;
                std::vector<uint32_t> part[8];
                for (uint32_t s : S)
                {
                    boxOf(s).centroid(c);
                    int o = 0;
                    for (int i = 0; i < 3; i++) if (c[i] >= origin[i]) o |= (4 >> i);
                    part[o].push_back(s);
                }
                for (int o = 0; o < 8; o++)
                {
                    if (part[o].empty()) continue;
                    Box child_cell;
                    for (int i = 0; i < 3; i++)
                    {
                        const double no = origin[i] + half[i] * ((o & (4 >> i)) ? 0.5 : -0.5), h = half[i] * 0.5;
                        child_cell.mn[i] = no - h; child_cell.mx[i] = no + h;
                    }
                    node->children.push_back(std::make_unique<BuildNode>());
                    node->children.back()->surfaces = std::move(part[o]);
                    octree(node->children.back().get(), child_cell);
                    BB.merge(node->children.back()->BB);
                }
            }
            node->BB = BB;
        }
    };

    struct BvhOut
    {
        std::vector<double> bounds;
        std::vector<uint32_t> first, count, next, order;
    };

    void compactBvh(const BuildNode* node, uint32_t next_sibling, BvhOut& out)   // BVH::compact, bvh.cpp:434-456
    {
        const uint32_t i = node->df_idx;
        for (int k = 0; k < 3; k++) { out.bounds[6 * (size_t)i + k] = node->BB.mn[k]; out.bounds[6 * (size_t)i + 3 + k] = node->BB.mx[k]; }
        out.next[i] = next_sibling;
        out.first[i] = (uint32_t)out.order.size();
        out.count[i] = (uint32_t)node->surfaces.size();
        for (uint32_t s : node->surfaces) out.order.push_back(s);
        for (size_t k = 0; k < node->children.size(); k++)
            compactBvh(node->children[k].get(), k + 1 < node->children.size() ? node->children[k + 1]->df_idx : 0u, out);
    }
}

// prim_bounds [n][6], scene_bounds = Scene::BB(); type / bins as mcrt_bvh_build. *out points into
// memory owned by *handle (oracle_bvh_free).
void oracle_bvh_build(const double* prim_bounds, uint32_t n, const double* scene_bounds, int type, int bins_per_axis, void** handle,
                      mcrt_bvh_desc* out)
{
    BvhBuilder b;
    b.bounds = prim_bounds;
    b.bins_per_axis = bins_per_axis > 0 ? bins_per_axis : (type == MCRT_BVH_BINARY_SAH ? 16 : 8);
    BuildNode root;
    for (int i = 0; i < 3; i++) { root.BB.mn[i] = scene_bounds[i]; root.BB.mx[i] = scene_bounds[3 + i]; }
    root.surfaces.resize(n);
    for (uint32_t i = 0; i < n; i++) root.surfaces[i] = i;
    if (type == MCRT_BVH_QUATERNARY_SAH) b.quaternary(&root);
    else if (type == MCRT_BVH_BINARY_SAH) b.binary(&root);
    else
    {
        // bvh.cpp:44-47: cube around the scene box
        double c[3], m = 0.0;
        root.BB.centroid(c);
        for (int i = 0; i < 3; i++) m = std::max(m, root.BB.mx[i] - root.BB.mn[i]);
        const double half_max = m / 2.0;
        Box cube;
        for (int i = 0; i < 3; i++) { cube.mn[i] = c[i] - half_max; cube.mx[i] = c[i] + half_max; }
        b.octree(&root, cube);
    }
    auto* o = new BvhOut();
    const uint32_t n_nodes = b.df_idx;
    o->bounds.resize(6 * (size_t)n_nodes); o->first.resize(n_nodes); o->count.resize(n_nodes); o->next.resize(n_nodes);
    compactBvh(&root, 0u, *o);
    std::memset(out, 0, sizeof(*out));
    out->n_nodes = n_nodes; out->n_prims = n;
    out->node_bounds = o->bounds.data(); out->node_first_prim = o->first.data(); out->node_prim_count = o->count.data();
    out->node_next_sibling = o->next.data(); out->prim_order = o->order.data();
    *handle = o;
}

void oracle_bvh_free(void* handle) { delete static_cast<BvhOut*>(handle); }

// Octree<Photon> insertion + LinearOctree::compact (octree.cpp:34-81, linear-octree.cpp:201-244),
// restated top-down. The reference inserts photons one by one; a node ends up internal exactly when
// more than max_node_data photons fall into its box, and child boxes follow from the parent's by
// fixed arithmetic, so the finished tree is a function of the photon set alone: partition the
// node's photons into octants (stable), recurse in octant order = the order compact() emits.
namespace
{
    struct OctreeOut
    {
        std::vector<double> bounds;
        std::vector<uint64_t> start, count;
        std::vector<uint32_t> next;
        std::vector<uint8_t> leaf;
        std::vector<float> photons;
        std::vector<uint64_t> tags;
    };

    // tags: optional per-photon values (the path that stored the photon) moved along with the photons
    void octreeBuild(OctreeOut& out, std::vector<float>& data, std::vector<float>& scratch, std::vector<uint64_t>* tags, uint64_t begin,
                     uint64_t end, const double* bmin, const double* bmax, uint32_t max_node_data, bool last, int depth)
    {
        const uint64_t count = end - begin;
        const uint32_t idx = (uint32_t)out.leaf.size();
        // (the reference recurses without bound when > max_node_data photons coincide; stop at 64 levels)
        const bool split = count > max_node_data && depth < 64;
        out.leaf.push_back(split ? 0 : 1);
        out.start.push_back(begin);
        out.count.push_back(count);                 // LinearOctant::contained_data: everything below
        out.next.push_back(0xFFFFFFFFu);
        out.bounds.resize(out.bounds.size() + 6);
        double lo[3] = { 1.7976931348623157e308, 1.7976931348623157e308, 1.7976931348623157e308 };
        double hi[3] = { -1.7976931348623157e308, -1.7976931348623157e308, -1.7976931348623157e308 };
        for (uint64_t i = begin; i < end; i++)
            for (int c = 0; c < 3; c++)
            {
                const double v = (double)data[8 * i + 3 + c];
                if (lo[c] > v) lo[c] = v;
                if (hi[c] < v) hi[c] = v;
            }
        if (split)
        {
            // BoundingBox::centroid / dimensions (bounding-box.cpp:25-33), child boxes octree.cpp:51-60
            double centroid[3], half[3];
            for (int c = 0; c < 3; c++) { centroid[c] = (bmax[c] + bmin[c]) / 2.0; half[c] = (bmax[c] - bmin[c]) / 2.0; }
            auto octantOf = [&](const float* ph)
            {
                int o = 0;
                for (int c = 0; c < 3; c++) if ((double)ph[3 + c] >= centroid[c]) o |= (4 >> c);   // octree.cpp:73-79
                return o;
            };
            uint64_t counts[8] = { 0 }, starts[9], cursor[8];
            for (uint64_t i = begin; i < end; i++) counts[octantOf(&data[8 * i])]++;
            starts[0] = begin;
            for (int o = 0; o < 8; o++) starts[o + 1] = starts[o] + counts[o];
            scratch.resize(8 * count);
            std::vector<uint64_t> moved(tags ? count : 0);
            for (int o = 0; o < 8; o++) cursor[o] = starts[o] - begin;
            for (uint64_t i = begin; i < end; i++)
            {
                const int o = octantOf(&data[8 * i]);
                if (tags) moved[cursor[o]] = (*tags)[i];
                std::memcpy(&scratch[8 * cursor[o]++], &data[8 * i], 32);
            }
            std::memcpy(&data[8 * begin], scratch.data(), 32 * count);
            if (tags) std::copy(moved.begin(), moved.end(), tags->begin() + begin);
            int last_used = -1;
            for (int o = 0; o < 8; o++) if (counts[o]) last_used = o;
            for (int o = 0; o < 8; o++)
            {
                if (!counts[o]) continue;   // empty leaves are dropped (linear-octree.cpp:222-229)
                double cmin[3], cmax[3];
                for (int c = 0; c < 3; c++)
                {
                    const double new_origin = centroid[c] + half[c] * ((o & (4 >> c)) ? 0.5 : -0.5);
                    const double h = half[c] * 0.5;
                    cmin[c] = new_origin - h; cmax[c] = new_origin + h;
                }
                octreeBuild(out, data, scratch, tags, starts[o], starts[o + 1], cmin, cmax, max_node_data, o == last_used, depth + 1);
            }
        }
        for (int c = 0; c < 3; c++) { out.bounds[6 * idx + c] = lo[c]; out.bounds[6 * idx + 3 + c] = hi[c]; }
        out.next[idx] = last ? 0xFFFFFFFFu : (uint32_t)out.leaf.size();
    }
}

// photons: [n][8] floats {flux.xyz, pos.xyz, phi, theta}; scene_bounds6 = the root Octree box
// (photon-mapper.cpp:49-51). *out points into memory owned by *handle (oracle_octree_free).
void oracle_octree_build(const float* photons, uint64_t n, uint32_t max_node_data, const double* scene_bounds6, void** handle,
                         mcrt_photon_map_desc* out)
{
    auto* o = new OctreeOut();
    o->photons.assign(photons, photons + 8 * n);
    std::vector<float> scratch;
    if (n) octreeBuild(*o, o->photons, scratch, nullptr, 0, n, scene_bounds6, scene_bounds6 + 3, max_node_data, true, 0);
    std::memset(out, 0, sizeof(*out));
    out->n_octants = (uint32_t)o->leaf.size();
    out->octant_bounds = o->bounds.data(); out->octant_start = o->start.data(); out->octant_count = o->count.data();
    out->octant_next_sibling = o->next.data(); out->octant_leaf = o->leaf.data();
    out->n_photons = n; out->photons = o->photons.data();
    *handle = o;
}

void oracle_octree_free(void* handle) { delete static_cast<OctreeOut*>(handle); }

// ---------------------------------------------------------------- photon mapper (photon-mapper.cpp, photon.hpp)
namespace
{
    enum { PM_LIGHT = 0, PM_REJECT = 2 };                        // sampling.hpp:59-76
    enum { PM_EMISSION, PM_DIRECT, PM_CAUSTIC, PM_GLOBAL };      // the four terms sampleRay adds up

    struct PhotonList
    {
        std::vector<float> photons;      // [n][8] {flux.xyz, pos.xyz, phi, theta}
        std::vector<uint64_t> emission;  // light << 32 | the light's emission index: the path that stored each photon
    };

    void storePhoton(PhotonList& list, D3 flux, D3 pos, D3 dir, uint64_t emission) // Photon::Photon, photon.hpp:7-12
    {
        const float theta = (float)std::atan2(std::sqrt(dir.x * dir.x + dir.y * dir.y), dir.z);
        const float phi = (float)std::atan2(dir.y, dir.x);
        const float v[8] = { (float)flux.x, (float)flux.y, (float)flux.z, (float)pos.x, (float)pos.y, (float)pos.z, phi, theta };
        list.photons.insert(list.photons.end(), v, v + 8);
        list.emission.push_back(emission);
    }

    D3 photonDir(float phi, float theta) // Photon::dir, photon.hpp:19-27: glibc's float sinf / cosf
    {
        const float sin_theta = std::sin(theta);
        return D3((double)std::cos(phi) * sin_theta, (double)std::sin(phi) * sin_theta, (double)std::cos(theta));
    }

    void updateIORs(std::vector<double>& iors, const Ray& ray) // RefractionHistory::update, ray.cpp:80-93
    {
        if (ray.refraction_level > 0)
        {
            if (ray.refraction_level == (int)iors.size()) iors.push_back(ray.medium_ior);
            else if (ray.refraction_level < (int)iors.size() - 1) iors.pop_back();
        }
    }

    // PhotonMapper::emitPhoton, photon-mapper.cpp:225-277
    void emitPhoton(const Scene& s, Ray ray, D3 flux, Sampler& smp, double non_caustic_reject, uint64_t emission, PhotonList& caustic,
                    PhotonList& global)
    {
        std::vector<double> iors(1, ray.medium_ior);
        while (true)
        {
            smp.shuffle();
            Isect is = intersect(s, ray, nullptr);
            if (is.prim == 0xFFFFFFFFu) return;
            int ext = std::min(std::max(ray.refraction_level - 1, 0), (int)iors.size() - 1);
            Interaction ia = makeInteraction(s, is, ray, iors[ext], smp);
            if (!ia.material->dirac_delta) // :245-256: only where a non-delta interaction is possible
            {
                if (ray.dirac_delta) storePhoton(caustic, flux, ia.position, -ray.direction, emission);
                else if (non_caustic_reject > smp.get(PM_REJECT)) storePhoton(global, flux / non_caustic_reject, ia.position, -ray.direction, emission);
            }
            D3 f; double pdf; Ray nr;
            if (!sampleBSDF(ia, smp, f, pdf, nr, true)) return;
            f = f / pdf;
            double survive = std::min(compMax(f), 0.95); // :265-272: survival probability instead of flux scaling
            if (survive == 0.0 || survive <= smp.get(ABSORB)) return;
            flux = flux * (f / survive);
            ray = nr;
            updateIORs(iors, ray);
        }
    }

    struct PhotonPass { OctreeOut maps[2]; uint64_t emissions = 0; };

    // PhotonMapper::PhotonMapper's first pass, photon-mapper.cpp:24-110: emissions per light in proportion to its flux, emission
    // j of light l drawn from the sampler at (l, j), every photon appended in emission order as a single thread does.
    // Pass `pass` of progressive photon mapping (mcrt_photon_emit_pass) draws light l's emission j at (l, pass * n_l + j),
    // computed in 64 bits and cast to the sampler's 32-bit index, with the flux of a one-pass map; pass 0 is the
    // reference's pass. false, and nothing emitted, when a light's indices of the pass do not fit 32 bits.
    bool photonPass(const Scene& s, uint64_t emissions, double caustic_factor, uint32_t pass, uint32_t seed, PhotonList& caustic,
                    PhotonList& global, uint64_t& total)
    {
        const size_t n_lights = s.light_prim.size();
        const size_t photon_emissions = (size_t)((double)emissions * caustic_factor);
        std::vector<D3> light_flux(n_lights);
        double total_flux = 0.0;
        for (size_t l = 0; l < n_lights; l++)
        {
            const uint32_t prim = s.light_prim[l];
            light_flux[l] = D3(s.materials[s.prim_material[prim]].emittance) * s.prim_area[prim];
            total_flux += 0.0 + light_flux[l].x + light_flux[l].y + light_flux[l].z; // glm::compAdd
        }
        std::vector<size_t> counts(n_lights);
        for (size_t l = 0; l < n_lights; l++)
        {
            const double share = (0.0 + light_flux[l].x + light_flux[l].y + light_flux[l].z) / total_flux;
            counts[l] = (size_t)((double)photon_emissions * share);
            if (((uint64_t)pass + 1) * (uint64_t)counts[l] > 0x100000000ull) return false;
        }
        const double non_caustic_reject = 1.0 / caustic_factor;
        Sampler smp(seed);
        total = 0;
        for (size_t l = 0; l < n_lights; l++)
        {
            const uint32_t prim = s.light_prim[l];
            const size_t n = counts[l];
            const D3 photon_flux = light_flux[l] / (double)n;
            total += n;
            smp.initiate((uint32_t)l);
            for (size_t j = 0; j < n; j++)
            {
                const uint32_t index = (uint32_t)((uint64_t)pass * n + j);
                smp.setIndex(index);
                const double u0 = smp.get(PM_LIGHT), u1 = smp.get(PM_LIGHT + 1), u2 = smp.get(PM_LIGHT + 2), u3 = smp.get(PM_LIGHT + 3);
                const D3 pos = lightPoint(s, prim, u0, u1), normal = primNormal(s, prim, pos);
                const double r = std::sqrt(u2), az = u3 * TWO_PI; // Sampling::cosWeightedHemi
                const D3 dir = Frame(normal).from(D3(r * std::cos(az), r * std::sin(az), std::sqrt(1 - u2)));
                emitPhoton(s, makeRay(pos + normal * EPS, dir, s.d.scene_ior), photon_flux, smp, non_caustic_reject, (uint64_t)l << 32 | index,
                           caustic, global);
            }
        }
        return true;
    }

    struct PhotonMaps
    {
        const Scene* s;
        std::vector<float> photons[2];
        uint32_t k;
        bool direct_visualization;
        double gather_r2[2] = { 0.0, 0.0 };   // fixed gather radius^2 of the caustic / global map (k_gather); 0: k-NN
    };

    // queries: photon-map queries, ties: k-NN queries with a tie at the k-th distance, empty: queries that took no photon,
    // photons: photons taken by all queries
    struct PMCounts { uint64_t rays = 0, shadow_rays = 0, queries = 0, ties = 0, empty = 0, photons = 0; };

    // LinearOctree::knnSearch as a brute-force float64 search over the whole map, then the estimates of photon-mapper.cpp:343-391.
    // A photon at the k-th distance that is not taken while another at the same distance is counts a tie: the reference's choice
    // between them depends on its octree walk, which this search does not restate.
    // -> the min(k, n) nearest photons (distance2, index), farthest first, as the reference pops its max-heap of results
    std::vector<std::pair<double, uint32_t>> knnBrute(const PhotonMaps& pm, int which, D3 p, PMCounts& cnt)
    {
        const std::vector<float>& ph = pm.photons[which];
        const size_t n = ph.size() / 8;
        cnt.queries++;
        std::vector<std::pair<double, uint32_t>> d(n);
        if (n == 0) return d;
        for (size_t i = 0; i < n; i++)
        {
            const D3 v = p - D3(ph[8 * i + 3], ph[8 * i + 4], ph[8 * i + 5]); // glm::distance2
            d[i] = { dot(v, v), (uint32_t)i };
        }
        const size_t k = std::min<size_t>(pm.k, n);
        std::nth_element(d.begin(), d.begin() + (k - 1), d.end());
        const double kth = d[k - 1].first;
        for (size_t i = k; i < n; i++) if (d[i].first == kth) { cnt.ties++; break; }
        d.resize(k);
        std::sort(d.begin(), d.end(), [](const std::pair<double, uint32_t>& a, const std::pair<double, uint32_t>& b) { return a.first > b.first; });
        return d;
    }

    // The fixed-radius search of progressive photon mapping (gatherWarp, k_gather_user) as a brute force: every photon whose
    // float64 distance2 is <= r2, the same inclusive test. -> (distance2, index), farthest first, as knnBrute
    std::vector<std::pair<double, uint32_t>> gatherBrute(const PhotonMaps& pm, int which, D3 p, double r2, PMCounts& cnt)
    {
        const std::vector<float>& ph = pm.photons[which];
        const size_t n = ph.size() / 8;
        cnt.queries++;
        std::vector<std::pair<double, uint32_t>> d;
        for (size_t i = 0; i < n; i++)
        {
            const D3 v = p - D3(ph[8 * i + 3], ph[8 * i + 4], ph[8 * i + 5]);
            const double d2 = dot(v, v);
            if (d2 <= r2) d.push_back({ d2, (uint32_t)i });
        }
        std::sort(d.begin(), d.end(), [](const std::pair<double, uint32_t>& a, const std::pair<double, uint32_t>& b) { return a.first > b.first; });
        return d;
    }

    double coneWeight(double d2, double inv_r2) { return std::max(0.0, 1.0 - std::sqrt(d2 * inv_r2)); } // :383-386

    // The estimates of photon-mapper.cpp:343-391 over the photons a query takes: with gather_r2 0 the k nearest (knnBrute),
    // normalised by the k-th distance2; otherwise every photon within the fixed radius (gatherBrute), normalised by r^2, as
    // k_gather does. Only the selection and the normaliser r2 differ between the two. A query that takes no photon adds nothing.
    D3 photonEstimate(const PhotonMaps& pm, int which, const Interaction& ia, double gather_r2, PMCounts& cnt)
    {
        const std::vector<float>& ph = pm.photons[which];
        const std::vector<std::pair<double, uint32_t>> d = gather_r2 > 0.0 ? gatherBrute(pm, which, ia.position, gather_r2, cnt)
                                                                            : knnBrute(pm, which, ia.position, cnt);
        cnt.photons += d.size();
        if (d.empty()) { cnt.empty++; return D3(); }
        const double r2 = gather_r2 > 0.0 ? gather_r2 : d[0].first, inv_r2 = 1.0 / r2;
        D3 radiance;
        for (const auto& r : d)
        {
            const float* p = &ph[8 * (size_t)r.second];
            D3 f; double pdf;
            if (!ia.bsdfWorld(f, photonDir(p[6], p[7]), pdf)) continue;
            const D3 flux((double)p[0], (double)p[1], (double)p[2]);
            if (which == 0) radiance = radiance + (flux * f * coneWeight(r.first, inv_r2)) / pdf; // cone filter
            else radiance = radiance + flux * f / pdf;
        }
        if (which == 0) return 3.0 * radiance * inv_r2 * INV_PI;
        return radiance / (r2 * PI);
    }

    // PhotonMapper::sampleRay, photon-mapper.cpp:279-341. comp: the radiance split into PM_EMISSION (emission seen directly or
    // through delta vertices), PM_DIRECT (next-event estimation and its MIS partner), PM_CAUSTIC and PM_GLOBAL; the return value
    // is the reference's running sum.
    D3 pmSampleRay(const PhotonMaps& pm, Ray ray, Sampler& smp, D3 comp[4], PMCounts& cnt)
    {
        const Scene& s = *pm.s;
        D3 radiance, throughput(1, 1, 1);
        std::vector<double> iors(1, ray.medium_ior);
        LightSample ls;
        for (int c = 0; c < 4; c++) comp[c] = D3();
        auto add = [&](int c, D3 v) { v = v * throughput; comp[c] = comp[c] + v; radiance = radiance + v; };
        while (true)
        {
            smp.shuffle();
            Isect is = intersect(s, ray, &cnt.rays);
            if (is.prim == 0xFFFFFFFFu) return radiance; // no sky, :292-295
            int ext = std::min(std::max(ray.refraction_level - 1, 0), (int)iors.size() - 1);
            Interaction ia = makeInteraction(s, is, ray, iors[ext], smp);
            add(ray.depth == 0 || ray.dirac_delta ? PM_EMISSION : PM_DIRECT, sampleEmissive(s, ia, ls));
            if (ia.dirac_delta)
            {
                if (!ray.dirac_delta && ray.depth != 0) return radiance;
            }
            else
            {
                add(PM_CAUSTIC, photonEstimate(pm, 0, ia, pm.gather_r2[0], cnt));
                if (pm.direct_visualization || !(ray.dirac_delta || ray.depth == 0))
                {
                    add(PM_GLOBAL, photonEstimate(pm, 1, ia, pm.gather_r2[1], cnt));
                    return radiance;
                }
                uint64_t shadow = 0;
                add(PM_DIRECT, sampleDirect(s, ia, ls, smp, &shadow));
                cnt.shadow_rays += shadow; cnt.rays += shadow;
            }
            D3 f;
            if (!sampleBSDF(ia, smp, f, ls.bsdf_pdf, ray)) return radiance;
            throughput = throughput * (f / ls.bsdf_pdf);
            double survive = compMax(throughput) * ray.refraction_scale; // Integrator::absorb, integrator.cpp:112-129
            if (survive == 0.0) return radiance;
            if (ray.diffuse_depth > 3 || ray.depth > 16)
            {
                survive = std::min(0.95, survive);
                if (survive <= smp.get(ABSORB)) return radiance;
                throughput = throughput / survive;
            }
            updateIORs(iors, ray);
        }
    }
}

// The photon pass: emissions * caustic_factor emissions over the scene's lights, the caustic and global photons built into
// octrees (max_node_data photons per leaf, root box scene_bounds6) as oracle_octree_build does; emission[which] (n_photons of the
// map): light << 32 | the light's emission index, the path that stored each photon, in map order. Memory owned by *handle
// (oracle_photon_pass_free). pass_index: the photon pass of progressive photon mapping (photonPass); returns 0, or -1 and
// no handle when the pass's emission indices do not fit 32 bits.
int oracle_photon_pass(void* h, uint64_t emissions, double caustic_factor, uint32_t max_node_data, const double* scene_bounds6,
                       uint32_t pass_index, uint32_t seed, void** handle, mcrt_photon_map_desc* caustic_out, mcrt_photon_map_desc* global_out,
                       const uint64_t** emission, uint64_t* total_emissions)
{
    const Scene& s = *static_cast<Scene*>(h);
    PhotonList lists[2];
    uint64_t total = 0;
    *handle = nullptr;
    if (!photonPass(s, emissions, caustic_factor, pass_index, seed, lists[0], lists[1], total)) return -1;
    auto* pass = new PhotonPass();
    pass->emissions = total;
    mcrt_photon_map_desc* out[2] = { caustic_out, global_out };
    for (int w = 0; w < 2; w++)
    {
        OctreeOut& o = pass->maps[w];
        // the reference inserts its photons into the octree last first: every leaf of its maps holds them in reverse
        // emission order (pm_hexagon_room_64's maps, bit for bit)
        const uint64_t n = lists[w].emission.size();
        o.photons.resize(8 * n); o.tags.resize(n);
        for (uint64_t i = 0; i < n; i++)
        {
            std::memcpy(&o.photons[8 * i], &lists[w].photons[8 * (n - 1 - i)], 32);
            o.tags[i] = lists[w].emission[n - 1 - i];
        }
        std::vector<float> scratch;
        if (n) octreeBuild(o, o.photons, scratch, &o.tags, 0, n, scene_bounds6, scene_bounds6 + 3, max_node_data, true, 0);
        std::memset(out[w], 0, sizeof(*out[w]));
        out[w]->n_octants = (uint32_t)o.leaf.size();
        out[w]->octant_bounds = o.bounds.data(); out[w]->octant_start = o.start.data(); out[w]->octant_count = o.count.data();
        out[w]->octant_next_sibling = o.next.data(); out[w]->octant_leaf = o.leaf.data();
        out[w]->n_photons = n; out[w]->photons = o.photons.data();
        emission[w] = o.tags.data();
    }
    *total_emissions = pass->emissions;
    *handle = pass;
    return 0;
}

void oracle_photon_pass_free(void* handle) { delete static_cast<PhotonPass*>(handle); }

// PhotonMapper's second pass over given maps (only their photons are read): k nearest photons, direct_visualization
void* oracle_pm_create(void* h, const mcrt_photon_map_desc* caustic, const mcrt_photon_map_desc* global, uint32_t k, uint32_t direct_visualization)
{
    auto* pm = new PhotonMaps();
    pm->s = static_cast<Scene*>(h);
    const mcrt_photon_map_desc* m[2] = { caustic, global };
    for (int w = 0; w < 2; w++) copyv(pm->photons[w], m[w]->photons, 8 * (size_t)m[w]->n_photons);
    pm->k = k;
    pm->direct_visualization = direct_visualization != 0;
    return pm;
}

void oracle_pm_destroy(void* pm) { delete static_cast<PhotonMaps*>(pm); }

// Following estimates gather every photon within r_caustic / r_global (k_gather, mcrt_photon_gather_radius); (0, 0): k-NN.
// Returns -1, and changes nothing, for radii mcrt_photon_gather_radius refuses.
int oracle_pm_gather_radius(void* pmh, double r_caustic, double r_global)
{
    PhotonMaps& pm = *static_cast<PhotonMaps*>(pmh);
    if (r_caustic == 0.0 && r_global == 0.0) { pm.gather_r2[0] = pm.gather_r2[1] = 0.0; return 0; }
    const double r[2] = { r_caustic, r_global };
    for (int w = 0; w < 2; w++)
        if (!(r[w] > 0.0) || !std::isfinite(r[w] * r[w])) return -1;
    pm.gather_r2[0] = r_caustic * r_caustic; pm.gather_r2[1] = r_global * r_global;
    return 0;
}

// The fixed-radius search on caller points, as mcrt_photon_gather_search: per point the number of photons of map `which`
// within radius, the float64 sums of their flux and of their flux times the cone weight
void oracle_pm_gather(void* pmh, int which, const double* points, size_t n, double radius, uint32_t* out_count, double* out_flux,
                      double* out_cone)
{
    const PhotonMaps& pm = *static_cast<PhotonMaps*>(pmh);
    const std::vector<float>& ph = pm.photons[which];
    const double r2 = radius * radius, inv_r2 = 1.0 / r2;
    PMCounts cnt;
    for (size_t i = 0; i < n; i++)
    {
        const std::vector<std::pair<double, uint32_t>> d = gatherBrute(pm, which, D3(points + 3 * i), r2, cnt);
        D3 f, c;
        for (const auto& r : d)
        {
            const float* p = &ph[8 * (size_t)r.second];
            const D3 flux((double)p[0], (double)p[1], (double)p[2]);
            f = f + flux;
            c = c + flux * coneWeight(r.first, inv_r2);
        }
        out_count[i] = (uint32_t)d.size();
        const double v[6] = { f.x, f.y, f.z, c.x, c.y, c.z };
        std::memcpy(out_flux + 3 * i, v, 24); std::memcpy(out_cone + 3 * i, v + 3, 24);
    }
}

// The estimate of map `which` at the first vertex of each (ray, pixel, sample), as pmSampleRay makes it there, with
// gather radius radius[i] (0: the k-NN estimate). out [n][3]: the estimate (0 where the ray misses or the vertex is a delta
// one), position [n][3]: the vertex (NaN where the ray misses), estimated [n]: 1 where the estimate ran
void oracle_pm_first_estimate(void* pmh, int which, const mcrt_ray* rays, const uint32_t* pixel, const uint32_t* sample, size_t n,
                              uint32_t seed, const double* radius, double* out, double* position, uint8_t* estimated)
{
    const PhotonMaps& pm = *static_cast<PhotonMaps*>(pmh);
    const Scene& s = *pm.s;
    Sampler smp(seed);
    PMCounts cnt;
    for (size_t i = 0; i < n; i++)
    {
        smp.initiate(pixel[i]); smp.setIndex(sample[i]);
        const Ray ray = makeRay(D3(rays[i].origin), D3(rays[i].direction), s.d.scene_ior);
        smp.shuffle();
        const Isect is = intersect(s, ray, nullptr);
        D3 e, pos(std::nan(""), std::nan(""), std::nan(""));
        estimated[i] = 0;
        if (is.prim != 0xFFFFFFFFu)
        {
            const Interaction ia = makeInteraction(s, is, ray, ray.medium_ior, smp);
            pos = ia.position;
            if (!ia.dirac_delta)
            {
                e = photonEstimate(pm, which, ia, radius[i] * radius[i], cnt);
                estimated[i] = 1;
            }
        }
        const double v[6] = { e.x, e.y, e.z, pos.x, pos.y, pos.z };
        std::memcpy(out + 3 * i, v, 24); std::memcpy(position + 3 * i, v + 3, 24);
    }
}

namespace
{
    void storeSample(const D3& r, const D3 comp[4], size_t i, double* rgb, double* comp_out)
    {
        rgb[3 * i] = r.x; rgb[3 * i + 1] = r.y; rgb[3 * i + 2] = r.z;
        if (comp_out)
            for (int c = 0; c < 4; c++) { double* o = comp_out + (4 * i + c) * 3; o[0] = comp[c].x; o[1] = comp[c].y; o[2] = comp[c].z; }
    }
    void storeCounts(const PMCounts& c, uint64_t* counts)
    {
        if (counts)
        {
            counts[0] = c.rays; counts[1] = c.shadow_rays; counts[2] = c.queries; counts[3] = c.ties; counts[4] = c.empty;
            counts[5] = c.photons;
        }
    }

    // body(first, last, smp, counts) over [0, n) in contiguous chunks on up to hardware_concurrency threads, each with its own
    // sampler; -> the chunks' counts added up. Every sample sets its sampler's state from (pixel, sample), and the maps and
    // the scene are only read, so the results do not depend on the split.
    PMCounts parallelSamples(size_t n, uint32_t seed, const std::function<void(size_t, size_t, Sampler&, PMCounts&)>& body)
    {
        const size_t t_max = std::max(1u, std::thread::hardware_concurrency());
        const size_t T = std::max<size_t>(1, std::min<size_t>(t_max, n / 64));
        std::vector<PMCounts> cnt(T);
        std::vector<std::thread> threads;
        for (size_t t = 0; t < T; t++)
            threads.emplace_back([&, t] { Sampler smp(seed); body(n * t / T, n * (t + 1) / T, smp, cnt[t]); });
        for (std::thread& th : threads) th.join();
        PMCounts total;
        for (const PMCounts& c : cnt)
        {
            total.rays += c.rays; total.shadow_rays += c.shadow_rays; total.queries += c.queries; total.ties += c.ties;
            total.empty += c.empty; total.photons += c.photons;
        }
        return total;
    }
}

// per (ray, pixel, sample): rgb [n][3], comp [n][4][3] (may be null); counts: rays, shadow rays, k-NN queries, k-th distance ties
void oracle_pm_sample_rays(void* pmh, const mcrt_ray* rays, const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t seed,
                           double* rgb, double* comp, uint64_t* counts)
{
    const PhotonMaps& pm = *static_cast<PhotonMaps*>(pmh);
    storeCounts(parallelSamples(n, seed, [&](size_t first, size_t last, Sampler& smp, PMCounts& cnt)
    {
        for (size_t i = first; i < last; i++)
        {
            smp.initiate(pixel[i]); smp.setIndex(sample[i]);
            D3 c[4];
            const D3 r = pmSampleRay(pm, makeRay(D3(rays[i].origin), D3(rays[i].direction), pm.s->d.scene_ior), smp, c, cnt);
            storeSample(r, c, i, rgb, comp);
        }
    }), counts);
}

// the brute-force k-NN search on caller points: out_d2 / out_index [n][k] nearest first (unused slots: +inf / 0xFFFFFFFF),
// out_count [n]; *ties: queries with a tie at the k-th distance
void oracle_pm_knn(void* pmh, int which, const double* points, size_t n, double* out_d2, uint32_t* out_index, uint32_t* out_count, uint64_t* ties)
{
    const PhotonMaps& pm = *static_cast<PhotonMaps*>(pmh);
    PMCounts cnt;
    for (size_t i = 0; i < n; i++)
    {
        const std::vector<std::pair<double, uint32_t>> d = knnBrute(pm, which, D3(points + 3 * i), cnt);
        out_count[i] = (uint32_t)d.size();
        for (uint32_t j = 0; j < pm.k; j++)
        {
            const bool have = j < d.size();
            out_d2[i * pm.k + j] = have ? d[d.size() - 1 - j].first : std::numeric_limits<double>::infinity();
            out_index[i * pm.k + j] = have ? d[d.size() - 1 - j].second : 0xFFFFFFFFu;
        }
    }
    *ties = cnt.ties;
}

// Camera::samplePixel for (pixel, sample) pairs, as oracle_sample_pixels; rays6 (may be null): the camera rays
void oracle_pm_sample_pixels(void* pmh, const mcrt_camera* cam, const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t seed,
                             double* rgb, double* comp, double* rays6, uint64_t* counts)
{
    const PhotonMaps& pm = *static_cast<PhotonMaps*>(pmh);
    storeCounts(parallelSamples(n, seed, [&](size_t first, size_t last, Sampler& smp, PMCounts& cnt)
    {
        for (size_t i = first; i < last; i++)
        {
            smp.initiate(pixel[i]); smp.setIndex(sample[i]);
            const Ray ray = cameraRay(*cam, pm.s->d.scene_ior, pixel[i], smp);
            if (rays6)
            {
                const double v[6] = { ray.start.x, ray.start.y, ray.start.z, ray.direction.x, ray.direction.y, ray.direction.z };
                std::memcpy(rays6 + 6 * i, v, sizeof(v));
            }
            D3 c[4];
            const D3 r = pmSampleRay(pm, ray, smp, c, cnt);
            storeSample(r, c, i, rgb, comp);
        }
    }), counts);
}

// rows [y0, y1) with the default box film, as oracle_render_rows; comp (may be null): [4][y1 - y0][width][3], each term's
// mean over the pixel's samples (not clamped)
void oracle_pm_render_rows(void* pmh, const mcrt_camera* cam, uint32_t y0, uint32_t y1, uint32_t sqrtspp, uint32_t seed, double* out,
                           double* comp, uint64_t* counts)
{
    const PhotonMaps& pm = *static_cast<PhotonMaps*>(pmh);
    const uint32_t spp = sqrtspp * sqrtspp;
    const size_t plane = (size_t)(y1 - y0) * cam->width * 3;
    storeCounts(parallelSamples((size_t)(y1 - y0) * cam->width, seed, [&](size_t first, size_t last, Sampler& smp, PMCounts& cnt)
    {
        for (size_t p = first; p < last; p++)
        {
            const uint32_t pixel = y0 * cam->width + (uint32_t)p;
            smp.initiate(pixel);
            D3 sum, csum[4];
            for (uint32_t i = 0; i < spp; i++)
            {
                smp.setIndex(i);
                D3 c[4];
                const D3 r = pmSampleRay(pm, cameraRay(*cam, pm.s->d.scene_ior, pixel, smp), smp, c, cnt);
                sum = sum + r * 1.0; // Film::Splat::update, weight 1
                for (int k = 0; k < 4; k++) csum[k] = csum[k] + c[k];
            }
            const size_t at = p * 3;
            const D3 v = sum / (double)spp;
            out[at] = v.x < 0.0 ? 0.0 : v.x; out[at + 1] = v.y < 0.0 ? 0.0 : v.y; out[at + 2] = v.z < 0.0 ? 0.0 : v.z;
            if (comp)
                for (int k = 0; k < 4; k++)
                {
                    const D3 m = csum[k] / (double)spp;
                    comp[k * plane + at] = m.x; comp[k * plane + at + 1] = m.y; comp[k * plane + at + 2] = m.z;
                }
        }
    }), counts);
}

// Image::save without the file (image.cpp:37-88, histogram.cpp, pixel-operators.cpp, srgb.hpp:54-62)
namespace
{
    void tonemapOp(uint32_t op, const double in[3], double out[3])
    {
        if (op == MCRT_TONEMAP_LINEAR) { for (int c = 0; c < 3; c++) out[c] = in[c]; return; }
        if (op == MCRT_TONEMAP_ACES)
        {
            const double v[3] = {0.59719 * in[0] + 0.35458 * in[1] + 0.04823 * in[2], 0.07600 * in[0] + 0.90834 * in[1] + 0.01566 * in[2],
                                 0.02840 * in[0] + 0.13383 * in[1] + 0.83777 * in[2]};
            double r[3];
            for (int c = 0; c < 3; c++) r[c] = (v[c] * (v[c] + 0.0245786) - 0.000090537) / (v[c] * (0.983729 * v[c] + 0.4329510) + 0.238081);
            const double o[3] = {1.60475 * r[0] + -0.53108 * r[1] + -0.07367 * r[2], -0.10208 * r[0] + 1.10813 * r[1] + -0.00605 * r[2],
                                 -0.00327 * r[0] + -0.07276 * r[1] + 1.07602 * r[2]};
            for (int c = 0; c < 3; c++) out[c] = std::min(std::max(o[c], 0.0), 1.0);
            return;
        }
        const double A = 0.15, B = 0.50, Cc = 0.10, D = 0.20, E = 0.02, F = 0.30, W = 11.2;
        auto f = [&](double x) { return ((x * (A * x + Cc * B) + D * E) / (x * (A * x + B) + D * F)) - E / F; };
        for (int c = 0; c < 3; c++) out[c] = f(in[c]) / f(W);
    }

    double histogramLevel(const std::vector<double>& data, double pct)
    {
        const size_t bins = 65536;
        double mx = std::numeric_limits<double>::lowest();
        for (double v : data) { if (v < 0.0) return 0.0; if (mx < v) mx = v; }
        if (!(mx > 0.0)) return 0.0;
        const double bin_size = mx / bins;
        std::vector<size_t> counts(bins, 0);
        for (double v : data) counts[std::min((size_t)(v / bin_size), bins - 1)]++;
        const size_t num = (size_t)(data.size() * pct);
        size_t count = 0;
        for (size_t i = 0; i < bins; i++) { count += counts[i]; if (count >= num) return (i + 1) * bin_size; }
        return 0.0;
    }
}

void oracle_image_tonemap(const double* rgb, uint32_t width, uint32_t height, const mcrt_image_params* prm, uint8_t* out_bgr,
                          double* exposure_factor, double* gain_factor)
{
    const size_t n = (size_t)width * height;
    const uint32_t op = prm->plain ? (uint32_t)MCRT_TONEMAP_LINEAR : prm->tonemapper;
    double exposure = 1.0, gain = 1.0;
    if (!prm->plain)
    {
        std::vector<double> b(n);
        for (size_t i = 0; i < n; i++) b[i] = (rgb[3 * i] + rgb[3 * i + 1] + rgb[3 * i + 2]) / 3.0;
        double L = histogramLevel(b, 0.5);
        exposure = (L > 0.0 ? 0.5 / L : 1.0) * prm->exposure_scale;
        for (size_t i = 0; i < n; i++)
        {
            const double q[3] = {rgb[3 * i] * exposure, rgb[3 * i + 1] * exposure, rgb[3 * i + 2] * exposure};
            double t[3];
            tonemapOp(op, q, t);
            b[i] = (t[0] + t[1] + t[2]) / 3.0;
        }
        L = histogramLevel(b, 0.99);
        gain = (L > 0.0 ? 0.99 / L : 1.0) * prm->gain_scale;
    }
    for (size_t i = 0; i < n; i++)
    {
        const double q[3] = {rgb[3 * i] * exposure, rgb[3 * i + 1] * exposure, rgb[3 * i + 2] * exposure};
        double t[3];
        tonemapOp(op, q, t);
        for (int c = 0; c < 3; c++)
        {
            const double x = t[c] * gain;
            const double g = x <= 0.0031308 ? 12.92 * x : 1.055 * std::pow(x, 1.0 / 2.4) - 0.055;
            out_bgr[3 * i + (2 - c)] = (uint8_t)(std::min(std::max(g, 0.0), 1.0) * std::nextafter(256.0, 0.0));
        }
    }
    if (exposure_factor) *exposure_factor = exposure;
    if (gain_factor) *gain_factor = gain;
}

} // extern "C"
