// Small vector algebra for the device path, templated on the arithmetic type R (double = parity
// mode, float = fast mode). Every compound operation spells out the evaluation order GLM 0.9.9.8
// uses in the reference (lib/glm/glm/detail/func_geometric.inl:48-55,66-78,88,104-108;
// func_common.inl:17-30,104-112; type_mat3x3.inl:468-474), because in parity mode the float64
// result must round exactly like the CPU's: dot = (x+y)+z of the products, cross with the same
// operand pairing, normalize = v * (1/sqrt(dot)), min/max as ternaries (NaN-propagation of the
// slab test depends on it), mix = x*(1-a) + y*a. The f64 translation unit is compiled with
// --fmad=false since the reference build has no FMA contraction (CMakeLists.txt:16-21: -O3 only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#define MCRT_HD __host__ __device__ __forceinline__
#define MCRT_D __device__ __forceinline__

namespace mcrt
{
    template <class R> struct V3
    {
        R x, y, z;
        MCRT_HD V3() { }
        MCRT_HD V3(R a) : x(a), y(a), z(a) { }
        MCRT_HD V3(R a, R b, R c) : x(a), y(b), z(c) { }
        MCRT_HD R operator[](int i) const { return i == 0 ? x : (i == 1 ? y : z); }
    };

    // 4 * sizeof(R) alignment: a record never straddles a 32-byte sector, so a float64 record is two 128-bit
    // accesses to one sector - the path state, hit and shadow records are all V4<double>
    template <class R> struct alignas(4 * sizeof(R)) V4
    {
        R x, y, z, w;
        MCRT_HD V4() { }
        MCRT_HD V4(R a, R b, R c, R d) : x(a), y(b), z(c), w(d) { }
        MCRT_HD V4(const V3<R>& v, R d) : x(v.x), y(v.y), z(v.z), w(d) { }
        MCRT_HD V3<R> xyz() const { return V3<R>(x, y, z); }
    };

    // Streaming access to the wavefront queues (path state, hits, shadow records: written once, read once per
    // bounce, 6.5 GB per pool): the cache-streaming forms (ld.global.cs / st.global.cs = evict-first), so that
    // the 50 MB L2 keeps the scene arrays every ray reads (BVH nodes, float64 triangle records) instead of
    // queue records nobody will touch again. sm_90 has no 256-bit global access: a float64 record is two
    // 128-bit ones.
#if defined(__CUDACC__) && defined(MCRT_NO_STREAM)   // A/B switch: plain accesses
    template <class T> MCRT_D T ldStream(const T* p) { return *p; }
    template <class T> MCRT_D void stStream(T* p, const T& v) { *p = v; }
#elif defined(__CUDACC__)
    MCRT_D V4<double> ldStream(const V4<double>* p)
    {
        const double2 a = __ldcs(reinterpret_cast<const double2*>(p));
        const double2 b = __ldcs(reinterpret_cast<const double2*>(p) + 1);
        return V4<double>(a.x, a.y, b.x, b.y);
    }
    MCRT_D void stStream(V4<double>* p, const V4<double>& v)
    {
        __stcs(reinterpret_cast<double2*>(p), make_double2(v.x, v.y));
        __stcs(reinterpret_cast<double2*>(p) + 1, make_double2(v.z, v.w));
    }
    MCRT_D V4<float> ldStream(const V4<float>* p)
    {
        const float4 f = __ldcs(reinterpret_cast<const float4*>(p));
        return V4<float>(f.x, f.y, f.z, f.w);
    }
    MCRT_D void stStream(V4<float>* p, const V4<float>& v) { __stcs(reinterpret_cast<float4*>(p), make_float4(v.x, v.y, v.z, v.w)); }
    MCRT_D uint4 ldStream(const uint4* p) { return __ldcs(p); }
    MCRT_D void stStream(uint4* p, const uint4& v) { __stcs(p, v); }
#endif

    template <class R> MCRT_HD V3<R> operator+(const V3<R>& a, const V3<R>& b) { return V3<R>(a.x + b.x, a.y + b.y, a.z + b.z); }
    template <class R> MCRT_HD V3<R> operator-(const V3<R>& a, const V3<R>& b) { return V3<R>(a.x - b.x, a.y - b.y, a.z - b.z); }
    template <class R> MCRT_HD V3<R> operator*(const V3<R>& a, const V3<R>& b) { return V3<R>(a.x * b.x, a.y * b.y, a.z * b.z); }
    template <class R> MCRT_HD V3<R> operator/(const V3<R>& a, const V3<R>& b) { return V3<R>(a.x / b.x, a.y / b.y, a.z / b.z); }
    template <class R> MCRT_HD V3<R> operator*(const V3<R>& a, R s) { return V3<R>(a.x * s, a.y * s, a.z * s); }
    template <class R> MCRT_HD V3<R> operator*(R s, const V3<R>& a) { return V3<R>(s * a.x, s * a.y, s * a.z); }
    template <class R> MCRT_HD V3<R> operator/(const V3<R>& a, R s) { return V3<R>(a.x / s, a.y / s, a.z / s); }
    template <class R> MCRT_HD V3<R> operator/(R s, const V3<R>& a) { return V3<R>(s / a.x, s / a.y, s / a.z); }
    template <class R> MCRT_HD V3<R> operator-(const V3<R>& a) { return V3<R>(-a.x, -a.y, -a.z); }
    template <class R> MCRT_HD V3<R>& operator+=(V3<R>& a, const V3<R>& b) { a = a + b; return a; }
    template <class R> MCRT_HD V3<R>& operator-=(V3<R>& a, const V3<R>& b) { a = a - b; return a; }
    template <class R> MCRT_HD V3<R>& operator*=(V3<R>& a, const V3<R>& b) { a = a * b; return a; }
    template <class R> MCRT_HD V3<R>& operator*=(V3<R>& a, R s) { a = a * s; return a; }
    template <class R> MCRT_HD V3<R>& operator/=(V3<R>& a, R s) { a = a / s; return a; }

    // glm::min / glm::max / std::min / std::max: ternaries, not fmin/fmax
    template <class R> MCRT_HD R gmin(R x, R y) { return (y < x) ? y : x; }
    template <class R> MCRT_HD R gmax(R x, R y) { return (x < y) ? y : x; }
    template <class R> MCRT_HD R gclamp(R x, R lo, R hi) { return gmin(gmax(x, lo), hi); }
    template <class R> MCRT_HD V3<R> vmin(const V3<R>& a, const V3<R>& b) { return V3<R>(gmin(a.x, b.x), gmin(a.y, b.y), gmin(a.z, b.z)); }
    template <class R> MCRT_HD V3<R> vmax(const V3<R>& a, const V3<R>& b) { return V3<R>(gmax(a.x, b.x), gmax(a.y, b.y), gmax(a.z, b.z)); }
    template <class R> MCRT_HD R compMax(const V3<R>& v) { return gmax(gmax(v.x, v.y), v.z); }
    template <class R> MCRT_HD R compMin(const V3<R>& v) { return gmin(gmin(v.x, v.y), v.z); }

    template <class R> MCRT_HD R dot(const V3<R>& a, const V3<R>& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
    template <class R> MCRT_HD V3<R> cross(const V3<R>& x, const V3<R>& y)
    {
        return V3<R>(x.y * y.z - y.y * x.z, x.z * y.x - y.z * x.x, x.x * y.y - y.x * x.y);
    }

    MCRT_HD double rsqrt_ieee(double x) { return 1.0 / sqrt(x); }
    MCRT_HD float rsqrt_ieee(float x) { return 1.0f / sqrtf(x); }
    MCRT_HD double msqrt(double x) { return sqrt(x); }
    MCRT_HD float msqrt(float x) { return sqrtf(x); }
    MCRT_HD double mabs(double x) { return fabs(x); }
    MCRT_HD float mabs(float x) { return fabsf(x); }
    MCRT_HD double mcopysign(double a, double b) { return copysign(a, b); }
    MCRT_HD float mcopysign(float a, float b) { return copysignf(a, b); }
    MCRT_D void msincos(double a, double* s, double* c) { sincos(a, s, c); }
    MCRT_D void msincos(float a, float* s, float* c) { sincosf(a, s, c); }
    MCRT_D double masin(double x) { return asin(x); }
    MCRT_D float masin(float x) { return asinf(x); }

    template <class R> MCRT_HD V3<R> normalize(const V3<R>& v) { return v * rsqrt_ieee(dot(v, v)); }
    template <class R> MCRT_HD R length(const V3<R>& v) { return msqrt(dot(v, v)); }
    template <class R> MCRT_HD V3<R> reflect(const V3<R>& I, const V3<R>& N) { return I - N * dot(N, I) * R(2); }
    template <class R> MCRT_HD R mix(R x, R y, R a) { return x * (R(1) - a) + y * a; }
    template <class R> MCRT_HD V3<R> mix(const V3<R>& x, const V3<R>& y, R a) { return x * (R(1) - a) + y * a; }
    template <class R> MCRT_HD R pow2(R x) { return x * x; }

    template <class R> struct Consts;
    template <> struct Consts<double>
    {
        static constexpr double PI = 3.14159265358979323846;
        static constexpr double INV_PI = 0.31830988618379067154;
        static constexpr double TWO_PI = 6.283185307179586476925;
        static constexpr double EPSILON = 1e-9; // source/common/constants.hpp:9
        static constexpr double MAXV = 1.7976931348623157e308;
    };
    template <> struct Consts<float>
    {
        static constexpr float PI = 3.14159265358979323846f;
        static constexpr float INV_PI = 0.31830988618379067154f;
        static constexpr float TWO_PI = 6.283185307179586476925f;
        static constexpr float EPSILON = 1e-9f; // thresholds on material parameters only
        static constexpr float MAXV = 3.402823466e38f;
    };

    // Duff et al. orthonormal basis exactly as source/common/coordinate-system.cpp:7-40.
    template <class R> struct Frame
    {
        V3<R> c0, c1, c2; // columns of T; c2 = normal

        MCRT_HD Frame() { }
        MCRT_HD explicit Frame(const V3<R>& N)
        {
            R sign = mcopysign(R(1), N.z);
            R a = R(-1) / (sign + N.z);
            R b = N.x * N.y * a;
            c0 = V3<R>(R(1) + sign * N.x * N.x * a, sign * b, -sign * N.x);
            c1 = V3<R>(b, sign + N.y * N.y * a, -N.y);
            c2 = N;
        }
        // T * v
        MCRT_HD V3<R> from(const V3<R>& v) const
        {
            return V3<R>(c0.x * v.x + c1.x * v.y + c2.x * v.z,
                         c0.y * v.x + c1.y * v.y + c2.y * v.z,
                         c0.z * v.x + c1.z * v.y + c2.z * v.z);
        }
        // transpose(T) * v
        MCRT_HD V3<R> to(const V3<R>& v) const
        {
            return V3<R>(c0.x * v.x + c0.y * v.y + c0.z * v.z,
                         c1.x * v.x + c1.y * v.y + c1.z * v.z,
                         c2.x * v.x + c2.y * v.y + c2.z * v.z);
        }
    };
}
