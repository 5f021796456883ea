// Device-side scene layout, templated on the arithmetic type R.
//
// HBM layout (all arrays are built once in mcrt_scene_upload from the float64 description):
//   wide      the BVH (source/bvh/bvh.hpp:68-82) re-laid as one record per *child* {min.xyz,
//             max.xyz, a, b}: the children of an inner node are contiguous, in next_sibling order,
//             so one inner visit is n independent loads (2×float4 each in float = the "32 B per
//             box" of the roofline formula, SURVEY.md §8d; 64 B in double). (a,b) = (first child
//             record, child count) for inner children and (first prim, count | LEAF) for leaves.
//             Both traversals use it: the reference-order best-first one (parity) keeps the
//             reference's child order, the depth-first one (fast mode) sorts children by distance.
//   geom      3 × V4<R> per ordered primitive = the 48 B (float) / 96 B (double) intersection
//             record: triangle {v0,type | E1 | E2}, sphere {origin,type | radius | -},
//             quadric {index,type | - | -}. Indexed by ordered-primitive id: no indirection.
//   bvh4_geom the same records in the order of the BVH4's leaf references, so that a leaf's primitives
//             are contiguous also where spatial splits give a primitive several references (bvh4.cuh);
//             bvh4_prim maps each reference back to its ordered primitive.
//   shade     per ordered primitive: geometric normal (triangles), material id, vertex-normal id,
//             area, light id.
//   vnormals  3 × V4<R> per smooth triangle.
//   quadrics  Q (4x4), G (4x3) and clip box per quadric.
//   materials mcrt_material fields converted to R.
//   lights    per emissive: prim id, CDF value, sampling geometry, area, radiosity.
#pragma once

#include "vec.cuh"

namespace mcrt
{
    constexpr uint32_t NO_PRIM = 0xFFFFFFFFu;
    constexpr uint32_t WIDE_LEAF = 0x80000000u;

    enum PrimType : uint32_t { PRIM_TRIANGLE = 0, PRIM_SPHERE = 1, PRIM_QUADRIC = 2 };

    // One record per *child*: the children of an inner node are stored contiguously in the order of
    // the reference's next_sibling chain (bvh.cpp:109-118), so one inner-node visit is n independent
    // loads instead of n dependent pointer hops. (a, b) = (first child record, child count) for an
    // inner child, (first primitive, count | WIDE_LEAF) for a leaf. 32 B in float, 64 B in double.
    template <class R> struct WideChild;
    template <> struct alignas(16) WideChild<float>
    {
        float bmin[3];
        float bmax[3];
        uint32_t a, b;
    };
    template <> struct alignas(16) WideChild<double>
    {
        double bmin[3];
        double bmax[3];
        uint32_t a, b;
        uint32_t _pad[2];
    };

    template <class R> struct alignas(16) PrimShade
    {
        R nx, ny, nz;   // Triangle::normal_
        R area;         // Surface::Base::area_
        uint32_t material;
        int32_t vn_index;   // -1: no vertex normals
        uint32_t type;
        uint32_t light;     // index into lights or NO_PRIM
    };

    template <class R> struct alignas(16) Quadric
    {
        R Q[16];  // column-major
        R G[12];  // column-major 4 columns x 3 rows
        R bmin[3], bmax[3];
    };

    template <class R> struct alignas(16) Material
    {
        V3<R> reflectance, specular_reflectance, transmittance, emittance;
        V3<R> ior_real, ior_imag;
        R roughness, specular_roughness, ior, transparency;
        R A, B, ax, ay;
        uint32_t flags;
    };

    enum MaterialFlags : uint32_t
    {
        MAT_COMPLEX_IOR = 1u, MAT_PERFECT_MIRROR = 2u, MAT_ROUGH = 4u, MAT_ROUGH_SPECULAR = 8u,
        MAT_OPAQUE = 16u, MAT_EMISSIVE = 32u, MAT_DIRAC_DELTA = 64u
    };

    template <class R> struct alignas(16) Light
    {
        V3<R> p0, p1, p2;   // triangle v0,v1,v2  |  sphere origin, (radius,0,0), -
        V3<R> normal;       // triangle face normal
        V3<R> emittance;    // radiosity
        R area;
        R cdf;
        uint32_t prim;
        uint32_t type;
    };

    struct Bvh4Node;   // bvh4.cuh

    template <class R> struct DeviceScene
    {
        const Bvh4Node* bvh4;    // 4-wide float-box BVH of the order-free search (parity mode); null: replay traversal only
        const V4<R>* bvh4_geom;      // geom records in the order of bvh4's leaf references (geom itself when no primitive is split)
        const uint32_t* bvh4_prim;   // ordered primitive of each leaf reference of bvh4
        const WideChild<R>* wide;
        const V4<R>* geom;
        const PrimShade<R>* shade;
        const V4<R>* vnormals;
        const Quadric<R>* quadrics;
        const Material<R>* materials;
        const Light<R>* lights;
        const uint8_t* shade_class;   // per ordered primitive: 1 + index of its material's flag combination (+ vertex normals) among
                                      // those present in the scene (< 64); the shade-coherence sort groups paths by it
        uint32_t n_nodes, n_prims, n_lights, n_wide_root; // n_wide_root: children of the root
        uint32_t root_is_leaf, root_first_prim, root_prim_count;
        uint32_t prims_class;     // PRIMS_ALL / PRIMS_TRI_SPHERE / PRIMS_TRI: selects the pruned traversal kernels
        uint32_t dynamic_fetch;   // k_extend / k_shadow take rays per lane as lanes finish (bvh4.cuh traceManyFast)
        uint32_t _pad3[2];
        uint32_t material_flags_any;   // OR of Material::flags over the scene: selects the k_shade feature set
        R root_bmin[3], root_bmax[3];
        R scene_ior;
        R scene_scale;  // max |coordinate| of the scene bounds; fast-mode ray offsets scale with it
    };

    template <class R> struct DeviceCamera
    {
        V3<R> eye, forward, left, up;
        R focal_length, sensor_width, aperture_radius, focus_distance;
        uint32_t width, height, thin_lens, _pad;
    };

    template <class R> struct Hit
    {
        R t, u, v;
        uint32_t prim;       // NO_PRIM = miss
        uint32_t interpolate;
    };
}
