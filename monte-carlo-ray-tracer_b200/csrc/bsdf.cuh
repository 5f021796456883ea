// Material / BSDF evaluation and sampling on the device. Same lobe algebra and — in double —
// the same expression order as the reference:
//   Fresnel::dielectric / conductor            source/material/fresnel.cpp:16-49
//   GGX::{D,DV,Lambda,SmithG1,SmithG2,reflection,transmission,visibleMicrofacet}
//                                              source/material/ggx.cpp:21-89
//   Material::{diffuse,specular}Reflection, specularTransmission, OrenNayar
//                                              source/material/material.cpp:17-95
//   Interaction ctor / selectType / BSDF / sampleBSDF / specularNormal
//                                              source/ray/interaction.cpp:12-193
//   Ray(const Interaction&)                    source/ray/ray.cpp:16-67
#pragma once

#include "scene.cuh"
#include "sampler.cuh"

namespace mcrt
{
    template <class R>
    MCRT_D R fresnelDielectric(R n1, R n2, R cos_theta)
    {
        R g2 = pow2(n2 / n1) + pow2(cos_theta) - R(1);
        if (g2 < R(0)) return R(1);
        R g = msqrt(g2);
        R g_p_c = g + cos_theta;
        R g_m_c = g - cos_theta;
        return R(0.5) * pow2(g_m_c / g_p_c) * (R(1) + pow2((g_p_c * cos_theta - R(1)) / (g_m_c * cos_theta + R(1))));
    }

    template <class R> MCRT_D V3<R> vsqrt(const V3<R>& v) { return V3<R>(msqrt(v.x), msqrt(v.y), msqrt(v.z)); }
    template <class R> MCRT_D V3<R> operator+(const V3<R>& a, R s) { return V3<R>(a.x + s, a.y + s, a.z + s); }
    template <class R> MCRT_D V3<R> operator-(const V3<R>& a, R s) { return V3<R>(a.x - s, a.y - s, a.z - s); }

    template <class R>
    MCRT_D V3<R> fresnelConductor(R n1, const V3<R>& real, const V3<R>& imag, R cos_theta)
    {
        R cos_theta2 = pow2(cos_theta);
        R sin_theta2 = R(1) - cos_theta2;
        V3<R> er = real / n1, ei = imag / n1;
        V3<R> eta2 = er * er;
        V3<R> eta_k2 = ei * ei;
        V3<R> t0 = eta2 - eta_k2 - sin_theta2;
        V3<R> a2_p_b2 = vsqrt(t0 * t0 + R(4) * eta2 * eta_k2);
        V3<R> t1 = a2_p_b2 + cos_theta2;
        V3<R> t2 = R(2) * cos_theta * vsqrt(R(0.5) * (a2_p_b2 + t0));
        V3<R> r_perp = (t1 - t2) / (t1 + t2);
        V3<R> t3 = cos_theta2 * a2_p_b2 + pow2(sin_theta2);
        V3<R> t4 = t2 * sin_theta2;
        V3<R> r_par = r_perp * (t3 - t4) / (t3 + t4);
        return (r_par + r_perp) * R(0.5);
    }

    // ---------------------------------------------------------------------------- GGX
    template <class R> MCRT_D R ggxD(const V3<R>& m, R ax, R ay)
    {
        return R(1) / (Consts<R>::PI * ax * ay * pow2(pow2(m.x / ax) + pow2(m.y / ay) + pow2(m.z)));
    }
    template <class R> MCRT_D R ggxLambda(const V3<R>& w, R ax, R ay)
    {
        return (R(-1) + msqrt(R(1) + (pow2(ax * w.x) + pow2(ay * w.y)) / (pow2(w.z)))) / R(2);
    }
    template <class R> MCRT_D R ggxG1(const V3<R>& w, R ax, R ay) { return R(1) / (R(1) + ggxLambda(w, ax, ay)); }
    template <class R> MCRT_D R ggxG2(const V3<R>& wi, const V3<R>& wo, R ax, R ay)
    {
        return R(1) / (R(1) + ggxLambda(wo, ax, ay) + ggxLambda(wi, ax, ay));
    }
    template <class R> MCRT_D R ggxDV(const V3<R>& m, const V3<R>& wo, R ax, R ay)
    {
        return ggxG1(wo, ax, ay) * dot(wo, m) * ggxD(m, ax, ay) / wo.z;
    }
    template <class R> MCRT_D R ggxReflection(const V3<R>& wi, const V3<R>& wo, R ax, R ay, R& pdf)
    {
        V3<R> m = normalize(wo + wi);
        pdf = ggxDV(m, wo, ax, ay) / (R(4) * dot(m, wo));
        return ggxD(m, ax, ay) * ggxG2(wi, wo, ax, ay) / (R(4) * wo.z * wi.z);
    }
    template <class R> MCRT_D R ggxTransmission(const V3<R>& wi, const V3<R>& wo, R n1, R n2, R ax, R ay, R& pdf)
    {
        V3<R> m = wo * n1 + wi * n2;
        R m_length2 = dot(m, m);
        m /= msqrt(m_length2);
        if (n1 < n2) m = -m;
        R dm_dwi = pow2(n2) * mabs(dot(wi, m)) / m_length2;
        pdf = ggxDV(m, wo, ax, ay) * dm_dwi;
        return mabs(ggxG2(wi, wo, ax, ay) * ggxD(m, ax, ay) * dot(wo, m) * dm_dwi / (wo.z * wi.z));
    }
    template <class R> MCRT_D V3<R> ggxVisibleMicrofacet(R u, R v, const V3<R>& wo, R ax, R ay)
    {
        V3<R> Vh = normalize(V3<R>(ax * wo.x, ay * wo.y, wo.z));
        R len2 = pow2(Vh.x) + pow2(Vh.y);
        V3<R> T1 = len2 > R(0) ? V3<R>(-Vh.y, Vh.x, R(0)) * rsqrt_ieee(len2) : V3<R>(R(1), R(0), R(0));
        V3<R> T2 = cross(Vh, T1);
        R r = msqrt(u);
        R phi = v * Consts<R>::TWO_PI;
        R sn, cs;
        msincos(phi, &sn, &cs);
        R t1 = r * cs;
        R t2 = r * sn;
        R s = R(0.5) * (R(1) + Vh.z);
        t2 = (R(1) - s) * msqrt(R(1) - pow2(t1)) + s * t2;
        V3<R> Nh = t1 * T1 + t2 * T2 + msqrt(gmax(R(0), R(1) - pow2(t1) - pow2(t2))) * Vh;
        return normalize(V3<R>(ax * Nh.x, ay * Nh.y, gmax(R(0), Nh.z)));
    }

    // ---------------------------------------------------------------------------- Material
    template <class R> MCRT_D V3<R> matDiffuseReflection(const Material<R>& m, uint32_t flags, const V3<R>& wi, const V3<R>& wo, R& pdf)
    {
        if (wi.z < R(0)) { pdf = R(0); return V3<R>(R(0)); }
        pdf = wi.z * Consts<R>::INV_PI;
        V3<R> lambert = m.reflectance * Consts<R>::INV_PI;
        if (!(flags & MAT_ROUGH)) return lambert;
        if constexpr (sizeof(R) == 4)
        {
            // float32: a unit vector's z can round to a hair above 1 and its xy part to exactly 0 (normal incidence), where
            // the float64 expressions below give sqrt(< 0) and 0 / 0; both limits of the term are 0
            const R sin2 = (pow2(wi.x) + pow2(wi.y)) * (pow2(wo.x) + pow2(wo.y));
            const R cos_delta_phi = sin2 > R(0) ? gclamp((wi.x * wo.x + wi.y * wo.y) / msqrt(sin2), R(0), R(1)) : R(0);
            const R D = msqrt(gmax(R(0), (R(1) - pow2(wi.z)) * (R(1) - pow2(wo.z)))) / gmax(wi.z, wo.z);
            return lambert * (m.A + m.B * cos_delta_phi * D);
        }
        R cos_delta_phi = gclamp((wi.x * wo.x + wi.y * wo.y) /
                                 msqrt((pow2(wi.x) + pow2(wi.y)) * (pow2(wo.x) + pow2(wo.y))), R(0), R(1));
        R D = msqrt((R(1) - pow2(wi.z)) * (R(1) - pow2(wo.z))) / gmax(wi.z, wo.z);
        return lambert * (m.A + m.B * cos_delta_phi * D);
    }

    template <class R> MCRT_D V3<R> matSpecularReflection(const Material<R>& m, uint32_t flags, const V3<R>& wi, const V3<R>& wo, R& pdf)
    {
        if (wi.z < R(0)) { pdf = R(0); return V3<R>(R(0)); }
        if (flags & MAT_ROUGH_SPECULAR) return m.specular_reflectance * ggxReflection(wi, wo, m.ax, m.ay, pdf);
        pdf = R(1);
        return m.specular_reflectance / mabs(wi.z);
    }

    template <class R> MCRT_D V3<R> matSpecularTransmission(const Material<R>& m, uint32_t flags, const V3<R>& wi, const V3<R>& wo,
                                                            R n1, R n2, R& pdf, bool inside, bool flux)
    {
        if (wi.z > R(0)) { pdf = R(0); return V3<R>(R(0)); }
        V3<R> btdf = !inside ? m.transmittance : V3<R>(R(1));
        if (flags & MAT_ROUGH_SPECULAR)
        {
            btdf *= ggxTransmission(wi, wo, n1, n2, m.ax, m.ay, pdf);
            if (flux) btdf *= pow2(n2 / n1);
        }
        else
        {
            pdf = R(1);
            btdf *= m.transmittance / mabs(wi.z);
            if (!flux) btdf *= pow2(n1 / n2);
        }
        return btdf;
    }

    // ---------------------------------------------------------------------------- Ray / Interaction
    // Ray record of source/ray/ray.hpp:18-25 (inv_direction is recomputed where needed).
    template <class R> struct PathRay
    {
        V3<R> start, direction;
        R medium_ior, refraction_scale;
        uint32_t depth, diffuse_depth;
        int32_t refraction_level;
        bool dirac_delta, refraction;
    };

    enum InteractionType : uint32_t { IA_REFLECT = 0, IA_REFRACT = 1, IA_DIFFUSE = 2 };

    template <class R> struct Interaction
    {
        uint32_t type;
        R t, n1, n2, T, Rf;
        const Material<R>* material;
        // Feature set of the kernel instantiation (k_shade<.., FEATS>), a compile-time constant after
        // inlining: scenes without GGX / Oren-Nayar / conductors run kernels from which that code is
        // pruned, because (flags & fmask) & bit folds to 0 for the bits the mask lacks.
        uint32_t fmask;
        MCRT_D uint32_t flags() const { return material->flags & fmask; }
        uint32_t prim;
        V3<R> position, normal, out;
        Frame<R> shading_cs;
        bool inside, dirac_delta;

        // Interaction::BSDF (private overload), interaction.cpp:84-153. Kept inline: a __noinline__
        // version shrinks k_shade<double> from 9176 to 6864 SASS instructions but measured 17 % slower
        // (call ABI spills the Interaction).
        MCRT_D V3<R> bsdfLocal(const V3<R>& wo, const V3<R>& wi, R& pdf, bool flux, bool wi_dirac_delta) const
        {
            const Material<R>& m = *material;
            R cos_theta = wo.z;
            if (flags() & MAT_ROUGH_SPECULAR)
            {
                if (wi.z > R(0))
                {
                    cos_theta = dot(wo, normalize(wo + wi));
                }
                else
                {
                    V3<R> hm = normalize(wo * n1 + wi * n2);
                    cos_theta = dot(wo, hm);
                    if (n1 < n2) cos_theta = -cos_theta;
                }
            }

            if (flags() & (MAT_PERFECT_MIRROR | MAT_COMPLEX_IOR))
            {
                V3<R> brdf = matSpecularReflection(m, flags(), wi, wo, pdf);
                if (flags() & MAT_COMPLEX_IOR) brdf *= fresnelConductor(n1, m.ior_real, m.ior_imag, cos_theta);
                return brdf;
            }

            if (n2 < R(1)) return matDiffuseReflection(m, flags(), wi, wo, pdf);

            R F = fresnelDielectric(n1, n2, cos_theta);

            R pdf_s, pdf_d;
            V3<R> brdf_s = matSpecularReflection(m, flags(), wi, wo, pdf_s);
            V3<R> brdf_d = matDiffuseReflection(m, flags(), wi, wo, pdf_d);

            R pdf_t = pdf_s;
            V3<R> btdf = brdf_s;
            if (F < R(1)) btdf = matSpecularTransmission(m, flags(), wi, wo, n1, n2, pdf_t, inside, flux);

            if (wi_dirac_delta)
            {
                if (type == IA_REFLECT)
                {
                    pdf = Rf;
                    return brdf_s * F;
                }
                else
                {
                    pdf = T * (R(1) - Rf);
                    return btdf * T * (R(1) - F);
                }
            }
            else if (!(flags() & MAT_ROUGH_SPECULAR))
            {
                pdf = pdf_d * (R(1) - Rf) * (R(1) - T);
                return brdf_d * (R(1) - F) * (R(1) - T);
            }

            pdf = mix(mix(pdf_d, pdf_t, T), pdf_s, Rf);
            return mix(mix(brdf_d, btdf, T), brdf_s, F);
        }

        // public Interaction::BSDF for a world-space direction, interaction.cpp:74-82
        MCRT_D bool bsdfWorld(V3<R>& bsdf_absIdotN, const V3<R>& world_wi, R& pdf) const
        {
            V3<R> wi = shading_cs.to(world_wi);
            V3<R> wo = shading_cs.to(out);
            bsdf_absIdotN = bsdfLocal(wo, wi, pdf, false, false) * mabs(wi.z);
            return pdf > R(0);
        }
    };

    // Surface::normal(position) and the shading normal: the interpolated vertex normal where the triangle has them, the
    // face normal where it has none or where the two disagree on the side the ray comes from; both are flipped to face
    // the ray. -> dot(direction, face normal) before the flip. The same computation as buildInteraction's, kept
    // separate for k_features: calling it from buildInteraction changed the registers and spills of k_shade and
    // k_emit_shade (DESIGN.md §3).
    template <class R>
    MCRT_D R surfaceNormals(const DeviceScene<R>& sc, const PrimShade<R>& ps, const Hit<R>& hit, const V3<R>& position,
                            const V3<R>& direction, V3<R>& normal, V3<R>& shading_normal)
    {
        if (ps.type == PRIM_TRIANGLE)
        {
            normal = V3<R>(ps.nx, ps.ny, ps.nz);
        }
        else if (ps.type == PRIM_SPHERE)
        {
            const V4<R> g0 = sc.geom[3 * hit.prim];
            const V4<R> g1 = sc.geom[3 * hit.prim + 1];
            normal = (position - g0.xyz()) / g1.x;
        }
        else
        {
            const Quadric<R>& q = sc.quadrics[(uint32_t)sc.geom[3 * hit.prim].x];
            const V3<R>& p = position;
            // G * vec4(pos, 1): 4x3 matrix, type_mat4x3.inl:474-477
            normal = normalize(V3<R>(q.G[0] * p.x + q.G[3] * p.y + q.G[6] * p.z + q.G[9] * R(1),
                                     q.G[1] * p.x + q.G[4] * p.y + q.G[7] * p.z + q.G[10] * R(1),
                                     q.G[2] * p.x + q.G[5] * p.y + q.G[8] * p.z + q.G[11] * R(1)));
        }

        const R cos_theta = dot(direction, normal);
        shading_normal = normal;
        if (ps.type == PRIM_TRIANGLE && ps.vn_index >= 0)
        {
            const V3<R> n0 = sc.vnormals[3 * ps.vn_index + 0].xyz();
            const V3<R> nA = sc.vnormals[3 * ps.vn_index + 1].xyz();
            const V3<R> nB = sc.vnormals[3 * ps.vn_index + 2].xyz();
            shading_normal = normalize((R(1) - hit.u - hit.v) * n0 + hit.u * nA + hit.v * nB);
            if ((cos_theta < R(0)) != (dot(direction, shading_normal) < R(0))) shading_normal = normal;
        }

        if (cos_theta > R(0))
        {
            normal = -normal;
            shading_normal = -shading_normal;
        }
        return cos_theta;
    }

    // Interaction::Interaction + selectType. `ray_dir`/`ray_start` are the incoming ray.
    // normal_geo: Surface::normal(position); shading normal resolved by the caller's callback data.
    template <uint32_t FEATS = 0xFFFFFFFFu, class R>
    MCRT_D void buildInteraction(Interaction<R>& ia, const DeviceScene<R>& sc, const Hit<R>& hit, const PathRay<R>& ray,
                                 R external_ior, const SamplerState& smp)
    {
        ia.t = hit.t;
        ia.out = -ray.direction;
        ia.n1 = ray.medium_ior;
        ia.prim = hit.prim;
        const PrimShade<R> ps = sc.shade[hit.prim];
        ia.material = &sc.materials[ps.material];
        const Material<R>& m = *ia.material;
        ia.fmask = FEATS;
        ia.position = ray.start + ray.direction * hit.t;

        // Surface::normal(position)
        V3<R> normal;
        if (ps.type == PRIM_TRIANGLE)
        {
            normal = V3<R>(ps.nx, ps.ny, ps.nz);
        }
        else if (ps.type == PRIM_SPHERE)
        {
            const V4<R> g0 = sc.geom[3 * hit.prim];
            const V4<R> g1 = sc.geom[3 * hit.prim + 1];
            normal = (ia.position - g0.xyz()) / g1.x;
        }
        else
        {
            const Quadric<R>& q = sc.quadrics[(uint32_t)sc.geom[3 * hit.prim].x];
            const V3<R>& p = ia.position;
            // G * vec4(pos, 1): 4x3 matrix, type_mat4x3.inl:474-477
            normal = normalize(V3<R>(q.G[0] * p.x + q.G[3] * p.y + q.G[6] * p.z + q.G[9] * R(1),
                                     q.G[1] * p.x + q.G[4] * p.y + q.G[7] * p.z + q.G[10] * R(1),
                                     q.G[2] * p.x + q.G[5] * p.y + q.G[8] * p.z + q.G[11] * R(1)));
        }

        R cos_theta = dot(ray.direction, normal);
        ia.inside = cos_theta > R(0);
        ia.n2 = (ia.inside && !(ia.flags() & MAT_OPAQUE)) ? external_ior : m.ior;

        V3<R> shading_normal = normal;
        if (ps.type == PRIM_TRIANGLE && ps.vn_index >= 0)
        {
            const V3<R> n0 = sc.vnormals[3 * ps.vn_index + 0].xyz();
            const V3<R> nA = sc.vnormals[3 * ps.vn_index + 1].xyz();
            const V3<R> nB = sc.vnormals[3 * ps.vn_index + 2].xyz();
            shading_normal = normalize((R(1) - hit.u - hit.v) * n0 + hit.u * nA + hit.v * nB);
            if ((cos_theta < R(0)) != (dot(ray.direction, shading_normal) < R(0))) shading_normal = normal;
        }

        if (cos_theta > R(0))
        {
            normal = -normal;
            shading_normal = -shading_normal;
        }
        ia.normal = normal;
        ia.shading_cs = Frame<R>(shading_normal);

        ia.Rf = fresnelDielectric(ia.n1, ia.n2, dot(shading_normal, ia.out));
        ia.T = m.transparency;
        if (ia.flags() & MAT_ROUGH_SPECULAR) ia.Rf = gclamp(ia.Rf, R(0.1), R(0.9));

        // selectType, interaction.cpp:156-183
        if (ia.flags() & (MAT_PERFECT_MIRROR | MAT_COMPLEX_IOR))
        {
            ia.type = IA_REFLECT;
        }
        else if (ia.n2 < R(1))
        {
            ia.type = IA_DIFFUSE;
        }
        else
        {
            R p;
            samplerGet<R, DIM_INTERACTION, 1>(smp, &p);
            if (ia.Rf > p) ia.type = IA_REFLECT;
            else if (ia.Rf + (R(1) - ia.Rf) * ia.T > p) ia.type = IA_REFRACT;
            else ia.type = IA_DIFFUSE;
        }
        ia.dirac_delta = ia.type != IA_DIFFUSE && !(ia.flags() & MAT_ROUGH_SPECULAR);
    }

    template <class R>
    MCRT_D V3<R> cosWeightedHemi(R u, R v)
    {
        R r = msqrt(u);
        R azimuth = v * Consts<R>::TWO_PI;
        R sn, cs;
        msincos(azimuth, &sn, &cs);
        return V3<R>(r * cs, r * sn, msqrt(R(1) - u));
    }

    // Ray::Ray(const Interaction&), ray.cpp:16-67. eps = C::EPSILON in parity mode.
    template <class R>
    MCRT_D void spawnRay(PathRay<R>& nr, const Interaction<R>& ia, const PathRay<R>& in, const SamplerState& smp, R eps)
    {
        const Material<R>& m = *ia.material;
        nr.depth = in.depth + 1;
        nr.diffuse_depth = in.diffuse_depth;
        nr.refraction_scale = in.refraction_scale;
        nr.start = ia.position;
        nr.refraction_level = in.refraction_level;
        nr.dirac_delta = ia.dirac_delta;
        nr.refraction = false;

        V3<R> specular_normal;
        if (ia.type != IA_DIFFUSE)
        {
            if (ia.flags() & MAT_ROUGH_SPECULAR)
            {
                R u[2];
                samplerGet<R, DIM_BSDF, 2>(smp, u);
                specular_normal = ia.shading_cs.from(ggxVisibleMicrofacet(u[0], u[1], ia.shading_cs.to(ia.out), m.ax, m.ay));
            }
            else
            {
                specular_normal = ia.shading_cs.c2;
            }
        }

        if (ia.type == IA_REFLECT)
        {
            nr.direction = reflect(in.direction, specular_normal);
            nr.medium_ior = ia.n1;
            nr.start += ia.normal * eps;
        }
        else if (ia.type == IA_REFRACT)
        {
            R inv_eta = ia.n1 / ia.n2;
            R cos_theta = dot(specular_normal, in.direction);
            R k = R(1) - pow2(inv_eta) * (R(1) - pow2(cos_theta));
            if (k >= R(0))
            {
                nr.direction = inv_eta * in.direction - (inv_eta * cos_theta + msqrt(k)) * specular_normal;
                nr.medium_ior = ia.n2;
                nr.start -= ia.normal * eps;
                if (ia.inside) nr.refraction_level--; else nr.refraction_level++;
                nr.refraction_scale *= pow2(R(1) / inv_eta);
                nr.refraction = true;
            }
            else
            {
                nr.direction = in.direction - specular_normal * cos_theta * R(2);
                nr.medium_ior = ia.n1;
                nr.start += ia.normal * eps;
            }
        }
        else
        {
            nr.diffuse_depth++;
            R u[2];
            samplerGet<R, DIM_BSDF, 2>(smp, u);
            nr.direction = ia.shading_cs.from(cosWeightedHemi(u[0], u[1]));
            nr.medium_ior = ia.n1;
            nr.start += ia.normal * eps;
        }
    }

    // Interaction::sampleBSDF, interaction.cpp:56-72
    template <class R>
    MCRT_D bool sampleBSDF(const Interaction<R>& ia, const PathRay<R>& in, const SamplerState& smp, R eps, bool flux,
                           V3<R>& bsdf_absIdotN, R& pdf, PathRay<R>& new_ray)
    {
        spawnRay(new_ray, ia, in, smp, eps);
        V3<R> wi = ia.shading_cs.to(new_ray.direction);
        if ((new_ray.refraction && wi.z >= R(0)) || (!new_ray.refraction && wi.z <= R(0))) return false;
        V3<R> wo = ia.shading_cs.to(ia.out);
        bsdf_absIdotN = ia.bsdfLocal(wo, wi, pdf, flux, new_ray.dirac_delta) * mabs(wi.z);
        return pdf > R(0);
    }
}
