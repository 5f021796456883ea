// TEST INFRASTRUCTURE - the chain of mcrt_render_features_chain_dev restated on the CPU, on top of the scalar float64
// restatement of the reference (oracle/mcrt_oracle.cpp, included unchanged so that its sampler, Scene::intersect,
// Interaction, sampleBSDF and RefractionHistory are the very ones the path-tracing parity tests pin). Built by
// tests/specular_chain_ref.py into a temporary directory; never linked into the product.
#include "../oracle/mcrt_oracle.cpp"

extern "C"
{

// Denoiser guides after perfectly specular bounces (mcrt_render_features_chain_dev), per (pixel, sample): sampleRay's
// loop without emission, light sampling or Russian roulette, walked through at most max_depth hits on dirac_delta
// materials with throughput T and distance L. The end vertex (a hit on any other material, the hit at max_depth, or a
// hit whose sampleBSDF fails or leaves T at 0) gives out8[i] = {T * albedo, shading normal facing the ray, L + t, 1};
// a miss anywhere gives zeros. end3 (optional): {primitive of the last hit or miss (0xFFFFFFFF), its depth, 1 if the
// chain stopped there because the bounce was rejected or T became 0}.
void oracle_specular_chain(void* h, const mcrt_camera* cam, const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t seed,
                           uint32_t max_depth, double* out8, uint32_t* end3)
{
    const Scene& s = *static_cast<Scene*>(h);
    Sampler smp(seed);
    for (size_t i = 0; i < n; i++)
    {
        double* o = out8 + 8 * i;
        for (int k = 0; k < 8; k++) o[k] = 0.0;
        uint32_t end[3] = { 0xFFFFFFFFu, 0u, 0u };
        smp.initiate(pixel[i]);
        smp.setIndex(sample[i]);
        Ray ray = cameraRay(*cam, s.d.scene_ior, pixel[i], smp);
        std::vector<double> iors(1, ray.medium_ior);
        D3 T(1, 1, 1);
        double L = 0.0;
        for (uint32_t depth = 0;; depth++)
        {
            smp.shuffle();
            const Isect is = intersect(s, ray, nullptr);
            end[0] = is.prim; end[1] = depth;
            if (is.prim == 0xFFFFFFFFu) break;
            const mcrt_material& m = s.materials[s.prim_material[is.prim]];
            if (m.dirac_delta && depth < max_depth)
            {
                end[2] = 1u;
                const int ext = std::min(std::max(ray.refraction_level - 1, 0), (int)iors.size() - 1);
                const Interaction ia = makeInteraction(s, is, ray, iors[ext], smp);
                D3 f; double pdf; Ray nr;
                if (sampleBSDF(ia, smp, f, pdf, nr))
                {
                    const D3 Tn = T * (f / pdf);
                    if (compMax(Tn) != 0.0)
                    {
                        T = Tn; L += is.t; ray = nr;
                        if (ray.refraction_level > 0) // RefractionHistory::update
                        {
                            if (ray.refraction_level == (int)iors.size()) iors.push_back(ray.medium_ior);
                            else if (ray.refraction_level < (int)iors.size() - 1) iors.pop_back();
                        }
                        end[2] = 0u;
                        continue;
                    }
                }
            }
            // the shading normal of makeInteraction, flipped to face the ray
            const D3 position = ray.at(is.t);
            const D3 normal = primNormal(s, is.prim, position);
            const double cos_theta = dot(ray.direction, normal);
            D3 sn = normal;
            if (is.interpolate)
            {
                const double* N = &s.vn[9 * s.tri_vn[s.prim_index[is.prim]]];
                sn = normalize((1.0 - is.u - is.v) * D3(N) + is.u * D3(N + 3) + is.v * D3(N + 6));
                if ((cos_theta < 0.0) != (dot(ray.direction, sn) < 0.0)) sn = normal;
            }
            if (cos_theta > 0.0) sn = -sn;
            const D3 albedo = T * D3((m.perfect_mirror || m.has_complex_ior) ? m.specular_reflectance : m.reflectance);
            o[0] = albedo.x; o[1] = albedo.y; o[2] = albedo.z;
            o[3] = sn.x; o[4] = sn.y; o[5] = sn.z;
            o[6] = L + is.t;
            o[7] = 1.0;
            break;
        }
        if (end3) for (int k = 0; k < 3; k++) end3[3 * i + k] = end[k];
    }
}


} // extern "C"
