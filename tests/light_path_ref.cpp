// TEST INFRASTRUCTURE - the light-path AOVs of mcrt_render_accumulate_aovs_dev restated on the CPU, on top of the scalar
// float64 restatement of the reference (oracle/mcrt_oracle.cpp, included unchanged so that its sampler, Scene::intersect,
// Interaction, sampleDirect, sampleEmissive and sampleBSDF are the very ones the path-tracing parity tests pin). Built by
// tests/light_path_ref.py into a temporary directory; never linked into the product.
#include "../oracle/mcrt_oracle.cpp"

namespace
{
    // MCRT_AOV_* of include/mcrt_abi.h
    uint32_t directPlane(int type)
    {
        return type == DIFFUSE ? MCRT_AOV_DIFFUSE_DIRECT : (type == REFLECT ? MCRT_AOV_REFLECTION_DIRECT : MCRT_AOV_TRANSMISSION_DIRECT);
    }

    // sampleRay (mcrt_oracle.cpp) with each contribution added into its plane instead of one radiance: the camera ray's
    // sky goes to the background plane and its emitter to the emission plane; everything else goes to the plane of the
    // first vertex's interaction type, direct when the light path has one scattering vertex (light sampled at depth 0,
    // the sky or an emitter reached at depth 1) and indirect otherwise
    void sampleRayPlanes(const Scene& s, Ray ray, Sampler& smp, D3* planes)
    {
        D3 throughput(1, 1, 1);
        std::vector<double> iors(1, ray.medium_ior);
        LightSample ls;
        uint32_t first = 0;   // direct plane of the first vertex
        while (true)
        {
            smp.shuffle();
            const uint32_t depth = ray.depth;
            Isect is = intersect(s, ray, nullptr);
            if (is.prim == 0xFFFFFFFFu)
            {
                const uint32_t plane = depth == 0 ? (uint32_t)MCRT_AOV_BACKGROUND : first + (depth > 1 ? 1u : 0u);
                planes[plane] = planes[plane] + skyColor(ray) * throughput;
                return;
            }
            int ext = std::min(std::max(ray.refraction_level - 1, 0), (int)iors.size() - 1);
            Interaction ia = makeInteraction(s, is, ray, iors[ext], smp);
            if (depth == 0) first = directPlane(ia.type);
            const uint32_t emitted = depth == 0 ? (uint32_t)MCRT_AOV_EMISSION : first + (depth > 1 ? 1u : 0u);
            planes[emitted] = planes[emitted] + sampleEmissive(s, ia, ls) * throughput;
            const uint32_t sampled = first + (depth > 0 ? 1u : 0u);
            planes[sampled] = planes[sampled] + sampleDirect(s, ia, ls, smp, nullptr) * throughput;
            D3 f;
            if (!sampleBSDF(ia, smp, f, ls.bsdf_pdf, ray)) return;
            throughput = throughput * (f / ls.bsdf_pdf);
            double survive = compMax(throughput) * ray.refraction_scale;
            if (survive == 0.0) return;
            if (ray.diffuse_depth > 3 || ray.depth > 16)
            {
                survive = std::min(0.95, survive);
                if (survive <= smp.get(ABSORB)) return;
                throughput = throughput / survive;
            }
            if (ray.refraction_level > 0)
            {
                if (ray.refraction_level == (int)iors.size()) iors.push_back(ray.medium_ior);
                else if (ray.refraction_level < (int)iors.size() - 1) iors.pop_back();
            }
        }
    }
}

extern "C"
{

// oracle_render_rows split into the MCRT_AOV_COUNT planes: out[plane][(y - y0) * width + x][3], each the mean over the
// sqrtspp^2 samples of the pixel of that plane's contributions
void oracle_render_rows_aovs(void* h, const mcrt_camera* cam, uint32_t y0, uint32_t y1, uint32_t sqrtspp, uint32_t seed, double* out)
{
    const Scene& s = *static_cast<Scene*>(h);
    Sampler smp(seed);
    const uint32_t spp = sqrtspp * sqrtspp;
    const size_t plane_values = (size_t)(y1 - y0) * cam->width * 3;
    for (uint32_t y = y0; y < y1; y++)
        for (uint32_t x = 0; x < cam->width; x++)
        {
            const uint32_t pixel = y * cam->width + x;
            smp.initiate(pixel);
            D3 sum[MCRT_AOV_COUNT];
            for (uint32_t i = 0; i < spp; i++)
            {
                smp.setIndex(i);
                D3 planes[MCRT_AOV_COUNT];
                sampleRayPlanes(s, cameraRay(*cam, s.d.scene_ior, pixel, smp), smp, planes);
                for (int k = 0; k < MCRT_AOV_COUNT; k++) sum[k] = sum[k] + planes[k];
            }
            for (int k = 0; k < MCRT_AOV_COUNT; k++)
            {
                double* o = out + k * plane_values + ((size_t)(y - y0) * cam->width + x) * 3;
                o[0] = sum[k].x / (double)spp; o[1] = sum[k].y / (double)spp; o[2] = sum[k].z / (double)spp;
            }
        }
}

} // extern "C"
