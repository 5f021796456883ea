// TEST INFRASTRUCTURE - the event strings of light path expressions (mcrt_render_accumulate_lpe_dev) restated on the
// CPU, on top of the scalar float64 restatement of the reference (oracle/mcrt_oracle.cpp, included unchanged so that its
// sampler, Scene::intersect, Interaction, sampleDirect, sampleEmissive and sampleBSDF are the very ones the path-tracing
// parity tests pin). Every contribution of sampleRay is summed per pixel under its own event string; which strings an
// expression matches is decided in Python (tests/lpe_ref.py), independently of the product's compiler. Built by
// tests/lpe_ref.py into a temporary directory; never linked into the product.
#include "../oracle/mcrt_oracle.cpp"

#include <map>
#include <string>

namespace
{
    // One character per event: the camera 'C', the vertex events 'a' <RD>, 'b' <RS>, 'c' <RG>, 'd' <TS>, 'e' <TG>, the
    // sky 'B', an emitter of light group g the byte 0x80 + g (read as latin-1, so no group collides with another event
    // or with a character of Python's re), an emitter without a group (not a listed light, or a light the caller's table
    // leaves out) '*'
    char vertexChar(const Interaction& ia)
    {
        if (ia.type == DIFFUSE) return 'a';
        if (ia.type == REFLECT) return ia.dirac_delta ? 'b' : 'c';
        return ia.dirac_delta ? 'd' : 'e';
    }

    char groupChar(uint32_t g) { return (char)(0x80u + g); }

    struct LpeStrings
    {
        std::map<std::string, uint32_t> index;
        std::vector<std::string> strings;
        std::vector<std::map<uint32_t, D3>> pixels;   // per pixel: string index -> sum over its samples
        uint64_t entries = 0;
    };

    struct Labels
    {
        std::map<uint32_t, char> of_prim;   // light primitive -> its group's character (LightSample::light is the primitive)
        char operator()(uint32_t prim) const
        {
            auto it = of_prim.find(prim);
            return it == of_prim.end() ? '*' : it->second;
        }
    };

    void add(LpeStrings& out, std::map<uint32_t, D3>& px, const std::string& s, const D3& v)
    {
        if (v.x == 0.0 && v.y == 0.0 && v.z == 0.0) return;
        auto it = out.index.find(s);
        uint32_t k;
        if (it == out.index.end())
        {
            k = (uint32_t)out.strings.size();
            out.index.emplace(s, k);
            out.strings.push_back(s);
        }
        else k = it->second;
        auto p = px.find(k);
        if (p == px.end()) { px.emplace(k, v); out.entries++; }
        else p->second = p->second + v;
    }

    // sampleRay (mcrt_oracle.cpp) with each contribution added under its event string: the vertices before it, then its
    // source. An emitter hit takes the string of the vertices before the hit; light sampled at a vertex takes that
    // vertex's event, the interaction type its BSDF sample uses too.
    void sampleRayStrings(const Scene& s, const Labels& label, Ray ray, Sampler& smp, LpeStrings& out, std::map<uint32_t, D3>& px)
    {
        D3 throughput(1, 1, 1);
        std::vector<double> iors(1, ray.medium_ior);
        LightSample ls;
        std::string prefix = "C";
        while (true)
        {
            smp.shuffle();
            Isect is = intersect(s, ray, nullptr);
            if (is.prim == 0xFFFFFFFFu)
            {
                add(out, px, prefix + 'B', skyColor(ray) * throughput);
                return;
            }
            int ext = std::min(std::max(ray.refraction_level - 1, 0), (int)iors.size() - 1);
            Interaction ia = makeInteraction(s, is, ray, iors[ext], smp);
            add(out, px, prefix + label(ia.prim), sampleEmissive(s, ia, ls) * throughput);
            prefix += vertexChar(ia);
            const D3 direct = sampleDirect(s, ia, ls, smp, nullptr) * throughput;
            add(out, px, prefix + label(ls.light), direct);
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

// The per-pixel means (over the sqrtspp^2 samples) of the contributions of each distinct event string of rows [y0, y1).
// group_of_light[n_lights]: light l (the scene's l-th light_prim) is in group group_of_light[l] (< 128); NULL: no groups.
// -> a handle for oracle_lpe_sizes / oracle_lpe_get / oracle_lpe_free.
void* oracle_lpe_render(void* h, const mcrt_camera* cam, uint32_t y0, uint32_t y1, uint32_t sqrtspp, uint32_t seed,
                        const uint32_t* group_of_light, uint32_t n_lights)
{
    const Scene& s = *static_cast<Scene*>(h);
    Labels label;
    if (group_of_light)
        for (uint32_t l = 0; l < n_lights && l < s.light_prim.size(); l++) label.of_prim[s.light_prim[l]] = groupChar(group_of_light[l]);
    auto* out = new LpeStrings();
    out->pixels.resize((size_t)(y1 - y0) * cam->width);
    Sampler smp(seed);
    const uint32_t spp = sqrtspp * sqrtspp;
    for (uint32_t y = y0; y < y1; y++)
        for (uint32_t x = 0; x < cam->width; x++)
        {
            const uint32_t pixel = y * cam->width + x;
            std::map<uint32_t, D3>& px = out->pixels[(size_t)(y - y0) * cam->width + x];
            smp.initiate(pixel);
            for (uint32_t i = 0; i < spp; i++)
            {
                smp.setIndex(i);
                sampleRayStrings(s, label, cameraRay(*cam, s.d.scene_ior, pixel, smp), smp, *out, px);
            }
            for (auto& kv : px) kv.second = kv.second / (double)spp;
        }
    return out;
}

// entries: (pixel, string) pairs with a nonzero sum; strings: distinct strings; chars: their lengths + 1 each
void oracle_lpe_sizes(void* handle, uint64_t* entries, uint64_t* strings, uint64_t* chars)
{
    const LpeStrings& o = *static_cast<LpeStrings*>(handle);
    *entries = o.entries;
    *strings = o.strings.size();
    uint64_t c = 0;
    for (const std::string& str : o.strings) c += str.size() + 1;
    *chars = c;
}

// pixel[entries] (index in the rows' y-major order), string[entries], value[entries][3]; chars: the strings in order,
// each ended by '\0'
void oracle_lpe_get(void* handle, uint32_t* pixel, uint32_t* string, double* value, char* chars)
{
    const LpeStrings& o = *static_cast<LpeStrings*>(handle);
    uint64_t e = 0;
    for (size_t p = 0; p < o.pixels.size(); p++)
        for (const auto& kv : o.pixels[p])
        {
            pixel[e] = (uint32_t)p;
            string[e] = kv.first;
            value[3 * e] = kv.second.x; value[3 * e + 1] = kv.second.y; value[3 * e + 2] = kv.second.z;
            e++;
        }
    for (const std::string& str : o.strings)
    {
        std::memcpy(chars, str.c_str(), str.size() + 1);
        chars += str.size() + 1;
    }
}

void oracle_lpe_free(void* handle) { delete static_cast<LpeStrings*>(handle); }

} // extern "C"
