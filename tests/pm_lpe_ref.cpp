// TEST INFRASTRUCTURE - the event strings of the photon mapper's light path expressions restated on the CPU, on top of
// the scalar float64 restatement of the reference (oracle/mcrt_oracle.cpp, included unchanged so that its photonPass,
// emitPhoton's sampler use, knnBrute / gatherBrute, photonEstimate's terms and pmSampleRay's control flow are the very
// ones the photon-mapping parity tests pin). Built by tests/pm_lpe_ref.py into a temporary directory; never linked into
// the product.
//
// 1. oracle_pm_photon_events: photonPass, then every stored photon's emission path (PhotonList::emission) walked again
//    with the same sampler draws, recording the event of each vertex before the one that stored it. The walk's photons
//    must equal photonPass's bit for bit (the count of those that do not is returned).
// 2. oracle_pm_lpe_render: pmSampleRay over given maps, each contribution summed per pixel under its own event string -
//    an emitter hit or next-event estimation as tests/lpe_ref.cpp, and every photon term of a caustic or global
//    estimate separately, under the camera prefix up to the gather vertex x, x's event, then the photon's history.
#include "../oracle/mcrt_oracle.cpp"

#include <map>
#include <string>

namespace
{
    // the encoding of tests/lpe_ref.cpp: 'C', the vertex events 'a' <RD>, 'b' <RS>, 'c' <RG>, 'd' <TS>, 'e' <TG>, a light
    // of group g chr('0' + g), an emitter without a group '*'
    char eventChar(const Interaction& ia)
    {
        if (ia.type == DIFFUSE) return 'a';
        if (ia.type == REFLECT) return ia.dirac_delta ? 'b' : 'c';
        return ia.dirac_delta ? 'd' : 'e';
    }

    // emitPhoton (mcrt_oracle.cpp) with each stored photon's events e1..em recorded (emission order, the storing vertex
    // excluded)
    void emitPhotonEvents(const Scene& s, Ray ray, D3 flux, Sampler& smp, double non_caustic_reject, PhotonList lists[2],
                          std::vector<std::string> events[2])
    {
        std::vector<double> iors(1, ray.medium_ior);
        std::string walked;
        while (true)
        {
            smp.shuffle();
            Isect is = intersect(s, ray, nullptr);
            if (is.prim == 0xFFFFFFFFu) return;
            int ext = std::min(std::max(ray.refraction_level - 1, 0), (int)iors.size() - 1);
            Interaction ia = makeInteraction(s, is, ray, iors[ext], smp);
            if (!ia.material->dirac_delta)
            {
                if (ray.dirac_delta) { storePhoton(lists[0], flux, ia.position, -ray.direction, 0); events[0].push_back(walked); }
                else if (non_caustic_reject > smp.get(PM_REJECT))
                {
                    storePhoton(lists[1], flux / non_caustic_reject, ia.position, -ray.direction, 0);
                    events[1].push_back(walked);
                }
            }
            walked += eventChar(ia);
            D3 f; double pdf; Ray nr;
            if (!sampleBSDF(ia, smp, f, pdf, nr, true)) return;
            f = f / pdf;
            double survive = std::min(compMax(f), 0.95);
            if (survive == 0.0 || survive <= smp.get(ABSORB)) return;
            flux = flux * (f / survive);
            ray = nr;
            updateIORs(iors, ray);
        }
    }

    struct PhotonEvents
    {
        PhotonList lists[2];                  // photonPass's photons, emission order
        std::vector<std::string> events[2];   // each photon's e1..em (emission order)
        std::vector<uint32_t> lights[2];
        std::string chars[2];                 // events, each ended by '\0'
        uint64_t mismatched = 0;              // walked photons that differ from photonPass's
    };

    struct LpeStrings
    {
        std::map<std::string, uint32_t> index;
        std::vector<std::string> strings;
        std::vector<std::map<uint32_t, D3>> pixels;
        uint64_t entries = 0;
    };

    void add(LpeStrings& out, std::map<uint32_t, D3>& px, const std::string& str, const D3& v)
    {
        if (v.x == 0.0 && v.y == 0.0 && v.z == 0.0) return;
        auto it = out.index.find(str);
        uint32_t k;
        if (it == out.index.end())
        {
            k = (uint32_t)out.strings.size();
            out.index.emplace(str, k);
            out.strings.push_back(str);
        }
        else k = it->second;
        auto p = px.find(k);
        if (p == px.end()) { px.emplace(k, v); out.entries++; }
        else p->second = p->second + v;
    }

    struct Labels
    {
        std::map<uint32_t, char> of_prim;
        char operator()(uint32_t prim) const
        {
            auto it = of_prim.find(prim);
            return it == of_prim.end() ? '*' : it->second;
        }
    };

    // photonEstimate (mcrt_oracle.cpp), each photon's term scaled as the estimate scales the sum and added under
    // prefix + the photon's history (string order: e_m..e_1, then its light)
    void photonTerms(const PhotonMaps& pm, int which, const Interaction& ia, double gather_r2, PMCounts& cnt,
                     const std::vector<std::string>& history, const std::string& prefix, const D3& throughput, LpeStrings& out,
                     std::map<uint32_t, D3>& px)
    {
        const std::vector<float>& ph = pm.photons[which];
        const std::vector<std::pair<double, uint32_t>> d = gather_r2 > 0.0 ? gatherBrute(pm, which, ia.position, gather_r2, cnt)
                                                                            : knnBrute(pm, which, ia.position, cnt);
        if (d.empty()) return;
        const double r2 = gather_r2 > 0.0 ? gather_r2 : d[0].first, inv_r2 = 1.0 / r2;
        for (const auto& r : d)
        {
            const float* p = &ph[8 * (size_t)r.second];
            D3 f; double pdf;
            if (!ia.bsdfWorld(f, photonDir(p[6], p[7]), pdf)) continue;
            const D3 flux((double)p[0], (double)p[1], (double)p[2]);
            const D3 term = which == 0 ? 3.0 * ((flux * f * coneWeight(r.first, inv_r2)) / pdf) * inv_r2 * INV_PI
                                       : (flux * f / pdf) / (r2 * PI);
            add(out, px, prefix + history[r.second], term * throughput);
        }
    }

    // pmSampleRay (mcrt_oracle.cpp) with each contribution under its string
    void pmSampleRayStrings(const PhotonMaps& pm, const std::vector<std::string> history[2], const Labels& label, Ray ray,
                            Sampler& smp, PMCounts& cnt, LpeStrings& out, std::map<uint32_t, D3>& px)
    {
        const Scene& s = *pm.s;
        D3 throughput(1, 1, 1);
        std::vector<double> iors(1, ray.medium_ior);
        LightSample ls;
        std::string prefix = "C";
        while (true)
        {
            smp.shuffle();
            Isect is = intersect(s, ray, &cnt.rays);
            if (is.prim == 0xFFFFFFFFu) return;
            int ext = std::min(std::max(ray.refraction_level - 1, 0), (int)iors.size() - 1);
            Interaction ia = makeInteraction(s, is, ray, iors[ext], smp);
            add(out, px, prefix + label(ia.prim), sampleEmissive(s, ia, ls) * throughput);
            prefix += eventChar(ia);
            if (ia.dirac_delta)
            {
                if (!ray.dirac_delta && ray.depth != 0) return;
            }
            else
            {
                photonTerms(pm, 0, ia, pm.gather_r2[0], cnt, history[0], prefix, throughput, out, px);
                if (pm.direct_visualization || !(ray.dirac_delta || ray.depth == 0))
                {
                    photonTerms(pm, 1, ia, pm.gather_r2[1], cnt, history[1], prefix, throughput, out, px);
                    return;
                }
                uint64_t shadow = 0;
                add(out, px, prefix + label(ls.light), sampleDirect(s, ia, ls, smp, &shadow) * throughput);
            }
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
            updateIORs(iors, ray);
        }
    }
}

extern "C"
{

// photonPass (emissions, caustic_factor, pass, seed) and each photon's events: -> a handle for oracle_pm_photon_events_get
// / _free, or null when the pass's indices do not fit 32 bits. n[2]: photons per map; chars[2]: bytes of each map's
// events (each ended by '\0'); mismatched: walked photons that differ from photonPass's.
void* oracle_pm_photon_events(void* h, uint64_t emissions, double caustic_factor, uint32_t pass, uint32_t seed, uint64_t n[2],
                              uint64_t chars[2], uint64_t* mismatched)
{
    const Scene& s = *static_cast<Scene*>(h);
    auto* o = new PhotonEvents();
    uint64_t total = 0;
    if (!photonPass(s, emissions, caustic_factor, pass, seed, o->lists[0], o->lists[1], total)) { delete o; return nullptr; }
    // the per-light plan of photonPass, to walk each stored photon's emission again
    const size_t n_lights = s.light_prim.size();
    const size_t photon_emissions = (size_t)((double)emissions * caustic_factor);
    std::vector<D3> light_flux(n_lights);
    double total_flux = 0.0;
    for (size_t l = 0; l < n_lights; l++)
    {
        const uint32_t prim = s.light_prim[l];
        light_flux[l] = D3(s.materials[s.prim_material[prim]].emittance) * s.prim_area[prim];
        total_flux += 0.0 + light_flux[l].x + light_flux[l].y + light_flux[l].z;
    }
    std::vector<uint64_t> paths;
    for (int w = 0; w < 2; w++) paths.insert(paths.end(), o->lists[w].emission.begin(), o->lists[w].emission.end());
    std::sort(paths.begin(), paths.end());
    paths.erase(std::unique(paths.begin(), paths.end()), paths.end());
    PhotonList walked[2];
    std::vector<std::string> ev[2];
    Sampler smp(seed);
    for (uint64_t tag : paths)
    {
        const uint32_t l = (uint32_t)(tag >> 32), index = (uint32_t)tag;
        const double share = (0.0 + light_flux[l].x + light_flux[l].y + light_flux[l].z) / total_flux;
        const size_t n_l = (size_t)((double)photon_emissions * share);
        const uint32_t prim = s.light_prim[l];
        smp.initiate(l);
        smp.setIndex(index);
        const double u0 = smp.get(PM_LIGHT), u1 = smp.get(PM_LIGHT + 1), u2 = smp.get(PM_LIGHT + 2), u3 = smp.get(PM_LIGHT + 3);
        const D3 pos = lightPoint(s, prim, u0, u1), normal = primNormal(s, prim, pos);
        const double r = std::sqrt(u2), az = u3 * TWO_PI;
        const D3 dir = Frame(normal).from(D3(r * std::cos(az), r * std::sin(az), std::sqrt(1 - u2)));
        const size_t before[2] = { walked[0].photons.size(), walked[1].photons.size() };
        emitPhotonEvents(s, makeRay(pos + normal * EPS, dir, s.d.scene_ior), light_flux[l] / (double)n_l, smp, 1.0 / caustic_factor,
                         walked, ev);
        for (int w = 0; w < 2; w++)
            for (size_t k = before[w] / 8; k < walked[w].photons.size() / 8; k++) walked[w].emission[k] = tag;
    }
    for (int w = 0; w < 2; w++)
    {
        // photonPass's photons in its order, each with the events of the walked photon of the same path and rank
        std::map<uint64_t, std::vector<size_t>> of_path;
        for (size_t k = 0; k < walked[w].emission.size(); k++) of_path[walked[w].emission[k]].push_back(k);
        std::map<uint64_t, size_t> used;
        const PhotonList& L = o->lists[w];
        for (size_t i = 0; i < L.emission.size(); i++)
        {
            const uint64_t tag = L.emission[i];
            const std::vector<size_t>& ks = of_path[tag];
            const size_t rank = used[tag]++;
            if (rank >= ks.size() || std::memcmp(&walked[w].photons[8 * ks[rank]], &L.photons[8 * i], 32) != 0)
            {
                o->mismatched++;
                o->events[w].push_back("?");
            }
            else o->events[w].push_back(ev[w][ks[rank]]);
            o->lights[w].push_back((uint32_t)(tag >> 32));
            o->chars[w] += o->events[w].back();
            o->chars[w] += '\0';
        }
        for (const auto& kv : of_path) if (used[kv.first] != kv.second.size()) o->mismatched += kv.second.size() - std::min(kv.second.size(), used[kv.first]);
        n[w] = L.emission.size();
        chars[w] = o->chars[w].size();
    }
    *mismatched = o->mismatched;
    return o;
}

// photons[n][8] (float32, emission order), lights[n], events: the strings e1..em, each ended by '\0'
void oracle_pm_photon_events_get(void* handle, int which, float* photons, uint32_t* lights, char* events)
{
    const PhotonEvents& o = *static_cast<PhotonEvents*>(handle);
    std::memcpy(photons, o.lists[which].photons.data(), o.lists[which].photons.size() * sizeof(float));
    std::memcpy(lights, o.lights[which].data(), o.lights[which].size() * sizeof(uint32_t));
    std::memcpy(events, o.chars[which].data(), o.chars[which].size());
}

void oracle_pm_photon_events_free(void* handle) { delete static_cast<PhotonEvents*>(handle); }

// pmSampleRay over the maps (caustic, global: photons [n][8]) whose photons have the histories hist_c / hist_g (the
// string after x, e_m..e_1 then the light's character, each ended by '\0'), k nearest (gather_r2 > 0: fixed radius),
// rows [y0, y1), strings summed per pixel and averaged over the sqrtspp^2 samples. group_of_light as tests/lpe_ref.cpp.
// -> a handle for tests/lpe_ref.cpp's layout: oracle_pm_lpe_sizes / _get / _free.
void* oracle_pm_lpe_render(void* h, const float* caustic, uint64_t n_caustic, const char* hist_c, const float* global, uint64_t n_global,
                           const char* hist_g, uint32_t k, uint32_t direct_visualization, const double gather_r2[2],
                           const mcrt_camera* cam, uint32_t y0, uint32_t y1, uint32_t sqrtspp, uint32_t seed,
                           const uint32_t* group_of_light, uint32_t n_lights)
{
    const Scene& s = *static_cast<Scene*>(h);
    PhotonMaps pm;
    pm.s = &s;
    pm.photons[0].assign(caustic, caustic + 8 * n_caustic);
    pm.photons[1].assign(global, global + 8 * n_global);
    pm.k = k;
    pm.direct_visualization = direct_visualization != 0;
    pm.gather_r2[0] = gather_r2[0]; pm.gather_r2[1] = gather_r2[1];
    std::vector<std::string> history[2];
    const char* src[2] = { hist_c, hist_g };
    const uint64_t cnts[2] = { n_caustic, n_global };
    for (int w = 0; w < 2; w++)
        for (uint64_t i = 0; i < cnts[w]; i++) { history[w].emplace_back(src[w]); src[w] += history[w].back().size() + 1; }
    Labels label;
    if (group_of_light)
        for (uint32_t l = 0; l < n_lights && l < s.light_prim.size(); l++) label.of_prim[s.light_prim[l]] = (char)('0' + group_of_light[l]);
    auto* out = new LpeStrings();
    out->pixels.resize((size_t)(y1 - y0) * cam->width);
    Sampler smp(seed);
    PMCounts cnt;
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
                pmSampleRayStrings(pm, history, label, cameraRay(*cam, s.d.scene_ior, pixel, smp), smp, cnt, *out, px);
            }
            for (auto& kv : px) kv.second = kv.second / (double)spp;
        }
    return out;
}

void oracle_pm_lpe_sizes(void* handle, uint64_t* entries, uint64_t* strings, uint64_t* chars)
{
    const LpeStrings& o = *static_cast<LpeStrings*>(handle);
    *entries = o.entries;
    *strings = o.strings.size();
    uint64_t c = 0;
    for (const std::string& str : o.strings) c += str.size() + 1;
    *chars = c;
}

void oracle_pm_lpe_get(void* handle, uint32_t* pixel, uint32_t* string, double* value, char* chars)
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

void oracle_pm_lpe_free(void* handle) { delete static_cast<LpeStrings*>(handle); }

} // extern "C"
