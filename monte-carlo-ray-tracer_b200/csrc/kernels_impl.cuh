// Shared body of kernels_f64.cu / kernels_f32.cu: defines Launch<MCRT_REAL>.
#include <type_traits>

#include "launch.h"

namespace mcrt
{
    template <int V> using Int = std::integral_constant<int, V>;
    template <uint32_t V> using Feats = std::integral_constant<uint32_t, V>;

    // f(Int<V>{}) for the first V of Vs equal to v, or for the last V when none is: turns a run-time value into a
    // template argument, instantiating f for every V listed
    template <int V, int... Vs, class F> static void pick(int v, F&& f)
    {
        if constexpr (sizeof...(Vs) == 0) f(Int<V>{});
        else if (v == V) f(Int<V>{});
        else pick<Vs...>(v, f);
    }

    // f(film mode): the one runWavefront stored, for the launchers of every depositing kernel
    template <class F> static void withFilmMode(const WaveParams<MCRT_REAL>& p, F&& f)
    {
        pick<FILM_MODE_BOX, FILM_MODE_SPLAT, FILM_MODE_GROUPS, FILM_MODE_AOV, FILM_MODE_LPE>((int)p.film_mode, f);
    }

    // f(film mode, shade features) of the kernels that shade. Scenes whose materials use no Oren-Nayar / GGX / conductor
    // Fresnel run the instantiation without that code; the filtered film, the rare configuration, has one generic
    // instantiation.
    template <class F> static void withFilm(const WaveParams<MCRT_REAL>& p, F&& f)
    {
        const bool lite = (p.scene.material_flags_any & ~SHADE_FEATS_LITE) == 0;
        withFilmMode(p, [&](auto film) {
            if constexpr (film == FILM_MODE_SPLAT) f(film, Feats<SHADE_FEATS_ALL>{});
            else if (lite) f(film, Feats<SHADE_FEATS_LITE>{});
            else f(film, Feats<SHADE_FEATS_ALL>{});
        });
    }

    // f(prims, traversal, dynamic shared bytes) of k_extend / k_shadow: triangle-only scenes (every OBJ scene) run the
    // traversal without sphere / quadric code; parity mode takes the order-free BVH4 search whenever the scene has that
    // BVH (2: with dynamic fetch), fast mode always the plain traversal (0)
    template <class F> static void withTraversal(const WaveParams<MCRT_REAL>& p, F&& f)
    {
        const auto prims = [&](auto fast) {
            const size_t smem = fast ? fastStackSharedBytes(256) : 0;
            pick<PRIMS_TRI, PRIMS_TRI_SPHERE, PRIMS_ALL>((int)p.scene.prims_class, [&](auto pr) { f(pr, fast, smem); });
        };
        if constexpr (Mode<MCRT_REAL>::parity)
        {
            if (p.scene.bvh4 && p.scene.dynamic_fetch) return prims(Int<2>{});
            if (p.scene.bvh4) return prims(Int<1>{});
        }
        prims(Int<0>{});
    }

    template <> void Launch<MCRT_REAL>::generate(const WaveParams<MCRT_REAL>& p, int next, int grid, cudaStream_t s)
    {
        const bool filtered = p.film_mode == FILM_MODE_SPLAT;
        if (p.pixel_list)
        {
            if (filtered) k_generate<MCRT_REAL, true, true><<<grid, 256, 0, s>>>(p, next);
            else k_generate<MCRT_REAL, false, true><<<grid, 256, 0, s>>>(p, next);
            return;
        }
        if (filtered) k_generate<MCRT_REAL, true, false><<<grid, 256, 0, s>>>(p, next);
        else k_generate<MCRT_REAL, false, false><<<grid, 256, 0, s>>>(p, next);
    }
    template <> void Launch<MCRT_REAL>::extend(const WaveParams<MCRT_REAL>& p, int cur, int grid, cudaStream_t s)
    {
        withTraversal(p, [&](auto prims, auto fast, size_t smem) { k_extend<MCRT_REAL, prims, fast><<<grid, 256, smem, s>>>(p, cur); });
    }
    // KIND 0: PathTracer loop body, 1: PhotonMapper loop body
    template <int KIND> static void launchShade(const WaveParams<MCRT_REAL>& p, int cur, int grid, cudaStream_t s)
    {
        withFilm(p, [&](auto film, auto feats) { k_shade<MCRT_REAL, KIND, film, feats><<<grid * 2, 128, 0, s>>>(p, cur); });
    }
    template <> void Launch<MCRT_REAL>::shade(const WaveParams<MCRT_REAL>& p, int cur, int grid, cudaStream_t s)
    {
        launchShade<0>(p, cur, grid, s);
    }
    template <> void Launch<MCRT_REAL>::shadePhoton(const WaveParams<MCRT_REAL>& p, int cur, int grid, cudaStream_t s)
    {
        launchShade<1>(p, cur, grid, s);
    }
    template <int SLOTS, int FILM, uint32_t FEATS>
    static void launchKnn(const WaveParams<MCRT_REAL>& p, dim3 g, dim3 b, size_t smem, cudaStream_t s)
    {
        // k > 672 needs more than the default 48 KB of dynamic shared memory (knnSharedBytes)
        static bool attr_set = false;
        if (!attr_set)
        {
            cudaFuncSetAttribute(k_knn<MCRT_REAL, SLOTS, FILM, FEATS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)knnSharedBytes(1024));
            attr_set = true;
        }
        k_knn<MCRT_REAL, SLOTS, FILM, FEATS><<<g, b, smem, s>>>(p);
    }
    template <> void Launch<MCRT_REAL>::knn(const WaveParams<MCRT_REAL>& p, int grid, cudaStream_t s)
    {
        const dim3 g(grid * 2), b(32 * KNN_WARPS_PER_BLOCK);
        if (p.pm.gather_r2[0] > 0.0)
        {
            // fixed-radius gather (mcrt_photon_gather_radius) in place of the k-NN estimate
            withFilm(p, [&](auto film, auto feats) { k_gather<MCRT_REAL, film, feats><<<g, b, 0, s>>>(p); });
            return;
        }
        const size_t smem = knnSharedBytes(p.pm.k_nearest);
        // the photon maps hold at least k photons in every render that matters; if a map is smaller the
        // search clamps k itself and the register slots are simply not all used
        withFilm(p, [&](auto film, auto feats) {
            if constexpr (film == FILM_MODE_SPLAT) launchKnn<0, film, feats>(p, g, b, smem, s);   // the generic instantiation only
            else pick<1, 2, 4, 8, 0>(knnSlotsFor(p.pm.k_nearest), [&](auto slots) { launchKnn<slots, film, feats>(p, g, b, smem, s); });
        });
    }
    template <> void Launch<MCRT_REAL>::shadow(const WaveParams<MCRT_REAL>& p, int grid, cudaStream_t s)
    {
        withFilmMode(p, [&](auto film) {
            if constexpr (film == FILM_MODE_SPLAT)
            {
                // filtered film: the rare configuration, the generic traversal only
                if constexpr (Mode<MCRT_REAL>::parity)
                {
                    if (p.scene.bvh4) { k_shadow<MCRT_REAL, film, PRIMS_ALL, 1><<<grid, 256, fastStackSharedBytes(256), s>>>(p); return; }
                }
                k_shadow<MCRT_REAL, film, PRIMS_ALL, 0><<<grid, 256, 0, s>>>(p);
            }
            else withTraversal(p, [&](auto prims, auto fast, size_t smem) { k_shadow<MCRT_REAL, film, prims, fast><<<grid, 256, smem, s>>>(p); });
        });
    }
    template <> void Launch<MCRT_REAL>::shadeKey(const WaveParams<MCRT_REAL>& p, int grid, cudaStream_t s)
    {
        k_shade_key<MCRT_REAL><<<grid, 256, 0, s>>>(p);
    }
    template <> void Launch<MCRT_REAL>::emitGenerate(const WaveParams<MCRT_REAL>& p, int next, int grid, cudaStream_t s)
    {
        if (p.emit.lpe_states[0]) k_emit_generate<MCRT_REAL, true><<<grid, 256, 0, s>>>(p, next);
        else k_emit_generate<MCRT_REAL, false><<<grid, 256, 0, s>>>(p, next);
    }
    template <> void Launch<MCRT_REAL>::emitShade(const WaveParams<MCRT_REAL>& p, int cur, int grid, cudaStream_t s)
    {
        if (p.emit.lpe_states[0]) k_emit_shade<MCRT_REAL, true><<<grid * 2, 128, 0, s>>>(p, cur);
        else k_emit_shade<MCRT_REAL, false><<<grid * 2, 128, 0, s>>>(p, cur);
    }
    template <> void Launch<MCRT_REAL>::traceUser(const DeviceScene<MCRT_REAL>& sc, const double* rays6, size_t n,
                                                  double* out_tuv, uint32_t* out_prim, Counters* c, int grid, cudaStream_t s)
    {
        if constexpr (Mode<MCRT_REAL>::parity)
        {
            if (sc.bvh4) { k_trace_user<MCRT_REAL, true><<<grid, 256, fastStackSharedBytes(256), s>>>(sc, rays6, n, out_tuv, out_prim, c); return; }
        }
        k_trace_user<MCRT_REAL, false><<<grid, 256, 0, s>>>(sc, rays6, n, out_tuv, out_prim, c);
    }
    template <> void Launch<MCRT_REAL>::features(const DeviceScene<MCRT_REAL>& sc, const DeviceCamera<MCRT_REAL>& cam, uint32_t global_seed,
                                                 uint32_t sample_first, uint32_t sample_count, double* out, Counters* c, int grid,
                                                 cudaStream_t s)
    {
        if constexpr (Mode<MCRT_REAL>::parity)
        {
            if (sc.bvh4) { k_features<MCRT_REAL, true><<<grid, 256, fastStackSharedBytes(256), s>>>(sc, cam, global_seed, sample_first, sample_count, out, c); return; }
        }
        k_features<MCRT_REAL, false><<<grid, 256, 0, s>>>(sc, cam, global_seed, sample_first, sample_count, out, c);
    }
    template <> void Launch<MCRT_REAL>::featuresChain(const DeviceScene<MCRT_REAL>& sc, const DeviceCamera<MCRT_REAL>& cam, uint32_t global_seed,
                                                      uint32_t sample_first, uint32_t sample_count, uint32_t specular_depth,
                                                      MCRT_REAL ray_eps, double* out, Counters* c, int grid, cudaStream_t s)
    {
        if constexpr (Mode<MCRT_REAL>::parity)
        {
            if (sc.bvh4)
            {
                k_features_chain<MCRT_REAL, true><<<grid, 256, fastStackSharedBytes(256), s>>>(sc, cam, global_seed, sample_first, sample_count,
                                                                                              specular_depth, ray_eps, out, c);
                return;
            }
        }
        k_features_chain<MCRT_REAL, false><<<grid, 256, 0, s>>>(sc, cam, global_seed, sample_first, sample_count, specular_depth, ray_eps, out, c);
    }
}
