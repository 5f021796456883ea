// Shared body of kernels_f64.cu / kernels_f32.cu: defines Launch<MCRT_REAL>.
#include "launch.h"

namespace mcrt
{
    template <> void Launch<MCRT_REAL>::generate(const WaveParams<MCRT_REAL>& p, int next, int grid, cudaStream_t s)
    {
        if (p.pixel_list)
        {
            if (p.filmp.is_default_box) k_generate<MCRT_REAL, false, true><<<grid, 256, 0, s>>>(p, next);
            else k_generate<MCRT_REAL, true, true><<<grid, 256, 0, s>>>(p, next);
            return;
        }
        if (p.filmp.is_default_box) k_generate<MCRT_REAL, false, false><<<grid, 256, 0, s>>>(p, next);
        else k_generate<MCRT_REAL, true, false><<<grid, 256, 0, s>>>(p, next);
    }
    template <> void Launch<MCRT_REAL>::extend(const WaveParams<MCRT_REAL>& p, int cur, int grid, cudaStream_t s)
    {
        // triangle-only scenes (every OBJ scene) run the traversal without sphere / quadric code
        if constexpr (Mode<MCRT_REAL>::parity)
        {
            if (p.scene.bvh4 && p.scene.dynamic_fetch)
            {
                if (p.scene.prims_class == PRIMS_TRI) k_extend<MCRT_REAL, PRIMS_TRI, 2><<<grid, 256, fastStackSharedBytes(256), s>>>(p, cur);
                else if (p.scene.prims_class == PRIMS_TRI_SPHERE) k_extend<MCRT_REAL, PRIMS_TRI_SPHERE, 2><<<grid, 256, fastStackSharedBytes(256), s>>>(p, cur);
                else k_extend<MCRT_REAL, PRIMS_ALL, 2><<<grid, 256, fastStackSharedBytes(256), s>>>(p, cur);
                return;
            }
            if (p.scene.bvh4)
            {
                if (p.scene.prims_class == PRIMS_TRI) k_extend<MCRT_REAL, PRIMS_TRI, 1><<<grid, 256, fastStackSharedBytes(256), s>>>(p, cur);
                else if (p.scene.prims_class == PRIMS_TRI_SPHERE) k_extend<MCRT_REAL, PRIMS_TRI_SPHERE, 1><<<grid, 256, fastStackSharedBytes(256), s>>>(p, cur);
                else k_extend<MCRT_REAL, PRIMS_ALL, 1><<<grid, 256, fastStackSharedBytes(256), s>>>(p, cur);
                return;
            }
        }
        if (p.scene.prims_class == PRIMS_TRI) k_extend<MCRT_REAL, PRIMS_TRI, 0><<<grid, 256, 0, s>>>(p, cur);
        else if (p.scene.prims_class == PRIMS_TRI_SPHERE) k_extend<MCRT_REAL, PRIMS_TRI_SPHERE, 0><<<grid, 256, 0, s>>>(p, cur);
        else k_extend<MCRT_REAL, PRIMS_ALL, 0><<<grid, 256, 0, s>>>(p, cur);
    }
    template <> void Launch<MCRT_REAL>::shade(const WaveParams<MCRT_REAL>& p, int cur, int grid, cudaStream_t s)
    {
        // scenes whose materials use no Oren-Nayar / GGX / conductor Fresnel run the instantiation without that code
        const bool lite = (p.scene.material_flags_any & ~SHADE_FEATS_LITE) == 0;
        if (!p.filmp.is_default_box) k_shade<MCRT_REAL, 0, FILM_MODE_SPLAT, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
        else if (p.n_planes && p.lpe_next)
        {
            if (lite) k_shade<MCRT_REAL, 0, FILM_MODE_LPE, SHADE_FEATS_LITE><<<grid * 2, 128, 0, s>>>(p, cur);
            else k_shade<MCRT_REAL, 0, FILM_MODE_LPE, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
        }
        else if (p.n_planes && p.aovs)
        {
            if (lite) k_shade<MCRT_REAL, 0, FILM_MODE_AOV, SHADE_FEATS_LITE><<<grid * 2, 128, 0, s>>>(p, cur);
            else k_shade<MCRT_REAL, 0, FILM_MODE_AOV, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
        }
        else if (p.n_planes)
        {
            if (lite) k_shade<MCRT_REAL, 0, FILM_MODE_GROUPS, SHADE_FEATS_LITE><<<grid * 2, 128, 0, s>>>(p, cur);
            else k_shade<MCRT_REAL, 0, FILM_MODE_GROUPS, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
        }
        else if (lite) k_shade<MCRT_REAL, 0, FILM_MODE_BOX, SHADE_FEATS_LITE><<<grid * 2, 128, 0, s>>>(p, cur);
        else k_shade<MCRT_REAL, 0, FILM_MODE_BOX, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
    }
    template <> void Launch<MCRT_REAL>::shadePhoton(const WaveParams<MCRT_REAL>& p, int cur, int grid, cudaStream_t s)
    {
        const bool lite = (p.scene.material_flags_any & ~SHADE_FEATS_LITE) == 0;
        if (!p.filmp.is_default_box) k_shade<MCRT_REAL, 1, FILM_MODE_SPLAT, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
        else if (p.n_planes && p.lpe_next)
        {
            if (lite) k_shade<MCRT_REAL, 1, FILM_MODE_LPE, SHADE_FEATS_LITE><<<grid * 2, 128, 0, s>>>(p, cur);
            else k_shade<MCRT_REAL, 1, FILM_MODE_LPE, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
        }
        else if (p.n_planes && p.aovs)
        {
            // photon-mapper components: FILM_MODE_AOV deposits into the plane each site names (MCRT_PM_*)
            if (lite) k_shade<MCRT_REAL, 1, FILM_MODE_AOV, SHADE_FEATS_LITE><<<grid * 2, 128, 0, s>>>(p, cur);
            else k_shade<MCRT_REAL, 1, FILM_MODE_AOV, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
        }
        else if (p.n_planes)
        {
            if (lite) k_shade<MCRT_REAL, 1, FILM_MODE_GROUPS, SHADE_FEATS_LITE><<<grid * 2, 128, 0, s>>>(p, cur);
            else k_shade<MCRT_REAL, 1, FILM_MODE_GROUPS, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
        }
        else if (lite) k_shade<MCRT_REAL, 1, FILM_MODE_BOX, SHADE_FEATS_LITE><<<grid * 2, 128, 0, s>>>(p, cur);
        else k_shade<MCRT_REAL, 1, FILM_MODE_BOX, SHADE_FEATS_ALL><<<grid * 2, 128, 0, s>>>(p, cur);
    }
    template <> void Launch<MCRT_REAL>::knn(const WaveParams<MCRT_REAL>& p, int grid, cudaStream_t s)
    {
        const dim3 g(grid * 2), b(32 * KNN_WARPS_PER_BLOCK);
        if (p.pm.gather_r2[0] > 0.0)
        {
            // fixed-radius gather (mcrt_photon_gather_radius) in place of the k-NN estimate
            const bool lite = (p.scene.material_flags_any & ~SHADE_FEATS_LITE) == 0;
            if (!p.filmp.is_default_box) k_gather<MCRT_REAL, FILM_MODE_SPLAT, SHADE_FEATS_ALL><<<g, b, 0, s>>>(p);
            else if (p.n_planes && p.lpe_next)
            {
                if (lite) k_gather<MCRT_REAL, FILM_MODE_LPE, SHADE_FEATS_LITE><<<g, b, 0, s>>>(p);
                else k_gather<MCRT_REAL, FILM_MODE_LPE, SHADE_FEATS_ALL><<<g, b, 0, s>>>(p);
            }
            else if (p.n_planes && p.aovs)
            {
                if (lite) k_gather<MCRT_REAL, FILM_MODE_AOV, SHADE_FEATS_LITE><<<g, b, 0, s>>>(p);
                else k_gather<MCRT_REAL, FILM_MODE_AOV, SHADE_FEATS_ALL><<<g, b, 0, s>>>(p);
            }
            else if (p.n_planes)
            {
                if (lite) k_gather<MCRT_REAL, FILM_MODE_GROUPS, SHADE_FEATS_LITE><<<g, b, 0, s>>>(p);
                else k_gather<MCRT_REAL, FILM_MODE_GROUPS, SHADE_FEATS_ALL><<<g, b, 0, s>>>(p);
            }
            else if (lite) k_gather<MCRT_REAL, FILM_MODE_BOX, SHADE_FEATS_LITE><<<g, b, 0, s>>>(p);
            else k_gather<MCRT_REAL, FILM_MODE_BOX, SHADE_FEATS_ALL><<<g, b, 0, s>>>(p);
            return;
        }
        const size_t smem = knnSharedBytes(p.pm.k_nearest);
        // the photon maps hold at least k photons in every render that matters; if a map is smaller the
        // search clamps k itself and the register slots are simply not all used
        if (!p.filmp.is_default_box)
        {
            // filtered film: the rare configuration, one generic instantiation
            static bool attr_set = false;
            if (!attr_set) { cudaFuncSetAttribute(k_knn<MCRT_REAL, 0, FILM_MODE_SPLAT, SHADE_FEATS_ALL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)knnSharedBytes(1024)); attr_set = true; }
            k_knn<MCRT_REAL, 0, FILM_MODE_SPLAT, SHADE_FEATS_ALL><<<g, b, smem, s>>>(p);
            return;
        }
        const bool lite = (p.scene.material_flags_any & ~SHADE_FEATS_LITE) == 0;
        // film mode of the box film: one plane, light-group planes, the photon mapper's component planes (FILM_MODE_AOV)
        // or LPE planes
        const int film_mode = !p.n_planes ? FILM_MODE_BOX : (p.lpe_next ? FILM_MODE_LPE : (p.aovs ? FILM_MODE_AOV : FILM_MODE_GROUPS));
        const int slots = knnSlotsFor(p.pm.k_nearest);
        // k > 672 needs more than the default 48 KB of dynamic shared memory (knnSharedBytes)
        #define MCRT_KNN_LAUNCH2(SL, FM, FE) \
            do { static bool attr_set = false; \
                 if (!attr_set) { cudaFuncSetAttribute(k_knn<MCRT_REAL, SL, FM, FE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)knnSharedBytes(1024)); attr_set = true; } \
                 k_knn<MCRT_REAL, SL, FM, FE><<<g, b, smem, s>>>(p); } while (0)
        #define MCRT_KNN_LAUNCH1(SL, FE) \
            do { if (film_mode == FILM_MODE_GROUPS) MCRT_KNN_LAUNCH2(SL, FILM_MODE_GROUPS, FE); \
                 else if (film_mode == FILM_MODE_AOV) MCRT_KNN_LAUNCH2(SL, FILM_MODE_AOV, FE); \
                 else if (film_mode == FILM_MODE_LPE) MCRT_KNN_LAUNCH2(SL, FILM_MODE_LPE, FE); \
                 else MCRT_KNN_LAUNCH2(SL, FILM_MODE_BOX, FE); } while (0)
        #define MCRT_KNN_LAUNCH(SL) \
            do { if (lite) MCRT_KNN_LAUNCH1(SL, SHADE_FEATS_LITE); else MCRT_KNN_LAUNCH1(SL, SHADE_FEATS_ALL); } while (0)
        switch (slots)
        {
            case 1: MCRT_KNN_LAUNCH(1); break;
            case 2: MCRT_KNN_LAUNCH(2); break;
            case 4: MCRT_KNN_LAUNCH(4); break;
            case 8: MCRT_KNN_LAUNCH(8); break;
            default: MCRT_KNN_LAUNCH(0); break;
        }
        #undef MCRT_KNN_LAUNCH
        #undef MCRT_KNN_LAUNCH1
        #undef MCRT_KNN_LAUNCH2
    }
    // k_shadow of the box film (one plane, light-group planes, AOV / photon-mapper component planes, or LPE planes) with the
    // scene-specialised traversal
    template <int FILM> static void launchShadowBox(const WaveParams<MCRT_REAL>& p, int grid, cudaStream_t s)
    {
        if constexpr (Mode<MCRT_REAL>::parity)
        {
            if (p.scene.bvh4 && p.scene.dynamic_fetch)
            {
                if (p.scene.prims_class == PRIMS_TRI) k_shadow<MCRT_REAL, FILM, PRIMS_TRI, 2><<<grid, 256, fastStackSharedBytes(256), s>>>(p);
                else if (p.scene.prims_class == PRIMS_TRI_SPHERE) k_shadow<MCRT_REAL, FILM, PRIMS_TRI_SPHERE, 2><<<grid, 256, fastStackSharedBytes(256), s>>>(p);
                else k_shadow<MCRT_REAL, FILM, PRIMS_ALL, 2><<<grid, 256, fastStackSharedBytes(256), s>>>(p);
                return;
            }
            if (p.scene.bvh4)
            {
                if (p.scene.prims_class == PRIMS_TRI) k_shadow<MCRT_REAL, FILM, PRIMS_TRI, 1><<<grid, 256, fastStackSharedBytes(256), s>>>(p);
                else if (p.scene.prims_class == PRIMS_TRI_SPHERE) k_shadow<MCRT_REAL, FILM, PRIMS_TRI_SPHERE, 1><<<grid, 256, fastStackSharedBytes(256), s>>>(p);
                else k_shadow<MCRT_REAL, FILM, PRIMS_ALL, 1><<<grid, 256, fastStackSharedBytes(256), s>>>(p);
                return;
            }
        }
        if (p.scene.prims_class == PRIMS_TRI) k_shadow<MCRT_REAL, FILM, PRIMS_TRI, 0><<<grid, 256, 0, s>>>(p);
        else if (p.scene.prims_class == PRIMS_TRI_SPHERE) k_shadow<MCRT_REAL, FILM, PRIMS_TRI_SPHERE, 0><<<grid, 256, 0, s>>>(p);
        else k_shadow<MCRT_REAL, FILM, PRIMS_ALL, 0><<<grid, 256, 0, s>>>(p);
    }
    template <> void Launch<MCRT_REAL>::shadow(const WaveParams<MCRT_REAL>& p, int grid, cudaStream_t s)
    {
        if (!p.filmp.is_default_box)
        {
            // filtered film: the rare configuration, the generic traversal only
            if constexpr (Mode<MCRT_REAL>::parity)
            {
                if (p.scene.bvh4) { k_shadow<MCRT_REAL, FILM_MODE_SPLAT, PRIMS_ALL, 1><<<grid, 256, fastStackSharedBytes(256), s>>>(p); return; }
            }
            k_shadow<MCRT_REAL, FILM_MODE_SPLAT, PRIMS_ALL, 0><<<grid, 256, 0, s>>>(p);
        }
        else if (p.n_planes && p.lpe_next) launchShadowBox<FILM_MODE_LPE>(p, grid, s);
        else if (p.n_planes && p.aovs) launchShadowBox<FILM_MODE_AOV>(p, grid, s);
        else if (p.n_planes) launchShadowBox<FILM_MODE_GROUPS>(p, grid, s);
        else launchShadowBox<FILM_MODE_BOX>(p, grid, s);
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
