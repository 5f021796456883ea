// Host-callable launch wrappers; Launch<double> is instantiated in kernels_f64.cu (compiled with
// --fmad=false), Launch<float> in kernels_f32.cu.
#pragma once

#include "integrator.cuh"

namespace mcrt
{
    template <class R> struct Launch
    {
        static void generate(const WaveParams<R>& p, int next, int grid, cudaStream_t s);
        static void extend(const WaveParams<R>& p, int cur, int grid, cudaStream_t s);
        static void shade(const WaveParams<R>& p, int cur, int grid, cudaStream_t s);   // PathTracer loop body
        static void shadePhoton(const WaveParams<R>& p, int cur, int grid, cudaStream_t s); // PhotonMapper loop body
        static void knn(const WaveParams<R>& p, int grid, cudaStream_t s);
        static void emitGenerate(const WaveParams<R>& p, int next, int grid, cudaStream_t s);
        static void emitShade(const WaveParams<R>& p, int cur, int grid, cudaStream_t s);
        static void shadow(const WaveParams<R>& p, int grid, cudaStream_t s);
        static void shadeKey(const WaveParams<R>& p, int grid, cudaStream_t s);
        static void traceUser(const DeviceScene<R>& sc, const double* rays6, size_t n, double* out_tuv,
                              uint32_t* out_prim, Counters* c, int grid, cudaStream_t s);
        static void features(const DeviceScene<R>& sc, const DeviceCamera<R>& cam, uint32_t global_seed, uint32_t sample_first,
                             uint32_t sample_count, double* out, Counters* c, int grid, cudaStream_t s);
        static void featuresChain(const DeviceScene<R>& sc, const DeviceCamera<R>& cam, uint32_t global_seed, uint32_t sample_first,
                                  uint32_t sample_count, uint32_t specular_depth, R ray_eps, double* out, Counters* c, int grid,
                                  cudaStream_t s);
    };

    void launchAdvance(Counters* c, cudaStream_t s);
    void launchSortScan(uint32_t* hist, const RaySort& rs, cudaStream_t s);
    void launchSortScatter(const uint32_t* key, const uint32_t* rank, const RaySort& rs, uint32_t* order,
                           const uint32_t* n_ptr, int grid, cudaStream_t s);
    void launchResolveFilmWeighted(const double* film, const double* wsum, double* out, size_t n_pixels, int grid, cudaStream_t s);
    void launchResolveFilm(const double* film, double* out, size_t n_values, double weight, int grid, cudaStream_t s);
    void launchResolveFilmPeers(const double* film, const PeerFrames& pf, size_t n_values, double weight, int grid, cudaStream_t s);
    // Resolves a+b into out and adds {sum v, sum I^2} of each tile into sums[2*tile..] and of the frame into
    // sums[2*n_tiles..] (zeroed by the caller); tile_error (optional) receives the per-tile relative errors.
    // tile_counts (device, optional): per-tile {nA, nB}[n_tiles] in place of a.samples, b.samples.
    void launchProgressiveResolve(const ProgressiveHalf& a, const ProgressiveHalf& b, bool weighted, uint32_t width, uint32_t rows,
                                  uint32_t tile, uint32_t tiles_x, double* out, double* sums, double* tile_error, uint32_t n_tiles,
                                  int grid, cudaStream_t s, const double* tile_counts = nullptr);
    // out[i] = sum_g weights[g][i % 3] * planes[g * n_values + i], summed over g in order (mcrt_light_groups_combine_dev)
    void launchLightGroupsCombine(const double* planes, uint32_t n_planes, uint64_t n_values, const double* weights, double* out,
                                  int grid, cudaStream_t s);
    void launchFp64Peak(double* sink, int iterations, int grid, cudaStream_t s);
    void launchKnnUser(const DevicePhotonMap& map, uint32_t k, const double* points, size_t n, uint32_t* out_index,
                       double* out_d2, uint32_t* out_count, uint32_t* overflow_flag, int grid, cudaStream_t s);
    void launchGatherUser(const DevicePhotonMap& map, const double* points, size_t n, double r2, uint32_t* out_count,
                          double* out_flux, double* out_cone, uint32_t* overflow_flag, int grid, cudaStream_t s);
    void launchSamplerStream(const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t n_shuffles,
                             uint32_t global_seed, uint32_t* out, cudaStream_t s);
}
