// Parity mode: float64, reference operation order. Compiled with --fmad=false (the reference's
// CPU build performs no FMA contraction, /root/reference/CMakeLists.txt:16-21).
#define MCRT_REAL double
#include "kernels_impl.cuh"

namespace mcrt
{
    void launchAdvance(Counters* c, cudaStream_t s) { k_advance<<<1, 1, 0, s>>>(c); }

    void launchSortScan(uint32_t* hist, const RaySort& rs, cudaStream_t s)
    {
        k_sort_scan<<<SORT_SCAN_BLOCKS, 256, 0, s>>>(hist, rs.bin_start, rs.block_offset, rs.done_counter);
    }

    void launchSortScatter(const uint32_t* key, const uint32_t* rank, const RaySort& rs, uint32_t* order,
                           const uint32_t* n_ptr, int grid, cudaStream_t s)
    {
        k_sort_scatter<<<grid, 256, 0, s>>>(key, rank, rs.bin_start, rs.block_offset, order, n_ptr);
    }

    void launchResolveFilmWeighted(const double* film, const double* wsum, double* out, size_t n_pixels, int grid, cudaStream_t s)
    {
        k_resolve_film_weighted<<<grid, 256, 0, s>>>(film, wsum, out, n_pixels);
    }

    void launchResolveFilm(const double* film, double* out, size_t n_values, double weight, int grid, cudaStream_t s)
    {
        k_resolve_film<<<grid, 256, 0, s>>>(film, out, n_values, weight);
    }

    void launchResolveFilmPeers(const double* film, const PeerFrames& pf, size_t n_values, double weight, int grid, cudaStream_t s)
    {
        k_resolve_film_peers<<<grid, 256, 0, s>>>(film, pf, n_values, weight);
    }

    // Progressive resolve: frame = max((A+B) / (wA+wB), 0) as Film::Splat::get (film.cpp:106-113), and per pixel and
    // channel v = (I_A - I_B)^2 nA nB / (nA+nB)^2 with I_A = A/wA, I_B = B/wB: for independent halves an unbiased
    // estimate of the variance of the combined mean. v and I^2 are summed per tile x tile block of the buffer's
    // rows x width (one atomic per warp and tile) and over the frame (one atomic per warp).
    // TILE_COUNTS (adaptive sampling): nA, nB are those of the pixel's tile, tile_counts[tile][2], instead of
    // a.samples, b.samples. With a filter a pixel near a tile's border also holds splats of samples of neighbouring
    // tiles, which may have other counts; its own tile's counts in the scale are then an approximation.
    template <bool TILE_COUNTS>
    static __global__ void __launch_bounds__(256) k_progressive_resolve(ProgressiveHalf a, ProgressiveHalf b, uint32_t weighted,
                                                                        uint32_t width, uint32_t rows, uint32_t tile,
                                                                        uint32_t tiles_x, uint32_t n_tiles, double* out, double* sums,
                                                                        const double* tile_counts)
    {
        const uint64_t n = (uint64_t)width * rows;
        const bool both = a.samples > 0.0 && b.samples > 0.0;
        const double scale = both ? a.samples * b.samples / ((a.samples + b.samples) * (a.samples + b.samples)) : 0.0;
        const unsigned lane = threadIdx.x & 31u;
        // stride and bound are multiples of 32: the lanes of a warp leave the loop together
        const uint64_t n_rounded = (n + 31u) & ~31ull;
        for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_rounded; i += (uint64_t)gridDim.x * blockDim.x)
        {
            double v = 0.0, i2 = 0.0;
            uint32_t key = 0xFFFFFFFFu;
            if (i < n)
            {
                double na = a.samples, nb = b.samples, pixel_scale = scale;
                bool pixel_both = both;
                if constexpr (TILE_COUNTS)
                {
                    const uint32_t y = (uint32_t)(i / width), x = (uint32_t)(i - (uint64_t)y * width);
                    const size_t t = (size_t)(y / tile) * tiles_x + x / tile;
                    na = tile_counts[2 * t]; nb = tile_counts[2 * t + 1];
                    pixel_both = na > 0.0 && nb > 0.0;
                    pixel_scale = pixel_both ? na * nb / ((na + nb) * (na + nb)) : 0.0;
                }
                const double wa = !a.rgb ? 0.0 : (weighted ? a.wsum[i] : na);
                const double wb = !b.rgb ? 0.0 : (weighted ? b.wsum[i] : nb);
                const double w = wa + wb;
                const bool compare = pixel_both && wa != 0.0 && wb != 0.0;
                for (int c = 0; c < 3; c++)
                {
                    const double sa = a.rgb ? a.rgb[3 * i + c] : 0.0, sb = b.rgb ? b.rgb[3 * i + c] : 0.0;
                    double value = w == 0.0 ? 0.0 : (sa + sb) / w;
                    value = value < 0.0 ? 0.0 : value;
                    out[3 * i + c] = value;
                    i2 += value * value;
                    if (compare)
                    {
                        const double d = sa / wa - sb / wb;
                        v += d * d * pixel_scale;
                    }
                }
                const uint32_t y = (uint32_t)(i / width), x = (uint32_t)(i - (uint64_t)y * width);
                key = (y / tile) * tiles_x + x / tile;
            }
            double fv = v, fi = i2;
            for (int off = 16; off > 0; off >>= 1)
            {
                fv += __shfl_xor_sync(0xFFFFFFFFu, fv, off);
                fi += __shfl_xor_sync(0xFFFFFFFFu, fi, off);
            }
            if (lane == 0)
            {
                if (fv != 0.0) atomicAdd(&sums[2 * (size_t)n_tiles], fv);
                if (fi != 0.0) atomicAdd(&sums[2 * (size_t)n_tiles + 1], fi);
            }
            // one group of lanes per tile the warp touches
            unsigned pending = __ballot_sync(0xFFFFFFFFu, key != 0xFFFFFFFFu);
            while (pending)
            {
                const int leader = __ffs(pending) - 1;
                const uint32_t k = __shfl_sync(0xFFFFFFFFu, key, leader);
                const bool mine = key == k;
                double gv = mine ? v : 0.0, gi = mine ? i2 : 0.0;
                for (int off = 16; off > 0; off >>= 1)
                {
                    gv += __shfl_xor_sync(0xFFFFFFFFu, gv, off);
                    gi += __shfl_xor_sync(0xFFFFFFFFu, gi, off);
                }
                if ((int)lane == leader)
                {
                    if (gv != 0.0) atomicAdd(&sums[2 * (size_t)k], gv);
                    if (gi != 0.0) atomicAdd(&sums[2 * (size_t)k + 1], gi);
                }
                pending &= ~__ballot_sync(0xFFFFFFFFu, mine);
            }
        }
    }

    // TILE_COUNTS: a tile has both halves when its own counts tile_counts[t][2] are both nonzero
    template <bool TILE_COUNTS>
    static __global__ void k_progressive_tile_error(const double* sums, uint32_t n_tiles, bool both_halves, double* tile_error,
                                                    const double* tile_counts)
    {
        for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n_tiles; t += gridDim.x * blockDim.x)
        {
            bool both = both_halves;
            if constexpr (TILE_COUNTS) both = tile_counts[2 * (size_t)t] > 0.0 && tile_counts[2 * (size_t)t + 1] > 0.0;
            tile_error[t] = progressiveRelativeError(sums[2 * (size_t)t], sums[2 * (size_t)t + 1], both);
        }
    }

    void launchProgressiveResolve(const ProgressiveHalf& a, const ProgressiveHalf& b, bool weighted, uint32_t width, uint32_t rows,
                                  uint32_t tile, uint32_t tiles_x, double* out, double* sums, double* tile_error, uint32_t n_tiles,
                                  int grid, cudaStream_t s, const double* tile_counts)
    {
        const uint32_t w = weighted ? 1u : 0u;
        if (tile_counts) k_progressive_resolve<true><<<grid, 256, 0, s>>>(a, b, w, width, rows, tile, tiles_x, n_tiles, out, sums, tile_counts);
        else k_progressive_resolve<false><<<grid, 256, 0, s>>>(a, b, w, width, rows, tile, tiles_x, n_tiles, out, sums, nullptr);
        if (!tile_error) return;
        const uint32_t tile_grid = (n_tiles + 255) / 256 < (uint32_t)grid ? (n_tiles + 255) / 256 : (uint32_t)grid;
        const bool both = a.samples > 0.0 && b.samples > 0.0;
        if (tile_counts) k_progressive_tile_error<true><<<tile_grid, 256, 0, s>>>(sums, n_tiles, both, tile_error, tile_counts);
        else k_progressive_tile_error<false><<<tile_grid, 256, 0, s>>>(sums, n_tiles, both, tile_error, nullptr);
    }

    // Relighting of light-group planes: out[i] = sum over g of weights[g][i % 3] * planes[g][i], g = 0, 1, ... in order,
    // each product rounded before its addition (this unit has no FMA contraction), so numpy reproduces it bit for bit
    static __global__ void __launch_bounds__(256) k_light_groups_combine(const double* planes, uint32_t n_planes, uint64_t n_values,
                                                                         const double* weights, double* out)
    {
        for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_values; i += (uint64_t)gridDim.x * blockDim.x)
        {
            const uint32_t c = (uint32_t)(i % 3u);
            double acc = weights[c] * planes[i];
            for (uint32_t g = 1; g < n_planes; g++) acc = acc + weights[3 * g + c] * planes[g * n_values + i];
            out[i] = acc;
        }
    }

    void launchLightGroupsCombine(const double* planes, uint32_t n_planes, uint64_t n_values, const double* weights, double* out,
                                  int grid, cudaStream_t s)
    {
        k_light_groups_combine<<<grid, 256, 0, s>>>(planes, n_planes, n_values, weights, out);
    }

    void launchFp64Peak(double* sink, int iterations, int grid, cudaStream_t s)
    {
        k_fp64_peak<<<grid, 256, 0, s>>>(sink, iterations);
    }

    void launchKnnUser(const DevicePhotonMap& map, uint32_t k, const double* points, size_t n, uint32_t* out_index,
                       double* out_d2, uint32_t* out_count, uint32_t* overflow_flag, int grid, cudaStream_t s)
    {
        const dim3 g(grid), b(32 * KNN_WARPS_PER_BLOCK);
        const size_t smem = knnSharedBytes(k);
        static bool attr_set = false;
        if (!attr_set)
        {
            const int max_smem = (int)knnSharedBytes(1024);   // k > 672 exceeds the default 48 KB
            cudaFuncSetAttribute(k_knn_user<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
            cudaFuncSetAttribute(k_knn_user<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
            cudaFuncSetAttribute(k_knn_user<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
            cudaFuncSetAttribute(k_knn_user<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
            cudaFuncSetAttribute(k_knn_user<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
            attr_set = true;
        }
        switch (knnSlotsFor(k))
        {
            case 1: k_knn_user<1><<<g, b, smem, s>>>(map, k, points, n, out_index, out_d2, out_count, overflow_flag); break;
            case 2: k_knn_user<2><<<g, b, smem, s>>>(map, k, points, n, out_index, out_d2, out_count, overflow_flag); break;
            case 4: k_knn_user<4><<<g, b, smem, s>>>(map, k, points, n, out_index, out_d2, out_count, overflow_flag); break;
            case 8: k_knn_user<8><<<g, b, smem, s>>>(map, k, points, n, out_index, out_d2, out_count, overflow_flag); break;
            default: k_knn_user<0><<<g, b, smem, s>>>(map, k, points, n, out_index, out_d2, out_count, overflow_flag); break;
        }
    }

    // Fixed-radius search on caller points (mcrt_photon_gather_search), the traversal of k_gather: per point the
    // number of photons within r and the float64 sums of their float32 flux, plain and cone-weighted (1 - d/r).
    __global__ void __launch_bounds__(32 * KNN_WARPS_PER_BLOCK) k_gather_user(DevicePhotonMap map, const double* points, size_t n,
                                                                             double r2, uint32_t* out_count, double* out_flux,
                                                                             double* out_cone, uint32_t* overflow_flag)
    {
        __shared__ uint32_t gather_stack[KNN_WARPS_PER_BLOCK][GATHER_STACK];
        uint32_t* const stack = gather_stack[threadIdx.x >> 5];
        const unsigned lane = threadIdx.x & 31u;
        const size_t warps_total = (size_t)gridDim.x * KNN_WARPS_PER_BLOCK;
        const double inv_r2 = 1.0 / r2;
        uint32_t overflow = 0;
        for (size_t q = (size_t)blockIdx.x * KNN_WARPS_PER_BLOCK + (threadIdx.x >> 5); q < n; q += warps_total)
        {
            uint32_t count = 0;
            double f[3] = { 0.0, 0.0, 0.0 }, c[3] = { 0.0, 0.0, 0.0 };
            gatherWarp(map, points[3 * q], points[3 * q + 1], points[3 * q + 2], r2, stack, &overflow,
                       [&](unsigned long long, double d2, const float4& a, const float4&)
                       {
                           const double wp = fmax(0.0, 1.0 - sqrt(d2 * inv_r2));
                           count++;
                           f[0] += (double)a.x; f[1] += (double)a.y; f[2] += (double)a.z;
                           c[0] += (double)a.x * wp; c[1] += (double)a.y * wp; c[2] += (double)a.z * wp;
                       });
            count = __reduce_add_sync(0xFFFFFFFFu, count);
            for (int off = 16; off > 0; off >>= 1)
                for (int j = 0; j < 3; j++)
                {
                    f[j] += __shfl_xor_sync(0xFFFFFFFFu, f[j], off);
                    c[j] += __shfl_xor_sync(0xFFFFFFFFu, c[j], off);
                }
            if (lane == 0)
            {
                out_count[q] = count;
                for (int j = 0; j < 3; j++) { out_flux[3 * q + j] = f[j]; out_cone[3 * q + j] = c[j]; }
            }
            __syncwarp();
        }
        if (overflow && lane == 0) atomicOr(overflow_flag, 1u);
    }

    void launchGatherUser(const DevicePhotonMap& map, const double* points, size_t n, double r2, uint32_t* out_count,
                          double* out_flux, double* out_cone, uint32_t* overflow_flag, int grid, cudaStream_t s)
    {
        k_gather_user<<<grid, 32 * KNN_WARPS_PER_BLOCK, 0, s>>>(map, points, n, r2, out_count, out_flux, out_cone, overflow_flag);
    }

    __global__ void k_sampler_stream(const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t n_shuffles,
                                     uint32_t global_seed, uint32_t* out)
    {
        for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        {
            SamplerState s = SamplerState::make(global_seed, pixel[i], sample[i], n_shuffles);
            uint32_t raw[7];
            s.raw<0x7Fu>(raw);
            for (int d = 0; d < 7; d++) out[7 * i + d] = raw[d];
        }
    }

    void launchSamplerStream(const uint32_t* pixel, const uint32_t* sample, size_t n, uint32_t n_shuffles,
                             uint32_t global_seed, uint32_t* out, cudaStream_t s)
    {
        int grid = (int)((n + 255) / 256);
        if (grid > 1184) grid = 1184;
        if (grid < 1) grid = 1;
        k_sampler_stream<<<grid, 256, 0, s>>>(pixel, sample, n, n_shuffles, global_seed, out);
    }
}
