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
