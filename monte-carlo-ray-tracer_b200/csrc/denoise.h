// Cross-filtered à-trous denoiser over the two halves of a progressive frame (mcrt_denoise_dev, denoise.cu).
#pragma once

#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace mcrt
{
    struct DenoiseInput
    {
        const double* a_rgb;         // [height*width][3] sums of half A
        const double* a_weight;      // [height*width] weight sums of a reconstruction filter; null with the box film
        const double* b_rgb;
        const double* b_weight;
        const double* tile_counts;   // device {nA, nB}[n_tiles]: a pixel's box-film weight in each half
        const double* features;      // [height*width][8] {albedo.rgb, normal.xyz, t, hits} sums (k_features)
        uint32_t width, height, tile, tiles_x;
    };

    struct DenoiseSigmas
    {
        double color, normal, depth, albedo;   // 0 switches a term off
    };

    // doubles of scratch launchDenoise needs for a frame of n_pixels
    size_t denoiseScratchValues(size_t n_pixels);

    // Writes the denoised frame into out [height*width][3] and adds {sum v', sum out^2} into sums[0..1] (zeroed by the
    // caller). scratch: denoiseScratchValues(width * height) doubles.
    void launchDenoise(const DenoiseInput& in, const DenoiseSigmas& sigma, uint32_t iterations, double* scratch, double* out,
                       double* sums, cudaStream_t s);
}
