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

    struct DenoisePlanes
    {
        const double* a;   // [n][height*width][3] box-film sums of half A of each plane
        const double* b;
        double* a_out;     // filtered sums, same layout; must not overlap a, b or each other
        double* b_out;
        uint32_t n;
    };

    // doubles of planes_scratch launchDenoisePlanes needs: the tap weights, 2 halves x 25 taps per pixel (400 B, 0.83 GB
    // at 1920x1080), and one plane state set, {a[3], b[3]} per pixel per plane (48 B, 3.1 GB for 31 planes at 1920x1080)
    size_t denoisePlanesScratchValues(size_t n_pixels, uint32_t n_planes);

    // Filters every plane with the weights launchDenoise computes for the guide frame `in` (box film) and writes the
    // filtered sums into planes.a_out / b_out; an invalid pixel keeps its input sums. out (optional) and sums receive what
    // launchDenoise writes. scratch: denoiseScratchValues(width * height) doubles; planes_scratch:
    // denoisePlanesScratchValues(width * height, planes.n).
    void launchDenoisePlanes(const DenoiseInput& in, const DenoisePlanes& planes, const DenoiseSigmas& sigma, uint32_t iterations,
                             double* scratch, double* planes_scratch, double* out, double* sums, cudaStream_t s);
}
