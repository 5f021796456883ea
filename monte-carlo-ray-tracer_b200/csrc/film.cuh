// Film reconstruction on the device (widened scope, SURVEY.md §8f-4): Film::deposit with the
// reference's reconstruction filters (source/camera/film.cpp:61-113, source/camera/filter.hpp:8-66).
// The default box film (radius 0.5) deposits every sample into exactly one pixel with weight 1 and
// keeps the fast path: one RED.ADD.F64 per channel, resolve = sum / spp. For the other filters a
// radiance contribution v of sample (pixel, s) is splatted as v * wy * wx over the filter window
// around the sample's jittered film position, and the weights are accumulated once per sample in
// k_generate; resolve = rgb_sum / weight_sum, clamped at 0. By linearity, splatting each
// contribution of a path separately equals the reference's single deposit of the path's radiance.
#pragma once

#include "sampler.cuh"

namespace mcrt
{
    enum FilmFilter : uint32_t
    {
        FILM_BOX = 0, FILM_MITCHELL_NETRAVALI = 1, FILM_CATMULL_ROM = 2, FILM_B_SPLINE = 3, FILM_HERMITE = 4,
        FILM_GAUSSIAN = 5, FILM_LANCZOS = 6
    };

    struct FilmParams
    {
        double* rgb;            // [pixels][3]
        double* wsum;           // [pixels] (filters other than the default box)
        const double* cache;    // Film::filter_cache or null
        double radius, two_inv_radius, inv_dx;
        uint32_t filter, cache_size, width, height;
        uint32_t _pad[2];
    };

    // Filter::MitchellNetravali<B, C>, filter.hpp:15-38 (same constant expressions, evaluated at compile time)
    template <int VARIANT>
    MCRT_HD double mitchellNetravali(double x)
    {
        constexpr double B = VARIANT == 0 ? 1.0 / 3.0 : (VARIANT == 2 ? 1.0 : 0.0);
        constexpr double C = VARIANT == 0 ? 1.0 / 3.0 : (VARIANT == 1 ? 0.5 : 0.0);
        constexpr double k = 6.0 / (6.0 - 2.0 * B);
        if (x < 1.0)
        {
            constexpr double a = k * (12.0 - 9.0 * B - 6.0 * C) / 6.0;
            constexpr double b = k * (-18.0 + 12.0 * B + 6.0 * C) / 6.0;
            constexpr double d = k * (6.0 - 2.0 * B) / 6.0;
            return d + (b + a * x) * x * x;
        }
        else
        {
            constexpr double a = k * (-B - 6.0 * C) / 6.0;
            constexpr double b = k * (6.0 * B + 30.0 * C) / 6.0;
            constexpr double c = k * (-12.0 * B - 48.0 * C) / 6.0;
            constexpr double d = k * (8.0 * B + 24.0 * C) / 6.0;
            return d + (c + (b + a * x) * x) * x;
        }
    }

    // the filter_function of Film (film.cpp:25-43), x in [0, 2]
    MCRT_HD double filmFilterFunction(uint32_t filter, double x)
    {
        switch (filter)
        {
            case FILM_MITCHELL_NETRAVALI: return mitchellNetravali<0>(x);
            case FILM_CATMULL_ROM: return mitchellNetravali<1>(x);         // B = 0, C = 0.5
            case FILM_B_SPLINE: return mitchellNetravali<2>(x);            // B = 1, C = 0
            case FILM_HERMITE: return mitchellNetravali<3>(x * 0.5);       // B = C = 0, stretched (filter.hpp:50-54)
            case FILM_GAUSSIAN: return exp(-2.0 * x * x) - exp(-2.0 * 2.0 * 2.0);
            case FILM_LANCZOS:
                if (x == 0.0) return 1.0;
                return 2.0 * sin(3.14159265358979323846 * x) * sin(3.14159265358979323846 * x / 2.0) / (3.14159265358979323846 * 3.14159265358979323846 * x * x);
            default: return 1.0;
        }
    }

    // Film::filter, film.cpp:86-97
    MCRT_D double filmFilter(const FilmParams& f, double x)
    {
        const double ax = fabs(x);
        if (f.cache_size == 0) return filmFilterFunction(f.filter, f.two_inv_radius * ax);
        return f.cache[(size_t)(f.inv_dx * ax + 0.5)];
    }

    // jittered film position of (pixel, sample): camera.cpp:79-80
    MCRT_D void filmPosition(uint32_t global_seed, uint32_t width, uint32_t pixel, uint32_t sample, double& px, double& py)
    {
        const SamplerState smp = SamplerState::make(global_seed, pixel, sample, 0u);
        double u[2];
        samplerGet<double, DIM_PIXEL, 2>(smp, u);
        px = (double)(pixel % width) + u[0];
        py = (double)(pixel / width) + u[1];
    }

    // window of Film::deposit, film.cpp:63-64 (ivec2 conversion truncates toward zero)
    MCRT_D void filmWindow(const FilmParams& f, double px, double py, long long& x0, long long& x1, long long& y0, long long& y1)
    {
        x0 = (long long)(px + 0.5 - f.radius); if (x0 < 0) x0 = 0;
        y0 = (long long)(py + 0.5 - f.radius); if (y0 < 0) y0 = 0;
        x1 = (long long)(px - 0.5 + f.radius); if (x1 > (long long)f.width - 1) x1 = (long long)f.width - 1;
        y1 = (long long)(py - 0.5 + f.radius); if (y1 > (long long)f.height - 1) y1 = (long long)f.height - 1;
    }

    // Film::deposit of one contribution (general filters)
    MCRT_D void filmSplatInline(const FilmParams& f, double px, double py, double r, double g, double b)
    {
        long long x0, x1, y0, y1;
        filmWindow(f, px, py, x0, x1, y0, y1);
        for (long long y = y0; y <= y1; y++)
        {
            const double wy = filmFilter(f, (double)y + 0.5 - py);
            for (long long x = x0; x <= x1; x++)
            {
                const double w = wy * filmFilter(f, (double)x + 0.5 - px);
                const size_t pix = (size_t)y * f.width + (size_t)x;
                if (r != 0.0) atomicAdd(&f.rgb[3 * pix + 0], r * w);
                if (g != 0.0) atomicAdd(&f.rgb[3 * pix + 1], g * w);
                if (b != 0.0) atomicAdd(&f.rgb[3 * pix + 2], b * w);
            }
        }
    }

    // weight_sum += weight, once per camera sample (film.cpp:99-104)
    MCRT_D void filmSplatWeightInline(const FilmParams& f, double px, double py)
    {
        long long x0, x1, y0, y1;
        filmWindow(f, px, py, x0, x1, y0, y1);
        for (long long y = y0; y <= y1; y++)
        {
            const double wy = filmFilter(f, (double)y + 0.5 - py);
            for (long long x = x0; x <= x1; x++)
                atomicAdd(&f.wsum[(size_t)y * f.width + (size_t)x], wy * filmFilter(f, (double)x + 0.5 - px));
        }
    }

    // Out-of-line entry points: the filtered film is the rare configuration, and inlining the splat
    // loops into k_shade / k_generate costs the default box path registers (measured: +58..280 B of
    // spills in the f64 shade kernels). FilmParams travels by value so the kernel parameter block
    // is never addressed.
    static __device__ __noinline__ void filmSplatSample(FilmParams f, uint32_t global_seed, uint32_t pixel, uint32_t sample,
                                                        double r, double g, double b)
    {
        double px, py;
        filmPosition(global_seed, f.width, pixel, sample, px, py);
        filmSplatInline(f, px, py, r, g, b);
    }

    static __device__ __noinline__ void filmSplatSampleWeight(FilmParams f, uint32_t global_seed, uint32_t pixel, uint32_t sample)
    {
        double px, py;
        filmPosition(global_seed, f.width, pixel, sample, px, py);
        filmSplatWeightInline(f, px, py);
    }
}
