// Cross-filtered à-trous denoiser for progressive frames (mcrt_denoise_dev), float64 throughout.
//
// Halves A and B of a frame are filtered separately, and the colour term of each half's weights is measured on the
// other half (cross-filtering, after Rousselle, Knaus & Zwicker, "Adaptive Rendering with Non-Local Means
// Filtering", 2012), so the weights do not correlate with the noise they remove and the difference of the two
// filtered halves still estimates the residual noise. oracle/denoise_ref.py restates these kernels in numpy.
//
// With w_X a pixel's weight in half X (box film: its tile's count; filter: its weight sum) and I_X = S_X / w_X:
// - prep: I_A, I_B; var_A = mean_c (I_A - I_B)^2 w_B / (w_A + w_B) and var_B = ... w_A / (w_A + w_B), each smoothed
//   by a 3x3 [1,2,1]x[1,2,1] kernel normalised over the valid in-image pixels it covers; the guide record.
//   A pixel with zero weight in either half is invalid: it is output as its plain resolve and is never a neighbour.
// - K a-trous iterations of step 2^k: 5x5 taps of h = (1,4,6,4,1)/16 separable, weight h w_n w_z w_a w_c with the
//   colour term w_c on the partner half; X' = sum w X_q / sum w, var_X' = sum w^2 var_X,q / (sum w)^2.
// - final: out = max(0, (w_A A + w_B B) / (w_A + w_B)), v' = sum_c (A - B)^2 w_A w_B / (w_A + w_B)^2, and the
//   frame sums {sum v', sum out^2}.
//
// Planes (mcrt_denoise_planes_dev): the filter is linear in the data once its weights are fixed, so every plane is
// filtered with the weights of the beauty frame. k_denoise_atrous_weights is k_denoise_atrous plus a store of each
// tap's weights; k_denoise_atrous_planes applies them to the planes' per-half means, and k_denoise_planes_prep / _final
// turn sums into means and back. Planes that sum to the beauty then have filtered sums that sum to its filtered sums,
// up to rounding.
#include <cmath>

#include "denoise.h"

// planes per thread of k_denoise_atrous_planes: each tap weight it loads serves this many planes (DESIGN.md §3)
#ifndef MCRT_DENOISE_PLANE_CHUNK
#define MCRT_DENOISE_PLANE_CHUNK 8
#endif

namespace mcrt
{
    namespace
    {
        constexpr int BX = 32, BY = 8;   // a warp is 32 pixels of one row: the taps of a row share lines
        constexpr int DENOISE_PLANE_CHUNK = MCRT_DENOISE_PLANE_CHUNK;

        enum : uint32_t { GUIDE_SURFACE = 0u, GUIDE_BACKGROUND = 1u, GUIDE_INVALID = 2u };

        struct alignas(16) State
        {
            double a[3], b[3];
            double var_a, var_b;
        };

        struct alignas(16) Guide
        {
            double n[3];
            double z;
            double albedo[3];
            double flag;   // GUIDE_*
        };

        __device__ __forceinline__ void halfWeights(const DenoiseInput& in, uint32_t x, uint32_t y, size_t i, double& wa, double& wb)
        {
            if (in.a_weight)
            {
                wa = in.a_weight[i];
                wb = in.b_weight[i];
            }
            else
            {
                const size_t t = (size_t)(y / in.tile) * in.tiles_x + x / in.tile;
                wa = in.tile_counts[2 * t];
                wb = in.tile_counts[2 * t + 1];
            }
        }

        // unfiltered per-half variances of pixel i; false for an invalid pixel
        __device__ __forceinline__ bool rawVariance(const DenoiseInput& in, uint32_t x, uint32_t y, double& va, double& vb)
        {
            const size_t i = (size_t)y * in.width + x;
            double wa, wb;
            halfWeights(in, x, y, i, wa, wb);
            if (wa == 0.0 || wb == 0.0) return false;
            double d2 = 0.0;
            for (int c = 0; c < 3; c++)
            {
                const double d = in.a_rgb[3 * i + c] / wa - in.b_rgb[3 * i + c] / wb;
                d2 += d * d;
            }
            d2 = d2 / 3.0;
            va = d2 * (wb / (wa + wb));
            vb = d2 * (wa / (wa + wb));
            return true;
        }

        __global__ void __launch_bounds__(BX * BY) k_denoise_prep(DenoiseInput in, State* state, Guide* guide)
        {
            const uint32_t x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
            if (x >= in.width || y >= in.height) return;
            const size_t i = (size_t)y * in.width + x;
            Guide& g = guide[i];
            State& st = state[i];
            for (int k = 0; k < 3; k++) { g.n[k] = 0.0; g.albedo[k] = 0.0; }
            g.z = 0.0;
            double sa = 0.0, sb = 0.0, sk = 0.0;
            for (int dy = -1; dy <= 1; dy++)
            {
                const int qy = (int)y + dy;
                if (qy < 0 || qy >= (int)in.height) continue;
                for (int dx = -1; dx <= 1; dx++)
                {
                    const int qx = (int)x + dx;
                    if (qx < 0 || qx >= (int)in.width) continue;
                    double va, vb;
                    if (!rawVariance(in, (uint32_t)qx, (uint32_t)qy, va, vb)) continue;
                    const double k = (double)((2 - (dx < 0 ? -dx : dx)) * (2 - (dy < 0 ? -dy : dy)));
                    sa += k * va; sb += k * vb; sk += k;
                }
            }
            double wa, wb;
            halfWeights(in, x, y, i, wa, wb);
            if (wa == 0.0 || wb == 0.0)
            {
                g.flag = GUIDE_INVALID;
                for (int c = 0; c < 3; c++) { st.a[c] = 0.0; st.b[c] = 0.0; }
                st.var_a = st.var_b = 0.0;
                return;
            }
            st.var_a = sa / sk;   // sk > 0: the pixel itself is valid
            st.var_b = sb / sk;
            for (int c = 0; c < 3; c++)
            {
                st.a[c] = in.a_rgb[3 * i + c] / wa;
                st.b[c] = in.b_rgb[3 * i + c] / wb;
            }
            const double* f = in.features + 8 * i;
            const double hits = f[7];
            if (hits == 0.0) { g.flag = GUIDE_BACKGROUND; return; }
            g.flag = GUIDE_SURFACE;
            const double len2 = f[3] * f[3] + f[4] * f[4] + f[5] * f[5];
            if (len2 > 0.0)
            {
                const double inv = 1.0 / sqrt(len2);
                for (int k = 0; k < 3; k++) g.n[k] = f[3 + k] * inv;
            }
            g.z = f[6] / hits;
            for (int k = 0; k < 3; k++) g.albedo[k] = f[k] / hits;
        }

        // (1, 4, 6, 4, 1) / 16
        __device__ __forceinline__ double binomial5(int k) { return (k == 2 ? 6.0 : (k == 1 || k == 3 ? 4.0 : 1.0)) / 16.0; }

        __device__ __forceinline__ double colorWeight(double d2, double var_sum, double sigma)
        {
            if (sigma == 0.0) return 1.0;
            const double num = fmax(0.0, d2 - var_sum);
            if (num == 0.0) return 1.0;
            if (var_sum == 0.0) return 0.0;
            return exp(-num / (sigma * sigma * var_sum));
        }

        __global__ void __launch_bounds__(BX * BY) k_denoise_atrous(uint32_t width, uint32_t height, uint32_t step, DenoiseSigmas sg,
                                                                    const Guide* __restrict__ guide, const State* __restrict__ src,
                                                                    State* __restrict__ dst)
        {
            const uint32_t x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
            if (x >= width || y >= height) return;
            const size_t i = (size_t)y * width + x;
            const Guide gp = guide[i];
            const State sp = src[i];
            if (gp.flag == GUIDE_INVALID) { dst[i] = sp; return; }
            double acc_a[3] = { 0.0, 0.0, 0.0 }, acc_b[3] = { 0.0, 0.0, 0.0 };
            double wsum_a = 0.0, wsum_b = 0.0, vsum_a = 0.0, vsum_b = 0.0;
            for (int ky = 0; ky < 5; ky++)
            {
                const long long qy = (long long)y + (long long)(ky - 2) * step;
                if (qy < 0 || qy >= (long long)height) continue;
                for (int kx = 0; kx < 5; kx++)
                {
                    const long long qx = (long long)x + (long long)(kx - 2) * step;
                    if (qx < 0 || qx >= (long long)width) continue;
                    const size_t q = (size_t)qy * width + (size_t)qx;
                    const double hw = binomial5(ky) * binomial5(kx);
                    double wa = hw, wb = hw;
                    const State sq = src[q];
                    if (q != i)
                    {
                        const Guide gq = guide[q];
                        if (gq.flag == GUIDE_INVALID) continue;
                        double wf = 1.0;
                        if (gp.flag != gq.flag) wf = 0.0;   // background against surface
                        else if (gp.flag == GUIDE_SURFACE)
                        {
                            if (sg.normal != 0.0)
                                wf *= pow(fmax(0.0, gp.n[0] * gq.n[0] + gp.n[1] * gq.n[1] + gp.n[2] * gq.n[2]), sg.normal);
                            if (sg.depth != 0.0)
                                wf *= exp(-fabs(gp.z - gq.z) / (sg.depth * fmax(gp.z, gq.z)));
                            if (sg.albedo != 0.0)
                            {
                                double d2 = 0.0;
                                for (int c = 0; c < 3; c++) { const double d = gp.albedo[c] - gq.albedo[c]; d2 += d * d; }
                                wf *= exp(-d2 / (sg.albedo * sg.albedo));
                            }
                        }
                        if (wf == 0.0) continue;
                        double d2a = 0.0, d2b = 0.0;
                        for (int c = 0; c < 3; c++)
                        {
                            const double da = sp.a[c] - sq.a[c], db = sp.b[c] - sq.b[c];
                            d2a += da * da; d2b += db * db;
                        }
                        // each half's colour term is measured on its partner
                        wa = hw * wf * colorWeight(d2b / 3.0, sp.var_b + sq.var_b, sg.color);
                        wb = hw * wf * colorWeight(d2a / 3.0, sp.var_a + sq.var_a, sg.color);
                    }
                    for (int c = 0; c < 3; c++) { acc_a[c] += wa * sq.a[c]; acc_b[c] += wb * sq.b[c]; }
                    wsum_a += wa; wsum_b += wb;
                    vsum_a += wa * wa * sq.var_a; vsum_b += wb * wb * sq.var_b;
                }
            }
            State o;
            for (int c = 0; c < 3; c++) { o.a[c] = acc_a[c] / wsum_a; o.b[c] = acc_b[c] / wsum_b; }
            o.var_a = vsum_a / (wsum_a * wsum_a);
            o.var_b = vsum_b / (wsum_b * wsum_b);
            dst[i] = o;
        }

        __global__ void __launch_bounds__(BX * BY) k_denoise_final(DenoiseInput in, const Guide* guide, const State* state, double* out,
                                                                   double* sums)
        {
            const uint32_t x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
            double v = 0.0, i2 = 0.0;
            if (x < in.width && y < in.height)
            {
                const size_t i = (size_t)y * in.width + x;
                double wa, wb;
                halfWeights(in, x, y, i, wa, wb);
                const double w = wa + wb;
                if (guide[i].flag == GUIDE_INVALID)
                {
                    // the plain resolve, as k_progressive_resolve writes it
                    for (int c = 0; c < 3; c++)
                    {
                        double value = w == 0.0 ? 0.0 : (in.a_rgb[3 * i + c] + in.b_rgb[3 * i + c]) / w;
                        value = value < 0.0 ? 0.0 : value;
                        out[3 * i + c] = value;
                        i2 += value * value;
                    }
                }
                else
                {
                    const State st = state[i];
                    const double scale = wa * wb / (w * w);
                    for (int c = 0; c < 3; c++)
                    {
                        double value = (wa * st.a[c] + wb * st.b[c]) / w;
                        value = value < 0.0 ? 0.0 : value;
                        out[3 * i + c] = value;
                        i2 += value * value;
                        const double d = st.a[c] - st.b[c];
                        v += d * d * scale;
                    }
                }
            }
            for (int off = 16; off > 0; off >>= 1)
            {
                v += __shfl_xor_sync(0xFFFFFFFFu, v, off);
                i2 += __shfl_xor_sync(0xFFFFFFFFu, i2, off);
            }
            if (threadIdx.x == 0)
            {
                if (v != 0.0) atomicAdd(&sums[0], v);
                if (i2 != 0.0) atomicAdd(&sums[1], i2);
            }
        }

        // ------------------------------------------------------------------------------------------ denoising planes
        // Each pass's tap weights are computed once, on the beauty frame, and applied to every plane. taps holds them
        // [tap][half][pixel] (tap = 5 ky + kx), so a warp's loads of one tap are 32 consecutive doubles; a tap that
        // k_denoise_atrous skips, and every tap of an invalid pixel, is 0.

        // k_denoise_atrous, which it must equal bit for bit (same operations in the same order), plus the tap weights
        __global__ void __launch_bounds__(BX * BY) k_denoise_atrous_weights(uint32_t width, uint32_t height, uint32_t step, DenoiseSigmas sg,
                                                                            const Guide* __restrict__ guide, const State* __restrict__ src,
                                                                            State* __restrict__ dst, double* __restrict__ taps)
        {
            const uint32_t x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
            if (x >= width || y >= height) return;
            const size_t i = (size_t)y * width + x, n = (size_t)width * height;
            const Guide gp = guide[i];
            const State sp = src[i];
            if (gp.flag == GUIDE_INVALID)
            {
                dst[i] = sp;
                for (int t = 0; t < 50; t++) taps[t * n + i] = 0.0;
                return;
            }
            double acc_a[3] = { 0.0, 0.0, 0.0 }, acc_b[3] = { 0.0, 0.0, 0.0 };
            double wsum_a = 0.0, wsum_b = 0.0, vsum_a = 0.0, vsum_b = 0.0;
            for (int ky = 0; ky < 5; ky++)
            {
                const long long qy = (long long)y + (long long)(ky - 2) * step;
                if (qy < 0 || qy >= (long long)height)
                {
                    for (int kx = 0; kx < 5; kx++) { taps[2 * (5 * ky + kx) * n + i] = 0.0; taps[(2 * (5 * ky + kx) + 1) * n + i] = 0.0; }
                    continue;
                }
                for (int kx = 0; kx < 5; kx++)
                {
                    double* ta = taps + 2 * (5 * ky + kx) * n + i;   // wa; wb at ta[n]
                    const long long qx = (long long)x + (long long)(kx - 2) * step;
                    if (qx < 0 || qx >= (long long)width) { ta[0] = 0.0; ta[n] = 0.0; continue; }
                    const size_t q = (size_t)qy * width + (size_t)qx;
                    const double hw = binomial5(ky) * binomial5(kx);
                    double wa = hw, wb = hw;
                    const State sq = src[q];
                    if (q != i)
                    {
                        const Guide gq = guide[q];
                        if (gq.flag == GUIDE_INVALID) { ta[0] = 0.0; ta[n] = 0.0; continue; }
                        double wf = 1.0;
                        if (gp.flag != gq.flag) wf = 0.0;   // background against surface
                        else if (gp.flag == GUIDE_SURFACE)
                        {
                            if (sg.normal != 0.0)
                                wf *= pow(fmax(0.0, gp.n[0] * gq.n[0] + gp.n[1] * gq.n[1] + gp.n[2] * gq.n[2]), sg.normal);
                            if (sg.depth != 0.0)
                                wf *= exp(-fabs(gp.z - gq.z) / (sg.depth * fmax(gp.z, gq.z)));
                            if (sg.albedo != 0.0)
                            {
                                double d2 = 0.0;
                                for (int c = 0; c < 3; c++) { const double d = gp.albedo[c] - gq.albedo[c]; d2 += d * d; }
                                wf *= exp(-d2 / (sg.albedo * sg.albedo));
                            }
                        }
                        if (wf == 0.0) { ta[0] = 0.0; ta[n] = 0.0; continue; }
                        double d2a = 0.0, d2b = 0.0;
                        for (int c = 0; c < 3; c++)
                        {
                            const double da = sp.a[c] - sq.a[c], db = sp.b[c] - sq.b[c];
                            d2a += da * da; d2b += db * db;
                        }
                        wa = hw * wf * colorWeight(d2b / 3.0, sp.var_b + sq.var_b, sg.color);
                        wb = hw * wf * colorWeight(d2a / 3.0, sp.var_a + sq.var_a, sg.color);
                    }
                    ta[0] = wa; ta[n] = wb;
                    for (int c = 0; c < 3; c++) { acc_a[c] += wa * sq.a[c]; acc_b[c] += wb * sq.b[c]; }
                    wsum_a += wa; wsum_b += wb;
                    vsum_a += wa * wa * sq.var_a; vsum_b += wb * wb * sq.var_b;
                }
            }
            State o;
            for (int c = 0; c < 3; c++) { o.a[c] = acc_a[c] / wsum_a; o.b[c] = acc_b[c] / wsum_b; }
            o.var_a = vsum_a / (wsum_a * wsum_a);
            o.var_b = vsum_b / (wsum_b * wsum_b);
            dst[i] = o;
        }

        // Plane states are the per-half means, a [n_planes][pixel][3] and b alike.
        struct PlaneSet
        {
            double* a;
            double* b;
        };

        // means S_X / w_X of every plane, as k_denoise_prep takes the beauty's; 0 at invalid pixels, which no pass reads
        __global__ void __launch_bounds__(BX * BY) k_denoise_planes_prep(DenoiseInput in, const double* __restrict__ a,
                                                                         const double* __restrict__ b, uint32_t n_planes, PlaneSet dst)
        {
            const uint32_t x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
            if (x >= in.width || y >= in.height) return;
            const size_t i = (size_t)y * in.width + x, n = (size_t)in.width * in.height;
            double wa, wb;
            halfWeights(in, x, y, i, wa, wb);
            const bool valid = wa != 0.0 && wb != 0.0;
            for (uint32_t k = blockIdx.z; k < n_planes; k += gridDim.z)
            {
                const size_t o = 3 * ((size_t)k * n + i);
                for (int c = 0; c < 3; c++)
                {
                    dst.a[o + c] = valid ? a[o + c] / wa : 0.0;
                    dst.b[o + c] = valid ? b[o + c] / wb : 0.0;
                }
            }
        }

        // One pass over planes [C z, C z + C) for each z: X' = sum w X_q / sum w with the beauty pass's tap weights,
        // summed in its tap order, so that a plane equal to the beauty gets its values exactly. A thread's C planes share
        // each weight it loads.
        template <int C>
        __global__ void __launch_bounds__(BX * BY) k_denoise_atrous_planes(uint32_t width, uint32_t height, uint32_t step, uint32_t n_planes,
                                                                           const double* __restrict__ taps, PlaneSet src, PlaneSet dst)
        {
            const uint32_t x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
            if (x >= width || y >= height) return;
            const size_t i = (size_t)y * width + x, n = (size_t)width * height;
            const uint32_t n_chunks = (n_planes + C - 1) / C;
            // the centre tap's weight is h(2)^2 > 0 at every valid pixel; an invalid pixel is no tap's neighbour, and
            // k_denoise_planes_final gives it its input sums, so its state is never read
            if (taps[2 * 12 * n + i] == 0.0) return;
            for (uint32_t z = blockIdx.z; z < n_chunks; z += gridDim.z)
            {
                const uint32_t k0 = z * C;
                double acc_a[C][3], acc_b[C][3];
#pragma unroll
                for (int k = 0; k < C; k++)
                    for (int c = 0; c < 3; c++) { acc_a[k][c] = 0.0; acc_b[k][c] = 0.0; }
                double wsum_a = 0.0, wsum_b = 0.0;
                for (int ky = 0; ky < 5; ky++)
                {
                    for (int kx = 0; kx < 5; kx++)
                    {
                        const double* ta = taps + 2 * (5 * ky + kx) * n + i;
                        const double wa = ta[0], wb = ta[n];
                        if (wa == 0.0 && wb == 0.0) continue;   // outside the image, invalid or cut by the guides
                        const size_t q = (size_t)((long long)y + (long long)(ky - 2) * step) * width +
                                         (size_t)((long long)x + (long long)(kx - 2) * step);
#pragma unroll
                        for (int k = 0; k < C; k++)
                        {
                            if (k0 + k >= n_planes) break;
                            const size_t o = 3 * ((size_t)(k0 + k) * n + q);
                            for (int c = 0; c < 3; c++) { acc_a[k][c] += wa * src.a[o + c]; acc_b[k][c] += wb * src.b[o + c]; }
                        }
                        wsum_a += wa; wsum_b += wb;
                    }
                }
#pragma unroll
                for (int k = 0; k < C; k++)
                {
                    if (k0 + k >= n_planes) break;
                    const size_t o = 3 * ((size_t)(k0 + k) * n + i);
                    for (int c = 0; c < 3; c++) { dst.a[o + c] = acc_a[k][c] / wsum_a; dst.b[o + c] = acc_b[k][c] / wsum_b; }
                }
            }
        }

        // in place: the filtered means become sums w_X X~ in the input's layout; an invalid pixel keeps its input sums
        __global__ void __launch_bounds__(BX * BY) k_denoise_planes_final(DenoiseInput in, const double* __restrict__ a,
                                                                          const double* __restrict__ b, uint32_t n_planes, PlaneSet out)
        {
            const uint32_t x = blockIdx.x * BX + threadIdx.x, y = blockIdx.y * BY + threadIdx.y;
            if (x >= in.width || y >= in.height) return;
            const size_t i = (size_t)y * in.width + x, n = (size_t)in.width * in.height;
            double wa, wb;
            halfWeights(in, x, y, i, wa, wb);
            const bool valid = wa != 0.0 && wb != 0.0;
            for (uint32_t k = blockIdx.z; k < n_planes; k += gridDim.z)
            {
                const size_t o = 3 * ((size_t)k * n + i);
                for (int c = 0; c < 3; c++)
                {
                    out.a[o + c] = valid ? wa * out.a[o + c] : a[o + c];
                    out.b[o + c] = valid ? wb * out.b[o + c] : b[o + c];
                }
            }
        }
    }

    size_t denoiseScratchValues(size_t n_pixels)
    {
        static_assert(sizeof(State) == 8 * sizeof(double) && sizeof(Guide) == 8 * sizeof(double), "scratch layout");
        return 3 * 8 * n_pixels;   // two states (ping-pong) and the guides
    }

    void launchDenoise(const DenoiseInput& in, const DenoiseSigmas& sigma, uint32_t iterations, double* scratch, double* out,
                       double* sums, cudaStream_t s)
    {
        const size_t n = (size_t)in.width * in.height;
        State* state[2] = { reinterpret_cast<State*>(scratch), reinterpret_cast<State*>(scratch + 8 * n) };
        Guide* guide = reinterpret_cast<Guide*>(scratch + 16 * n);
        const dim3 block(BX, BY), grid((in.width + BX - 1) / BX, (in.height + BY - 1) / BY);
        k_denoise_prep<<<grid, block, 0, s>>>(in, state[0], guide);
        int cur = 0;
        for (uint32_t k = 0; k < iterations; k++, cur ^= 1)
            k_denoise_atrous<<<grid, block, 0, s>>>(in.width, in.height, 1u << k, sigma, guide, state[cur], state[cur ^ 1]);
        k_denoise_final<<<grid, block, 0, s>>>(in, guide, state[cur], out, sums);
    }

    size_t denoisePlanesScratchValues(size_t n_pixels, uint32_t n_planes)
    {
        return 50 * n_pixels + 6 * n_pixels * n_planes;   // the tap weights, then one plane state set
    }

    void launchDenoisePlanes(const DenoiseInput& in, const DenoisePlanes& planes, const DenoiseSigmas& sigma, uint32_t iterations,
                             double* scratch, double* planes_scratch, double* out, double* sums, cudaStream_t s)
    {
        const size_t n = (size_t)in.width * in.height;
        State* state[2] = { reinterpret_cast<State*>(scratch), reinterpret_cast<State*>(scratch + 8 * n) };
        Guide* guide = reinterpret_cast<Guide*>(scratch + 16 * n);
        double* taps = planes_scratch;
        // the plane passes ping-pong between the scratch set and the caller's buffers, starting where the last lands in them
        PlaneSet set[2] = { { planes_scratch + 50 * n, planes_scratch + 50 * n + 3 * n * planes.n },
                            { planes.a_out, planes.b_out } };
        int pc = iterations % 2 == 0 ? 1 : 0;
        constexpr uint32_t MAX_Z = 65535;
        const uint32_t chunks = (planes.n + DENOISE_PLANE_CHUNK - 1) / DENOISE_PLANE_CHUNK;
        const dim3 block(BX, BY), grid((in.width + BX - 1) / BX, (in.height + BY - 1) / BY);
        const dim3 plane_grid(grid.x, grid.y, planes.n < MAX_Z ? planes.n : MAX_Z);
        const dim3 chunk_grid(grid.x, grid.y, chunks < MAX_Z ? chunks : MAX_Z);
        k_denoise_prep<<<grid, block, 0, s>>>(in, state[0], guide);
        k_denoise_planes_prep<<<plane_grid, block, 0, s>>>(in, planes.a, planes.b, planes.n, set[pc]);
        int cur = 0;
        for (uint32_t k = 0; k < iterations; k++, cur ^= 1, pc ^= 1)
        {
            k_denoise_atrous_weights<<<grid, block, 0, s>>>(in.width, in.height, 1u << k, sigma, guide, state[cur], state[cur ^ 1], taps);
            k_denoise_atrous_planes<DENOISE_PLANE_CHUNK><<<chunk_grid, block, 0, s>>>(in.width, in.height, 1u << k, planes.n, taps, set[pc],
                                                                                       set[pc ^ 1]);
        }
        k_denoise_planes_final<<<plane_grid, block, 0, s>>>(in, planes.a, planes.b, planes.n, set[1]);
        if (out) k_denoise_final<<<grid, block, 0, s>>>(in, guide, state[cur], out, sums);
    }
}
