// Random-gather bandwidth probe (built and run by tools/gather_probe.py).
//
// The wavefront kernels read their queues through a sort permutation, so every record they read is at a
// random position in a multi-GB array. This times warp-wide random gathers of one record per lane, with the
// same 128-bit evict-first loads (ld.global.cs) that ldStream uses, over a buffer far larger than L2:
//   rec S    one S-byte record per gather, S = 16, 32, 64, 128
//   soa5     one path's state in the old structure-of-arrays layout: five separate reads of 32+32+32+16+16 B
//   aos128   the same 128 B as one aligned record
// and prints one JSON line per case: useful GB/s (bytes the kernel asked for) and records per second.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ uint64_t mix64(uint64_t x)
{
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}

// VEC 128-bit loads from one record of VEC*16 bytes
template <int VEC>
__global__ void __launch_bounds__(256) k_gather(const uint4* base, uint64_t n_records, uint64_t n_gathers, uint32_t seed, uint4* sink)
{
    uint32_t acc = 0;
    for (uint64_t g = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; g < n_gathers; g += (uint64_t)gridDim.x * blockDim.x)
    {
        const uint64_t r = mix64(g * 0x9E3779B97F4A7C15ull + seed) % n_records;
        const uint4* p = base + r * VEC;
        #pragma unroll
        for (int k = 0; k < VEC; k++) { const uint4 v = __ldcs(p + k); acc ^= v.x ^ v.y ^ v.z ^ v.w; }
    }
    if (acc == 0x12345678u) sink[0] = make_uint4(acc, 0, 0, 0);   // keeps the loads alive
}

// the old path-state layout: five arrays, 2/2/2/1/1 128-bit loads per path at the same random index
__global__ void __launch_bounds__(256) k_gather_soa5(const uint4* base, uint64_t n_records, uint64_t n_gathers, uint32_t seed, uint4* sink)
{
    const uint4* a0 = base;                  // 32 B per path
    const uint4* a1 = a0 + 2 * n_records;    // 32 B
    const uint4* a2 = a1 + 2 * n_records;    // 32 B
    const uint4* a3 = a2 + 2 * n_records;    // 16 B
    const uint4* a4 = a3 + n_records;        // 16 B
    uint32_t acc = 0;
    for (uint64_t g = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; g < n_gathers; g += (uint64_t)gridDim.x * blockDim.x)
    {
        const uint64_t r = mix64(g * 0x9E3779B97F4A7C15ull + seed) % n_records;
        uint4 v[8];
        v[0] = __ldcs(a0 + 2 * r); v[1] = __ldcs(a0 + 2 * r + 1);
        v[2] = __ldcs(a1 + 2 * r); v[3] = __ldcs(a1 + 2 * r + 1);
        v[4] = __ldcs(a2 + 2 * r); v[5] = __ldcs(a2 + 2 * r + 1);
        v[6] = __ldcs(a3 + r); v[7] = __ldcs(a4 + r);
        #pragma unroll
        for (int k = 0; k < 8; k++) acc ^= v[k].x ^ v[k].y ^ v[k].z ^ v[k].w;
    }
    if (acc == 0x12345678u) sink[0] = make_uint4(acc, 0, 0, 0);
}

typedef void (*Kern)(const uint4*, uint64_t, uint64_t, uint32_t, uint4*);

int main(int argc, char** argv)
{
    const double gib = argc > 1 ? atof(argv[1]) : 16.0;
    const int reps = argc > 2 ? atoi(argv[2]) : 20;
    const uint64_t bytes = (uint64_t)(gib * 1073741824.0) & ~(uint64_t)127;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    uint4* buf = nullptr; uint4* sink = nullptr;
    CK(cudaMalloc(&buf, bytes));
    CK(cudaMalloc(&sink, sizeof(uint4)));
    CK(cudaMemset(buf, 1, bytes));
    const int grid = prop.multiProcessorCount * 8;
    const uint64_t n_gathers = 1ull << 26;   // 64 Mi records per launch (0.5 s of work at most)
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));

    struct Case { const char* name; Kern k; int bytes; };
    const Case cases[] = {
        { "rec16", k_gather<1>, 16 }, { "rec32", k_gather<2>, 32 }, { "rec64", k_gather<4>, 64 }, { "rec128", k_gather<8>, 128 },
        { "soa5_128", k_gather_soa5, 128 }, { "aos128", k_gather<8>, 128 },
    };
    for (const Case& c : cases)
    {
        const uint64_t n_records = bytes / (uint64_t)c.bytes;
        for (int w = 0; w < 3; w++) c.k<<<grid, 256>>>(buf, n_records, n_gathers, 1000u + w, sink);
        CK(cudaEventRecord(e0));
        for (int r = 0; r < reps; r++) c.k<<<grid, 256>>>(buf, n_records, n_gathers, (uint32_t)r, sink);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaGetLastError());
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        const double recs = (double)n_gathers * reps, s = ms * 1e-3;
        printf("{\"case\": \"%s\", \"record_bytes\": %d, \"array_gib\": %.2f, \"launches\": %d, \"ms_per_launch\": %.3f, "
               "\"useful_gbs\": %.1f, \"grecords_per_s\": %.3f, \"device\": \"%s\"}\n",
               c.name, c.bytes, bytes / 1073741824.0, reps, ms / reps, recs * c.bytes / s / 1e9, recs / s / 1e9, prop.name);
    }
    CK(cudaFree(buf)); CK(cudaFree(sink));
    return 0;
}
