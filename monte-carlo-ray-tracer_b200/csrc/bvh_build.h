// BVH construction on the device (widened scope, SURVEY.md §8f-2). See bvh_build.cu.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "photon.cuh"

namespace mcrt
{
    struct BvhBuildResult
    {
        // BVH::linear_tree in depth-first order (bvh.hpp:68-82) + BVH::ordered_surfaces as indices
        // into the caller's primitive array
        std::vector<double> node_bounds;
        std::vector<uint32_t> node_first_prim, node_prim_count, node_next_sibling, prim_order;
        double gpu_ms = 0.0;          // first kernel to last kernel, copies of the result excluded
        uint32_t iterations = 0;      // breadth-first build rounds
        uint32_t kernel_launches = 0;
    };

    // LinearOctree<Photon> built on the device, in the layout k_knn walks; memory is pushed to `keep`
    struct PhotonOctreeDevice
    {
        const DeviceOctant* octants = nullptr;
        const uint32_t* next_sibling = nullptr;   // LinearOctant::next_sibling (OCTANT_NULL terminated), for downloads
        const float4* photons = nullptr;          // LinearOctree::ordered_data, 2 float4 per photon
        const uint32_t* lights = nullptr;         // the emitting light of each photon, in the same order (built with lights only)
        const uint32_t* lpe_states = nullptr;     // the reverse-DFA state of each photon, in the same order (built with states only)
        uint32_t n_octants = 0, rounds = 0;
        uint64_t n_photons = 0;
        double gpu_ms = 0.0;
    };

    // d_photons: device, 2 float4 per photon as k_emit_shade stores them; cell: the root Octree box;
    // d_lights / d_lpe_states: null, or device, the emitting light / reverse-DFA state of each photon (k_emit_shade),
    // reordered with the photons
    int buildPhotonOctreeOnDevice(const float4* d_photons, uint32_t n_photons, const double cell[6], uint32_t max_node_data,
                                  int sm_count, cudaStream_t stream, std::vector<void*>& keep, PhotonOctreeDevice& out,
                                  std::string& error, const uint32_t* d_lights = nullptr, const uint32_t* d_lpe_states = nullptr);

    // type: MCRT_BVH_*; returns an mcrt_status code, message in `error`
    int buildBvhOnDevice(const double* prim_bounds_host, uint32_t n_prims, const double scene_bounds[6], int type,
                         int bins_per_axis, int sm_count, cudaStream_t stream, BvhBuildResult& out, std::string& error);
}
