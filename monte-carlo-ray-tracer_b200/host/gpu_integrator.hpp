// GpuPathTracer / GpuPhotonMapper: the reference-side adapters that put the GPU path behind the
// reference's own Integrator interface (source/integrator/integrator.hpp:7-30).
//
//   Camera camera(j, option);                       // unchanged reference code: loads the Scene,
//                                                   // builds the BVH (+ photon maps) on the CPU
//   mcrt_host::GpuRenderer gpu(camera);             // flattens + uploads what the reference built
//   gpu.sampleImage(camera);                        // replaces Camera::sampleImage (camera.cpp:101-145)
//   camera.saveImage();                             // unchanged: exposure, tonemap, TGA
//
// Compiled with -fno-access-control against the reference headers (Camera::integrator, Camera::film
// and Sampler::global_seed are private there).
#pragma once

#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "mcrt_abi.h"
#include "exporter.hpp"

class Camera;

namespace mcrt_host
{
    // The scene JSON's "bvh" object (bvh.cpp:24-56) when the hierarchy is to be built on the GPU:
    // construct the reference's Scene from a JSON with "bvh" erased (no CPU build) and pass this.
    struct GpuBvh
    {
        int type = MCRT_BVH_OCTREE;     // MCRT_BVH_*
        int bins_per_axis = 0;          // <= 0: the reference's default for the type
        static GpuBvh fromTypeName(std::string type, int bins_per_axis);
    };

    class GpuRenderer
    {
    public:
        // Takes the Scene (and photon maps, if the camera was built with a PhotonMapper) that the
        // reference constructed and uploads them to CUDA device `device`.
        // gpu_bvh: build the BVH with mcrt_bvh_build instead of taking the one the reference built
        // (the Scene must then have none).
        explicit GpuRenderer(const Camera& camera, int device = 0, int precision = MCRT_PRECISION_F64,
                             const GpuBvh* gpu_bvh = nullptr);
        ~GpuRenderer();
        GpuRenderer(const GpuRenderer&) = delete;
        GpuRenderer& operator=(const GpuRenderer&) = delete;

        // Camera::sampleImage: renders every row and stores Film::scan-equivalent values in
        // camera.image(x, y), through the camera's own Film filter (mcrt_set_film).
        void sampleImage(Camera& camera);

        // First pass of PhotonMapper::PhotonMapper (photon-mapper.cpp:24-277) on the GPU instead of the CPU:
        // photon emission and both photon octrees (mcrt_photon_emit). The camera is built WITHOUT photon
        // mapping (a PathTracer, so the reference runs no CPU pass); afterwards this renderer renders
        // photon-mapped. Arguments = the scene JSON's "photon_map" object (photon-mapper.cpp:28-36).
        void emitPhotons(const Camera& camera, uint64_t emissions, double caustic_factor, uint32_t max_photons_per_octree_leaf = 200,
                         uint32_t k_nearest_photons = 50, bool direct_visualization = false);

        // Camera::saveImage / Image::save (image.cpp:37-51) with exposure, tone mapping, gain, gamma and
        // byte conversion on the GPU (mcrt_image_tonemap); writes camera.savename + ".tga".
        void saveImage(const Camera& camera);

        // Rows [y0, y1) as float64 RGB, row-major.
        std::vector<double> renderRows(const Camera& camera, uint32_t y0, uint32_t y1);

        // Batched Integrator::sampleRay: ray i is sample `sample[i]` of pixel `pixel[i]`.
        std::vector<double> sampleRays(const std::vector<mcrt_ray>& rays, const std::vector<uint32_t>& pixel,
                                       const std::vector<uint32_t>& sample);

        const mcrt_stats& lastStats() const { return stats_; }
        uint64_t uploadedBytes() const { return h2d_bytes_; }
        double bvhBuildMs() const { return bvh_build_ms_; }   // device time of mcrt_bvh_build (0: not used)

    private:
        void check(int rc, const char* what) const;

        mcrt_ctx* ctx_ = nullptr;
        int precision_;
        int integrator_kind_;
        uint32_t global_seed_;
        mcrt_stats stats_{};
        uint64_t h2d_bytes_ = 0;
        double bvh_build_ms_ = 0.0;
    };
}
