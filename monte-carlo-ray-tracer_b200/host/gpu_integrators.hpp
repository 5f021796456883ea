// GpuPathTracer / GpuPhotonMapper: the GPU path behind the reference's own Integrator interface
// (source/integrator/integrator.hpp:7-30). They are drop-in replacements for the objects Camera::Camera
// creates at source/camera/camera.cpp:22-29:
//
//     integrator = std::make_shared<GpuPathTracer>(j);      // instead of std::make_shared<PathTracer>(j)
//     integrator = std::make_shared<GpuPhotonMapper>(j);    // instead of std::make_shared<PhotonMapper>(j)
//
// The base-class constructor Integrator(j) is the reference's: it loads the Scene and builds the BVH
// on the CPU, unchanged. The derived constructor flattens what was built (exporter.cpp) and uploads it
// (mcrt_scene_upload); GpuPhotonMapper then runs the photon pass on the GPU (mcrt_photon_emit) with
// the parameters of the scene's "photon_map" object (photon-mapper.cpp:28-36).
//
// sampleRay(Ray) keeps the reference's one-ray-per-call contract by forwarding a batch of one through
// mcrt_sample_rays. The sampler state the reference keeps thread_local (sampler.hpp:55: which pixel,
// which sample) is read back from it: base_seed = hashCombine(global_seed, hash(pixel)) is inverted
// (both hashes are bijections), the sample index is the bit-reversed `bit_reversed_index`. One ray per
// launch cannot feed a GPU - it is the compatibility path; renders go through sampleRows(), the
// batched body of Camera::sampleImage (GpuRenderer in gpu_integrator.hpp wraps it for whole frames).
//
// Compiled with -fno-access-control against the reference headers (Sampler's state is private).
#pragma once

#include <cstdint>
#include <mutex>
#include <vector>

#include <nlohmann/json.hpp>

#include "integrator/integrator.hpp"

#include "mcrt_abi.h"

class Camera;

namespace mcrt_host
{
    // (pixel, sample) of the calling thread's Sampler, as set by Sampler::initiate / setIndex
    void currentSamplerPixelAndSample(uint32_t& pixel, uint32_t& sample);
}

class GpuPathTracer : public Integrator
{
public:
    explicit GpuPathTracer(const nlohmann::json& j, int device = 0, int precision = MCRT_PRECISION_F64);
    ~GpuPathTracer() override;
    GpuPathTracer(const GpuPathTracer&) = delete;
    GpuPathTracer& operator=(const GpuPathTracer&) = delete;

    // Integrator::sampleRay for the camera ray of the sample the calling thread's Sampler is set to
    glm::dvec3 sampleRay(Ray ray) override;

    // Batched: rows [y0, y1) of `camera` (Camera::sampleImage's body for those rows), float64 RGB row-major
    std::vector<double> sampleRows(const Camera& camera, uint32_t y0, uint32_t y1);

    const mcrt_stats& lastStats() const { return stats_; }
    mcrt_ctx* context() { return ctx_; }

protected:
    void check(int rc, const char* what) const;

    mcrt_ctx* ctx_ = nullptr;
    int precision_;
    int kind_ = MCRT_INTEGRATOR_PATH;
    mcrt_stats stats_{};
    std::mutex mutex_;    // the reference calls sampleRay from num_threads threads; a context is single-threaded
};

class GpuPhotonMapper : public GpuPathTracer
{
public:
    explicit GpuPhotonMapper(const nlohmann::json& j, int device = 0, int precision = MCRT_PRECISION_F64);
    uint64_t causticPhotons() const { return n_caustic_; }
    uint64_t globalPhotons() const { return n_global_; }

private:
    uint64_t n_caustic_ = 0, n_global_ = 0;
};
