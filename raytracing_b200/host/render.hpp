/*
 * Headless mirror of the reference's Render (/root/reference/src/render.hpp:37-94, render.cpp:38-204):
 * owns the acceleration structure, the integrator, the camera and the frame image; the backend is picked
 * from RenderBackend exactly where the reference switches between OpenCL and OpenGL (render.cpp:70-79) —
 * kCUDA is the new arm.  Window, GUI, GL framebuffer and kernel hot-reload are out of scope; RenderFrame()
 * is the reference's RenderFrame minus presentation: SetCameraData, RequestReset if the camera moved,
 * Integrate.
 */
#pragma once

#include <memory>
#include <vector>

#include "bvh.hpp"
#include "camera_controller.hpp"
#include "cuda_pt_integrator.hpp"
#include "reference_api.hpp"

namespace rt_host
{

class Render
{
public:
    enum class RenderBackend { kOpenCL, kOpenGL, kCUDA };

    Render(std::uint32_t width, std::uint32_t height, RenderBackend backend, Scene& scene,
           const char* env_map_path = "assets/ibl/CGSkies_0036_free.hdr", int device = 0);
    // kCUDA over several devices of the node (empty list = all of them): one integrator, the image partitioned by scanline
    Render(std::uint32_t width, std::uint32_t height, RenderBackend backend, Scene& scene,
           const char* env_map_path, std::vector<int> const& devices);
    // headless: the environment image is handed over decoded (RGBA32F rows) instead of being read from an .hdr file
    Render(std::uint32_t width, std::uint32_t height, RenderBackend backend, Scene& scene,
           Image const& env_image, std::vector<int> const& devices);

    void RenderFrame();
    Integrator& GetIntegrator() { return *integrator_; }
    CameraController& GetCamera() { return *camera_controller_; }
    AccelerationStructure& GetAccelerationStructure() { return *acc_structure_; }
    std::vector<float> const& GetImage() const { return image_; }     // resolved RGBA32F, width*height
    void SetMaxBounces(std::uint32_t b) { integrator_->SetMaxBounces(b); }
    // progressive samples accumulated by one RenderFrame() (CUDAPathTraceIntegrator::SetSamplesPerFrame), default 1
    void SetSamplesPerFrame(std::uint32_t n) { Cuda().SetSamplesPerFrame(n); }
    // adaptive sampling (CUDAPathTraceIntegrator::SetAdaptiveSampling): applies from the next RenderFrame(), which starts over
    void SetAdaptiveSampling(float max_error, std::uint32_t min_samples) { Cuda().SetAdaptiveSampling(max_error, min_samples); }
    // spatial denoiser (CUDAPathTraceIntegrator::SetSpatialDenoiser): filters the image of every later RenderFrame()
    void SetSpatialDenoiser(std::uint32_t iterations, float sigma_color, float sigma_normal, float sigma_depth)
    {
        Cuda().SetSpatialDenoiser(iterations, sigma_color, sigma_normal, sigma_depth);
    }
    std::uint32_t ActivePixels() const { return static_cast<CUDAPathTraceIntegrator const&>(*integrator_).ActivePixels(); }
    void NotifyCameraChanged() { camera_changed_ = true; }

private:
    CUDAPathTraceIntegrator& Cuda() { return static_cast<CUDAPathTraceIntegrator&>(*integrator_); }
    void Init(RenderBackend backend, const char* env_map_path, const Image* env_image, const std::vector<int>* devices, int device);
    Scene& scene_;
    std::uint32_t width_, height_;
    std::unique_ptr<Integrator> integrator_;
    std::unique_ptr<AccelerationStructure> acc_structure_;
    std::unique_ptr<CameraController> camera_controller_;
    std::vector<float> image_;
    bool camera_changed_ = true;
};

} // namespace rt_host
