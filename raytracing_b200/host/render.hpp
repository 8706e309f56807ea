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
    // emitter sampling (CUDAPathTraceIntegrator::SetEmitterSampling): applies from the next RenderFrame(), keeps the accumulation
    void SetEmitterSampling(bool on) { Cuda().SetEmitterSampling(on); }
    // object motion vectors (CUDAPathTraceIntegrator::SetObjectMotion): AOV view 4 and the temporal denoiser follow UpdateTriangles
    void SetObjectMotion(bool on) { Cuda().SetObjectMotion(on); }
    // environment sampling and light-kind weights (CUDAPathTraceIntegrator): apply from the next RenderFrame(), keep the accumulation
    void SetEnvironmentSampling(bool on) { Cuda().SetEnvironmentSampling(on); }
    void SetLightSelection(float analytic, float emitters, float environment) { Cuda().SetLightSelection(analytic, emitters, environment); }
    // geometry update (CUDAPathTraceIntegrator::UpdateTriangles): the scene's triangles in leaf order, moved; the next RenderFrame()
    // renders them into the same accumulation unless the caller calls NotifyCameraChanged()
    void UpdateTriangles(const Triangle* triangles, size_t count) { Cuda().UpdateTriangles(triangles, count); }
    // BVH rebuild (CUDAPathTraceIntegrator::RebuildBvh): a device-built tree over the current triangles; returns its node count.
    // Keeps the accumulation, as above
    using BvhBuild = CUDAPathTraceIntegrator::BvhBuild;
    std::uint64_t RebuildBvh(BvhBuild build = BvhBuild::kLinear) { return Cuda().RebuildBvh(build); }
    // instanced scene (CUDAPathTraceIntegrator::UploadInstancedScene / SetInstances): shared meshes in place of the scene's
    // triangles, with the scene's materials, lights and environment; then the instance list
    void UploadInstancedScene(const RtTriangle* triangles, size_t n_triangles, const RtLinearBVHNode* nodes, size_t n_nodes,
                              const RtMeshDesc* meshes, std::uint32_t n_meshes)
    {
        Cuda().UploadInstancedScene(scene_, triangles, n_triangles, nodes, n_nodes, meshes, n_meshes);
    }
    void SetInstances(const RtInstance* instances, std::uint32_t count) { Cuda().SetInstances(instances, count); }
    // mesh update in an instanced scene (CUDAPathTraceIntegrator::UpdateMeshTriangles); keeps the accumulation, as UpdateTriangles
    void UpdateMeshTriangles(std::uint32_t mesh, const RtTriangle* triangles, size_t count) { Cuda().UpdateMeshTriangles(mesh, triangles, count); }
    // per-instance materials (CUDAPathTraceIntegrator::SetInstanceMaterials); keeps the accumulation, as SetInstances
    void SetInstanceMaterials(const std::uint32_t* remaps, std::uint32_t n_remaps, const std::uint32_t* remap_of_instance, std::uint32_t n_instances)
    {
        Cuda().SetInstanceMaterials(remaps, n_remaps, remap_of_instance, n_instances);
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
