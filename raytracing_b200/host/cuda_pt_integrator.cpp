#include "cuda_pt_integrator.hpp"

#include <stdexcept>

#include "reference_api.hpp"

namespace rt_host
{

void CUDAPathTraceIntegrator::Check(int status, const char* what) const
{
    if (status != RT_OK)
        throw std::runtime_error(std::string(what) + ": " + rt_last_error(ctx_) + " (status " + std::to_string(status) + ")");
}

CUDAPathTraceIntegrator::CUDAPathTraceIntegrator(std::uint32_t width, std::uint32_t height, AccelerationStructure& acc_structure,
                                                 int device, Schedule schedule)
    : Integrator(width, height, acc_structure), schedule_(schedule)
{
    int status = rt_create(width, height, device, &ctx_);
    if (status != RT_OK)
        throw std::runtime_error(std::string("Failed to create the CUDA path tracing context: ") + rt_last_error(nullptr));
    CreateKernels();
    Reset();            // "Don't forget to reset frame index", cl_pt_integrator.cpp:257-258
}

CUDAPathTraceIntegrator::CUDAPathTraceIntegrator(std::uint32_t width, std::uint32_t height, AccelerationStructure& acc_structure,
                                                 std::vector<int> const& devices, Schedule schedule)
    : Integrator(width, height, acc_structure), schedule_(schedule)
{
    std::vector<int> list = devices;
    if (list.empty())
    {
        int n = 0;
        rt_device_count(&n);
        for (int i = 0; i < n; ++i) list.push_back(i);
    }
    int status = list.empty() ? RT_ERR_NO_DEVICE : rt_create_multi(width, height, list.data(), (std::uint32_t)list.size(), &ctx_);
    if (status != RT_OK)
        throw std::runtime_error(std::string("Failed to create the CUDA path tracing context: ") + (list.empty() ? "no CUDA device" : rt_last_error(nullptr)));
    CreateKernels();
    Reset();
}

CUDAPathTraceIntegrator::~CUDAPathTraceIntegrator()
{
    if (resolve_target_ && resolve_target_locked_) rt_host_unregister(resolve_target_);
    if (ctx_) rt_destroy(ctx_);
}

void CUDAPathTraceIntegrator::SetResolveTarget(float* host_rgba, bool page_lock)
{
    if (resolve_target_ && resolve_target_locked_) rt_host_unregister(resolve_target_);
    resolve_target_ = host_rgba;
    resolve_target_locked_ = host_rgba && page_lock && rt_host_register(host_rgba, (std::uint64_t)width_ * height_ * 16) == RT_OK;
}

// Kernel variants are compiled ahead of time for sm_90a (there is no runtime compilation / hot reload,
// cl_context.cpp:173-210); "creating the kernels" pushes the current option set to the context.
void CUDAPathTraceIntegrator::CreateKernels()
{
    Check(rt_set_option(ctx_, RT_OPT_WHITE_FURNACE, enable_white_furnace_ ? 1u : 0u), "EnableWhiteFurnace");
    Check(rt_set_option(ctx_, RT_OPT_SAMPLER, sampler_type_ == SamplerType::kBlueNoise ? 1u : 0u), "SetSamplerType");
    Check(rt_set_option(ctx_, RT_OPT_DENOISER, enable_denoiser_ ? 1u : 0u), "EnableDenoiser");
}

void CUDAPathTraceIntegrator::UploadGPUData(Scene const& scene, AccelerationStructure const& acc_structure)
{
    RtSceneDesc d = {};
    d.triangles = scene.GetTriangles().data();          d.n_triangles = scene.GetTriangles().size();
    d.nodes = acc_structure.GetNodes().data();          d.n_nodes = acc_structure.GetNodes().size();
    d.materials = scene.GetMaterials().data();          d.n_materials = scene.GetMaterials().size();
    d.lights = scene.GetLights().data();                d.n_lights = scene.GetLights().size();
    d.textures = scene.GetTextures().data();            d.n_textures = scene.GetTextures().size();
    d.texture_data = scene.GetTextureData().data();     d.n_texture_data = scene.GetTextureData().size();
    d.emissive_indices = scene.GetEmissiveIndices().data(); d.n_emissive = scene.GetEmissiveIndices().size();
    d.env_image = scene.GetEnvImage().data.data();      d.env_width = scene.GetEnvImage().width; d.env_height = scene.GetEnvImage().height;
    d.scene_info = scene.GetSceneInfo();
    Check(rt_upload_scene(ctx_, &d), "UploadGPUData");
}

void CUDAPathTraceIntegrator::SetCameraData(Camera const& camera)
{
    Check(rt_set_camera(ctx_, &camera), "SetCameraData");
    prev_camera_ = camera;
    camera_ = camera;
}

void CUDAPathTraceIntegrator::SetSamplerType(SamplerType sampler_type)
{
    if (sampler_type == sampler_type_) return;
    Check(rt_set_option(ctx_, RT_OPT_SAMPLER, sampler_type == SamplerType::kBlueNoise ? 1u : 0u), "SetSamplerType");
    sampler_type_ = sampler_type;
    RequestReset();
}

void CUDAPathTraceIntegrator::SetBlueNoiseTables(const int* sobol_256spp_256d, const int* scrambling_tile, const int* ranking_tile)
{
    Check(rt_upload_sampler_tables(ctx_, sobol_256spp_256d, scrambling_tile, ranking_tile), "SetBlueNoiseTables");
    if (sampler_type_ == SamplerType::kBlueNoise) RequestReset();
}

void CUDAPathTraceIntegrator::SetAOV(AOV aov)
{
    if (aov == aov_) return;
    Check(rt_set_option(ctx_, RT_OPT_AOV, (std::uint32_t)aov), "SetAOV");
    aov_ = aov;
    RequestReset();
}

void CUDAPathTraceIntegrator::EnableDenoiser(bool enable)
{
    if (enable == enable_denoiser_) return;
    Check(rt_set_option(ctx_, RT_OPT_DENOISER, enable ? 1u : 0u), "EnableDenoiser");
    enable_denoiser_ = enable;
    RequestReset();
}

void CUDAPathTraceIntegrator::Reset() { Check(rt_reset(ctx_), "Reset"); }

void CUDAPathTraceIntegrator::SetSamplesPerFrame(std::uint32_t n)
{
    if (n == 0) throw std::runtime_error("SetSamplesPerFrame: a frame renders at least one sample");
    samples_per_frame_ = n;
}

void CUDAPathTraceIntegrator::SetAdaptiveSampling(float max_error, std::uint32_t min_samples)
{
    Check(rt_set_adaptive_sampling(ctx_, max_error, min_samples), "SetAdaptiveSampling");
    RequestReset();
}

void CUDAPathTraceIntegrator::SetSpatialDenoiser(std::uint32_t iterations, float sigma_color, float sigma_normal, float sigma_depth)
{
    Check(rt_set_spatial_denoiser(ctx_, iterations, sigma_color, sigma_normal, sigma_depth), "SetSpatialDenoiser");
}

std::uint32_t CUDAPathTraceIntegrator::ActivePixels() const
{
    std::uint32_t n = 0;
    Check(rt_read_active_pixels(ctx_, &n), "ActivePixels");
    return n;
}

void CUDAPathTraceIntegrator::ReadPixelSamples(std::uint32_t* counts) const { Check(rt_read_pixel_samples(ctx_, counts), "ReadPixelSamples"); }

// ---- the per-frame steps.  kFrame: Integrate() (integrator.cpp:27-59, not virtual) calls them in a fixed order; they are
// checked against that order and the frame is submitted as a whole in AdvanceSampleCount().
void CUDAPathTraceIntegrator::GenerateRays()
{
    if (samples_per_frame_ > 1 && schedule_ != Schedule::kFrame)
        throw std::runtime_error("GenerateRays: several samples per frame (SetSamplesPerFrame) need the kFrame schedule");
    if (samples_per_frame_ > 1 && enable_denoiser_)
        throw std::runtime_error("GenerateRays: several samples per frame (SetSamplesPerFrame) are not available with the denoiser, which runs once per sample");
    if (schedule_ == Schedule::kFrame) { frame_deferred_ = true; deferred_shaded_ = deferred_accumulated_ = 0; return; }
    Check(rt_generate_rays(ctx_), "GenerateRays");
}

void CUDAPathTraceIntegrator::FlushDeferredFrame()
{
    if (!frame_deferred_) return;
    frame_deferred_ = false;
    if (samples_per_frame_ > 1)
        throw std::runtime_error("several samples per frame (SetSamplesPerFrame) need the call order of Integrate(); this frame's steps arrived in another order");
    Check(rt_generate_rays(ctx_), "GenerateRays");
    for (std::uint32_t b = 0; b < deferred_shaded_; ++b)
    {
        Check(rt_extend_shade(ctx_, b), "ShadeSurfaceHits (fused intersect+miss+shade)");
        if (b < deferred_accumulated_) Check(rt_shadow_accumulate(ctx_, b), "AccumulateDirectSamples (fused shadow trace+accumulate)");
    }
}

void CUDAPathTraceIntegrator::AdvanceSampleCount()
{
    if (frame_deferred_)
    {
        if (deferred_shaded_ == max_bounces_ + 1 && deferred_accumulated_ == max_bounces_ + 1)
        {   // the canonical frame: one call, rt_integrate advances the sample count itself
            frame_deferred_ = false;
            if (samples_per_frame_ > 1) Check(rt_integrate_samples(ctx_, max_bounces_, samples_per_frame_), "Integrate (whole frame, several samples)");
            else Check(rt_integrate(ctx_, max_bounces_), "Integrate (whole frame)");
            return;
        }
        FlushDeferredFrame();
    }
    Check(rt_advance_sample_count(ctx_), "AdvanceSampleCount");
}

void CUDAPathTraceIntegrator::IntersectRays(std::uint32_t bounce)
{
    current_bounce_ = bounce;
    if (schedule_ == Schedule::kStepwise) Check(rt_intersect(ctx_, bounce), "IntersectRays");
}

void CUDAPathTraceIntegrator::ComputeAOVs() { Check(rt_compute_aovs(ctx_), "ComputeAOVs"); }

void CUDAPathTraceIntegrator::ShadeMissedRays(std::uint32_t bounce)
{
    if (schedule_ == Schedule::kStepwise) Check(rt_shade_miss(ctx_, bounce), "ShadeMissedRays");
}

void CUDAPathTraceIntegrator::ClearOutgoingRayCounter(std::uint32_t bounce) { Check(rt_clear_outgoing_counter(ctx_, bounce), "ClearOutgoingRayCounter"); }
void CUDAPathTraceIntegrator::ClearShadowRayCounter() { Check(rt_clear_shadow_counter(ctx_), "ClearShadowRayCounter"); }

void CUDAPathTraceIntegrator::ShadeSurfaceHits(std::uint32_t bounce)
{
    current_bounce_ = bounce;
    if (frame_deferred_)
    {
        if (bounce == deferred_shaded_ && deferred_accumulated_ == deferred_shaded_) { ++deferred_shaded_; return; }
        FlushDeferredFrame();                 // not the canonical order: run what was recorded, continue call by call
    }
    if (schedule_ == Schedule::kStepwise) Check(rt_shade_hits(ctx_, bounce), "ShadeSurfaceHits");
    else Check(rt_extend_shade(ctx_, bounce), "ShadeSurfaceHits (fused intersect+miss+shade)");
}

void CUDAPathTraceIntegrator::IntersectShadowRays()
{
    if (schedule_ == Schedule::kStepwise) Check(rt_intersect_shadow(ctx_), "IntersectShadowRays");
}

void CUDAPathTraceIntegrator::AccumulateDirectSamples()
{
    if (frame_deferred_)
    {
        if (deferred_accumulated_ + 1 == deferred_shaded_ && current_bounce_ + 1 == deferred_shaded_) { ++deferred_accumulated_; return; }
        FlushDeferredFrame();
    }
    if (schedule_ == Schedule::kStepwise) Check(rt_accumulate_direct(ctx_), "AccumulateDirectSamples");
    else Check(rt_shadow_accumulate(ctx_, current_bounce_), "AccumulateDirectSamples (fused shadow trace+accumulate)");
}

void CUDAPathTraceIntegrator::Denoise() { Check(rt_denoise(ctx_), "Denoise"); }
void CUDAPathTraceIntegrator::CopyHistoryBuffers() { Check(rt_copy_history(ctx_), "CopyHistoryBuffers"); }
void CUDAPathTraceIntegrator::ResolveRadiance() { Check(rt_resolve(ctx_, resolve_target_), "ResolveRadiance"); }

} // namespace rt_host
