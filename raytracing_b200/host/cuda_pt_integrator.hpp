/*
 * CUDAPathTraceIntegrator — the H100 backend behind the reference's Integrator interface, the
 * counterpart of CLPathTraceIntegrator (/root/reference/src/integrator/cl_pt_integrator.hpp:31-125).
 * It owns an opaque rt_ctx and forwards every virtual step to the C ABI (include/rt_b200.h), which
 * takes the place of CLContext/CLKernel.  Errors come back as status codes and are re-thrown as
 * std::runtime_error, the behaviour callers of the OpenCL backend see (CLException).
 *
 * Schedules:
 *   kFrame (default)  Integrate() is not virtual and calls the 15 virtuals in a fixed order (integrator.cpp:27-59); here the
 *                     steps between GenerateRays() and AdvanceSampleCount() only check that order, and AdvanceSampleCount()
 *                     submits the WHOLE frame with one rt_integrate call (one persistent kernel, or one graph replay of the
 *                     per-phase kernels: the schedule bench.py measures).  A caller that drives the virtuals in another
 *                     order falls back to kFused for that frame: the steps seen so far are replayed, the rest run as they come.
 *   kFused            the seven per-bounce virtuals map onto TWO kernels: ShadeSurfaceHits(b) launches
 *                     the fused intersect+miss+shade kernel, AccumulateDirectSamples() the fused
 *                     shadow-trace+accumulate kernel; IntersectRays, ShadeMissedRays, the two counter
 *                     clears and IntersectShadowRays are empty (the OpenGL backend of the reference
 *                     also leaves steps empty: gl_pt_integrator.cpp:230-243,354-357,466-474).  At the
 *                     end of each loop iteration of Integrate() the device state is the same as with
 *                     the stepwise schedule, bit for bit.
 *   kStepwise         one kernel per virtual, like the OpenCL backend.
 * SetSamplesPerFrame(n): Integrate() renders n progressive samples, the same bits as n calls with one sample each.  kFrame only:
 * AdvanceSampleCount() submits them with ONE rt_integrate_samples call (n frames on the device without a host round trip, or
 * one launch of the regenerating frame kernel with RT_OPT_FRAME_KERNEL 1).  With n > 1 the kFused / kStepwise schedules, a call order other than
 * Integrate()'s and the denoiser (it runs once per sample) throw std::runtime_error.
 * SetAdaptiveSampling(max_error, min_samples): pixels stop tracing once they have settled (include/rt_b200.h); ActivePixels() tells
 * a progressive loop when every pixel has.
 * SetSpatialDenoiser(iterations, sigmas): ResolveRadiance() filters the shaded colour (include/rt_b200.h states the rule).
 * AOVs (ComputeAOVs) are produced inside the bounce-0 shading pass, and only when SetAOV selected a view other than
 * the shaded colour or the denoiser is on.  SetSamplerType(kBlueNoise) needs the sampler's three tables first
 * (SetBlueNoiseTables; the OpenCL backend reads them from utils/blue_noise_sampler.hpp, cl_pt_integrator.cpp:222-235).
 * The last constructor argument of the OpenCL backend is a GL texture to resolve into
 * (cl_pt_integrator.hpp:33-34); here ResolveRadiance() writes to a host RGBA32F image instead
 * (SetResolveTarget), or only resolves on the device if none is set.
 */
#pragma once

#include <string>
#include <vector>

#include "reference_api.hpp"
#include "rt_b200.h"

namespace rt_host
{

class CUDAPathTraceIntegrator : public Integrator
{
public:
    enum class Schedule { kFrame, kFused, kStepwise };

    CUDAPathTraceIntegrator(std::uint32_t width, std::uint32_t height, AccelerationStructure& acc_structure,
                            int device = 0, Schedule schedule = Schedule::kFrame);
    // several devices of the node behind ONE integrator (rt_create_multi: device i renders the rows y % n == i); an empty
    // list means every CUDA device of the node, as CLContext enumerates every device of its platform (cl_context.cpp:64-89)
    CUDAPathTraceIntegrator(std::uint32_t width, std::uint32_t height, AccelerationStructure& acc_structure,
                            std::vector<int> const& devices, Schedule schedule = Schedule::kFrame);
    ~CUDAPathTraceIntegrator() override;

    void UploadGPUData(Scene const& scene, AccelerationStructure const& acc_structure) override;
    void SetCameraData(Camera const& camera) override;
    void SetSamplerType(SamplerType sampler_type) override;
    void SetAOV(AOV aov) override;
    void EnableDenoiser(bool enable) override;

    // sobol_256spp_256d[256*256], scramblingTile[128*128*8], rankingTile[128*128*8]; copied to the device
    void SetBlueNoiseTables(const int* sobol_256spp_256d, const int* scrambling_tile, const int* ranking_tile);
    // host RGBA32F image that ResolveRadiance() fills; page_lock = true registers it with the driver (rt_host_register) so that
    // the device->host copies are asynchronous (several devices then read back in parallel)
    void SetResolveTarget(float* host_rgba, bool page_lock = false);
    void SetSchedule(Schedule s) { schedule_ = s; }
    // samples rendered by one Integrate() (default 1); n > 1 needs the kFrame schedule and no denoiser
    void SetSamplesPerFrame(std::uint32_t n);
    std::uint32_t SamplesPerFrame() const { return samples_per_frame_; }
    // adaptive sampling (rt_set_adaptive_sampling): stop tracing pixels whose resolved luminance has a standard error <= max_error
    // after >= min_samples samples; max_error 0 turns it off.  Requests a reset, like SetMaxBounces: it applies from the next frame.
    void SetAdaptiveSampling(float max_error, std::uint32_t min_samples);
    // pixels that trace the next sample (all of them with adaptive sampling off); blocks
    std::uint32_t ActivePixels() const;
    // every pixel's sample count, width*height entries; blocks
    void ReadPixelSamples(std::uint32_t* counts) const;
    // spatial denoiser (rt_set_spatial_denoiser): an edge-avoiding a-trous filter on the resolved shaded colour, guided by the
    // bounce-0 normal and depth; iterations 0 turns it off.  No reset: the accumulation is unaffected.
    void SetSpatialDenoiser(std::uint32_t iterations, float sigma_color, float sigma_normal, float sigma_depth);
    rt_ctx* Context() const { return ctx_; }

protected:
    void CreateKernels() override;
    void Reset() override;
    void AdvanceSampleCount() override;
    void GenerateRays() override;
    void IntersectRays(std::uint32_t bounce) override;
    void ComputeAOVs() override;
    void ShadeMissedRays(std::uint32_t bounce) override;
    void ShadeSurfaceHits(std::uint32_t bounce) override;
    void IntersectShadowRays() override;
    void AccumulateDirectSamples() override;
    void ClearOutgoingRayCounter(std::uint32_t bounce) override;
    void ClearShadowRayCounter() override;
    void Denoise() override;
    void CopyHistoryBuffers() override;
    void ResolveRadiance() override;

private:
    void Check(int status, const char* what) const;

    void FlushDeferredFrame();     // kFrame: replay the recorded steps through the per-call API (order was not the canonical one)

    rt_ctx* ctx_ = nullptr;
    Schedule schedule_;
    std::uint32_t current_bounce_ = 0;
    std::uint32_t samples_per_frame_ = 1;
    float* resolve_target_ = nullptr;
    bool resolve_target_locked_ = false;
    // kFrame bookkeeping: a frame is "deferred" from GenerateRays() until AdvanceSampleCount()
    bool frame_deferred_ = false;
    std::uint32_t deferred_shaded_ = 0, deferred_accumulated_ = 0;   // bounces whose ShadeSurfaceHits / AccumulateDirectSamples were seen
};

} // namespace rt_host
