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
 * AdvanceSampleCount() submits them with ONE rt_integrate_samples call (n frames on the device without a host round trip).
 * With n > 1 the kFused / kStepwise schedules, a call order other than
 * Integrate()'s and the denoiser (it runs once per sample) throw std::runtime_error.
 * SetAdaptiveSampling(max_error, min_samples): pixels stop tracing once they have settled (include/rt_b200.h); ActivePixels() tells
 * a progressive loop when every pixel has.
 * SetSpatialDenoiser(iterations, sigmas): ResolveRadiance() filters the shaded colour (include/rt_b200.h states the rule).
 * SetEmitterSampling(on): next-event estimation on the emissive triangles as well, combined with BSDF sampling by MIS
 * (RT_OPT_EMITTER_SAMPLING; the image converges to the same expectation, so the accumulation is kept).
 * SetObjectMotion(on): motion vectors that follow UpdateTriangles as well as the camera (RT_OPT_OBJECT_MOTION).
 * SetEnvironmentSampling(on): the same for the environment map (RT_OPT_ENV_SAMPLING); SetLightSelection(a, e, v): relative weights of
 * the light kind drawn at each vertex (rt_set_light_selection).  Neither resets the accumulation.
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
    // RebuildBvh: kLinear a linear BVH (rt_rebuild_bvh, the faster build), kPloc clustering (rt_rebuild_bvh_ploc, the faster trace)
    enum class BvhBuild { kLinear, kPloc };

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
    // emitter sampling (RT_OPT_EMITTER_SAMPLING): sample the emissive triangles at every hit too, with MIS.  No reset: the estimator has
    // the same expectation, so it applies from the next frame and keeps the accumulation.
    void SetEmitterSampling(bool on);
    // object motion (RT_OPT_OBJECT_MOTION): the motion-vector AOV (view 4, the temporal denoiser's reprojection) follows
    // UpdateTriangles as well as the camera.  Changes no image until the next UpdateTriangles.
    void SetObjectMotion(bool on);
    // environment sampling (RT_OPT_ENV_SAMPLING): sample the environment map at every hit too, with MIS.  No reset, as above.
    void SetEnvironmentSampling(bool on);
    // light-kind weights (rt_set_light_selection): analytic, emitters, environment, each finite and > 0.  No reset, as above.
    void SetLightSelection(float analytic, float emitters, float environment);
    // geometry update (rt_update_triangles): new positions, normals and texcoords for the uploaded triangles (leaf order, same count;
    // materials are kept); the BVH is refit on the device.  No reset: like a camera move, whether the old samples are kept is the
    // caller's choice (RequestReset() starts over; an animation that keeps them gets motion blur).
    void UpdateTriangles(const Triangle* triangles, size_t count);
    // BVH rebuild (rt_rebuild_bvh, or rt_rebuild_bvh_ploc for BvhBuild::kPloc): replaces the tree by one over the current
    // triangles, built on the device, when a refit no longer traces well; returns the new node count (2n - 1).  Triangle ids do
    // not change.  No reset, as above.
    std::uint64_t RebuildBvh(BvhBuild build = BvhBuild::kLinear);
    // instanced scene (rt_upload_instanced_scene): the meshes' triangles (each mesh in its own leaf order) and nodes (each mesh's
    // own array), concatenated, with the materials, lights, textures and environment of `shared`; replaces the scene.  Place the
    // meshes with SetInstances (rt_set_instances: the whole list; no reset, as for UpdateTriangles).
    void UploadInstancedScene(Scene const& shared, const RtTriangle* triangles, size_t n_triangles, const RtLinearBVHNode* nodes,
                              size_t n_nodes, const RtMeshDesc* meshes, std::uint32_t n_meshes);
    void SetInstances(const RtInstance* instances, std::uint32_t count);
    // mesh update in an instanced scene (rt_update_mesh_triangles): new triangles for one mesh (its leaf order, same count); its
    // tree is refit on the device and the top-level tree rebuilt.  No reset, as for UpdateTriangles.
    void UpdateMeshTriangles(std::uint32_t mesh, const RtTriangle* triangles, size_t count);
    // per-instance materials (rt_set_instance_materials): n_remaps rows of one entry per scene material, and the row of each
    // instance index (RT_INVALID_ID: the mesh's own materials); replaces the assignment.  No reset, as for SetInstances.
    void SetInstanceMaterials(const std::uint32_t* remaps, std::uint32_t n_remaps, const std::uint32_t* remap_of_instance,
                              std::uint32_t n_instances);
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
