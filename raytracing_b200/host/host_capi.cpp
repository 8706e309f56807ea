/*
 * host_capi.cpp — small C façade over the C++ host classes so that the Python tests and bench.py can drive
 * them (ctypes): scene loading, BVH build, and the headless Render with RenderBackend::kCUDA.  Not part of
 * the reference-facing boundary (that is include/rt_b200.h + the C++ classes); test/bench plumbing only.
 */
#include "obj_reader.hpp"
#include <cstring>
#include <memory>
#include <string>

#include "bvh.hpp"
#include "render.hpp"
#include "reference_api.hpp"

using namespace rt_host;

namespace
{
thread_local std::string g_error;
struct SceneHandle { std::unique_ptr<Scene> scene; Bvh bvh; bool built = false; };
struct RenderHandle { std::unique_ptr<Render> render; };
}

extern "C" {

const char* rth_last_error() { return g_error.c_str(); }

void* rth_scene_load(const char* obj_path, float scale, int flip_yz)
{
    try { auto* h = new SceneHandle; h->scene.reset(new Scene(obj_path, scale, flip_yz != 0)); return h; }
    catch (std::exception& e) { g_error = e.what(); return nullptr; }
}
// Scene from arrays in the reference layout (a scene dump); the triangles are copied (Render's BVH build reorders them)
void* rth_scene_from_arrays(const RtTriangle* triangles, size_t n_triangles, const RtPackedMaterial* materials, size_t n_materials,
                            const RtLight* lights, size_t n_lights, const RtTexture* textures, size_t n_textures,
                            const std::uint32_t* texels, size_t n_texels)
{
    try
    {
        auto* h = new SceneHandle;
        h->scene.reset(new Scene(std::vector<Triangle>(triangles, triangles + n_triangles), std::vector<PackedMaterial>(materials, materials + n_materials),
                                 std::vector<Light>(lights, lights + n_lights), std::vector<Texture>(textures, textures + n_textures),
                                 std::vector<std::uint32_t>(texels, texels + n_texels)));
        return h;
    }
    catch (std::exception& e) { g_error = e.what(); return nullptr; }
}
void rth_scene_free(void* h) { delete (SceneHandle*)h; }

int rth_scene_add_directional_light(void* h, float dx, float dy, float dz, float r, float g, float b)
{
    ((SceneHandle*)h)->scene->AddDirectionalLight(make_float3(dx, dy, dz), make_float3(r, g, b)); return 0;
}
int rth_scene_add_point_light(void* h, float x, float y, float z, float r, float g, float b)
{
    ((SceneHandle*)h)->scene->AddPointLight(make_float3(x, y, z), make_float3(r, g, b)); return 0;
}
int rth_scene_build_bvh(void* h)
{
    try { auto* s = (SceneHandle*)h; s->bvh.BuildCPU(s->scene->GetTriangles()); s->built = true; return 0; }
    catch (std::exception& e) { g_error = e.what(); return -1; }
}
int rth_scene_finalize_hdr(void* h, const char* env_path)
{
    try { ((SceneHandle*)h)->scene->Finalize(env_path); return 0; }
    catch (std::exception& e) { g_error = e.what(); return -1; }
}
int rth_scene_finalize_image(void* h, const float* env, std::uint32_t w, std::uint32_t hgt)
{
    ((SceneHandle*)h)->scene->Finalize(env, w, hgt); return 0;
}
// which: 0 triangles 1 nodes 2 materials 3 lights 4 textures 5 texels 6 emissive 7 env 8 scene_info
int rth_scene_query(void* h, int which, const void** ptr, size_t* count, std::uint32_t* e0, std::uint32_t* e1)
{
    auto* s = (SceneHandle*)h;
    const Scene& sc = *s->scene;
    *e0 = *e1 = 0;
    switch (which)
    {
    case 0: *ptr = sc.GetTriangles().data(); *count = sc.GetTriangles().size(); return 0;
    case 1: *ptr = s->bvh.GetNodes().data(); *count = s->bvh.GetNodes().size(); return 0;
    case 2: *ptr = sc.GetMaterials().data(); *count = sc.GetMaterials().size(); return 0;
    case 3: *ptr = sc.GetLights().data(); *count = sc.GetLights().size(); return 0;
    case 4: *ptr = sc.GetTextures().data(); *count = sc.GetTextures().size(); return 0;
    case 5: *ptr = sc.GetTextureData().data(); *count = sc.GetTextureData().size(); return 0;
    case 6: *ptr = sc.GetEmissiveIndices().data(); *count = sc.GetEmissiveIndices().size(); return 0;
    case 7: *ptr = sc.GetEnvImage().data.data(); *count = sc.GetEnvImage().data.size(); *e0 = sc.GetEnvImage().width; *e1 = sc.GetEnvImage().height; return 0;
    case 8: *ptr = &sc.GetSceneInfo(); *count = 1; return 0;
    }
    return -1;
}

// Stand-alone BVH build over a caller-provided triangle array (reordered in place); nodes_out must hold 2*n entries.
int rth_bvh_build(RtTriangle* triangles, size_t n, RtLinearBVHNode* nodes_out, size_t* n_nodes, std::uint32_t* max_depth)
{
    try
    {
        static_assert(sizeof(Triangle) == sizeof(RtTriangle), "layout");
        Bvh bvh;
        bvh.Build(reinterpret_cast<Triangle*>(triangles), n);
        memcpy(nodes_out, bvh.GetNodes().data(), bvh.GetNodes().size() * sizeof(LinearBVHNode));
        *n_nodes = bvh.GetNodes().size();
        if (max_depth) *max_depth = bvh.MaxDepth();
        return 0;
    }
    catch (std::exception& e) { g_error = e.what(); return -1; }
}

// One number token in the OBJ reader's arithmetic (obj_reader.cpp ParseDouble): 1 = parsed, 0 = not a number
int rth_obj_parse_number(const char* text, double* out)
{
    return obj::ParseDouble(text, text + strlen(text), out) ? 1 : 0;
}

int rth_default_camera(std::uint32_t width, std::uint32_t height, RtCamera* out)
{
    CameraController c(width, height);
    *out = c.GetData();
    return 0;
}

// Headless Render with the CUDA backend; the scene handle must not have had its BVH built yet (Render builds it).
void* rth_render_create(void* scene_handle, std::uint32_t width, std::uint32_t height, const char* env_path, int device, int stepwise)
{
    try
    {
        auto* s = (SceneHandle*)scene_handle;
        auto* h = new RenderHandle;
        h->render.reset(new Render(width, height, Render::RenderBackend::kCUDA, *s->scene, env_path, device));
        if (stepwise) static_cast<CUDAPathTraceIntegrator&>(h->render->GetIntegrator()).SetSchedule(CUDAPathTraceIntegrator::Schedule::kStepwise);
        return h;
    }
    catch (std::exception& e) { g_error = e.what(); return nullptr; }
}
// Same over several devices (n_devices == 0: every CUDA device of the node); schedule: 0 whole frame (default), 1 fused per bounce, 2 stepwise
void* rth_render_create_multi(void* scene_handle, std::uint32_t width, std::uint32_t height, const char* env_path, const int* devices, std::uint32_t n_devices, int schedule)
{
    try
    {
        auto* s = (SceneHandle*)scene_handle;
        auto* h = new RenderHandle;
        std::vector<int> list(devices, devices + n_devices);
        h->render.reset(new Render(width, height, Render::RenderBackend::kCUDA, *s->scene, env_path, list));
        auto& it = static_cast<CUDAPathTraceIntegrator&>(h->render->GetIntegrator());
        it.SetSchedule(schedule == 2 ? CUDAPathTraceIntegrator::Schedule::kStepwise : (schedule == 1 ? CUDAPathTraceIntegrator::Schedule::kFused : CUDAPathTraceIntegrator::Schedule::kFrame));
        return h;
    }
    catch (std::exception& e) { g_error = e.what(); return nullptr; }
}
// Same with the environment image handed over decoded (RGBA32F, env_w x env_h)
void* rth_render_create_env(void* scene_handle, std::uint32_t width, std::uint32_t height, const float* env, std::uint32_t env_w, std::uint32_t env_h,
                            const int* devices, std::uint32_t n_devices, int schedule)
{
    try
    {
        auto* s = (SceneHandle*)scene_handle;
        auto* h = new RenderHandle;
        Image img; img.width = env_w; img.height = env_h; img.data.assign(env, env + (size_t)env_w * env_h * 4);
        h->render.reset(new Render(width, height, Render::RenderBackend::kCUDA, *s->scene, img, std::vector<int>(devices, devices + n_devices)));
        auto& it = static_cast<CUDAPathTraceIntegrator&>(h->render->GetIntegrator());
        it.SetSchedule(schedule == 2 ? CUDAPathTraceIntegrator::Schedule::kStepwise : (schedule == 1 ? CUDAPathTraceIntegrator::Schedule::kFused : CUDAPathTraceIntegrator::Schedule::kFrame));
        return h;
    }
    catch (std::exception& e) { g_error = e.what(); return nullptr; }
}
int rth_render_set_camera(void* h, const RtCamera* cam)
{
    ((RenderHandle*)h)->render->GetCamera().SetData(*cam); ((RenderHandle*)h)->render->NotifyCameraChanged(); return 0;
}
int rth_render_set_schedule(void* h, int schedule)
{
    auto& it = static_cast<CUDAPathTraceIntegrator&>(((RenderHandle*)h)->render->GetIntegrator());
    it.SetSchedule(schedule == 2 ? CUDAPathTraceIntegrator::Schedule::kStepwise : (schedule == 1 ? CUDAPathTraceIntegrator::Schedule::kFused : CUDAPathTraceIntegrator::Schedule::kFrame));
    return 0;
}
void rth_render_free(void* h) { delete (RenderHandle*)h; }
int rth_render_set_max_bounces(void* h, std::uint32_t b)
{
    try { ((RenderHandle*)h)->render->SetMaxBounces(b); return 0; } catch (std::exception& e) { g_error = e.what(); return -1; }
}
int rth_render_set_samples_per_frame(void* h, std::uint32_t n)
{
    try { ((RenderHandle*)h)->render->SetSamplesPerFrame(n); return 0; } catch (std::exception& e) { g_error = e.what(); return -1; }
}
int rth_render_set_adaptive_sampling(void* h, float max_error, std::uint32_t min_samples)
{
    try { ((RenderHandle*)h)->render->SetAdaptiveSampling(max_error, min_samples); return 0; } catch (std::exception& e) { g_error = e.what(); return -1; }
}
int rth_render_set_spatial_denoiser(void* h, std::uint32_t iterations, float sigma_color, float sigma_normal, float sigma_depth)
{
    try { ((RenderHandle*)h)->render->SetSpatialDenoiser(iterations, sigma_color, sigma_normal, sigma_depth); return 0; }
    catch (std::exception& e) { g_error = e.what(); return -1; }
}
int rth_render_active_pixels(void* h, std::uint32_t* n)
{
    try { *n = ((RenderHandle*)h)->render->ActivePixels(); return 0; } catch (std::exception& e) { g_error = e.what(); return -1; }
}
int rth_render_enable_white_furnace(void* h, int e)
{
    try { ((RenderHandle*)h)->render->GetIntegrator().EnableWhiteFurnace(e != 0); return 0; } catch (std::exception& ex) { g_error = ex.what(); return -1; }
}
int rth_render_set_sampler(void* h, int blue_noise)
{
    try { ((RenderHandle*)h)->render->GetIntegrator().SetSamplerType(blue_noise ? Integrator::SamplerType::kBlueNoise : Integrator::SamplerType::kRandom); return 0; }
    catch (std::exception& ex) { g_error = ex.what(); return -1; }
}
int rth_render_set_sampler_tables(void* h, const int* sobol, const int* scrambling, const int* ranking)
{
    try { static_cast<CUDAPathTraceIntegrator&>(((RenderHandle*)h)->render->GetIntegrator()).SetBlueNoiseTables(sobol, scrambling, ranking); return 0; }
    catch (std::exception& ex) { g_error = ex.what(); return -1; }
}
int rth_render_frame(void* h)
{
    try { ((RenderHandle*)h)->render->RenderFrame(); return 0; } catch (std::exception& e) { g_error = e.what(); return -1; }
}
int rth_render_request_reset(void* h) { ((RenderHandle*)h)->render->NotifyCameraChanged(); return 0; }
// nodes of the BVH that Render built (Render owns its acceleration structure, render.hpp:87)
int rth_render_nodes(void* h, const void** ptr, size_t* count)
{
    auto const& n = ((RenderHandle*)h)->render->GetAccelerationStructure().GetNodes();
    *ptr = n.data(); *count = n.size(); return 0;
}
const float* rth_render_image(void* h) { return ((RenderHandle*)h)->render->GetImage().data(); }
void* rth_render_context(void* h) { return static_cast<CUDAPathTraceIntegrator&>(((RenderHandle*)h)->render->GetIntegrator()).Context(); }

} // extern "C"
