/*
 * reference_api.hpp — the reference-facing C++ interface of the backend, in one header.
 *
 * The H100 backend is a drop-in behind the reference's own abstractions, so the host side mirrors three of them with
 * the same names, members and call contracts (paths relative to /root/reference/src):
 *   AccelerationStructure   acceleration_structure.hpp:31-38   BuildCPU reorders the triangles into leaf order
 *   Integrator              integrator/integrator.hpp:34-100, integrator.cpp:27-77
 *                           public interface + the 15 protected virtual steps + the fixed wavefront schedule Integrate()
 *   Scene                   scene/scene.hpp:34-67, scene/scene.cpp:46-361   OBJ/MTL -> the seven arrays the integrator uploads
 * A backend plugs in by deriving from Integrator (cuda_pt_integrator.hpp is the H100 one, next to the reference's
 * OpenCL and OpenGL backends); Bvh (bvh.hpp) derives from AccelerationStructure; Render (render.hpp) wires them up.
 */
#pragma once

#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "types.hpp"

namespace rt_host
{

class Scene;

// ---------------------------------------------------------------------------------------------------------------
// AccelerationStructure
// ---------------------------------------------------------------------------------------------------------------
class AccelerationStructure
{
public:
    virtual ~AccelerationStructure() = default;
    virtual void BuildCPU(std::vector<Triangle>& triangles) = 0;
    virtual std::vector<LinearBVHNode> const& GetNodes() const = 0;
};

// ---------------------------------------------------------------------------------------------------------------
// Integrator: same public interface, same protected virtual steps, same Integrate() as the reference.
// ---------------------------------------------------------------------------------------------------------------
class Integrator
{
public:
    enum class SamplerType { kRandom, kBlueNoise };
    enum AOV { kShadedColor, kDiffuseAlbedo, kDepth, kNormal, kMotionVectors };

    Integrator(std::uint32_t width, std::uint32_t height, AccelerationStructure& acc_structure)
        : width_(width), height_(height), acc_structure_(acc_structure) {}
    virtual ~Integrator() = default;

    void Integrate();
    virtual void UploadGPUData(Scene const& scene, AccelerationStructure const& acc_structure) = 0;
    virtual void SetCameraData(Camera const& camera) = 0;
    void RequestReset() { request_reset_ = true; }
    void EnableWhiteFurnace(bool enable);
    void SetMaxBounces(std::uint32_t max_bounces);
    virtual void SetSamplerType(SamplerType sampler_type) = 0;
    virtual void SetAOV(AOV aov) = 0;
    virtual void EnableDenoiser(bool enable) = 0;

protected:
    virtual void CreateKernels() = 0;
    virtual void Reset() = 0;
    virtual void AdvanceSampleCount() = 0;
    virtual void GenerateRays() = 0;
    virtual void IntersectRays(std::uint32_t bounce) = 0;
    virtual void ComputeAOVs() = 0;
    virtual void ShadeMissedRays(std::uint32_t bounce) = 0;
    virtual void ShadeSurfaceHits(std::uint32_t bounce) = 0;
    virtual void IntersectShadowRays() = 0;
    virtual void AccumulateDirectSamples() = 0;
    virtual void ClearOutgoingRayCounter(std::uint32_t bounce) = 0;
    virtual void ClearShadowRayCounter() = 0;
    virtual void Denoise() = 0;
    virtual void CopyHistoryBuffers() = 0;
    virtual void ResolveRadiance() = 0;

    std::uint32_t width_;
    std::uint32_t height_;
    AccelerationStructure& acc_structure_;
    Camera camera_ = {};
    Camera prev_camera_ = {};
    std::uint32_t max_bounces_ = 3u;
    SamplerType sampler_type_ = SamplerType::kRandom;
    AOV aov_ = AOV::kShadedColor;
    bool request_reset_ = false;
    bool enable_white_furnace_ = false;
    bool enable_denoiser_ = false;
};

// ---------------------------------------------------------------------------------------------------------------
// Scene.  The OBJ/MTL reader is a small purpose-built parser (triangulated faces with v//vn or v/vt/vn indices, the MTL
// keys the reference consumes: Kd Ks Ke Ni Tf Pr Pm map_Kd map_Ks map_Pr map_Pm map_Ke map_d), with tinyobjloader's defaults
// for absent keys (tiny_obj_loader.h:1331-1340).  Image textures are decoded by image_loader.cpp (PNG, TGA; the reference goes
// through stb_image, loaders/image_loader.cpp:30-63) into the reference's packed texel words; JPEG files fail loudly.
// ---------------------------------------------------------------------------------------------------------------
struct Image
{
    std::uint32_t width = 0, height = 0;
    std::vector<float> data;      // RGBA32F
};

// 8-bit texture image as the reference stores it (loaders/image_loader.hpp: Image with uint32 texels r | g<<8 | b<<16 | a<<24)
struct TextureImage
{
    std::uint32_t width = 0, height = 0;
    std::vector<std::uint32_t> data;
};
bool LoadTextureImage(const char* filename, TextureImage& result, std::string& error);
// JPEG file in memory -> interleaved 8-bit pixels, `channels` = 3 (colour) or 1 (greyscale), in the arithmetic of the reference's
// decoder (jpeg_decoder.cpp)
bool DecodeJpeg(const unsigned char* file, size_t size, int& w, int& h, int& channels, std::vector<unsigned char>& pixels, std::string& error);

// Radiance .hdr reader with the reference's conversion (loaders/hdr_loader.cpp:29-120):
// rows in file order, value = (mantissa / 256) * 2^(e - 128), alpha left 0.
bool LoadHDR(const char* filename, Image& result);

class Scene
{
public:
    Scene(const char* filename, float scale, bool flip_yz);
    // Headless construction from arrays that are already in the reference layout (a scene dump: Triangle[160 B], PackedMaterial[20 B],
    // Light[48 B], Texture[16 B] + texels) — the state a Scene is in after Load() and the Add*Light calls; bench/test plumbing.
    Scene(std::vector<Triangle> triangles, std::vector<PackedMaterial> materials, std::vector<Light> lights,
          std::vector<Texture> textures, std::vector<std::uint32_t> texture_data);

    std::vector<Triangle>& GetTriangles() { return triangles_; }
    std::vector<Triangle> const& GetTriangles() const { return triangles_; }
    std::vector<std::uint32_t> const& GetEmissiveIndices() const { return emissive_indices_; }
    std::vector<PackedMaterial> const& GetMaterials() const { return materials_; }
    std::vector<Texture> const& GetTextures() const { return textures_; }
    std::vector<std::uint32_t> const& GetTextureData() const { return texture_data_; }
    std::vector<Light> const& GetLights() const { return lights_; }
    SceneInfo const& GetSceneInfo() const { return scene_info_; }
    Image const& GetEnvImage() const { return env_image_; }
    // The reference hard-codes "assets/ibl/CGSkies_0036_free.hdr" relative to the CWD (scene.cpp:360);
    // the path is a parameter here, with that default.
    void Finalize(const char* env_map_path = "assets/ibl/CGSkies_0036_free.hdr");
    // Headless variant for callers that already hold the decoded environment image.
    void Finalize(const float* env_rgba, std::uint32_t env_width, std::uint32_t env_height);
    void AddPointLight(float3 origin, float3 radiance);
    void AddDirectionalLight(float3 direction, float3 radiance);

private:
    void Load(const char* filename, float scale, bool flip_yz);
    void CollectEmissiveTriangles();
    std::size_t LoadTexture(const std::string& filename);      // scene.cpp:276-323 (cached by file name)
    std::map<std::string, std::size_t> loaded_textures_;

    std::vector<Triangle> triangles_;
    std::vector<std::uint32_t> emissive_indices_;
    std::vector<PackedMaterial> materials_;
    std::vector<Light> lights_;
    std::vector<Texture> textures_;
    std::vector<std::uint32_t> texture_data_;
    SceneInfo scene_info_ = {};
    Image env_image_;
};

} // namespace rt_host
