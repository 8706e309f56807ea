/*
 * examples/headless_render.cpp — the reference's main.cpp (src/main.cpp:30-79) minus the window: load an OBJ scene,
 * add the directional light main.cpp:58 adds, create a Render with the CUDA backend, render N progressive samples with one
 * RenderFrame() (SetSamplesPerFrame: one rt_integrate_samples call, the same image as N frames of one sample) and write the
 * resolved image as a binary PFM.
 *
 *   g++ -std=c++17 -O2 -Iinclude -Iraytracing_b200/host examples/headless_render.cpp \
 *       -Lraytracing_b200 -lrt_host -lrt_b200 -Wl,-rpath,'$ORIGIN/../raytracing_b200' -o examples/headless_render
 *   examples/headless_render assets/CornellBox.obj assets/ibl/CGSkies_0036_free.hdr 1920 1080 64 out.pfm [all|d0,d1,...] [max_error=E] [denoise=ITER,SC,SN,SZ]
 *
 * The optional device list spreads the frame over several GPUs of the node behind the same Render / Integrator objects
 * ("all" = every CUDA device; the image is partitioned by scanline inside the library, rt_create_multi).
 * max_error=E turns on adaptive sampling (Render::SetAdaptiveSampling(E, 4)): `samples` becomes the budget, rendered in
 * RenderFrame() calls of 16 samples until no pixel is active any more or the budget is spent; the mean samples per pixel is printed.
 * denoise=ITER,SC,SN,SZ turns on the spatial denoiser (Render::SetSpatialDenoiser: ITER passes, the colour, normal and depth sigmas)
 * on a single-device render.
 *
 * Needs an H100 (there is no CPU fallback: Render's constructor throws without a CUDA device).
 */
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <exception>
#include <memory>
#include <string>
#include <vector>

#include "render.hpp"

int main(int argc, char** argv)
{
    if (argc < 7) { std::fprintf(stderr, "usage: %s scene.obj env.hdr width height samples out.pfm [all|d0,d1,...] [max_error=E] [denoise=ITER,SC,SN,SZ]\n", argv[0]); return 2; }
    const unsigned width = (unsigned)std::atoi(argv[3]), height = (unsigned)std::atoi(argv[4]), samples = (unsigned)std::atoi(argv[5]);
    float max_error = 0.0f;                                                                         // 0: every pixel takes every sample
    const char* device_arg = nullptr;
    unsigned denoise_iters = 0;                                                                     // 0: no spatial denoiser
    float sigma_color = 0.0f, sigma_normal = 0.0f, sigma_depth = 0.0f;
    for (int i = 7; i < argc; ++i)
    {
        if (std::string(argv[i]).rfind("max_error=", 0) == 0) max_error = (float)std::atof(argv[i] + 10);
        else if (std::string(argv[i]).rfind("denoise=", 0) == 0)
        {
            if (std::sscanf(argv[i] + 8, "%u,%f,%f,%f", &denoise_iters, &sigma_color, &sigma_normal, &sigma_depth) != 4)
            { std::fprintf(stderr, "denoise=ITER,SC,SN,SZ expects four numbers\n"); return 2; }
        }
        else device_arg = argv[i];
    }
    try
    {
        rt_host::Scene scene(argv[1], 1.0f, false);
        scene.AddDirectionalLight({ -0.6f, -1.5f, 3.5f }, { 15.0f, 10.0f, 5.0f });                 // main.cpp:58
        std::vector<int> devices;                                                                   // empty = every CUDA device of the node
        const bool multi = device_arg != nullptr;
        if (multi && std::string(device_arg) != "all")
            for (const char* p = device_arg; *p;) { devices.push_back(std::atoi(p)); while (*p && *p != ',') ++p; if (*p == ',') ++p; }
        std::unique_ptr<rt_host::Render> owner(multi ? new rt_host::Render(width, height, rt_host::Render::RenderBackend::kCUDA, scene, argv[2], devices)
                                                     : new rt_host::Render(width, height, rt_host::Render::RenderBackend::kCUDA, scene, argv[2]));
        rt_host::Render& render = *owner;
        render.SetMaxBounces(8);
        if (denoise_iters > 0) render.SetSpatialDenoiser(denoise_iters, sigma_color, sigma_normal, sigma_depth);
        if (samples > 0 && max_error > 0.0f)
        {   // progressive: chunks of 16 samples until every pixel has settled or the budget is spent
            render.SetAdaptiveSampling(max_error, 4);
            unsigned spent = 0;
            while (spent < samples)
            {
                const unsigned chunk = std::min(16u, samples - spent);
                render.SetSamplesPerFrame(chunk);
                render.RenderFrame();
                spent += chunk;
                if (render.ActivePixels() == 0) break;
            }
            std::vector<std::uint32_t> counts((size_t)width * height);
            static_cast<rt_host::CUDAPathTraceIntegrator&>(render.GetIntegrator()).ReadPixelSamples(counts.data());
            double sum = 0.0;
            for (std::uint32_t n : counts) sum += n;
            std::printf("adaptive sampling, max_error %g: %u samples spent, %.2f samples per pixel on average\n", max_error, spent,
                        sum / (double)counts.size());
        }
        else if (samples > 0)
        {
            render.SetSamplesPerFrame(samples);
            render.RenderFrame();                                                                  // every sample in one call, accumulated
        }
        std::FILE* f = std::fopen(argv[6], "wb");
        if (!f) { std::perror(argv[6]); return 1; }
        std::fprintf(f, "PF\n%u %u\n-1.0\n", width, height);
        const float* img = render.GetImage().data();
        for (unsigned y = height; y-- > 0;)                                                        // PFM rows go bottom-up
            for (unsigned x = 0; x < width; ++x) std::fwrite(img + ((size_t)y * width + x) * 4, sizeof(float), 3, f);
        std::fclose(f);
    }
    catch (std::exception const& e) { std::fprintf(stderr, "error: %s\n", e.what()); return 1; }   // same single catch as main.cpp:74-77
    return 0;
}
