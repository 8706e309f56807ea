/*
 * examples/headless_render.cpp — the reference's main.cpp (src/main.cpp:30-79) minus the window: load an OBJ scene,
 * add the directional light main.cpp:58 adds, create a Render with the CUDA backend, render N progressive samples and
 * write the resolved image as a binary PFM.
 *
 *   g++ -std=c++17 -O2 -Iinclude -Iraytracing_b200/host examples/headless_render.cpp \
 *       -Lraytracing_b200 -lrt_host -lrt_b200 -Wl,-rpath,'$ORIGIN/../raytracing_b200' -o examples/headless_render
 *   examples/headless_render assets/CornellBox.obj assets/ibl/CGSkies_0036_free.hdr 1920 1080 64 out.pfm [all|d0,d1,...]
 *
 * The optional last argument spreads the frame over several GPUs of the node behind the same Render / Integrator objects
 * ("all" = every CUDA device; the image is partitioned by scanline inside the library, rt_create_multi).
 *
 * Needs an H100 (there is no CPU fallback: Render's constructor throws without a CUDA device).
 */
#include <cstdio>
#include <cstdlib>
#include <exception>
#include <memory>
#include <string>
#include <vector>

#include "render.hpp"

int main(int argc, char** argv)
{
    if (argc < 7) { std::fprintf(stderr, "usage: %s scene.obj env.hdr width height samples out.pfm [all|d0,d1,...]\n", argv[0]); return 2; }
    const unsigned width = (unsigned)std::atoi(argv[3]), height = (unsigned)std::atoi(argv[4]), samples = (unsigned)std::atoi(argv[5]);
    try
    {
        rt_host::Scene scene(argv[1], 1.0f, false);
        scene.AddDirectionalLight({ -0.6f, -1.5f, 3.5f }, { 15.0f, 10.0f, 5.0f });                 // main.cpp:58
        std::vector<int> devices;                                                                   // empty = every CUDA device of the node
        bool multi = argc > 7;
        if (multi && std::string(argv[7]) != "all")
            for (const char* p = argv[7]; *p;) { devices.push_back(std::atoi(p)); while (*p && *p != ',') ++p; if (*p == ',') ++p; }
        std::unique_ptr<rt_host::Render> owner(multi ? new rt_host::Render(width, height, rt_host::Render::RenderBackend::kCUDA, scene, argv[2], devices)
                                                     : new rt_host::Render(width, height, rt_host::Render::RenderBackend::kCUDA, scene, argv[2]));
        rt_host::Render& render = *owner;
        render.SetMaxBounces(8);
        for (unsigned s = 0; s < samples; ++s) render.RenderFrame();                               // one sample per frame, accumulated
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
