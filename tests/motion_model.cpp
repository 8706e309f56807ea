/*
 * motion_model.cpp — TEST INFRASTRUCTURE.  CPU model of object motion vectors (RT_OPT_OBJECT_MOTION, include/rt_b200.h): the
 * oracle's GenerateAOV (oracle/oracle.cpp orc_aovs) with the previous hit position taken from a given array of previous triangle
 * positions at the hit's barycentrics.  It reuses the oracle's building blocks (ray generation, traversal, textures, the screen
 * projection) by compiling oracle.cpp into the same translation unit.  With the previous positions equal to the scene's it is
 * orc_aovs.  Built by tests/motion_model.py with -ffp-contract=off.
 */
#include "oracle.cpp"

extern "C" {

/* orc_aovs with prev = (q1 * w0 + q2 * u) + q3 * v, where prev_pos holds 3 float4 per triangle (q1, q2, q3; the .w words are not
 * read) in the scene's triangle order. */
void mv_aovs(const OrcScene* scene, const float* prev_pos, const RtCamera* cam, const RtCamera* prev_cam, uint32_t width,
             uint32_t height, uint32_t sample_idx, float* albedo, float* depth, float* normal, float* velocity)
{
    Scene sc = to_scene(scene);
    size_t n = (size_t)width * height;
#pragma omp parallel for schedule(dynamic, 256)
    for (long long i = 0; i < (long long)n; ++i)
    {
        albedo[4 * i] = albedo[4 * i + 1] = albedo[4 * i + 2] = 0.0f; albedo[4 * i + 3] = 0.0f;
        depth[i] = RT_MAX_RENDER_DIST;
        normal[4 * i] = normal[4 * i + 1] = normal[4 * i + 2] = 0.0f; normal[4 * i + 3] = 0.0f;
        velocity[2 * i] = velocity[2 * i + 1] = 0.0f;
        Ray ray = RayGeneration((uint32_t)i, width, height, *cam, sample_idx);
        RtHit hit;
        TraceBvh(sc, ray, false, &hit, nullptr);
        if (hit.primitive_id == RT_INVALID_ID) continue;
        const RtTriangle& tri = sc.triangles[hit.primitive_id];
        float u = hit.bc.x, v = hit.bc.y, w0 = 1.0f - u - v;
        V3 position = Interp(v3(tri.v1.position), v3(tri.v2.position), v3(tri.v3.position), u, v);
        V2 texcoord = { tri.v1.texcoord.x * w0 + tri.v2.texcoord.x * u + tri.v3.texcoord.x * v,
                        tri.v1.texcoord.y * w0 + tri.v2.texcoord.y * u + tri.v3.texcoord.y * v };
        V3 nrm = normalize(Interp(v3(tri.v1.normal), v3(tri.v2.normal), v3(tri.v3.normal), u, v));
        Material m = ApplyTextures(sc, sc.materials[tri.mtlIndex], texcoord);
        albedo[4 * i] = m.diffuse_albedo.x; albedo[4 * i + 1] = m.diffuse_albedo.y; albedo[4 * i + 2] = m.diffuse_albedo.z;
        depth[i] = length(ray.o - position);
        normal[4 * i] = nrm.x; normal[4 * i + 1] = nrm.y; normal[4 * i + 2] = nrm.z;
        const float* q = prev_pos + (size_t)hit.primitive_id * 12;
        V3 prev = Interp(V3{ q[0], q[1], q[2] }, V3{ q[4], q[5], q[6] }, V3{ q[8], q[9], q[10] }, u, v);
        V2 a = ProjectScreen(position, *cam), b = ProjectScreen(prev, *prev_cam);
        velocity[2 * i] = a.x - b.x; velocity[2 * i + 1] = a.y - b.y;
    }
}

} // extern "C"
