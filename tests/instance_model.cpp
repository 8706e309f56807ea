/*
 * instance_model.cpp — TEST INFRASTRUCTURE.  CPU model of instanced scenes (rt_upload_instanced_scene / rt_set_instances,
 * include/rt_b200.h): one sample of the oracle's frame (oracle/oracle.cpp orc_render) with the two-level traversal and instanced
 * shading.  It compiles oracle.cpp into the same translation unit for its building blocks (ray generation, sky, lights, materials,
 * BSDF sampling) and uses the library's own top-level builder (raytracing_b200/csrc/rt_instances.h), so the model and the device
 * trace the same tree.  The traversal restates trace_instanced: the top-level walk with trace_fast's slab test on boxes widened
 * by the ray's slack (rt_instances.h), near/far order and pop rule, the ray moved into object space by W, and the mesh traced by the reference-order traversal (which trace_fast equals
 * bit for bit) with the back-face test on det * sign(det M).  Built by tests/instance_model.py with -ffp-contract=off.
 */
#include "oracle.cpp"
#include "rt_instances.h"

namespace
{

struct Inst
{
    std::vector<rtinst::MeshInfo> meshes;
    rtinst::Prepared pr;
    uint32_t n = 0;
};

inline V3 XPoint(const float* m, V3 p)
{
    return v3(((m[0] * p.x + m[1] * p.y) + m[2] * p.z) + m[3], ((m[4] * p.x + m[5] * p.y) + m[6] * p.z) + m[7],
              ((m[8] * p.x + m[9] * p.y) + m[10] * p.z) + m[11]);
}
inline V3 XDir(const float* m, V3 d)
{
    return v3((m[0] * d.x + m[1] * d.y) + m[2] * d.z, (m[4] * d.x + m[5] * d.y) + m[6] * d.z, (m[8] * d.x + m[9] * d.y) + m[10] * d.z);
}
inline V3 XNormalT(const float* w, V3 n)     // W^T * n
{
    return v3((w[0] * n.x + w[4] * n.y) + w[8] * n.z, (w[1] * n.x + w[5] * n.y) + w[9] * n.z, (w[2] * n.x + w[6] * n.y) + w[10] * n.z);
}

// the slab test of the box (lo3, hi3) widened by e on each side
inline bool SlabHit(const float* lo3, const float* hi3, float e, V3 o, V3 inv, float t_min, float t_max, float* entry)
{
    V3 t0 = (v3(lo3[0] - e, lo3[1] - e, lo3[2] - e) - o) * inv, t1 = (v3(hi3[0] + e, hi3[1] + e, hi3[2] + e) - o) * inv;
    float lo = rt_fmaxf(rt_fmaxf(rt_fmaxf(rt_fminf(t0.x, t1.x), rt_fminf(t0.y, t1.y)), rt_fminf(t0.z, t1.z)), t_min);
    float hi = rt_fminf(rt_fminf(rt_fmaxf(t0.x, t1.x), rt_fmaxf(t0.y, t1.y)), rt_fmaxf(t0.z, t1.z));
    *entry = lo;
    return rt_fminf(hi, t_max) >= lo;
}

// TraceBvh (reference order) on one mesh, culling on det * cull
inline uint32_t MeshTrace(const Scene& sc, Ray ray, float cull, bool any_hit, float* bu, float* bv, float* bt)
{
    V3 inv_dir = splat(1.0f) / ray.d;
    int sign[3] = { inv_dir.x < 0, inv_dir.y < 0, inv_dir.z < 0 };
    uint32_t prim = RT_INVALID_ID;
    int to_visit = 0, cur = 0;
    int stack[64];
    for (;;)
    {
        const RtLinearBVHNode& node = sc.nodes[cur];
        if (RayBounds(node, ray.o, inv_dir, ray.tmin, ray.tmax))
        {
            int nprims = (int)(node.num_primitives_axis >> 16);
            if (nprims > 0)
            {
                for (int i = 0; i < nprims; ++i)
                {
                    const RtTriangle& t = sc.triangles[node.offset + i];
                    V3 p1 = v3(t.v1.position), p2 = v3(t.v2.position), p3 = v3(t.v3.position);
                    V3 e1 = p2 - p1, e2 = p3 - p1;
                    V3 pvec = cross(ray.d, e2);
                    float det = dot(e1, pvec);
                    float cdet = det * cull;
                    if (cdet < 1e-8f || -cdet > 1e-8f) continue;
                    float inv_det = 1.0f / det;
                    V3 tvec = ray.o - p1;
                    float u = dot(tvec, pvec) * inv_det;
                    if (u < 0.0f || u > 1.0f) continue;
                    V3 qvec = cross(tvec, e1);
                    float v = dot(ray.d, qvec) * inv_det;
                    if (v < 0.0f || u + v > 1.0f) continue;
                    float tt = dot(e2, qvec) * inv_det;
                    if (tt < ray.tmin || tt > ray.tmax) continue;
                    *bu = u; *bv = v; *bt = tt; prim = node.offset + i; ray.tmax = tt;
                    if (any_hit) return 0;
                }
                if (to_visit == 0) break;
                cur = stack[--to_visit];
            }
            else if (sign[node.num_primitives_axis & 0xFFFF]) { stack[to_visit++] = cur + 1; cur = (int)node.offset; }
            else { stack[to_visit++] = (int)node.offset; cur = cur + 1; }
        }
        else
        {
            if (to_visit == 0) break;
            cur = stack[--to_visit];
        }
    }
    return prim;
}

// trace_instanced: -> virtual id (closest) / 0 (any hit) / RT_INVALID_ID
inline uint32_t InstTrace(const Scene& sc, const Inst& I, Ray ray, bool any_hit, RtHit* hit)
{
    uint32_t prim = RT_INVALID_ID;
    float bu = 0.0f, bv = 0.0f, bt = 0.0f;
    if (hit) { hit->bc.x = 0.0f; hit->bc.y = 0.0f; hit->t = 0.0f; hit->primitive_id = RT_INVALID_ID; }
    if (I.n == 0) return prim;
    const V3 o = ray.o, d = ray.d;
    const V3 inv = splat(1.0f) / d;
    const bool sx = inv.x < 0, sy = inv.y < 0, sz = inv.z < 0;
    float t_max = ray.tmax;
    const rtinst::Tree& tr = I.pr.tree;
    const float e = rt_fmaxf(rt_fmaxf(std::fabs(o.x), std::fabs(o.y)), std::fabs(o.z)) * tr.slack[0] + tr.slack[1];
    {
        V3 t0 = (v3(tr.root.lo[0] - e, tr.root.lo[1] - e, tr.root.lo[2] - e) - o) * inv,
           t1 = (v3(tr.root.hi[0] + e, tr.root.hi[1] + e, tr.root.hi[2] + e) - o) * inv;
        float lo = rt_fmaxf(rt_fmaxf(rt_fminf(t0.x, t1.x), rt_fminf(t0.y, t1.y)), rt_fminf(t0.z, t1.z));
        float hi = rt_fminf(rt_fminf(rt_fmaxf(t0.x, t1.x), rt_fmaxf(t0.y, t1.y)), rt_fmaxf(t0.z, t1.z));
        if (!(rt_fminf(hi, t_max) >= rt_fmaxf(lo, ray.tmin))) return prim;
    }
    int cur = tr.root_ref, sp = 0;
    int stack_ref[64];
    float stack_t[64];
    for (;;)
    {
        while (cur >= 0)
        {
            const float* r = tr.records.data() + 16 * (size_t)cur;
            float lo0, lo1;
            bool h0 = SlabHit(r, r + 3, e, o, inv, ray.tmin, t_max, &lo0), h1 = SlabHit(r + 6, r + 9, e, o, inv, ray.tmin, t_max, &lo1);
            int r0, r1; uint32_t axis;
            memcpy(&r0, r + 12, 4); memcpy(&r1, r + 13, 4); memcpy(&axis, r + 14, 4);
            bool swap = axis == 0 ? sx : (axis == 1 ? sy : sz);
            int near_ref = swap ? r1 : r0, far_ref = swap ? r0 : r1;
            bool near_hit = swap ? h1 : h0, far_hit = swap ? h0 : h1;
            float far_lo = swap ? lo0 : lo1;
            if (near_hit)
            {
                if (far_hit) { stack_ref[sp] = far_ref; stack_t[sp] = far_lo; ++sp; }
                cur = near_ref;
            }
            else if (far_hit) cur = far_ref;
            else
            {
                bool found = false;
                while (sp > 0) { --sp; if (t_max >= stack_t[sp]) { cur = stack_ref[sp]; found = true; break; } }
                if (!found) goto done;
            }
        }
        {
            const uint32_t i = (uint32_t)(~cur);
            const float* rec = I.pr.rec.data() + 32 * (size_t)i;
            uint32_t mesh_first_tri, base, first_node;
            memcpy(&mesh_first_tri, rec + 26, 4); memcpy(&base, rec + 27, 4); memcpy(&first_node, rec + 29, 4);
            Scene view = sc;
            view.triangles = sc.triangles + mesh_first_tri;
            view.nodes = sc.nodes + first_node;
            Ray r;
            r.o = XPoint(rec, o); r.d = XDir(rec, d); r.tmin = ray.tmin; r.tmax = t_max;
            float u, v, t;
            const uint32_t p = MeshTrace(view, r, rec[28], any_hit, &u, &v, &t);
            if (p != RT_INVALID_ID)
            {
                if (any_hit) return 0;
                prim = base + p; bu = u; bv = v; bt = t; t_max = t;
            }
        }
        {
            bool found = false;
            while (sp > 0) { --sp; if (t_max >= stack_t[sp]) { cur = stack_ref[sp]; found = true; break; } }
            if (!found) break;
        }
    }
done:
    if (hit) { hit->bc.x = bu; hit->bc.y = bv; hit->t = bt; hit->primitive_id = prim; }
    return prim;
}

// the instance of a virtual id (the last base <= prim)
inline uint32_t InstanceOf(const Inst& I, uint32_t prim)
{
    return (uint32_t)(std::upper_bound(I.pr.base.begin(), I.pr.base.end(), prim) - I.pr.base.begin()) - 1u;
}

} // namespace

extern "C" {

/* One sample of the instanced frame, as orc_render: scene = the concatenated meshes and the shared arrays; meshes, instances as
 * rt_upload_instanced_scene / rt_set_instances take them; prev (12 floats per instance, may be NULL) the previous transforms for
 * velocity (float2 per pixel, bounce-0 hits, camera == previous camera; may be NULL).  Returns 0, or -1 for a rejected list. */
static bool make_inst(const Scene& sc, const RtMeshDesc* meshes, uint32_t n_meshes, const RtInstance* instances, uint32_t n_inst, Inst& I)
{
    for (uint32_t k = 0; k < n_meshes; ++k)
    {
        const RtMeshDesc& m = meshes[k];
        const RtLinearBVHNode& r = sc.nodes[m.first_node];
        rtinst::MeshInfo mi = { 0, 0, (uint32_t)m.first_triangle, (uint32_t)m.n_triangles, (uint32_t)m.first_node,
                                { r.bounds_min.x, r.bounds_min.y, r.bounds_min.z }, { r.bounds_max.x, r.bounds_max.y, r.bounds_max.z } };
        I.meshes.push_back(mi);
    }
    std::string err;
    if (!rtinst::prepare(instances, n_inst, I.meshes, I.pr, err)) return false;
    I.n = n_inst;
    return true;
}

/* The two-level traversal of n rays (origin.w = t_min, direction.w = t_max, as orc_trace takes them): closest hits (virtual ids)
 * into hits, or for any_hit 0 (occluded) / RT_INVALID_ID per ray into flags.  Returns 0, or -1 for a rejected list. */
int im_trace(const OrcScene* scene, const RtMeshDesc* meshes, uint32_t n_meshes, const RtInstance* instances, uint32_t n_inst,
             const RtRay* rays, uint32_t n, int any_hit, RtHit* hits, uint32_t* flags)
{
    Scene sc = to_scene(scene);
    Inst I;
    if (!make_inst(sc, meshes, n_meshes, instances, n_inst, I)) return -1;
#pragma omp parallel for schedule(dynamic, 256)
    for (long long i = 0; i < (long long)n; ++i)
    {
        Ray r; r.o = v3(rays[i].origin); r.tmin = rays[i].origin.w; r.d = v3(rays[i].direction); r.tmax = rays[i].direction.w;
        RtHit h;
        const uint32_t p = InstTrace(sc, I, r, any_hit != 0, any_hit ? nullptr : &h);
        if (any_hit) flags[i] = p;
        else hits[i] = h;
    }
    return 0;
}

/* Mesh `mesh`'s own tree alone (no top level) on n object-space rays, culling on det * cull: closest hits (mesh triangle ids). */
void im_trace_mesh(const OrcScene* scene, const RtMeshDesc* meshes, uint32_t mesh, const RtRay* rays, uint32_t n, float cull, RtHit* hits)
{
    Scene sc = to_scene(scene);
    Scene view = sc;
    view.triangles = sc.triangles + meshes[mesh].first_triangle;
    view.nodes = sc.nodes + meshes[mesh].first_node;
#pragma omp parallel for schedule(dynamic, 256)
    for (long long i = 0; i < (long long)n; ++i)
    {
        Ray r; r.o = v3(rays[i].origin); r.tmin = rays[i].origin.w; r.d = v3(rays[i].direction); r.tmax = rays[i].direction.w;
        float u = 0.0f, v = 0.0f, t = 0.0f;
        const uint32_t p = MeshTrace(view, r, cull, false, &u, &v, &t);
        hits[i].bc.x = u; hits[i].bc.y = v; hits[i].t = t; hits[i].primitive_id = p;
    }
}

int im_render(const OrcScene* scene, const RtMeshDesc* meshes, uint32_t n_meshes, const RtInstance* instances, uint32_t n_inst,
              const float* prev, const RtCamera* cam, uint32_t width, uint32_t height, uint32_t max_bounces, uint32_t sample_idx,
              float* radiance, RtHit* primary_hits, OrcStats* stats, float* velocity)
{
    Scene sc = to_scene(scene);
    Inst I;
    if (!make_inst(sc, meshes, n_meshes, instances, n_inst, I)) return -1;

    std::vector<uint32_t> pix;
    for (uint32_t y = 0; y < height; ++y)
        for (uint32_t x = 0; x < width; ++x) pix.push_back(y * width + x);
    size_t n_live = pix.size();
    std::vector<Ray> rays(n_live), next_rays(n_live);
    std::vector<uint32_t> next_pix(n_live);
    std::vector<V3> throughputs((size_t)width * height);
    std::vector<RtHit> hits(n_live);
    struct Shadow { Ray ray; uint32_t pixel; V3 sample; bool valid; };
    std::vector<Shadow> shadow(n_live);
    std::vector<uint8_t> cont(n_live);
    if (stats) memset(stats, 0, sizeof(*stats));
    if (velocity) memset(velocity, 0, sizeof(float) * 2 * width * height);
    for (size_t i = 0; i < n_live; ++i)
    {
        rays[i] = RayGeneration(pix[i], width, height, *cam, sample_idx);
        throughputs[pix[i]] = splat(1.0f);
    }
    for (uint32_t bounce = 0; bounce <= max_bounces; ++bounce)
    {
        uint32_t n_miss = 0, n_emis = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : n_miss, n_emis)
        for (long long i = 0; i < (long long)n_live; ++i)
        {
            RtHit hit;
            const Ray& ray = rays[i];
            InstTrace(sc, I, ray, false, &hit);
            hits[i] = hit;
            uint32_t pixel = pix[i];
            float* rad = radiance + (size_t)pixel * 4;
            shadow[i].valid = false; cont[i] = 0;
            if (hit.primitive_id == RT_INVALID_ID)
            {
                ++n_miss;
                V3 add = SampleSky(sc, ray.d) * throughputs[pixel];
                rad[0] += add.x; rad[1] += add.y; rad[2] += add.z;
                continue;
            }
            const uint32_t inst = InstanceOf(I, hit.primitive_id);
            const float* rec = I.pr.rec.data() + 32 * (size_t)inst;
            uint32_t first_tri;
            memcpy(&first_tri, rec + 26, 4);
            const RtTriangle& tri = sc.triangles[first_tri + (hit.primitive_id - I.pr.base[inst])];
            V3 incoming = -ray.d;
            uint32_t px = pixel % width, py = pixel / width;
            V3 p1 = v3(tri.v1.position), p2 = v3(tri.v2.position), p3 = v3(tri.v3.position);
            float u = hit.bc.x, v = hit.bc.y;
            V3 obj = Interp(p1, p2, p3, u, v);
            V3 position = XPoint(rec + 12, obj);
            V3 geometry_normal = normalize(XNormalT(rec, cross(p2 - p1, p3 - p1))) * rec[28];
            float w0 = 1.0f - u - v;
            V2 texcoord = { tri.v1.texcoord.x * w0 + tri.v2.texcoord.x * u + tri.v3.texcoord.x * v,
                            tri.v1.texcoord.y * w0 + tri.v2.texcoord.y * u + tri.v3.texcoord.y * v };
            V3 normal = normalize(XNormalT(rec, Interp(v3(tri.v1.normal), v3(tri.v2.normal), v3(tri.v3.normal), u, v)));
            Material material = ApplyTextures(sc, sc.materials[tri.mtlIndex], texcoord);
            if (bounce == 0 && velocity)
            {
                V3 was = prev ? XPoint(prev + 12 * (size_t)inst, obj) : position;
                V2 a = ProjectScreen(position, *cam), b = ProjectScreen(was, *cam);
                velocity[2 * pixel] = a.x - b.x; velocity[2 * pixel + 1] = a.y - b.y;
            }
            V3 hit_throughput = throughputs[pixel];
            if (dot(material.emission, splat(1.0f)) > 0.0f)
            {
                ++n_emis;
                V3 add = hit_throughput * material.emission;
                rad[0] += add.x; rad[1] += add.y; rad[2] += add.z;
            }
            {
                float s_light = SampleRandom(px, py, sample_idx, bounce, SAMPLE_LIGHT);
                V3 outgoing; float pdf;
                V3 light_radiance = Light_Sample(sc, position, s_light, &outgoing, &pdf);
                float distance_to_light = length(outgoing);
                outgoing = normalize(outgoing);
                V3 brdf = EvaluateMaterial(material, normal, incoming, outgoing);
                V3 light_sample = light_radiance * hit_throughput * brdf / pdf * rt_fmaxf(dot(outgoing, normal), 0.0f);
                if (pdf > 0.0f && dot(light_sample, light_sample) > 0.0f)
                {
                    Shadow& s = shadow[i];
                    s.valid = true; s.pixel = pixel; s.sample = light_sample;
                    s.ray.o = position + normal * RT_EPS; s.ray.tmin = 0.0f;
                    s.ray.d = outgoing; s.ray.tmax = distance_to_light;
                }
            }
            {
                V2 s = { SampleRandom(px, py, sample_idx, bounce, SAMPLE_U), SampleRandom(px, py, sample_idx, bounce, SAMPLE_V) };
                float s1 = SampleRandom(px, py, sample_idx, bounce, SAMPLE_LAYER);
                float pdf = 0.0f, offset;
                V3 outgoing = v3(0, 0, 0);
                V3 bxdf = SampleBxdf(s1, s, material, normal, incoming, false, &outgoing, &pdf, &offset);
                V3 throughput = splat(0.0f);
                if (pdf > 0.0f) throughput = bxdf / pdf;
                throughputs[pixel] = throughputs[pixel] * throughput;
                if (pdf > 0.0f)
                {
                    cont[i] = 1;
                    Ray& o = next_rays[i];
                    o.o = position + geometry_normal * RT_EPS * offset; o.tmin = 0.0f;
                    o.d = outgoing; o.tmax = RT_MAX_RENDER_DIST;
                }
            }
        }
        if (bounce == 0 && primary_hits)
            for (size_t i = 0; i < n_live; ++i) primary_hits[pix[i]] = hits[i];
        uint32_t n_shadow = 0, n_unocc = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : n_shadow, n_unocc)
        for (long long i = 0; i < (long long)n_live; ++i)
        {
            if (!shadow[i].valid) continue;
            ++n_shadow;
            if (InstTrace(sc, I, shadow[i].ray, true, nullptr) == RT_INVALID_ID)
            {
                ++n_unocc;
                float* rad = radiance + (size_t)shadow[i].pixel * 4;
                rad[0] += shadow[i].sample.x; rad[1] += shadow[i].sample.y; rad[2] += shadow[i].sample.z;
            }
        }
        size_t n_next = 0;
        for (size_t i = 0; i < n_live; ++i)
            if (cont[i]) { rays[n_next] = next_rays[i]; next_pix[n_next] = pix[i]; ++n_next; }
        if (stats && bounce < ORC_MAX_BOUNCES)
        {
            stats->n_ext[bounce] = (uint32_t)n_live; stats->n_miss[bounce] = n_miss; stats->n_hit[bounce] = (uint32_t)n_live - n_miss;
            stats->n_shadow[bounce] = n_shadow; stats->n_cont[bounce] = (uint32_t)n_next; stats->n_unoccluded[bounce] = n_unocc;
            stats->n_emissive_hits[bounce] = n_emis;
        }
        pix.swap(next_pix); pix.resize(n_next); next_pix.resize(n_live);
        n_live = n_next;
        if (n_live == 0) break;
    }
    return 0;
}

} // extern "C"
