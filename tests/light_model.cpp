/*
 * light_model.cpp — TEST INFRASTRUCTURE.  CPU model of the sampled lights (include/rt_b200.h: RT_OPT_EMITTER_SAMPLING,
 * RT_OPT_ENV_SAMPLING and rt_set_light_selection): one sample of the oracle's frame (oracle/oracle.cpp orc_render) with next-event
 * estimation on the emissive triangles and on the environment map, the light kind drawn with the selection weights, and the
 * MIS-weighted emission of BSDF hits and sky of BSDF misses.  It reuses the emitter model (emitter_model.cpp: the oracle compiled
 * into the same translation unit, EmitRandom, BxdfEvalSampled, MisPower) and the library's own table builders and environment
 * walk (raytracing_b200/csrc/rt_emitters.h, rt_envmap.h).  With both tables inactive it is orc_render; with the environment table
 * inactive and the default weights it is em_render.  Built by tests/light_model.py with -ffp-contract=off.
 */
#include "emitter_model.cpp"
#include "rt_envmap.h"

extern "C" {

/* The environment table of an RGBA32F image with P_v = p_v: returns whether it is active (T finite and > 0, white furnace off);
 * marg holds h entries, cond and pdf w * h. */
int lm_env_table(const float* rgba, uint32_t w, uint32_t h, float p_v, int white_furnace, float* marg, float* cond, float* pdf)
{
    rtenv::Table t;
    if (white_furnace || !rtenv::build(rgba, w, h, t)) return 0;
    rtenv::scale(t, p_v);
    for (uint32_t j = 0; j < h; ++j) marg[j] = t.marg[j];
    for (size_t k = 0; k < (size_t)w * h; ++k) { cond[k] = t.cond[k]; pdf[k] = t.pdf[k]; }
    return 1;
}

/* p_v of n directions (xyz) for a table pdf of w x h */
void lm_env_pdf(const float* pdf, uint32_t w, uint32_t h, const float* dirs, uint32_t n, float* out)
{
    for (uint32_t k = 0; k < n; ++k) out[k] = rtenv::pdf_dir(pdf, (int)w, (int)h, dirs[3 * k], dirs[3 * k + 1], dirs[3 * k + 2]);
}

/* n environment samples from draws r (4 per sample): directions (xyz) */
void lm_env_sample(const float* marg, const float* cond, uint32_t w, uint32_t h, const float* r, uint32_t n, float* dirs)
{
    for (uint32_t k = 0; k < n; ++k)
        rtenv::sample(marg, cond, (int)w, (int)h, r[4 * k], r[4 * k + 1], r[4 * k + 2], r[4 * k + 3], dirs[3 * k], dirs[3 * k + 1], dirs[3 * k + 2]);
}

/* rt_sinf of n floats (the row factor of the table) */
void lm_sinf(const float* x, uint32_t n, float* out)
{
    for (uint32_t k = 0; k < n; ++k) out[k] = rt_sinf(x[k]);
}

/* The light-kind probabilities: out = (P_e, P_v, P_e + P_v, no_analytic) */
void lm_select(int analytic, int emitters, int env, float wa, float we, float wv, float* out)
{
    const rtenv::Selection s = rtenv::select(analytic != 0, emitters != 0, env != 0, wa, we, wv);
    out[0] = s.p_e; out[1] = s.p_v; out[2] = s.p_ev; out[3] = s.no_analytic ? 1.0f : 0.0f;
}

/* orc_render with the sampled lights: emitters / env are the two options, weights the rt_set_light_selection weights (the
 * emitter list must be valid: em_table) */
void lm_render(const OrcScene* scene, const uint32_t* emissive, uint32_t n_emissive, const RtCamera* cam, uint32_t width, uint32_t height,
               uint32_t max_bounces, uint32_t sample_idx, int white_furnace, uint32_t row_first, uint32_t row_step,
               int emitters, int env, const float* weights, float* radiance, OrcStats* stats)
{
    Scene sc = to_scene(scene);
    auto tri_of = [&](uint64_t i) -> const RtTriangle& { return scene->triangles[emissive[i]]; };
    rtemit::Table tab;
    if (emitters)
        rtemit::build(tri_of, emissive, n_emissive, scene->n_triangles, scene->materials, scene->lights, scene->info.analytic_light_count,
                      white_furnace != 0, tab);
    const bool emit_active = tab.p_e > 0.0f;
    rtenv::Table vt;
    const bool env_active = env && !white_furnace && rtenv::build(sc.env, sc.env_w, sc.env_h, vt);
    const rtenv::Selection sel = rtenv::select(rtenv::analytic_lit(scene->lights, scene->info.analytic_light_count), emit_active, env_active,
                                               weights[0], weights[1], weights[2]);
    if (emit_active)
        rtemit::build(tri_of, emissive, n_emissive, scene->n_triangles, scene->materials, scene->lights, scene->info.analytic_light_count,
                      white_furnace != 0, tab, sel.p_e);
    if (env_active) rtenv::scale(vt, sel.p_v);
    const bool active = emit_active || env_active;
    const int ew = (int)sc.env_w, eh = (int)sc.env_h;

    if (row_step == 0) row_step = 1;
    std::vector<uint32_t> pix;
    for (uint32_t y = row_first; y < height; y += row_step)
        for (uint32_t x = 0; x < width; ++x) pix.push_back(y * width + x);
    size_t n_live = pix.size();
    std::vector<Ray> rays(n_live), next_rays(n_live);
    std::vector<float> cw(n_live, 0.0f), next_cw(n_live, 0.0f);      // C.w of the rays: p_b of their direction
    std::vector<uint32_t> next_pix(n_live);
    std::vector<V3> throughputs((size_t)width * height);
    struct Shadow { Ray ray; uint32_t pixel; V3 sample; bool valid; };
    std::vector<Shadow> shadow(n_live);
    std::vector<uint8_t> cont(n_live);
    if (stats) memset(stats, 0, sizeof(*stats));

    for (size_t i = 0; i < n_live; ++i)
    {
        rays[i] = RayGeneration(pix[i], width, height, *cam, sample_idx);
        throughputs[pix[i]] = splat(1.0f);
    }

    for (uint32_t bounce = 0; bounce <= max_bounces; ++bounce)
    {
        uint64_t nv = 0, nt = 0, nvs = 0, nts = 0;
        uint32_t n_miss = 0, n_emis = 0;
        const bool emit_on = active && bounce < max_bounces;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : nv, nt, n_miss, n_emis)
        for (long long i = 0; i < (long long)n_live; ++i)
        {
            TraceCounters c = { 0, 0 };
            RtHit hit;
            const Ray& ray = rays[i];
            TraceBvh(sc, ray, false, &hit, &c);
            nv += c.nodes_visited; nt += c.tris_tested;
            uint32_t pixel = pix[i];
            float* rad = radiance + (size_t)pixel * 4;
            shadow[i].valid = false; cont[i] = 0;
            if (hit.primitive_id == RT_INVALID_ID)
            {
                ++n_miss;
                V3 sky = white_furnace ? splat(0.5f) : SampleSky(sc, ray.d);
                V3 add = sky * throughputs[pixel];
                if (env_active && cw[i] > 0.0f)
                    add = add * MisPower(cw[i], rtenv::pdf_dir(vt.pdf.data(), ew, eh, ray.d.x, ray.d.y, ray.d.z));
                rad[0] += add.x; rad[1] += add.y; rad[2] += add.z;
                continue;
            }
            V3 incoming = -ray.d;
            uint32_t px = pixel % width, py = pixel / width;
            const RtTriangle& tri = sc.triangles[hit.primitive_id];
            V3 p1 = v3(tri.v1.position), p2 = v3(tri.v2.position), p3 = v3(tri.v3.position);
            float u = hit.bc.x, v = hit.bc.y;
            V3 position = Interp(p1, p2, p3, u, v);
            V3 geometry_normal = normalize(cross(p2 - p1, p3 - p1));
            float w0 = 1.0f - u - v;
            V2 texcoord = { tri.v1.texcoord.x * w0 + tri.v2.texcoord.x * u + tri.v3.texcoord.x * v,
                            tri.v1.texcoord.y * w0 + tri.v2.texcoord.y * u + tri.v3.texcoord.y * v };
            V3 normal = normalize(Interp(v3(tri.v1.normal), v3(tri.v2.normal), v3(tri.v3.normal), u, v));
            Material material = ApplyTextures(sc, sc.materials[tri.mtlIndex], texcoord);
            V3 hit_throughput = throughputs[pixel];
            if (!white_furnace && dot(material.emission, splat(1.0f)) > 0.0f)
            {
                ++n_emis;
                V3 add = hit_throughput * material.emission;
                if (emit_active && cw[i] > 0.0f && tab.pdfA[hit.primitive_id] > 0.0f)
                {
                    V3 dv = position - ray.o;
                    float cos_e = -dot(ray.d, geometry_normal);
                    float p_l = tab.pdfA[hit.primitive_id] * dot(dv, dv) / cos_e;
                    add = add * MisPower(cw[i], p_l);
                }
                rad[0] += add.x; rad[1] += add.y; rad[2] += add.z;
            }
            bool pick_emitter = false, pick_env = false;
            if (emit_on)
            {
                float ck = EmitRandom(px, py, sample_idx, 0x10000u + 4u * bounce);
                pick_emitter = sel.p_e >= 1.0f || ck < sel.p_e;
                pick_env = !pick_emitter && env_active && (sel.no_analytic || ck < sel.p_ev);
            }
            if (pick_emitter)
            {
                float k1 = EmitRandom(px, py, sample_idx, 0x10000u + 4u * bounce + 1u);
                float k2 = EmitRandom(px, py, sample_idx, 0x10000u + 4u * bounce + 2u);
                float k3 = EmitRandom(px, py, sample_idx, 0x10000u + 4u * bounce + 3u);
                k1 = rt_fminf(k1, 0.99999994f);
                size_t sel_i = 0;
                while (!(tab.cdf[sel_i] > k1)) ++sel_i;          // first CDF entry above k1
                const uint32_t t = tab.list[sel_i];
                const RtTriangle& et = sc.triangles[t];
                V3 q1 = v3(et.v1.position), q2 = v3(et.v2.position), q3 = v3(et.v3.position);
                float sq = sqrtf(k2);
                float b0 = 1.0f - sq, b1 = sq * (1.0f - k3), b2 = sq * k3;
                V3 y = q1 * b0 + q2 * b1 + q3 * b2;
                V2 euv = { et.v1.texcoord.x * b0 + et.v2.texcoord.x * b1 + et.v3.texcoord.x * b2,
                           et.v1.texcoord.y * b0 + et.v2.texcoord.y * b1 + et.v3.texcoord.y * b2 };
                V3 le = ApplyTextures(sc, sc.materials[et.mtlIndex], euv).emission;
                V3 gn = normalize(cross(q2 - q1, q3 - q1));
                V3 o = position + geometry_normal * RT_EPS;
                V3 dv = y - o;
                float d2 = dot(dv, dv);
                float d = sqrtf(d2);
                V3 w = normalize(dv);
                float cos_e = -dot(w, gn);
                if (cos_e > 0.0f)
                {
                    float p_l = tab.pdfA[t] * d2 / cos_e;
                    float p_b, spec_pdf, alpha;
                    V3 g = BxdfEvalSampled(material, normal, incoming, w, &p_b, &spec_pdf, &alpha);
                    V3 ls = hit_throughput * g * le * (MisPower(p_l, p_b) / p_l);
                    if (p_l > 0.0f && dot(ls, ls) > 0.0f)
                    {
                        Shadow& s = shadow[i];
                        s.valid = true; s.pixel = pixel; s.sample = ls;
                        s.ray.o = o; s.ray.tmin = 0.0f; s.ray.d = w; s.ray.tmax = 0.999f * d;
                    }
                }
            }
            else if (pick_env)
            {
                float k1 = EmitRandom(px, py, sample_idx, 0x10000u + 4u * bounce + 1u);
                float k2 = EmitRandom(px, py, sample_idx, 0x10000u + 4u * bounce + 2u);
                float k3 = EmitRandom(px, py, sample_idx, 0x10000u + 4u * bounce + 3u);
                float k4 = EmitRandom(px, py, sample_idx, 0x20000u + bounce);
                V3 w;
                rtenv::sample(vt.marg.data(), vt.cond.data(), ew, eh, k1, k2, k3, k4, w.x, w.y, w.z);
                float p_v = rtenv::pdf_dir(vt.pdf.data(), ew, eh, w.x, w.y, w.z);
                V3 le = SampleSky(sc, w);
                float p_b, spec_pdf, alpha;
                V3 g = BxdfEvalSampled(material, normal, incoming, w, &p_b, &spec_pdf, &alpha);
                V3 ls = hit_throughput * g * le * (MisPower(p_v, p_b) / p_v);
                if (p_v > 0.0f && dot(ls, ls) > 0.0f)
                {
                    Shadow& s = shadow[i];
                    s.valid = true; s.pixel = pixel; s.sample = ls;
                    s.ray.o = position + geometry_normal * RT_EPS; s.ray.tmin = 0.0f; s.ray.d = w; s.ray.tmax = RT_MAX_RENDER_DIST;
                }
            }
            else
            {
                float s_light = SampleRandom(px, py, sample_idx, bounce, SAMPLE_LIGHT);
                V3 outgoing; float pdf;
                V3 light_radiance = Light_Sample(sc, position, s_light, &outgoing, &pdf);
                float distance_to_light = length(outgoing);
                outgoing = normalize(outgoing);
                V3 brdf = EvaluateMaterial(material, normal, incoming, outgoing);
                V3 light_sample = light_radiance * hit_throughput * brdf / pdf * rt_fmaxf(dot(outgoing, normal), 0.0f);
                if (emit_on) light_sample = light_sample / (1.0f - sel.p_ev);
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
                V3 bxdf = SampleBxdf(s1, s, material, normal, incoming, white_furnace != 0, &outgoing, &pdf, &offset);
                V3 throughput = splat(0.0f);
                if (pdf > 0.0f) throughput = bxdf / pdf;
                throughputs[pixel] = throughputs[pixel] * throughput;
                if (pdf > 0.0f)
                {
                    cont[i] = 1;
                    Ray& o = next_rays[i];
                    o.o = position + geometry_normal * RT_EPS * offset; o.tmin = 0.0f;
                    o.d = outgoing; o.tmax = RT_MAX_RENDER_DIST;
                    next_cw[i] = 0.0f;
                    if (emit_on)
                    {
                        float p_b, spec_pdf, alpha;
                        BxdfEvalSampled(material, normal, incoming, outgoing, &p_b, &spec_pdf, &alpha);
                        bool delta = material.transparency < 0.5f || (s1 <= spec_pdf && alpha <= 1e-4f);
                        next_cw[i] = delta ? 0.0f : p_b;
                    }
                }
            }
        }

        uint32_t n_shadow = 0, n_unocc = 0;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : nvs, nts, n_shadow, n_unocc)
        for (long long i = 0; i < (long long)n_live; ++i)
        {
            if (!shadow[i].valid) continue;
            ++n_shadow;
            TraceCounters c = { 0, 0 };
            uint32_t f = TraceBvh(sc, shadow[i].ray, true, nullptr, &c);
            nvs += c.nodes_visited; nts += c.tris_tested;
            if (f == RT_INVALID_ID)
            {
                ++n_unocc;
                float* rad = radiance + (size_t)shadow[i].pixel * 4;
                rad[0] += shadow[i].sample.x; rad[1] += shadow[i].sample.y; rad[2] += shadow[i].sample.z;
            }
        }

        size_t n_next = 0;
        for (size_t i = 0; i < n_live; ++i)
            if (cont[i]) { rays[n_next] = next_rays[i]; cw[n_next] = next_cw[i]; next_pix[n_next] = pix[i]; ++n_next; }
        if (stats && bounce < ORC_MAX_BOUNCES)
        {
            stats->n_ext[bounce] = (uint32_t)n_live; stats->n_miss[bounce] = n_miss; stats->n_hit[bounce] = (uint32_t)n_live - n_miss;
            stats->n_shadow[bounce] = n_shadow; stats->n_cont[bounce] = (uint32_t)n_next; stats->n_unoccluded[bounce] = n_unocc;
            stats->n_emissive_hits[bounce] = n_emis;
            stats->nodes_ext[bounce] = nv; stats->tris_ext[bounce] = nt; stats->nodes_shadow[bounce] = nvs; stats->tris_shadow[bounce] = nts;
        }
        pix.swap(next_pix); pix.resize(n_next); next_pix.resize(n_live);
        n_live = n_next;
        if (n_live == 0) break;
    }
}

} // extern "C"
